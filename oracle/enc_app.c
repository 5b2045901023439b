/* oracle/enc_app.c -- TEST INFRASTRUCTURE.  A minimal application over the reference's public encoder API
 * (Source/API/EbSvtAv1Enc.h; the call sequence of Source/App/app_process_cmd.c:577-590,866-935, restated): encodes
 * raw planar 4:2:0 frames held in memory and returns the concatenated OBU packets.  Compiled into
 * oracle/_ref/libsvtav1_enc.so next to the UNMODIFIED reference library sources; with the environment variable
 * SVT_B200_DEVICE set, the rtcd hook (integration/svt_b200_rtcd.c) installs the H100 tier at enc_handle.c:1445, so
 * the same call encodes once on the C path and once with every hot-path DSP pointer served by libsvtav1_b200.so --
 * the bitstreams must be identical (SURVEY.md 8(c)(ii)). */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "EbSvtAv1Enc.h"

/* oracle/ref_driver.c is linked in as well (its frame / unit drivers then run the reference's process-level loops with
 * whatever the dispatch pointers currently hold); it expects this initialiser from ref_glue.c, which cannot be linked here
 * because the real Source/Lib/Globals objects are */
extern void svt_aom_setup_common_rtcd_internal(uint64_t flags);
extern void svt_aom_setup_rtcd_internal(uint64_t flags);
void ref_glue_init(void) {
    svt_aom_setup_common_rtcd_internal(0);
    svt_aom_setup_rtcd_internal(0);
}

/* returns the number of bitstream bytes written to `out` (<= cap), or a negative error */
int64_t ref_encode(const uint8_t* yuv, int width, int height, int n_frames, int bit_depth, int preset, int crf, int lp, int tune,
                   uint8_t* out, int64_t cap, int32_t* n_packets) {
    EbComponentType*         h = NULL;
    EbSvtAv1EncConfiguration cfg;
    if (svt_av1_enc_init_handle(&h, &cfg) != EB_ErrorNone) return -1;
    cfg.source_width           = (uint32_t)width;
    cfg.source_height          = (uint32_t)height;
    cfg.encoder_bit_depth      = (uint32_t)bit_depth;
    cfg.enc_mode               = (int8_t)preset;
    cfg.rate_control_mode      = 0; /* CRF */
    cfg.qp                     = (uint32_t)crf;
    cfg.frame_rate_numerator   = 30;
    cfg.frame_rate_denominator = 1;
    cfg.level_of_parallelism   = (uint32_t)lp;
    cfg.use_cpu_flags          = 0; /* "--asm c": these objects are built without ARCH_X86_64 anyway */
    if (tune >= 0) cfg.tune = (uint8_t)tune;
    if (svt_av1_enc_set_parameter(h, &cfg) != EB_ErrorNone) { svt_av1_enc_deinit_handle(h); return -2; }
    if (svt_av1_enc_init(h) != EB_ErrorNone) { svt_av1_enc_deinit_handle(h); return -3; }

    const size_t psz = bit_depth > 8 ? 2 : 1;
    const size_t luma = (size_t)width * height * psz, chroma = luma / 4, frame_bytes = luma + 2 * chroma;
    int64_t written = 0;
    int     packets = 0, sent = 0, done = 0, eos_sent = 0;
    while (!done) {
        if (sent < n_frames) {
            EbSvtIOFormat      io;
            EbBufferHeaderType in;
            memset(&io, 0, sizeof(io));
            memset(&in, 0, sizeof(in));
            const uint8_t* f = yuv + (size_t)sent * frame_bytes;
            io.luma = (uint8_t*)f; io.cb = (uint8_t*)f + luma; io.cr = (uint8_t*)f + luma + chroma;
            io.y_stride = (uint32_t)width; io.cb_stride = io.cr_stride = (uint32_t)width / 2;
            in.size = sizeof(in); in.p_buffer = (uint8_t*)&io; in.n_filled_len = (uint32_t)frame_bytes; in.n_alloc_len = (uint32_t)frame_bytes;
            in.pts = sent; in.pic_type = EB_AV1_INVALID_PICTURE;
            if (svt_av1_enc_send_picture(h, &in) != EB_ErrorNone) { written = -4; break; }
            sent++;
        } else if (!eos_sent) {
            EbBufferHeaderType eos;
            memset(&eos, 0, sizeof(eos));
            eos.size = sizeof(eos); eos.flags = EB_BUFFERFLAG_EOS; eos.pic_type = EB_AV1_INVALID_PICTURE;
            svt_av1_enc_send_picture(h, &eos);
            eos_sent = 1;
        }
        for (;;) { /* drain what is ready; once everything was sent the call blocks until the next packet */
            EbBufferHeaderType* pkt = NULL;
            const EbErrorType   st  = svt_av1_enc_get_packet(h, &pkt, (uint8_t)eos_sent);
            if (st == EB_ErrorMax) { written = -5; done = 1; break; }
            if (st == EB_NoErrorEmptyQueue) break;
            const uint32_t flags = pkt->flags;
            if (pkt->n_filled_len) {
                if (written + (int64_t)pkt->n_filled_len > cap) { svt_av1_enc_release_out_buffer(&pkt); written = -6; done = 1; break; }
                memcpy(out + written, pkt->p_buffer, pkt->n_filled_len);
                written += pkt->n_filled_len;
                packets++;
            }
            svt_av1_enc_release_out_buffer(&pkt);
            if (flags & EB_BUFFERFLAG_EOS) { done = 1; break; }
        }
    }
    if (n_packets) *n_packets = packets;
    svt_av1_enc_deinit(h);
    svt_av1_enc_deinit_handle(h);
    return written;
}
