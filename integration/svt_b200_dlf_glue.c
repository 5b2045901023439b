/* svt_b200_dlf_glue.c -- see svt_b200_dlf_glue.h.  Compiled against the reference headers with -Wall -Werror. */
#include <string.h>
#include "definitions.h"
#include "pcs.h"
#include "sequence_control_set.h"
#include "coding_unit.h"
#include "deblocking_common.h"
#include "svt_b200.h"
#include "svt_b200_dlf_glue.h"

static void lfthr_from(const LoopFilterInfoN* lfi, SvtB200DlfFrame* frame) {
    for (int l = 0; l <= MAX_LOOP_FILTER; l++) {
        frame->lfthr[l][0] = lfi->lfthr[l].mblim[0];
        frame->lfthr[l][1] = lfi->lfthr[l].lim[0];
        frame->lfthr[l][2] = lfi->lfthr[l].hev_thr[0];
    }
}

int svt_b200_dlf_frame_from_pcs(const PictureControlSet* pcs, const EbPictureBufferDesc* recon, SvtB200DlfFrame* frame, SvtB200DlfMi* mi) {
    const PictureParentControlSet* ppcs = pcs->ppcs;
    const SequenceControlSet*      scs  = pcs->scs;
    const FrameHeader*             fh   = &ppcs->frm_hdr;
    if (ppcs->frame_superres_enabled || ppcs->frame_resize_enabled || fh->delta_lf_params.delta_lf_present) return SVT_B200_ERR_BAD_ARG;
    memset(frame, 0, sizeof(*frame));
    /* deblocking_filter.c:556-570: 16-bit samples when the pipeline is 16-bit or the picture is high bit depth */
    const int pb = (scs->is_16bit_pipeline || recon->bit_depth > EB_EIGHT_BIT) ? 2 : 1;
    frame->plane[0] = recon->buffer_y + (((size_t)recon->org_y * recon->stride_y + recon->org_x) * pb);
    frame->plane[1] = recon->buffer_cb + (((size_t)(recon->org_y >> 1) * recon->stride_cb + (recon->org_x >> 1)) * pb);
    frame->plane[2] = recon->buffer_cr + (((size_t)(recon->org_y >> 1) * recon->stride_cr + (recon->org_x >> 1)) * pb);
    frame->stride[0] = recon->stride_y;
    frame->stride[1] = recon->stride_cb;
    frame->stride[2] = recon->stride_cr;
    /* the unpadded size (deblocking_filter.c:100-132) */
    frame->width       = scs->max_input_luma_width - scs->max_input_pad_right;
    frame->height      = scs->max_input_luma_height - scs->max_input_pad_bottom;
    frame->mi_rows     = ((ppcs->aligned_height + 7) & ~7) >> 2;
    frame->mi_cols     = ((ppcs->aligned_width + 7) & ~7) >> 2;
    frame->mi_stride   = pcs->mi_stride;
    frame->bit_depth   = (int32_t)scs->static_config.encoder_bit_depth;
    frame->pixel_bytes = pb;
    frame->filter_level[0] = fh->loop_filter_params.filter_level[0];
    frame->filter_level[1] = fh->loop_filter_params.filter_level[1];
    frame->filter_level_u  = fh->loop_filter_params.filter_level_u;
    frame->filter_level_v  = fh->loop_filter_params.filter_level_v;
    memcpy(frame->lvl, ppcs->lf_info.lvl, sizeof(frame->lvl));
    lfthr_from(&ppcs->lf_info, frame);
    if (mi) {
        for (int r = 0; r < frame->mi_rows; r++)
            for (int c = 0; c < frame->mi_stride; c++) {
                SvtB200DlfMi* o = &mi[(size_t)r * frame->mi_stride + c];
                memset(o, 0, sizeof(*o));
                if (c >= frame->mi_cols) continue;
                const ModeInfo* m = pcs->mi_grid_base[(size_t)r * pcs->mi_stride + c];
                if (!m) return SVT_B200_ERR_BAD_ARG;
                const BlockModeInfoEnc* b = &m->mbmi.block_mi;
                o->bsize      = (uint8_t)b->bsize;
                o->tx_depth   = b->tx_depth;
                o->skip       = b->skip;
                o->ref_frame0 = (int8_t)b->ref_frame[0];
                o->mode       = (uint8_t)b->mode;
                o->segment_id = b->segment_id;
            }
    }
    return SVT_B200_OK;
}

int svt_b200_dlf_level_sse_from_pcs(const PictureControlSet* pcs, const EbPictureBufferDesc* recon, int plane_mask, int n_levels,
                                    const uint8_t* levels, SvtB200DlfFrame* frame, SvtB200DlfLevelSse* s, uint8_t* lvl) {
    if (n_levels < 1 || n_levels > 64 || !(plane_mask & 7) || (plane_mask & ~7)) return SVT_B200_ERR_BAD_ARG;
    for (int i = 0; i < n_levels; i++)
        if (levels[i] > MAX_LOOP_FILTER) return SVT_B200_ERR_BAD_ARG;
    const int rc = svt_b200_dlf_frame_from_pcs(pcs, recon, frame, NULL);
    if (rc) return rc;
    const PictureParentControlSet* ppcs = pcs->ppcs;
    /* picture_sse_calculations (deblocking_filter.c:717) compares 8-bit pipelines with enhanced_pic, 16-bit ones with
     * input_frame16bit */
    const int pb = frame->pixel_bytes;
    if ((pb == 2) != (pcs->scs->is_16bit_pipeline != 0)) return SVT_B200_ERR_BAD_ARG;
    const EbPictureBufferDesc* src = pb == 2 ? pcs->input_frame16bit : ppcs->enhanced_pic;
    if (!src) return SVT_B200_ERR_BAD_ARG;
    memset(s, 0, sizeof(*s));
    s->src[0] = src->buffer_y + (((size_t)src->org_y * src->stride_y + src->org_x) * pb);
    s->src[1] = src->buffer_cb + (((size_t)(src->org_y >> 1) * src->stride_cb + (src->org_x >> 1)) * pb);
    s->src[2] = src->buffer_cr + (((size_t)(src->org_y >> 1) * src->stride_cr + (src->org_x >> 1)) * pb);
    s->src_stride[0] = src->stride_y;
    s->src_stride[1] = src->stride_cb;
    s->src_stride[2] = src->stride_cr;
    s->sse_width  = ppcs->aligned_width;
    s->sse_height = ppcs->aligned_height;
    s->plane_mask = plane_mask;
    s->n_levels   = n_levels;
    memcpy(s->level, levels, (size_t)n_levels);
    /* try_filter_frame (deblocking_filter.c:840) sets the plane's level in the frame header, and svt_av1_loop_filter_frame
     * derives the tables from it; done here on copies, so the pcs stays as it was */
    FrameHeader     fh  = ppcs->frm_hdr;
    LoopFilterInfoN lfi = ppcs->lf_info;
    for (int p = 0; p < 3; p++) {
        if (!((plane_mask >> p) & 1)) continue;
        for (int i = 0; i < n_levels; i++) {
            struct LoopFilter* lf = &fh.loop_filter_params;
            if (p == 0) lf->filter_level[0] = lf->filter_level[1] = levels[i];
            else if (p == 1) lf->filter_level_u = levels[i];
            else lf->filter_level_v = levels[i];
            svt_av1_loop_filter_frame_init(&fh, &lfi, p, p + 1);
            uint8_t* o = lvl + ((size_t)p * n_levels + i) * sizeof(lfi.lvl[p]);
            if (levels[i]) memcpy(o, lfi.lvl[p], sizeof(lfi.lvl[p]));
            else memset(o, 0, sizeof(lfi.lvl[p])); /* level 0 filters nothing: the reference leaves the table stale */
        }
    }
    lfthr_from(&lfi, frame); /* svt_av1_loop_filter_frame_init applied the frame header's sharpness */
    return SVT_B200_OK;
}
