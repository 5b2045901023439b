/* oracle/ref_dlf.c -- TEST / BASELINE INFRASTRUCTURE, compiled into oracle/_ref/libsvtav1_dlf.so (oracle/dlf.mk), which takes
 * every reference symbol from oracle/_ref/libsvtav1_ref.so.
 *
 * Deblocking of one picture through the reference's OWN loop filter: svt_av1_loop_filter_init + svt_av1_loop_filter_frame
 * (deblocking_filter.c:36, :625) run on the caller's planes, with a minimal SequenceControlSet / PictureParentControlSet /
 * PictureControlSet whose mode-info grid (one ModeInfo per 4x4 position) is built from flat SvtB200DlfMi records.  None
 * of the edge logic is restated here.  The derived lf_info tables and the records come back out through the integration
 * glue (integration/svt_b200_dlf_glue.c), so the parity tests exercise that mapping too.
 *
 * ref_dlf_frame(mode 1) replays the same picture as two whole-plane passes -- every vertical edge of every superblock,
 * then every horizontal edge -- with the reference's own per-superblock walks (svt_av1_filter_block_plane_vert / _horz,
 * which call the dispatched lpf pointers).  Equality of modes 0 and 1 is the claim the device's two-launch filter rests
 * on.  Nothing here is used by the product. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "definitions.h"
#include "pcs.h"
#include "sequence_control_set.h"
#include "coding_unit.h"
#include "deblocking_filter.h"
#include "deblocking_common.h"
#include "utility.h"

#include "svt_b200.h"
#include "../integration/svt_b200_dlf_glue.h"
#include "../svt-av1-psy_b200/csrc/dlf_tables.h"

void svt_av1_setup_dst_planes(PictureControlSet* pcs, struct MacroblockdPlane* planes, BlockSize bsize, const EbPictureBufferDesc* src,
                              int32_t mi_row, int32_t mi_col, const int32_t plane_start, const int32_t plane_end); /* deblocking_filter.c:79 */

/* the frame header fields the loop filter reads, and the picture geometry */
typedef struct RefDlfCfg {
    int32_t width, height;      /* luma, unpadded */
    int32_t sb_size;            /* 64 or 128 */
    int32_t bit_depth;          /* encoder bit depth */
    int32_t pixel_bytes;        /* 1: 8-bit pipeline; 2: 16-bit pipeline (is_16bit_pipeline) */
    int32_t filter_level[2], filter_level_u, filter_level_v;
    int32_t sharpness;
    int32_t mode_ref_delta_enabled;
    int32_t ref_deltas[8];
    int32_t mode_deltas[2];
    int32_t segmentation_enabled;
    int32_t seg_lf_enabled[8][4]; /* SEG_LVL_ALT_LF_Y_V, _Y_H, _U, _V */
    int32_t seg_lf_data[8][4];
    int32_t mi_rows, mi_cols, mi_stride;
    int32_t reserved;
} RefDlfCfg;

typedef struct DlfPic {
    SequenceControlSet*      scs;
    PictureParentControlSet* ppcs;
    PictureControlSet*       pcs;
    ModeInfo*                mip;
    EbPictureBufferDesc      fb;
} DlfPic;

static void pic_build(DlfPic* d, const RefDlfCfg* c, const SvtB200DlfMi* mi, void* y, void* cb, void* cr, int stride_y, int stride_c) {
    memset(d, 0, sizeof(*d));
    SequenceControlSet*      scs  = (SequenceControlSet*)calloc(1, sizeof(SequenceControlSet));
    PictureParentControlSet* ppcs = (PictureParentControlSet*)calloc(1, sizeof(PictureParentControlSet));
    PictureControlSet*       pcs  = (PictureControlSet*)calloc(1, sizeof(PictureControlSet));
    const int aw = (c->width + 7) & ~7, ah = (c->height + 7) & ~7;
    scs->seq_header.sb_size = c->sb_size == 128 ? BLOCK_128X128 : BLOCK_64X64;
    scs->sb_size = (uint16_t)c->sb_size;
    scs->is_16bit_pipeline = c->pixel_bytes == 2;
    scs->static_config.encoder_bit_depth = (EbBitDepth)c->bit_depth;
    scs->max_input_luma_width = (uint16_t)aw;
    scs->max_input_luma_height = (uint16_t)ah;
    scs->max_input_pad_right = (uint16_t)(aw - c->width);
    scs->max_input_pad_bottom = (uint16_t)(ah - c->height);
    ppcs->scs = scs;
    ppcs->aligned_width = (uint16_t)aw;
    ppcs->aligned_height = (uint16_t)ah;
    struct LoopFilter* lf = &ppcs->frm_hdr.loop_filter_params;
    lf->filter_level[0] = c->filter_level[0];
    lf->filter_level[1] = c->filter_level[1];
    lf->filter_level_u = c->filter_level_u;
    lf->filter_level_v = c->filter_level_v;
    lf->sharpness_level = c->sharpness;
    lf->mode_ref_delta_enabled = (uint8_t)c->mode_ref_delta_enabled;
    for (int i = 0; i < REF_FRAMES; i++) lf->ref_deltas[i] = (int8_t)c->ref_deltas[i];
    for (int i = 0; i < MAX_MODE_LF_DELTAS; i++) lf->mode_deltas[i] = (int8_t)c->mode_deltas[i];
    SegmentationParams* seg = &ppcs->frm_hdr.segmentation_params;
    seg->segmentation_enabled = (uint8_t)c->segmentation_enabled;
    for (int s = 0; s < MAX_SEGMENTS; s++)
        for (int k = 0; k < 4; k++) {
            seg->feature_enabled[s][SEG_LVL_ALT_LF_Y_V + k] = (int16_t)c->seg_lf_enabled[s][k];
            seg->feature_data[s][SEG_LVL_ALT_LF_Y_V + k] = (int16_t)c->seg_lf_data[s][k];
        }
    pcs->scs = scs;
    pcs->ppcs = ppcs;
    pcs->mi_stride = c->mi_stride;
    const size_t n = (size_t)c->mi_rows * c->mi_stride;
    d->mip = (ModeInfo*)calloc(n, sizeof(ModeInfo));
    pcs->mi_grid_base = (ModeInfo**)calloc(n, sizeof(ModeInfo*));
    for (size_t i = 0; i < n; i++) {
        BlockModeInfoEnc* b = &d->mip[i].mbmi.block_mi;
        b->bsize = (BlockSize)mi[i].bsize;
        b->tx_depth = mi[i].tx_depth;
        b->skip = mi[i].skip & 1;
        b->ref_frame[0] = (MvReferenceFrame)mi[i].ref_frame0;
        b->ref_frame[1] = NONE_FRAME;
        b->mode = (PredictionMode)mi[i].mode;
        b->segment_id = mi[i].segment_id;
        pcs->mi_grid_base[i] = &d->mip[i];
    }
    d->fb.buffer_y = (EbByte)y;
    d->fb.buffer_cb = (EbByte)cb;
    d->fb.buffer_cr = (EbByte)cr;
    d->fb.stride_y = (uint16_t)stride_y;
    d->fb.stride_cb = d->fb.stride_cr = (uint16_t)stride_c;
    d->fb.bit_depth = (EbBitDepth)c->bit_depth;
    d->fb.width = (uint16_t)aw;
    d->fb.height = (uint16_t)ah;
    d->scs = scs;
    d->ppcs = ppcs;
    d->pcs = pcs;
}

static void pic_free(DlfPic* d) {
    free(d->pcs->mi_grid_base);
    free(d->mip);
    free(d->pcs);
    free(d->ppcs);
    free(d->scs);
}

/* every vertical edge of the picture (dir 0) or every horizontal one (dir 1), superblock by superblock, with the reference's
 * own walks and the plane skips of svt_aom_loop_filter_sb (deblocking_filter.c:556-579) */
static void one_direction(DlfPic* d, int dir) {
    PictureControlSet* pcs = d->pcs;
    const FrameHeader* fh  = &d->ppcs->frm_hdr;
    const int sb = d->scs->sb_size, sbs = sb >> 2;
    struct MacroblockdPlane pd[3];
    memset(pd, 0, sizeof(pd));
    for (int p = 0; p < 3; p++) {
        pd[p].subsampling_x = pd[p].subsampling_y = p > 0;
        pd[p].plane_type = p ? PLANE_TYPE_UV : PLANE_TYPE_Y;
        pd[p].is_16bit = d->fb.bit_depth > 8 || d->scs->is_16bit_pipeline;
    }
    const int sb_cols = (d->ppcs->aligned_width + sb - 1) / sb, sb_rows = (d->ppcs->aligned_height + sb - 1) / sb;
    for (int p = 0; p < 3; p++) {
        if (p == 0 && !fh->loop_filter_params.filter_level[0] && !fh->loop_filter_params.filter_level[1]) break;
        if (p == 1 && !fh->loop_filter_params.filter_level_u) continue;
        if (p == 2 && !fh->loop_filter_params.filter_level_v) continue;
        for (int r = 0; r < sb_rows; r++)
            for (int c = 0; c < sb_cols; c++) {
                svt_av1_setup_dst_planes(pcs, pd, d->scs->seq_header.sb_size, &d->fb, r * sbs, c * sbs, p, p + 1);
                if (dir == 0) svt_av1_filter_block_plane_vert(pcs, p, &pd[p], r * sbs, c * sbs);
                else svt_av1_filter_block_plane_horz(pcs, p, &pd[p], r * sbs, c * sbs);
            }
    }
}

/* mode 0: svt_av1_loop_filter_frame (superblock order); 1: all vertical edges, then all horizontal edges; 2: derive the
 * tables only.  out_frame / out_mi (either may be NULL) receive what the glue makes of the picture afterwards. */
int ref_dlf_frame(const RefDlfCfg* cfg, const SvtB200DlfMi* mi, void* y, void* cb, void* cr, int stride_y, int stride_c, int mode,
                  SvtB200DlfFrame* out_frame, SvtB200DlfMi* out_mi) {
    DlfPic d;
    pic_build(&d, cfg, mi, y, cb, cr, stride_y, stride_c);
    svt_av1_loop_filter_init(d.pcs);
    if (mode == 0) {
        svt_av1_loop_filter_frame(&d.fb, d.pcs, 0, 3);
    } else {
        svt_av1_loop_filter_frame_init(&d.ppcs->frm_hdr, &d.ppcs->lf_info, 0, 3);
        if (mode == 1) {
            one_direction(&d, 0);
            one_direction(&d, 1);
        }
    }
    int rc = 0;
    if (out_frame || out_mi) {
        SvtB200DlfFrame f;
        rc = svt_b200_dlf_frame_from_pcs(d.pcs, &d.fb, &f, out_mi);
        if (out_frame) *out_frame = f;
    }
    pic_free(&d);
    return rc;
}

/* The tables dlf.cu uses (svt-av1-psy_b200/csrc/dlf_tables.h) against the reference's: returns the number of entries that
 * differ (each one is printed). */
int ref_dlf_table_mismatches(void) {
    static const uint8_t tx_depth[3][B200_DLF_N_BSIZE] = B200_DLF_TX_DEPTH_TO_TX_SIZE;
    static const uint8_t uv_tx[B200_DLF_N_BSIZE] = B200_DLF_UV_TX_SIZE_420;
    static const uint8_t horz[B200_DLF_N_TXSIZE] = B200_DLF_TXSIZE_HORZ_MAP;
    static const uint8_t vert[B200_DLF_N_TXSIZE] = B200_DLF_TXSIZE_VERT_MAP;
    static const uint8_t plane_bsize[B200_DLF_N_BSIZE] = B200_DLF_PLANE_BSIZE_420;
    static const uint8_t bw[B200_DLF_N_BSIZE] = B200_DLF_BLOCK_W;
    static const uint8_t bh[B200_DLF_N_BSIZE] = B200_DLF_BLOCK_H;
    static const uint8_t mode_lf[B200_DLF_N_MODES] = B200_DLF_MODE_LF_LUT;
    int bad = 0;
#define B200_CHECK(name, i, ours, theirs)                                                                  \
    if ((int)(ours) != (int)(theirs)) {                                                                    \
        fprintf(stderr, "[oracle] %s[%d]: dlf_tables.h %d, reference %d\n", name, i, (int)(ours), (int)(theirs)); \
        bad++;                                                                                             \
    }
    if (BlockSizeS_ALL != B200_DLF_N_BSIZE || TX_SIZES_ALL != B200_DLF_N_TXSIZE || sizeof(mode_lf_lut) / sizeof(mode_lf_lut[0]) != B200_DLF_N_MODES) {
        fprintf(stderr, "[oracle] table extents differ\n");
        return 1000;
    }
    for (int d = 0; d < 3; d++)
        for (int b = 0; b < B200_DLF_N_BSIZE; b++) B200_CHECK("tx_depth_to_tx_size", d * 100 + b, tx_depth[d][b], tx_depth_to_tx_size[d][b]);
    for (int b = 0; b < B200_DLF_N_BSIZE; b++) {
        B200_CHECK("uv_tx_size", b, uv_tx[b], av1_get_max_uv_txsize((BlockSize)b, 1, 1));
        B200_CHECK("plane_bsize", b, plane_bsize[b], get_plane_block_size((BlockSize)b, 1, 1));
        B200_CHECK("block_w", b, bw[b], block_size_wide[b]);
        B200_CHECK("block_h", b, bh[b], block_size_high[b]);
    }
    for (int t = 0; t < B200_DLF_N_TXSIZE; t++) {
        B200_CHECK("txsize_horz_map", t, horz[t], txsize_horz_map[t]);
        B200_CHECK("txsize_vert_map", t, vert[t], txsize_vert_map[t]);
    }
    for (int m = 0; m < B200_DLF_N_MODES; m++) B200_CHECK("mode_lf_lut", m, mode_lf[m], mode_lf_lut[m]);
#undef B200_CHECK
    return bad;
}
