/* svt_b200_dlf_glue.c -- see svt_b200_dlf_glue.h.  Compiled against the reference headers with -Wall -Werror. */
#include <string.h>
#include "definitions.h"
#include "pcs.h"
#include "sequence_control_set.h"
#include "coding_unit.h"
#include "svt_b200.h"
#include "svt_b200_dlf_glue.h"

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
    for (int l = 0; l <= MAX_LOOP_FILTER; l++) {
        frame->lfthr[l][0] = ppcs->lf_info.lfthr[l].mblim[0];
        frame->lfthr[l][1] = ppcs->lf_info.lfthr[l].lim[0];
        frame->lfthr[l][2] = ppcs->lf_info.lfthr[l].hev_thr[0];
    }
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
