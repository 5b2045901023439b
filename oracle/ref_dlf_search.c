/* oracle/ref_dlf_search.c -- TEST / BASELINE INFRASTRUCTURE, compiled into oracle/_ref/libsvtav1_dlf_search.so
 * (oracle/dlf_search.mk), which takes every reference symbol from oracle/_ref/libsvtav1_ref.so.
 *
 * The deblocking filter-level search through the reference's own functions, on the picture ref_dlf.c builds from flat
 * mode-info records and a RefDlfCfg (ref_dlf.c is included, so both checkers construct the picture the same way):
 *   - ref_dlf_level_sse runs the reference's steps of try_filter_frame (deblocking_filter.c:840) for a list of levels,
 *     each on the unfiltered picture, and hands the same search to the integration glue (svt_b200_dlf_level_sse_from_pcs);
 *   - ref_dlf_pick runs its whole search, svt_av1_pick_filter_level (deblocking_filter.c:1139).
 * Nothing here is used by the product. */
#include "ref_dlf.c"

/* ---- the filter-level search (svt_av1_pick_filter_level, deblocking_filter.c:1139-1296) ------------------------------
 * Inputs beyond RefDlfCfg: the source planes, and for ref_dlf_level_sse the planes and levels to try, for ref_dlf_pick
 * the controls svt_av1_pick_filter_level reads.  The hill-climb starts from cfg's filter levels. */
typedef struct RefDlfSearch {
    const void* src[3];          /* source planes at pixel (0, 0), the recon's pixel type */
    int32_t     src_stride[3];
    int32_t     plane_mask;      /* ref_dlf_level_sse: bit p = try plane p */
    int32_t     n_levels;
    int32_t     sharpness;       /* ref_dlf_pick: static_config.sharpness, tune, frame type, tx_mode, early exit */
    int32_t     tune;
    int32_t     frame_type;
    int32_t     tx_mode;
    int32_t     early_exit_convergence;
    uint8_t     level[64];
    int32_t     picked[4];       /* ref_dlf_pick's result: filter_level[0], filter_level[1], filter_level_u, filter_level_v */
    int64_t     zero_filt_sse;   /* pcs->zero_filt_sse / best_filt_sse after the search (-1: not set) */
    int64_t     best_filt_sse;
} RefDlfSearch;

/* What the filter may read of a plane (nothing left of or above (0, 0), at most 7 past the unpadded size): rows
 * [0, ah + 8) x columns [0, aw + 8), aw x ah = the aligned size.  The searches run on private copies of that region, so the
 * caller's planes are never written. */
typedef struct PlaneCopies {
    uint8_t* buf[3];
    int      w[3], h[3];  /* in pixels; the copy's stride is w */
    const uint8_t* from[3];
    int      from_stride[3];
    int      pb;
} PlaneCopies;

static void copies_make(PlaneCopies* pc, const RefDlfCfg* c, void* y, void* cb, void* cr, int stride_y, int stride_c) {
    const int aw = (c->width + 7) & ~7, ah = (c->height + 7) & ~7;
    void* from[3] = {y, cb, cr};
    pc->pb = c->pixel_bytes;
    for (int p = 0; p < 3; p++) {
        pc->w[p] = (p ? aw >> 1 : aw) + 8;
        pc->h[p] = (p ? ah >> 1 : ah) + 8;
        pc->from[p] = (const uint8_t*)from[p];
        pc->from_stride[p] = p ? stride_c : stride_y;
        pc->buf[p] = (uint8_t*)malloc((size_t)pc->w[p] * pc->h[p] * pc->pb);
    }
}

static void copies_refresh(PlaneCopies* pc, int p) {
    for (int r = 0; r < pc->h[p]; r++)
        memcpy(pc->buf[p] + (size_t)r * pc->w[p] * pc->pb, pc->from[p] + (size_t)r * pc->from_stride[p] * pc->pb, (size_t)pc->w[p] * pc->pb);
}

static void copies_free(PlaneCopies* pc) {
    for (int p = 0; p < 3; p++) free(pc->buf[p]);
}

/* the picture on the copies, with the source picture the SSE compares with (picture_sse_calculations reads enhanced_pic
 * in the 8-bit pipeline, input_frame16bit in the 16-bit one) */
static void search_pic_build(DlfPic* d, PlaneCopies* pc, EbPictureBufferDesc* sd, const RefDlfCfg* cfg, const SvtB200DlfMi* mi, void* y,
                             void* cb, void* cr, int stride_y, int stride_c, const RefDlfSearch* s) {
    copies_make(pc, cfg, y, cb, cr, stride_y, stride_c);
    for (int p = 0; p < 3; p++) copies_refresh(pc, p);
    pic_build(d, cfg, mi, pc->buf[0], pc->buf[1], pc->buf[2], pc->w[0], pc->w[1]);
    d->scs->subsampling_x = d->scs->subsampling_y = 1; /* the chroma SSE region (deblocking_filter.c:764-765, :813-814) */
    memset(sd, 0, sizeof(*sd));
    sd->buffer_y = (EbByte)s->src[0];
    sd->buffer_cb = (EbByte)s->src[1];
    sd->buffer_cr = (EbByte)s->src[2];
    sd->stride_y = (uint16_t)s->src_stride[0];
    sd->stride_cb = (uint16_t)s->src_stride[1];
    sd->stride_cr = (uint16_t)s->src_stride[2];
    sd->bit_depth = d->fb.bit_depth;
    sd->width = d->fb.width;
    sd->height = d->fb.height;
    d->ppcs->enhanced_pic = sd;
    d->pcs->input_frame16bit = sd;
}

/* sse[p * n_levels + i] = try_filter_frame (deblocking_filter.c:840) at s->level[i] for each plane p of s->plane_mask, each
 * on the unfiltered picture, through the reference's own steps: the plane's levels in the frame header,
 * svt_av1_loop_filter_frame(recon, pcs, p, p + 1), picture_sse_calculations(pcs, recon, p).  cfg->sharpness is the
 * sharpness the tries run at.  out_frame / out_s / out_lvl (all or none NULL) receive what the glue
 * (svt_b200_dlf_level_sse_from_pcs) makes of the same search; their plane pointers are the private copies'. */
int ref_dlf_level_sse(const RefDlfCfg* cfg, const SvtB200DlfMi* mi, void* y, void* cb, void* cr, int stride_y, int stride_c,
                      const RefDlfSearch* s, int64_t* sse, SvtB200DlfFrame* out_frame, SvtB200DlfLevelSse* out_s, uint8_t* out_lvl) {
    DlfPic              d;
    PlaneCopies         pc;
    EbPictureBufferDesc sd;
    search_pic_build(&d, &pc, &sd, cfg, mi, y, cb, cr, stride_y, stride_c, s);
    svt_av1_loop_filter_init(d.pcs);
    int rc = 0;
    if (out_frame) rc = svt_b200_dlf_level_sse_from_pcs(d.pcs, &d.fb, s->plane_mask, s->n_levels, s->level, out_frame, out_s, out_lvl);
    struct LoopFilter* lf = &d.ppcs->frm_hdr.loop_filter_params;
    for (int p = 0; p < 3 && !rc; p++) {
        if (!((s->plane_mask >> p) & 1)) continue;
        for (int i = 0; i < s->n_levels; i++) {
            copies_refresh(&pc, p);
            if (p == 0) lf->filter_level[0] = lf->filter_level[1] = s->level[i];
            else if (p == 1) lf->filter_level_u = s->level[i];
            else lf->filter_level_v = s->level[i];
            svt_av1_loop_filter_frame(&d.fb, d.pcs, p, p + 1);
            sse[p * s->n_levels + i] = (int64_t)picture_sse_calculations(d.pcs, &d.fb, p);
        }
    }
    pic_free(&d);
    copies_free(&pc);
    return rc;
}

/* The reference's own svt_av1_pick_filter_level(..., LPF_PICK_FROM_FULL_IMAGE) as dlf_process.c:109-110 runs it (after
 * svt_av1_loop_filter_init), on an intra picture without references (tot_ref_frame_types = 0, I_SLICE: no level
 * averaging, no ME-based skip, both searches run) and the recon as a non-reference picture's enc_dec recon.  Fills
 * s->picked, s->zero_filt_sse and s->best_filt_sse. */
int ref_dlf_pick(const RefDlfCfg* cfg, const SvtB200DlfMi* mi, void* y, void* cb, void* cr, int stride_y, int stride_c, RefDlfSearch* s) {
    DlfPic              d;
    PlaneCopies         pc;
    EbPictureBufferDesc sd;
    EncDecSet           eds;
    search_pic_build(&d, &pc, &sd, cfg, mi, y, cb, cr, stride_y, stride_c, s);
    SequenceControlSet*      scs  = d.scs;
    PictureParentControlSet* ppcs = d.ppcs;
    PictureControlSet*       pcs  = d.pcs;
    scs->super_block_size = (uint32_t)cfg->sb_size;
    scs->static_config.encoder_color_format = EB_YUV420;
    scs->static_config.sharpness = (int8_t)s->sharpness;
    scs->static_config.tune = (uint8_t)s->tune;
    ppcs->frm_hdr.frame_type = (FrameType)s->frame_type;
    ppcs->frm_hdr.tx_mode = (TxMode)s->tx_mode;
    ppcs->dlf_ctrls.early_exit_convergence = (uint8_t)s->early_exit_convergence;
    ppcs->tot_ref_frame_types = 0;
    pcs->slice_type = I_SLICE;
    memset(&eds, 0, sizeof(eds));
    eds.recon_pic = eds.recon_pic_16bit = &d.fb;
    ppcs->enc_dec_ptr = &eds;
    ppcs->is_ref = false;
    ppcs->render_width = d.fb.width; /* no rescale in svt_aom_get_recon_pic */
    ppcs->render_height = d.fb.height;
    pcs->zero_filt_sse = pcs->best_filt_sse = -1;
    svt_av1_loop_filter_init(pcs);
    const int rc = svt_av1_pick_filter_level(&sd, pcs, LPF_PICK_FROM_FULL_IMAGE) == EB_ErrorNone ? 0 : -1;
    const struct LoopFilter* lf = &ppcs->frm_hdr.loop_filter_params;
    s->picked[0] = lf->filter_level[0];
    s->picked[1] = lf->filter_level[1];
    s->picked[2] = lf->filter_level_u;
    s->picked[3] = lf->filter_level_v;
    s->zero_filt_sse = pcs->zero_filt_sse;
    s->best_filt_sse = pcs->best_filt_sse;
    pic_free(&d);
    copies_free(&pc);
    return rc;
}
