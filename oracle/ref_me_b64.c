/* oracle/ref_me_b64.c -- TEST / BASELINE INFRASTRUCTURE, compiled INTO oracle/_ref/libsvtav1_ref.so.
 *
 * Open-loop motion estimation of one picture through the reference's OWN driver: svt_aom_sig_deriv_me
 * (enc_mode_config.c:681) derives the MeContext controls of the preset, and svt_aom_motion_estimation_b64
 * (motion_estimation.c:3076) runs zz-SAD / pre-HME / HME L0-L2 / reference pruning / search-area adjustment /
 * full-pel search / candidate construction / distortion for every 64x64 block -- none of that control flow is
 * restated here.  What this file does is what the encoder's picture-level processes do around that call
 * (me_process.c:120-270): allocate a PictureParentControlSet / SequenceControlSet / MeContext, point them at the
 * caller's picture pyramids, and copy the results out.  The H100 T2 call svt_b200_me_b64_picture_dev is checked
 * against these outputs (tests/test_me_b64.py), and bench.py's reference arm times this function.
 * Nothing here is used by the product. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "definitions.h"
#include "pcs.h"
#include "sequence_control_set.h"
#include "me_context.h"
#include "motion_estimation.h"
#include "enc_mode_config.h"
#include "reference_object.h"

#include "ref_me_b64.h"

extern void svt_aom_get_max_allocated_me_refs(uint8_t ref_count_used_list0, uint8_t ref_count_used_list1, uint8_t* max_ref_to_alloc, uint8_t* max_cand_to_alloc); /* pcs.c:91 */
typedef void (*ParBody)(void* ctx, int i);
extern void ref_par_for(int n, int chunk, ParBody body, void* ctx); /* ref_driver.c's pool */

static void fill_desc(EbPictureBufferDesc* d, const RefMePicture* p, int level) {
    memset(d, 0, sizeof(*d));
    d->buffer_y = (uint8_t*)p->plane[level];
    d->stride_y = (uint16_t)p->stride[level];
    d->org_x    = (uint16_t)p->org_x[level];
    d->org_y    = (uint16_t)p->org_y[level];
    d->width    = (uint16_t)p->width[level];
    d->height   = (uint16_t)p->height[level];
    d->max_width = d->width; d->max_height = d->height;
    d->bit_depth = EB_EIGHT_BIT;
}

typedef struct {
    PictureParentControlSet* pcs;
    SequenceControlSet*      scs;
    EbPictureBufferDesc      cur[3];
    EbPictureBufferDesc      ref[2][4][3];
    const RefMeB64Cfg*       cfg;
    RefMeB64Out*             out;
    int                      b64_w, b64_h, n_pu;
} MeB64Job;

static void setup_me_ctx(MeB64Job* j, MeContext* me) {
    svt_aom_me_context_ctor(me);
    svt_aom_sig_deriv_me(j->scs, j->pcs, me);
    me->me_type               = ME_OPEN_LOOP;
    me->num_of_list_to_search = j->cfg->n_ref[1] > 0 ? 2 : 1;
    me->num_of_ref_pic_to_search[0] = (uint8_t)j->cfg->n_ref[0];
    me->num_of_ref_pic_to_search[1] = (uint8_t)j->cfg->n_ref[1];
    me->temporal_layer_index  = (uint8_t)j->cfg->temporal_layer_index;
    me->is_ref                = j->cfg->is_ref != 0;
    for (int l = 0; l < 2; l++)
        for (int r = 0; r < j->cfg->n_ref[l]; r++) {
            me->me_ds_ref_array[l][r].picture_ptr           = &j->ref[l][r][2];
            me->me_ds_ref_array[l][r].quarter_picture_ptr   = &j->ref[l][r][1];
            me->me_ds_ref_array[l][r].sixteenth_picture_ptr = &j->ref[l][r][0];
            me->me_ds_ref_array[l][r].picture_number        = (uint64_t)((int64_t)j->pcs->picture_number + j->cfg->ref_poc_dist_sign[l][r]);
        }
}

/* one row of 64x64 blocks per work item, its own MeContext (the encoder's ME segments do the same) */
static void me_b64_row(void* vctx, int by) {
    MeB64Job*  j = (MeB64Job*)vctx;
    MeContext* me = (MeContext*)calloc(1, sizeof(MeContext));
    setup_me_ctx(j, me);
    PictureParentControlSet* pcs = j->pcs;
    const int max_cand = pcs->pa_me_data->max_cand, max_refs = pcs->pa_me_data->max_refs;
    for (int bx = 0; bx < j->b64_w; bx++) {
        const uint32_t b = (uint32_t)(by * j->b64_w + bx), ox = (uint32_t)bx * 64, oy = (uint32_t)by * 64;
        /* me_process.c:176-214 */
        me->b64_src_ptr    = &j->cur[2].buffer_y[(j->cur[2].org_y + oy) * j->cur[2].stride_y + j->cur[2].org_x + ox];
        me->b64_src_stride = j->cur[2].stride_y;
        me->quarter_b64_buffer          = &j->cur[1].buffer_y[(j->cur[1].org_y + (oy >> 1)) * j->cur[1].stride_y + j->cur[1].org_x + (ox >> 1)];
        me->quarter_b64_buffer_stride   = j->cur[1].stride_y;
        me->sixteenth_b64_buffer        = &j->cur[0].buffer_y[(j->cur[0].org_y + (oy >> 2)) * j->cur[0].stride_y + j->cur[0].org_x + (ox >> 2)];
        me->sixteenth_b64_buffer_stride = j->cur[0].stride_y;
        svt_aom_motion_estimation_b64(pcs, b, ox, oy, me, &j->cur[2]);
        RefMeB64Out* o = j->out;
        const MeSbResults* res = pcs->pa_me_data->me_results[b];
        memcpy(o->total_me_candidate_index + (size_t)b * j->n_pu, res->total_me_candidate_index, (size_t)j->n_pu);
        memcpy(o->me_candidate_array + (size_t)b * j->n_pu * max_cand, res->me_candidate_array, (size_t)j->n_pu * max_cand);
        memcpy(o->me_mv_array + (size_t)b * j->n_pu * max_refs, res->me_mv_array, (size_t)j->n_pu * max_refs * 4);
        uint32_t* d = o->distortion + (size_t)b * 6;
        d[0] = pcs->rc_me_distortion[b]; d[1] = pcs->me_64x64_distortion[b]; d[2] = pcs->me_32x32_distortion[b];
        d[3] = pcs->me_16x16_distortion[b]; d[4] = pcs->me_8x8_distortion[b]; d[5] = pcs->me_8x8_cost_variance[b];
        o->flags[2 * b] = pcs->stationary_block_present_sb[b]; o->flags[2 * b + 1] = pcs->rc_me_allow_gm[b];
        for (int l = 0; l < 2; l++)
            for (int r = 0; r < 4; r++) {
                const size_t k = ((size_t)b * 2 + l) * 4 + r;
                const int live = l < me->num_of_list_to_search && r < me->num_of_ref_pic_to_search[l];
                o->do_ref[k] = live ? me->search_results[l][r].do_ref : 0;
                o->hme_centre[2 * k] = live ? me->search_results[l][r].hme_sc_x : 0;
                o->hme_centre[2 * k + 1] = live ? me->search_results[l][r].hme_sc_y : 0;
                o->zz_sad[k] = live ? me->zz_sad[l][r] : 0;
                if (o->best_sad && live && me->search_results[l][r].do_ref) {
                    memcpy(o->best_sad + k * 85, me->p_sb_best_sad[l][r], 85 * 4);
                    memcpy(o->best_mv + k * 85, me->p_sb_best_mv[l][r], 85 * 4);
                }
            }
    }
    free(me->p_eight_pos_sad16x16);
    free(me);
}

/* the flattened controls come from the integration glue a maintainer would ship (integration/svt_b200_me_glue.c): the parity
 * tests thereby check that mapping too.  RefMeControls and SvtB200MeControls are the same layout (static assert below). */
#include "../include/svt_b200.h"
#include "../integration/svt_b200_me_glue.h"
_Static_assert(sizeof(RefMeControls) == sizeof(SvtB200MeControls), "control struct mirrors differ");
static void flatten_controls(const MeB64Job* j, const MeContext* me, RefMeControls* c) {
    svt_b200_me_controls_from_context(j->pcs, me, (SvtB200MeControls*)c);
}

/* number of square PUs that carry candidates (me_sb_results_ctor, pcs.c:107-112) */
int ref_me_b64_num_pus(int enc_mode, int width, int height) {
    EbInputResolution res;
    svt_aom_derive_input_resolution(&res, (uint32_t)width * height);
    return svt_aom_get_enable_me_16x16((EncMode)enc_mode) ? (svt_aom_get_enable_me_8x8((EncMode)enc_mode, false, res) ? SQUARE_PU_COUNT : MAX_SB64_PU_COUNT_NO_8X8)
                                                          : MAX_SB64_PU_COUNT_WO_16X16;
}

/* array extents of the outputs for a configuration (without running anything) */
int ref_me_b64_sizes(const RefMeB64Cfg* cfg, int width, int height, int* n_pu, int* max_cand, int* max_refs) {
    uint8_t mr, mc;
    svt_aom_get_max_allocated_me_refs((uint8_t)cfg->max_l0, (uint8_t)cfg->max_l1, &mr, &mc);
    *n_pu = ref_me_b64_num_pus(cfg->enc_mode, width, height);
    *max_cand = mc;
    *max_refs = mr;
    return 0;
}

/* refs: [n_ref[0] + n_ref[1]] descriptors, list 0 first.  Returns 0; fills *ctrl with the derived controls; when `out` is NULL only
 * derives the controls. */
int ref_me_b64_picture(const RefMePicture* cur, const RefMePicture* refs, const RefMeB64Cfg* cfg, RefMeControls* ctrl, RefMeB64Out* out) {
    MeB64Job j;
    memset(&j, 0, sizeof(j));
    const int W = cur->width[2], H = cur->height[2];
    j.cfg = cfg; j.out = out;
    j.b64_w = (W + 63) >> 6; j.b64_h = (H + 63) >> 6;
    const int nb = j.b64_w * j.b64_h;
    SequenceControlSet*      scs = (SequenceControlSet*)calloc(1, sizeof(SequenceControlSet));
    PictureParentControlSet* pcs = (PictureParentControlSet*)calloc(1, sizeof(PictureParentControlSet));
    j.scs = scs; j.pcs = pcs;
    svt_aom_derive_input_resolution(&scs->input_resolution, (uint32_t)W * H);
    scs->static_config.pred_structure = SVT_AV1_PRED_RANDOM_ACCESS;
    scs->static_config.qp = (uint32_t)cfg->qp;
    scs->frame_rate = (uint32_t)cfg->frame_rate_q16;
    scs->b64_size = 64;
    scs->mrp_ctrls.only_l_bwd = (uint8_t)cfg->only_l_bwd;
    scs->mrp_ctrls.safe_limit_nref = (uint8_t)cfg->safe_limit_nref;
    scs->mrp_ctrls.safe_limit_zz_th = (uint32_t)cfg->safe_limit_zz_th;
    pcs->scs = scs;
    pcs->enc_mode = (EncMode)cfg->enc_mode;
    pcs->sc_class1 = (uint8_t)cfg->sc_class1;
    pcs->hierarchical_levels = (uint8_t)cfg->hierarchical_levels;
    pcs->temporal_layer_index = (uint8_t)cfg->temporal_layer_index;
    pcs->is_ref = cfg->is_ref != 0;
    pcs->picture_number = 64; /* any value: only differences to the reference pictures' numbers are used */
    pcs->aligned_width = (uint16_t)((W + 7) & ~7); pcs->aligned_height = (uint16_t)((H + 7) & ~7);
    pcs->enable_hme_flag = cfg->enable_hme_flag != 0; pcs->enable_hme_level0_flag = cfg->enable_hme_level0_flag != 0;
    pcs->enable_hme_level1_flag = cfg->enable_hme_level1_flag != 0; pcs->enable_hme_level2_flag = cfg->enable_hme_level2_flag != 0;
    pcs->enable_me_16x16 = svt_aom_get_enable_me_16x16(pcs->enc_mode);
    pcs->enable_me_8x8 = pcs->enable_me_16x16 ? svt_aom_get_enable_me_8x8(pcs->enc_mode, false, scs->input_resolution) : 0; /* pcs.c:1389-1394 */
    pcs->max_number_of_pus_per_sb = SQUARE_PU_COUNT; /* resource_coordination_process.c:425 */
    pcs->use_best_me_unipred_cand_only = cfg->enc_mode <= ENC_M3 ? 0 : 1; /* enc_mode_config.c:1841-1844 */
    pcs->similar_brightness_refs = cfg->similar_brightness_refs != 0;
    pcs->gm_ctrls.enabled = (uint8_t)cfg->gm_enabled;
    pcs->gm_ctrls.use_distance_based_active_th = (uint8_t)cfg->gm_use_distance_based_active_th;
    j.n_pu = ref_me_b64_num_pus(cfg->enc_mode, W, H);
    /* 64x64 block geometry (only width / height are read by compute_distortion) */
    pcs->b64_geom = (B64Geom*)calloc((size_t)nb, sizeof(B64Geom));
    for (int b = 0; b < nb; b++) {
        const int ox = (b % j.b64_w) * 64, oy = (b / j.b64_w) * 64;
        pcs->b64_geom[b].org_x = (uint16_t)ox; pcs->b64_geom[b].org_y = (uint16_t)oy;
        pcs->b64_geom[b].width = (uint8_t)(W - ox < 64 ? W - ox : 64); pcs->b64_geom[b].height = (uint8_t)(H - oy < 64 ? H - oy : 64);
    }
    pcs->rc_me_distortion = (uint32_t*)calloc((size_t)nb, 4); pcs->me_64x64_distortion = (uint32_t*)calloc((size_t)nb, 4);
    pcs->me_32x32_distortion = (uint32_t*)calloc((size_t)nb, 4); pcs->me_16x16_distortion = (uint32_t*)calloc((size_t)nb, 4);
    pcs->me_8x8_distortion = (uint32_t*)calloc((size_t)nb, 4); pcs->me_8x8_cost_variance = (uint32_t*)calloc((size_t)nb, 4);
    pcs->stationary_block_present_sb = (uint8_t*)calloc((size_t)nb, 1); pcs->rc_me_allow_gm = (uint8_t*)calloc((size_t)nb, 1);
    /* ME results storage, sized as pd_process.c:3503-3519 / pcs.c:91-117 */
    MotionEstimationData* pa = (MotionEstimationData*)calloc(1, sizeof(MotionEstimationData));
    uint8_t max_refs, max_cand;
    svt_aom_get_max_allocated_me_refs((uint8_t)cfg->max_l0, (uint8_t)cfg->max_l1, &max_refs, &max_cand);
    pa->max_cand = max_cand; pa->max_refs = max_refs; pa->max_l0 = (uint8_t)cfg->max_l0;
    pa->me_results = (MeSbResults**)calloc((size_t)nb, sizeof(MeSbResults*));
    for (int b = 0; b < nb; b++) {
        MeSbResults* r = (MeSbResults*)calloc(1, sizeof(MeSbResults));
        r->me_mv_array = (MvCandidate*)calloc((size_t)j.n_pu * max_refs, sizeof(MvCandidate));
        r->me_candidate_array = (MeCandidate*)calloc((size_t)j.n_pu * max_cand, sizeof(MeCandidate));
        r->total_me_candidate_index = (uint8_t*)calloc((size_t)j.n_pu, 1);
        pa->me_results[b] = r;
    }
    pcs->pa_me_data = pa;
    for (int lv = 0; lv < 3; lv++) fill_desc(&j.cur[lv], cur, lv);
    int k = 0;
    for (int l = 0; l < 2; l++)
        for (int r = 0; r < cfg->n_ref[l]; r++, k++)
            for (int lv = 0; lv < 3; lv++) fill_desc(&j.ref[l][r][lv], &refs[k], lv);
    {
        MeContext* me = (MeContext*)calloc(1, sizeof(MeContext));
        setup_me_ctx(&j, me);
        flatten_controls(&j, me, ctrl);
        free(me->p_eight_pos_sad16x16);
        free(me);
    }
    if (out) {
        ref_par_for(j.b64_h, 1, me_b64_row, &j);
        /* round trip through the integration glue: storing the copied-out results back must reproduce the reference's own state */
        uint8_t* t0 = (uint8_t*)malloc((size_t)nb * j.n_pu);
        for (int b = 0; b < nb; b++) memcpy(t0 + (size_t)b * j.n_pu, pa->me_results[b]->total_me_candidate_index, (size_t)j.n_pu);
        svt_b200_me_store_results(pcs, nb, j.n_pu, out->total_me_candidate_index, out->me_candidate_array, out->me_mv_array, out->distortion,
                                  out->flags);
        for (int b = 0; b < nb; b++)
            if (memcmp(t0 + (size_t)b * j.n_pu, pa->me_results[b]->total_me_candidate_index, (size_t)j.n_pu) ||
                pcs->rc_me_distortion[b] != out->distortion[(size_t)b * 6]) {
                fprintf(stderr, "[oracle] svt_b200_me_store_results round trip differs at block %d\n", b);
                abort();
            }
        free(t0);
    }
    for (int b = 0; b < nb; b++) {
        free(pa->me_results[b]->me_mv_array); free(pa->me_results[b]->me_candidate_array); free(pa->me_results[b]->total_me_candidate_index);
        free(pa->me_results[b]);
    }
    free(pa->me_results); free(pa);
    free(pcs->b64_geom); free(pcs->rc_me_distortion); free(pcs->me_64x64_distortion); free(pcs->me_32x32_distortion); free(pcs->me_16x16_distortion);
    free(pcs->me_8x8_distortion); free(pcs->me_8x8_cost_variance); free(pcs->stationary_block_present_sb); free(pcs->rc_me_allow_gm);
    free(pcs); free(scs);
    return 0;
}
