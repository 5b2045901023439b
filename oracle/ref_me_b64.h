/* oracle/ref_me_b64.h -- TEST / BASELINE INFRASTRUCTURE: the entry points of oracle/ref_me_b64.c and the structs they take beyond
 * include/svt_b200.h's (ctypes mirrors in oracle/support.py) */
#ifndef REF_ME_B64_H
#define REF_ME_B64_H
#include <stdint.h>
#include "../include/svt_b200.h"

/* what the caller chooses (the encoder derives these in resource coordination / picture decision) */
typedef struct {
    int32_t enc_mode, qp, hierarchical_levels, temporal_layer_index, is_ref, sc_class1;
    int32_t n_ref[2];                 /* ref_list0_count_try, ref_list1_count_try (0 in list 1: P picture) */
    int32_t ref_poc_dist_sign[2][4];  /* picture_number(ref) - picture_number(cur), per list / index */
    int32_t enable_hme_flag, enable_hme_level0_flag, enable_hme_level1_flag, enable_hme_level2_flag;
    int32_t max_l0, max_l1;           /* MRP allocation counts (pd_process.c:3503-3519): layout of me_mv_array / me_candidate_array */
    int32_t only_l_bwd, safe_limit_nref, safe_limit_zz_th, similar_brightness_refs;
    int32_t gm_enabled, gm_use_distance_based_active_th;
    int32_t frame_rate_q16;           /* scs->frame_rate (Q16) */
    int32_t reserved[3];
} RefMeB64Cfg;

typedef struct {
    uint8_t*  total_me_candidate_index; /* [n_b64][n_pu] */
    uint8_t*  me_candidate_array;       /* [n_b64][n_pu * max_cand]  (MeCandidate bit-field bytes) */
    uint32_t* me_mv_array;              /* [n_b64][n_pu * max_refs] */
    uint32_t* distortion;               /* [n_b64][6]: rc_me, 64x64, 32x32, 16x16, 8x8, 8x8 cost variance */
    uint8_t*  flags;                    /* [n_b64][2]: stationary_block_present_sb, rc_me_allow_gm */
    /* per list / reference index */
    uint8_t*  do_ref;                   /* [n_b64][2][4] */
    int16_t*  hme_centre;               /* [n_b64][2][4][2] */
    uint32_t* zz_sad;                   /* [n_b64][2][4] */
    uint32_t* best_sad;                 /* [n_b64][2][4][85]  (written where do_ref) -- may be NULL */
    uint32_t* best_mv;                  /* [n_b64][2][4][85]  -- may be NULL */
} RefMeB64Out;

int ref_me_b64_num_pus(int enc_mode, int width, int height);
int ref_me_b64_sizes(const RefMeB64Cfg* cfg, int width, int height, int* n_pu, int* max_cand, int* max_refs);
int ref_me_b64_picture(const SvtB200MePicture* cur, const SvtB200MePicture* refs, const RefMeB64Cfg* cfg, SvtB200MeControls* ctrl,
                       RefMeB64Out* out);
#endif
