// me_b64.cu -- T2, the COMPLETE open-loop ME driver of a picture (sm_90a): everything svt_aom_motion_estimation_b64 does for
// a 64x64 block, for all blocks and all reference pictures, in three launches.
//
// Reference behaviour restated (Source/Lib/Codec/motion_estimation.c):
//   svt_aom_motion_estimation_b64   :3076     order of the stages below
//   init_me_hme_data                :3012     per-block reset of the search state
//   init_zz_sad / get_zz_sad        :2391/:1670  zero-MV SAD per reference, zz-based reference pruning, "safe limit" of references
//   prehme_b64 / prehme_core        :1722/:1568  two elongated 1/16-resolution searches per reference, early exits, pruning
//   hme_level0/1/2_b64              :1906-2180   early exits, distance-scaled level-0 area, pre-HME replaces the worst quadrant
//   set_final_seach_centre_sb       :2182     (incl. the values that carry over from one reference to the next)
//   hme_prune_ref_and_adjust_sr     :2477
//   integer_search_b64              :1249     area = f(distance, HME MV, divisor, zz SAD, 8x8-SAD variance probe), clipping
//   me_prune_ref                    :1522
//   construct_me_candidate_array{,_mrp_off,_single_ref}  :2698/:2532/:2646
//   compute_distortion              :2964
//   perform_gm_detection            :2842
//
// Launches:  (A) me_b64_hme_kernel<PAR>  one CTA per 64x64 block, 4 * PAR warps.  The references are walked in the reference's
//                order, PAR at a time (1, or 2 from six references up: chosen on the previous target GPU, not re-measured on H100); inside the HME stages a warp is one
//                (reference, search region) pair, in the per-reference stages (zz SAD, pre-HME, window derivation) one reference.
//                Decisions that couple references (pruning, carried-over centres) are taken by one thread between barriers.
//                Writes one full-pel item per (reference, block) + the 85 SADs of the variance probe ("seed").
//            (B) fullpel_search_kernel<TMA> (me_pyramid.cu) over the items, best arrays seeded with the probe.
//            (C) me_b64_finish_kernel  one CTA per block: ME-based pruning, candidates, distortions, GM flags.
#include <map>

#include "common.cuh"
#include "sad_small.cuh"
#include "me_hme.cuh"
#include "../../include/svt_b200.h"

namespace b200 {
bool launch_fullpel_tma(const SvtB200MePicture* cur, const SvtB200MePicture* refs, int n_refs, int n_b64, const SvtB200FullpelItem* d_items,
                        int n_items, uint32_t* d_best_sad, uint32_t* d_best_mv, cudaStream_t st, const uint32_t* d_seed_sad);  // me_pyramid.cu

namespace {

constexpr int      kDepth   = 4;  // REF_LIST_MAX_DEPTH
constexpr uint32_t kMaxU32  = 0xffffffffu;
constexpr uint32_t kMaxSad  = 128u * 128u * 255u;  // MAX_SAD_VALUE

struct MeB64Table {  // by value with the launch
    SvtB200MePicture  cur;
    SvtB200MePicture  ref[2][kDepth];
    SvtB200MeControls c;
};

struct B64State {
    uint32_t zz[2][kDepth];
    uint8_t  do_ref[2][kDepth];
    int16_t  ph_x[2][kDepth][2], ph_y[2][kDepth][2];
    uint64_t ph_sad[2][kDepth][2];
    uint8_t  ph_valid[2][kDepth][2], ph_done[2][kDepth][2];
    int16_t  lx[3][2][kDepth][4], ly[3][2][kDepth][4];  // [level][list][ref][region = sr_w + 2 * sr_h]
    uint64_t lsad[3][2][kDepth][4];
    int16_t  sc_x[2][kDepth], sc_y[2][kDepth];
    uint64_t hme_sad[2][kDepth];
    uint32_t divisor[2][kDepth];
};

__device__ __forceinline__ int scaled_distance(int dist) { return (dist * 5) / 8 + ((dist % 8) == 0 ? 0 : 1); }  // svt_aom_get_scaled_picture_distance
__device__ __forceinline__ bool searched(const SvtB200MeControls& c, int l) { return c.temporal_layer_index > 0 || l == 0; }

// SAD of a bw x bh block on every other row (rows 0, 2, ...: bh >> 1 of them), lane = row; all lanes return the sum.
// svt_nxm_sad_kernel(src, stride << 1, ref, stride << 1, bh >> 1, bw) of get_zz_sad / check_00_center.
__device__ __forceinline__ uint32_t warp_sad_every_other_row(const uint8_t* src, int ss, const uint8_t* ref, int rs, int bw, int bh, int lane) {
    uint32_t acc = 0;
    if (lane < (bh >> 1)) {
        const int      yy = lane * 2, nw = (bw + 3) >> 2, tail = bw & 3;
        const uint32_t tailmask = tail ? ((1u << (tail * 8)) - 1u) : 0xffffffffu;
        const ByteRun  S(src + (size_t)yy * ss, bw), R(ref + (ptrdiff_t)yy * rs, bw);
        uint32_t       slo = S.raw(0), rlo = R.raw(0);
#pragma unroll 4
        for (int j = 0; j < nw; j++) {
            const uint32_t shi = S.raw(j + 1), rhi = R.raw(j + 1);
            const uint32_t m = j == nw - 1 ? tailmask : 0xffffffffu;
            acc = __vsadu4(__funnelshift_r(slo, shi, S.shift) & m, __funnelshift_r(rlo, rhi, R.shift) & m) + acc;
            slo = shi;
            rlo = rhi;
        }
    }
    return __reduce_add_sync(0xffffffffu, acc);
}

// the 85 SADs of ONE search position (src block vs ref block, both 64x64), written in the ME's PU order
// (64x64, 4 x 32x32, 16 x 16x16 and 64 x 8x8 in z order) -- what open_loop_me_fullpel_search_sblock(..., 1, 1) leaves in
// p_sb_best_sad.  lane handles the 8x8 blocks 2*lane and 2*lane+1 (z order), sub = rows 0,2,4,6 only, doubled.
// Returns, in every lane, the variance of the 64 8x8 SADs about their mean (sum / 64 of the squared deviations, 32-bit
// arithmetic as in the reference).  It is computed from registers: out85 is only for the search kernel that runs next, and
// a lane must not read another lane's stores there (the compiler may move such a load above the warp barrier).
__device__ __forceinline__ uint32_t warp_probe_sads(const uint8_t* src, int ss, const uint8_t* ref, int rs, bool sub, int lane, uint32_t* out85) {
    uint32_t s8[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const int z8 = 2 * lane + k, z16 = z8 >> 2, q = z16 >> 2, i = z16 & 3;
        const int y16 = 2 * (q >> 1) + (i >> 1), x16 = 2 * (q & 1) + (i & 1);
        const int by = 2 * y16 + ((z8 >> 1) & 1), bx = 2 * x16 + (z8 & 1);
        uint32_t  acc = 0;
        for (int r = 0; r < 8; r += (sub ? 2 : 1)) {
            const ByteRun S(src + (size_t)(8 * by + r) * ss + 8 * bx, 8), R(ref + (ptrdiff_t)(8 * by + r) * rs + 8 * bx, 8);
            const uint32_t s0 = S.raw(0), s1 = S.raw(1), s2 = S.raw(2), r0 = R.raw(0), r1 = R.raw(1), r2 = R.raw(2);
            acc = __vsadu4(__funnelshift_r(s0, s1, S.shift), __funnelshift_r(r0, r1, R.shift)) + acc;
            acc = __vsadu4(__funnelshift_r(s1, s2, S.shift), __funnelshift_r(r1, r2, R.shift)) + acc;
        }
        s8[k] = sub ? acc << 1 : acc;
        out85[21 + z8] = s8[k];
    }
    uint32_t v16 = s8[0] + s8[1];
    v16 += __shfl_xor_sync(0xffffffffu, v16, 1);  // lanes 2j, 2j+1 hold the four 8x8 of 16x16 z-index j
    uint32_t v32 = v16 + __shfl_xor_sync(0xffffffffu, v16, 2);
    v32 += __shfl_xor_sync(0xffffffffu, v32, 4);
    uint32_t v64 = v32 + __shfl_xor_sync(0xffffffffu, v32, 8);
    v64 += __shfl_xor_sync(0xffffffffu, v64, 16);
    if ((lane & 1) == 0) out85[5 + (lane >> 1)] = v16;
    if ((lane & 7) == 0) out85[1 + (lane >> 3)] = v32;
    if (lane == 0) out85[0] = v64;
    const uint32_t mean = v64 / 64u;
    const int32_t  d0 = (int32_t)s8[0] - (int32_t)mean, d1 = (int32_t)s8[1] - (int32_t)mean;
    return __reduce_add_sync(0xffffffffu, (uint32_t)(d0 * d0) + (uint32_t)(d1 * d1)) / 64u;
}

// integer_search_b64's clipping of the search window (same arithmetic as the HME levels, against the ALIGNED picture size)
__device__ __forceinline__ void clip_window(int16_t org, int16_t& o, int16_t& sa, int16_t pad, int16_t pic, bool round8) {
    const int16_t no = ((int16_t)(org + o) < -pad) ? (int16_t)(-pad - org) : o;
    sa = ((int16_t)(org + no) < -pad) ? (int16_t)(sa - (-pad - (org + no))) : sa;  // (sic) evaluated with the corrected origin
    o  = no;
    o  = ((int16_t)(org + o) > (int16_t)(pic - 1)) ? (int16_t)(o - ((org + o) - (pic - 1))) : o;
    sa = ((int16_t)(org + o + sa) > pic) ? (int16_t)max(1, sa - ((org + o + sa) - pic)) : sa;
    if (round8) sa = (sa < 8) ? sa : (int16_t)(sa & ~0x07);
}

template <int PAR>  // references whose HME runs concurrently in a CTA (4 warps each)
__global__ void __launch_bounds__(128 * PAR, PAR == 1 ? 4 : 3)
me_b64_hme_kernel(const __grid_constant__ MeB64Table tab, int n_b64, int b64_w, SvtB200FullpelItem* __restrict__ items,
                  uint32_t* __restrict__ seed_sad, uint8_t* __restrict__ st_do_ref /*[n_b64][8]*/, int16_t* __restrict__ out_centre,
                  uint32_t* __restrict__ out_zz) {
    __shared__ B64State s;
    const SvtB200MeControls& c = tab.c;
    const SvtB200MePicture&  cur = tab.cur;
    const int b = blockIdx.x, bx = b % b64_w, by = b / b64_w, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    const int W = cur.width[2], H = cur.height[2];
    const int16_t org_x = (int16_t)(bx * 64), org_y = (int16_t)(by * 64);
    // me_ctx->b64_width / b64_height come from the 8-aligned picture size (:3093-3100)
    const int aw = (W + 7) & ~7, ah = (H + 7) & ~7;
    const int blk_w = min(64, aw - org_x), blk_h = min(64, ah - org_y);
    const int n_pairs = c.n_ref[0] + (c.n_list > 1 ? c.n_ref[1] : 0);
    auto pair_l = [&](int p) { return p < c.n_ref[0] ? 0 : 1; };
    auto pair_r = [&](int p) { return p < c.n_ref[0] ? p : p - c.n_ref[0]; };
    const uint8_t* src_full = cur.plane[2] + (size_t)(cur.org_y[2] + org_y) * cur.stride[2] + cur.org_x[2] + org_x;

    // ---- init_me_hme_data ------------------------------------------------------------------------------------------
    for (int i = threadIdx.x; i < 2 * kDepth; i += blockDim.x) {
        const int l = i / kDepth, r = i % kDepth;
        s.zz[l][r] = kMaxU32;
        s.do_ref[l][r] = 1;
        s.hme_sad[l][r] = kMaxU32;
        s.divisor[l][r] = 1;
        s.sc_x[l][r] = s.sc_y[l][r] = 0;
        for (int k = 0; k < 2; k++) {
            s.ph_valid[l][r][k] = s.ph_done[l][r][k] = 0;
            s.ph_x[l][r][k] = s.ph_y[l][r][k] = 0;
            s.ph_sad[l][r][k] = 0;
        }
        for (int lv = 0; lv < 3; lv++)
            for (int g = 0; g < 4; g++) {
                s.lx[lv][l][r][g] = s.ly[lv][l][r][g] = 0;
                s.lsad[lv][l][r][g] = 0;
            }
    }
    __syncthreads();

    // ---- init_zz_sad -------------------------------------------------------------------------------------------------
    if (c.me_early_exit_th || c.me_safe_limit_zz_th) {
        for (int p = warp; p < n_pairs; p += n_warps) {
            const int l = pair_l(p), r = pair_r(p);
            if (!searched(c, l)) continue;
            const SvtB200MePicture& rp = tab.ref[l][r];
            const uint8_t* r0 = rp.plane[2] + (size_t)(rp.org_y[2] + org_y) * rp.stride[2] + rp.org_x[2] + org_x;
            uint32_t z = warp_sad_every_other_row(src_full, cur.stride[2], r0, rp.stride[2], blk_w, blk_h, lane) << 1;
            z = (z * 64u * 64u) / (uint32_t)(blk_w * blk_h);  // normalise an incomplete block (32-bit arithmetic as in the reference)
            if (lane == 0) s.zz[l][r] = z;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t best = kMaxU32;
            for (int p = 0; p < n_pairs; p++)
                if (searched(c, pair_l(p))) best = min(best, s.zz[pair_l(p)][pair_r(p)]);
            if (c.temporal_layer_index > 0 && best < (uint32_t)c.zz_sad_th)
                for (int p = 0; p < n_pairs; p++) {
                    const int l = pair_l(p), r = pair_r(p);
                    if (r == 0) continue;
                    if ((uint32_t)((s.zz[l][r] - best) * 100u) > (uint32_t)((uint32_t)c.zz_sad_pct * best)) s.do_ref[l][r] = 0;
                }
            const uint32_t safe = (uint32_t)c.me_safe_limit_zz_th;
            if (safe) {
                const bool limit = c.hierarchical_levels > 0 && c.n_list == 2 && c.temporal_layer_index >= c.hierarchical_levels &&
                                   c.similar_brightness_refs && s.zz[0][0] < safe && s.zz[1][0] < safe;
                if (limit)
                    for (int p = 0; p < n_pairs; p++)
                        if (pair_r(p) > 0) s.do_ref[pair_l(p)][pair_r(p)] = 0;
            }
        }
        __syncthreads();
    }

    // ---- prehme_b64 ----------------------------------------------------------------------------------------------------
    if (c.prehme_enable) {
        const int max_r = max(c.n_ref[0], c.n_list > 1 ? c.n_ref[1] : 0);
        // unit = (reference index, search region); the warp walks list 0 then list 1 of its unit: list 1 may copy list 0's result
        for (int u = warp; u < max_r * 2; u += n_warps) {
            const int r = u >> 1, sr = u & 1;
            for (int l = 0; l < c.n_list; l++) {
                if (r >= c.n_ref[l]) continue;
                if (!searched(c, l)) {  // base layer: list 1 mirrors list 0 (valid / performed flags are not touched)
                    if (lane == 0) {
                        s.ph_x[1][r][sr] = (int16_t)-s.ph_x[0][r][sr];
                        s.ph_y[1][r][sr] = (int16_t)-s.ph_y[0][r][sr];
                        s.ph_sad[1][r][sr] = s.ph_sad[0][r][sr];
                    }
                    __syncwarp();
                    continue;
                }
                // check_prehme_early_exit
                bool done = false;
                if (c.me_early_exit_th && s.zz[l][r] < (uint32_t)c.me_early_exit_th) {
                    if (lane == 0) { s.ph_x[l][r][sr] = s.ph_y[l][r][sr] = 0; s.ph_sad[l][r][sr] = 0; s.ph_valid[l][r][sr] = 1; }
                    done = true;
                } else if (c.prehme_l1_early_exit && l == 1 && s.ph_valid[0][r][sr] &&
                           (s.ph_sad[0][r][sr] < 32 * 32 || (abs((int)s.ph_x[0][r][sr]) < 16 && abs((int)s.ph_y[0][r][sr]) < 16))) {
                    if (lane == 0) {
                        s.ph_x[1][r][sr] = (int16_t)-s.ph_x[0][r][sr];
                        s.ph_y[1][r][sr] = (int16_t)-s.ph_y[0][r][sr];
                        s.ph_sad[1][r][sr] = s.ph_sad[0][r][sr];
                        s.ph_valid[1][r][sr] = 1;
                    }
                    done = true;
                } else if (!s.do_ref[l][r]) {
                    if (lane == 0) { s.ph_x[l][r][sr] = s.ph_y[l][r][sr] = 0; s.ph_sad[l][r][sr] = kMaxU32; }
                    done = true;
                }
                if (!done) {  // prehme_core
                    const SvtB200MePicture& rp = tab.ref[l][r];
                    const int     f = scaled_distance(c.dist[l][r]);
                    int16_t       sa_w = (int16_t)(uint16_t)min(c.prehme_sa[sr][0] * f, c.prehme_sa[sr][2]);
                    int16_t       sa_h = (int16_t)(uint16_t)min(c.prehme_sa[sr][1] * f, c.prehme_sa[sr][3]);
                    const int16_t ox16 = (int16_t)(org_x >> 2), oy16 = (int16_t)(org_y >> 2);
                    int16_t       ox = (int16_t)-(int16_t)(sa_w >> 1), oy = (int16_t)-(int16_t)(sa_h >> 1);
                    hme_clip(ox16, ox, sa_w, (int16_t)(rp.org_x[0] - 1), (int16_t)rp.width[0], false);
                    hme_clip(oy16, oy, sa_h, (int16_t)(rp.org_y[0] - 1), (int16_t)rp.height[0], false);
                    const int sub = c.hme_sub_sad ? 1 : 0;
                    SvtB200SadSearchItem it;
                    it.src_off = it.ref_off = 0;
                    it.src_stride = (uint32_t)(cur.stride[0] << sub);
                    it.ref_stride = (uint32_t)(rp.stride[0] << sub);
                    it.ref_step   = (uint32_t)rp.stride[0];
                    it.block_w    = (uint16_t)(blk_w >> 2);
                    it.block_h    = (uint16_t)((blk_h >> 2) >> sub);
                    it.sa_w = sa_w;
                    it.sa_h = sa_h;
                    it.skip_search_line = (uint16_t)c.prehme_skip_search_line;
                    it.reserved = 0;
                    const uint8_t* sp = cur.plane[0] + (size_t)(cur.org_y[0] + oy16) * cur.stride[0] + cur.org_x[0] + ox16;
                    const uint8_t* rq = rp.plane[0] + (ptrdiff_t)(rp.org_y[0] + oy16 + oy) * rp.stride[0] + rp.org_x[0] + ox16 + ox;
                    const SvtB200SadSearchResult q = sad_key_to_result(sad_search_warp(sp, rq, it, lane));
                    if (lane == 0) {
                        const bool none = q.x < 0;  // no line evaluated: the reference keeps the MV of an earlier block; (0,0) here (DESIGN 6)
                        uint64_t sad = q.best_sad;
                        if (sub) sad *= 2;
                        s.ph_sad[l][r][sr] = sad;
                        s.ph_x[l][r][sr] = (int16_t)((int16_t)((none ? 0 : q.x) + ox) * 4);
                        s.ph_y[l][r][sr] = (int16_t)((int16_t)((none ? 0 : q.y) + oy) * 4);
                        s.ph_valid[l][r][sr] = 1;
                        s.ph_done[l][r][sr] = 1;
                    }
                }
                __syncwarp();
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t best = kMaxU32;
            for (int p = 0; p < n_pairs; p++) {
                const int l = pair_l(p), r = pair_r(p);
                if (!searched(c, l)) continue;
                best = min(best, (uint32_t)min(s.ph_sad[l][r][0], s.ph_sad[l][r][1]));
            }
            if (c.temporal_layer_index > 0 && best < (uint32_t)c.phme_sad_th)
                for (int p = 0; p < n_pairs; p++) {
                    const int l = pair_l(p), r = pair_r(p);
                    if (!s.do_ref[l][r] || r == 0) continue;
                    const uint32_t ps = (uint32_t)min(s.ph_sad[l][r][0], s.ph_sad[l][r][1]);
                    if ((uint32_t)((ps - best) * 100u) > (uint32_t)((uint32_t)c.phme_sad_pct * best)) s.do_ref[l][r] = 0;
                }
        }
        __syncthreads();
    }

    // ---- HME level 0 / 1 / 2: warp = (reference, search region); `par` references at a time, in order ------------------------------
    // (the only coupling between references inside these stages is the low-delay "reduce_hme_l0_sr" rule, which reads the level-0
    //  centre of list 0 / reference 0: with it on, the references go one at a time)
    if (c.enable_hme) {
        const bool coupled = c.sr_enable && c.sr_distance_based_hme_resizing && c.reduce_hme_l0_sr_th_min && c.reduce_hme_l0_sr_th_max;
        const int  par = coupled ? 1 : max(1, n_warps >> 2), reg = warp & 3;
        // which branch of hme_level0_b64 a reference takes: 0 zz exit, 1 previous-stage exit, 2 pruned, 3 search, 4 not searched (base layer, list 1)
        auto l0_kind = [&](int li, int ri) {
            const int sr_i = s.ph_sad[li][ri][0] <= s.ph_sad[li][ri][1] ? 0 : 1;
            if (c.me_early_exit_th && s.zz[li][ri] < ((uint32_t)c.me_early_exit_th >> 2)) return 0;
            if (c.prev_me_stage_based_exit_th && s.ph_done[li][ri][sr_i] && s.ph_sad[li][ri][sr_i] < ((uint32_t)c.prev_me_stage_based_exit_th >> 4)) return 1;
            if (!s.do_ref[li][ri]) return 2;
            return searched(c, li) ? 3 : 4;
        };
        for (int p0 = 0; p0 < n_pairs; p0 += par) {
            const int  p = p0 + (warp >> 2);
            const bool on = (warp >> 2) < par && p < n_pairs;
            const int  l = on ? pair_l(p) : 0, r = on ? pair_r(p) : 0;
            const SvtB200MePicture& rp = tab.ref[l][r];
            SvtB200MeParams prm;
            prm.hme_l1_sa_w = c.hme_l1_w; prm.hme_l1_sa_h = c.hme_l1_h; prm.hme_l2_sa_w = c.hme_l2_w; prm.hme_l2_sa_h = c.hme_l2_h;
            prm.hme_sub_sad = c.hme_sub_sad; prm.me_sub_sad = c.me_sub_sad; prm.check_zero_centre = 0; prm.reserved = 0;
            prm.me_sa_w = prm.me_sa_h = 0;
            prm.hme_l0_sa_w = prm.hme_l0_sa_h = 0;
            const bool zz_exit = on && c.me_early_exit_th && s.zz[l][r] < ((uint32_t)c.me_early_exit_th >> 2);
            // ---- level 0 (hme_level0_b64)
            if (c.enable_l0) {
                if (on) {
                    const int kind = l0_kind(l, r);
                    const int sr_i = s.ph_sad[l][r][0] <= s.ph_sad[l][r][1] ? 0 : 1;
                    if (kind == 0) {
                        if (lane == 0) { s.lx[0][l][r][reg] = s.ly[0][l][r][reg] = 0; s.lsad[0][l][r][reg] = 0; }
                    } else if (kind == 1) {
                        if (lane == 0) { s.lx[0][l][r][reg] = s.ph_x[l][r][sr_i]; s.ly[0][l][r][reg] = s.ph_y[l][r][sr_i]; s.lsad[0][l][r][reg] = s.ph_sad[l][r][sr_i]; }
                    } else if (kind == 2) {
                        if (lane == 0) { s.lx[0][l][r][reg] = s.ly[0][l][r][reg] = 0; s.lsad[0][l][r][reg] = kMaxU32; }
                    } else if (kind == 3) {
                        // get_hme_l0_search_area
                        int min_w = c.hme_l0_min_w, min_h = c.hme_l0_min_h, max_w = c.hme_l0_max_w, max_h = c.hme_l0_max_h;
                        if (c.sr_enable && c.sr_distance_based_hme_resizing) {
                            bool is_hor = true, is_ver = true, is_still = false;
                            if (c.reduce_hme_l0_sr_th_min && c.reduce_hme_l0_sr_th_max && (l || r)) {
                                const int mx = abs((int)s.lx[0][0][0][0]), my = abs((int)s.ly[0][0][0][0]);
                                is_ver   = mx < c.reduce_hme_l0_sr_th_min && my > c.reduce_hme_l0_sr_th_max;
                                is_hor   = mx > c.reduce_hme_l0_sr_th_max && my < c.reduce_hme_l0_sr_th_min;
                                is_still = mx < c.reduce_hme_l0_sr_th_min * 3 && my < c.reduce_hme_l0_sr_th_min * 3;
                            }
                            int x_off = is_hor ? 1 : 2, y_off = is_ver ? 1 : 2;
                            if (c.sr_enable == 2 && is_still) x_off = y_off = 4;
                            min_w = (uint16_t)(min_w / (x_off + r)); min_h = (uint16_t)(min_h / (y_off + r));
                            max_w = (uint16_t)(max_w / (x_off + r)); max_h = (uint16_t)(max_h / (y_off + r));
                        }
                        const int f = scaled_distance(c.dist[l][r]);
                        int16_t sa_w = (int16_t)(min_w / 2);
                        sa_w = (int16_t)min(((sa_w * f) + 15) & ~0x0F, ((max_w / 2) + 15) & ~0x0F);
                        int16_t sa_h = (int16_t)(min_h / 2);
                        sa_h = (int16_t)min(sa_h * f, max_h / 2);
                        prm.hme_l0_sa_w = sa_w;
                        prm.hme_l0_sa_h = sa_h;
                        SvtB200SadSearchItem it;
                        HmeSide              sd;
                        hme_make_item(cur, rp, prm, 0, reg & 1, reg >> 1, bx, by, 0, 0, it, sd);
                        const SvtB200SadSearchResult q =
                            sad_key_to_result(sad_search_warp((const uint8_t*)(uintptr_t)it.src_off, (const uint8_t*)(uintptr_t)it.ref_off, it, lane));
                        int16_t  x, y;
                        uint64_t sad;
                        hme_finish_one(q, sd, prm, 0, x, y, sad);
                        if (lane == 0) { s.lx[0][l][r][reg] = x; s.ly[0][l][r][reg] = y; s.lsad[0][l][r][reg] = sad; }
                    }
                }
                __syncthreads();  // the four regions' level-0 results of these references are complete
                if (c.prehme_enable) {  // replace the worst quadrant of a searched reference by its better pre-HME result
                    if ((int)threadIdx.x < par && p0 + (int)threadIdx.x < n_pairs) {
                        const int li = pair_l(p0 + threadIdx.x), ri = pair_r(p0 + threadIdx.x);
                        if (l0_kind(li, ri) == 3) {
                            const int sr_i = s.ph_sad[li][ri][0] <= s.ph_sad[li][ri][1] ? 0 : 1;
                            uint64_t  mx = 0;
                            int       worst = 0;
                            for (int g = 0; g < 3; g++)
                                if (s.lsad[0][li][ri][g] > mx) { mx = s.lsad[0][li][ri][g]; worst = g; }
                            if (s.lsad[0][li][ri][3] > mx) worst = 3;
                            if (s.ph_sad[li][ri][sr_i] < s.lsad[0][li][ri][worst]) {
                                s.lsad[0][li][ri][worst] = s.ph_sad[li][ri][sr_i];
                                s.lx[0][li][ri][worst] = s.ph_x[li][ri][sr_i];
                                s.ly[0][li][ri][worst] = s.ph_y[li][ri][sr_i];
                            }
                        }
                    }
                    __syncthreads();
                }
            }
            // ---- level 1 (hme_level1_b64)
            if (on && c.enable_l1 && searched(c, l)) {
                if (zz_exit) {
                    if (lane == 0) { s.lx[1][l][r][reg] = s.ly[1][l][r][reg] = 0; s.lsad[1][l][r][reg] = 0; }
                } else if (!s.do_ref[l][r]) {
                    if (lane == 0) { s.lx[1][l][r][reg] = s.ly[1][l][r][reg] = 0; s.lsad[1][l][r][reg] = kMaxU32; }
                } else if (c.prev_me_stage_based_exit_th && s.lsad[0][l][r][reg] < ((uint32_t)c.prev_me_stage_based_exit_th >> 5)) {
                    if (lane == 0) { s.lx[1][l][r][reg] = s.lx[0][l][r][reg]; s.ly[1][l][r][reg] = s.ly[0][l][r][reg]; s.lsad[1][l][r][reg] = s.lsad[0][l][r][reg]; }
                } else {
                    SvtB200SadSearchItem it;
                    HmeSide              sd;
                    hme_make_item(cur, rp, prm, 1, reg & 1, reg >> 1, bx, by, s.lx[0][l][r][reg], s.ly[0][l][r][reg], it, sd);
                    const SvtB200SadSearchResult q =
                        sad_key_to_result(sad_search_warp((const uint8_t*)(uintptr_t)it.src_off, (const uint8_t*)(uintptr_t)it.ref_off, it, lane));
                    int16_t  x, y;
                    uint64_t sad;
                    hme_finish_one(q, sd, prm, 1, x, y, sad);
                    if (lane == 0) { s.lx[1][l][r][reg] = x; s.ly[1][l][r][reg] = y; s.lsad[1][l][r][reg] = sad; }
                }
                __syncwarp();
            }
            // ---- level 2 (hme_level2_b64): no early exit, pruned references are searched as well
            if (on && c.enable_l2 && searched(c, l)) {
                if (c.prev_me_stage_based_exit_th && s.lsad[1][l][r][reg] < ((uint32_t)c.prev_me_stage_based_exit_th >> 2)) {
                    if (lane == 0) { s.lx[2][l][r][reg] = s.lx[1][l][r][reg]; s.ly[2][l][r][reg] = s.ly[1][l][r][reg]; s.lsad[2][l][r][reg] = s.lsad[1][l][r][reg]; }
                } else {
                    SvtB200SadSearchItem it;
                    HmeSide              sd;
                    hme_make_item(cur, rp, prm, 2, reg & 1, reg >> 1, bx, by, s.lx[1][l][r][reg], s.ly[1][l][r][reg], it, sd);
                    const SvtB200SadSearchResult q =
                        sad_key_to_result(sad_search_warp((const uint8_t*)(uintptr_t)it.src_off, (const uint8_t*)(uintptr_t)it.ref_off, it, lane));
                    int16_t  x, y;
                    uint64_t sad;
                    hme_finish_one(q, sd, prm, 2, x, y, sad);
                    if (lane == 0) { s.lx[2][l][r][reg] = x; s.ly[2][l][r][reg] = y; s.lsad[2][l][r][reg] = sad; }
                }
                __syncwarp();
            }
        }
    }
    __syncthreads();

    // ---- set_final_seach_centre_sb + hme_prune_ref_and_adjust_sr (one thread: values carry over between references) ---------
    if (threadIdx.x == 0) {
        int16_t  x_hme = 0, y_hme = 0, x_sc = 0, y_sc = 0;
        uint64_t hme_mv_sad = 0;
        for (int p = 0; p < n_pairs; p++) {
            const int l = pair_l(p), r = pair_r(p);
            if (searched(c, l)) {
                if (c.enable_hme) {
                    int lv = -1;
                    if (c.enable_l0 && !c.enable_l1 && !c.enable_l2) lv = 0;
                    if (c.enable_l1 && !c.enable_l2) lv = 1;
                    if (c.enable_l2) lv = 2;
                    if (lv >= 0) {
                        x_hme = s.lx[lv][l][r][0]; y_hme = s.ly[lv][l][r][0]; hme_mv_sad = s.lsad[lv][l][r][0];
                        for (int g = 1; g < 4; g++)
                            if (s.lsad[lv][l][r][g] < hme_mv_sad) { x_hme = s.lx[lv][l][r][g]; y_hme = s.ly[lv][l][r][g]; hme_mv_sad = s.lsad[lv][l][r][g]; }
                    }
                    x_sc = x_hme;
                    y_sc = y_hme;
                }
            } else
                x_sc = y_sc = 0;
            s.sc_x[l][r] = x_sc;
            s.sc_y[l][r] = y_sc;
            s.hme_sad[l][r] = hme_mv_sad;
        }
        if (c.enable_hme) {  // prune_ref = enable_hme_flag (open-loop ME)
            const uint32_t th = (uint32_t)c.prune_hme_th & 0xffffu;
            if (c.prune_enable && th != 0xffffu) {
                uint64_t best = ~0ull;
                for (int l = 0; l < 2; l++)
                    for (int r = 0; r < kDepth; r++) best = min(best, s.hme_sad[l][r]);
                for (int l = 0; l < 2; l++)
                    for (int r = 1; r < kDepth; r++)
                        if ((s.hme_sad[l][r] - best) * 100ull > (unsigned long long)th * best) s.do_ref[l][r] = 0;
            }
            if (c.sr_enable)
                for (int l = 0; l < 2; l++)
                    for (int r = 0; r < kDepth; r++) {
                        if (abs((int)s.sc_x[l][r]) <= c.sr_mv_length_th && abs((int)s.sc_y[l][r]) <= c.sr_mv_length_th &&
                            s.hme_sad[l][r] < (uint64_t)(uint32_t)c.sr_stationary_hme_sad_abs_th)
                            s.divisor[l][r] = (uint32_t)c.sr_stationary_divisor;
                        else if (s.hme_sad[l][r] < (uint64_t)(uint32_t)c.sr_hme_sad_abs_th)
                            s.divisor[l][r] = (uint32_t)c.sr_low_hme_sad_divisor;
                    }
        }
    }
    __syncthreads();

    // ---- integer_search_b64: the search window of every live reference; warp = reference ------------------------------------------
    for (int p = warp; p < n_pairs; p += n_warps) {
        const int l = pair_l(p), r = pair_r(p);
        const SvtB200MePicture& rp = tab.ref[l][r];
        const size_t item_idx = (size_t)p * n_b64 + b;
        SvtB200FullpelItem it;
        it.src_off = (uint64_t)(uintptr_t)src_full;
        it.src_stride = (uint32_t)cur.stride[2];
        it.ref_stride = (uint32_t)rp.stride[2];
        it.sub_sad = (uint8_t)(c.me_sub_sad ? 1 : 0);
        it.seeded = 0;
        it.seed_x = it.seed_y = 0;
        it.reserved[0] = it.reserved[1] = 0;
        const uint8_t* r0 = rp.plane[2] + (size_t)(rp.org_y[2] + org_y) * rp.stride[2] + rp.org_x[2] + org_x;  // zero-MV position
        if (!s.do_ref[l][r]) {  // pruned: one position at the zero MV keeps the search kernel's item stream dense; the result is not used
            it.ref_off = (uint64_t)(uintptr_t)r0;
            it.sa_w = it.sa_h = 1;
            it.org_x = it.org_y = 0;
            if (lane == 0) items[item_idx] = it;
            continue;
        }
        int16_t sx = s.sc_x[l][r], sy = s.sc_y[l][r];
        const int dist = scaled_distance((int)(uint16_t)(int16_t)c.dist[l][r]);
        int16_t sa_w = (int16_t)min(c.me_min_w * dist, c.me_max_w), sa_h = (int16_t)min(c.me_min_h * dist, c.me_max_h);
        if (c.mvsa_enable && (!c.mvsa_nearest_ref_only || r == 0)) {
            if (abs((int)sx) > c.mvsa_mv_size_th) sa_w = (int16_t)(sa_w * c.mvsa_multiplier);
            if (abs((int)sy) > c.mvsa_mv_size_th) sa_h = (int16_t)(sa_h * c.mvsa_multiplier);
        }
        const int dv = (int)s.divisor[l][r];
        sa_w = (int16_t)((max(1, sa_w / dv) + 7) & ~0x07);
        sa_h = (int16_t)max(3, sa_h / dv);
        if (c.me_early_exit_th) {
            if (s.zz[l][r] < (uint32_t)c.me_early_exit_th / 6u) sa_w = sa_h = 1;
        } else if ((sx != 0 || sy != 0) && c.is_ref) {
            // check_00_center: keep the HME centre only if it beats the zero MV (SADs on every other row)
            const int16_t RW = (int16_t)rp.width[2], RH = (int16_t)rp.height[2];
            if ((int16_t)(org_x + sx) < -63) sx = (int16_t)(-63 - org_x);
            if ((int16_t)(org_x + sx) > (int16_t)(RW - 1)) sx = (int16_t)(sx - ((org_x + sx) - (RW - 1)));
            if ((int16_t)(org_y + sy) < -63) sy = (int16_t)(-63 - org_y);
            if ((int16_t)(org_y + sy) > (int16_t)(RH - 1)) sy = (int16_t)(sy - ((org_y + sy) - (RH - 1)));
            const uint32_t z = warp_sad_every_other_row(src_full, cur.stride[2], r0, rp.stride[2], blk_w, blk_h, lane) << 1;
            const uint32_t h = warp_sad_every_other_row(src_full, cur.stride[2], r0 + (ptrdiff_t)sy * rp.stride[2] + sx, rp.stride[2], blk_w, blk_h, lane) << 1;
            if (z <= h) sx = sy = 0;
        }
        // 8x8-SAD-variance probe at the search centre
        if (c.var_enable && (int)sa_w * (int)sa_h > 24) {
            const uint32_t var = warp_probe_sads(src_full, cur.stride[2], r0 + (ptrdiff_t)sy * rp.stride[2] + sx, rp.stride[2], c.me_sub_sad != 0,
                                                 lane, seed_sad + item_idx * 85);
            if (var > (uint32_t)c.var_mult2_th) {
                sa_w = (int16_t)((max(1, sa_w * 3 / 2) + 7) & ~0x7);
                sa_h = (int16_t)max(1, sa_h * 3 / 2);
            }
            if (var < (uint32_t)c.var_div4_th) {
                sa_w = (int16_t)((max(1, sa_w >> 2) + 7) & ~0x7);
                sa_h = (int16_t)max(3, max(1, sa_h >> 2));
            } else if (var < (uint32_t)c.var_div2_th) {
                sa_w = (int16_t)((min((int)sa_w, sa_w >> 1) + 7) & ~0x7);
                sa_h = (int16_t)max(3, min((int)sa_h, sa_h >> 1));
            }
            it.seeded = 1;
            it.seed_x = sx;
            it.seed_y = sy;
        }
        int16_t ox = (int16_t)(sx - (sa_w >> 1)), oy = (int16_t)(sy - (sa_h >> 1));
        clip_window(org_x, ox, sa_w, 63, (int16_t)aw, true);
        clip_window(org_y, oy, sa_h, 63, (int16_t)ah, false);
        it.ref_off = (uint64_t)(uintptr_t)(r0 + (ptrdiff_t)oy * rp.stride[2] + ox);
        it.sa_w = sa_w;
        it.sa_h = sa_h;
        it.org_x = ox;
        it.org_y = oy;
        if (lane == 0) items[item_idx] = it;
    }
    // state for the finishing kernel + diagnostics
    if (threadIdx.x < 2 * kDepth) {
        const int l = threadIdx.x / kDepth, r = threadIdx.x % kDepth;
        const bool live = l < c.n_list && r < c.n_ref[l];
        st_do_ref[(size_t)b * 8 + threadIdx.x] = live ? s.do_ref[l][r] : 0;
        out_centre[((size_t)b * 8 + threadIdx.x) * 2]     = live ? s.sc_x[l][r] : 0;
        out_centre[((size_t)b * 8 + threadIdx.x) * 2 + 1] = live ? s.sc_y[l][r] : 0;
        out_zz[(size_t)b * 8 + threadIdx.x] = live ? s.zz[l][r] : 0;
    }
}

__constant__ uint8_t kZToRaster[85] = {0,  1,  2,  3,  4,  5,  6,  9,  10, 7,  8,  11, 12, 13, 14, 17, 18, 15, 16, 19, 20, 21, 22, 29, 30, 23, 24, 31, 32,
                                       37, 38, 45, 46, 39, 40, 47, 48, 25, 26, 33, 34, 27, 28, 35, 36, 41, 42, 49, 50, 43, 44, 51, 52, 53, 54, 61, 62, 55,
                                       56, 63, 64, 69, 70, 77, 78, 71, 72, 79, 80, 57, 58, 65, 66, 59, 60, 67, 68, 73, 74, 81, 82, 75, 76, 83, 84};

__device__ __forceinline__ uint8_t cand_byte(int direction, int i0, int i1, int l0, int l1) {
    return (uint8_t)((direction & 3) | ((i0 & 3) << 2) | ((i1 & 3) << 4) | ((l0 & 1) << 6) | ((l1 & 1) << 7));
}

// (C) per 64x64 block: me_prune_ref, candidate construction, compute_distortion, perform_gm_detection.  thread = ME PU index (z order)
__global__ void __launch_bounds__(96)
me_b64_finish_kernel(const __grid_constant__ SvtB200MeControls c, int n_b64, int b64_w, int pic_w, int pic_h, int n_pu,
                     const uint32_t* __restrict__ best_sad, const uint32_t* __restrict__ best_mv, const uint8_t* __restrict__ st_do_ref,
                     uint8_t* __restrict__ out_total, uint8_t* __restrict__ out_cand, uint32_t* __restrict__ out_mv,
                     uint32_t* __restrict__ out_dist, uint8_t* __restrict__ out_flags, uint8_t* __restrict__ out_do_ref) {
    __shared__ uint8_t  do_ref[2][kDepth];
    __shared__ uint64_t me_sad[2][kDepth];
    __shared__ uint32_t me_distortion[85];
    const int b = blockIdx.x, t = threadIdx.x;
    const int n_list = c.n_list;
    const int n0 = c.n_ref[0], n1 = n_list > 1 ? c.n_ref[1] : 0;
    auto sad_of = [&](int l, int r, int n) { return best_sad[((size_t)(l ? n0 + r : r) * n_b64 + b) * 85 + n]; };
    auto mv_of  = [&](int l, int r, int n) { return best_mv[((size_t)(l ? n0 + r : r) * n_b64 + b) * 85 + n]; };
    if (t < 2 * kDepth) do_ref[t / kDepth][t % kDepth] = (t / kDepth < n_list && t % kDepth < c.n_ref[t / kDepth]) ? st_do_ref[(size_t)b * 8 + t] : 1;
    __syncthreads();
    // ---- me_prune_ref (prune_ref && enable_me_hme_ref_pruning)
    if (c.enable_hme && c.prune_enable) {
        if (t < 2 * kDepth) {
            const int l = t / kDepth, r = t % kDepth;
            // references that were never searched keep the MAX_U32 the HME stage left (they are not live and nothing reads do_ref of them)
            uint64_t v = kMaxU32;
            if (l < n_list && r < c.n_ref[l]) {
                v = 0;
                if (!do_ref[l][r]) v = (uint64_t)kMaxSad * 64;
                else
                    for (int k = 0; k < 64; k++) v += sad_of(l, r, 21 + k);
            }
            me_sad[l][r] = v;
        }
        __syncthreads();
        const uint32_t th = (uint32_t)c.prune_me_th & 0xffffu;
        if (t == 0 && th != 0xffffu) {
            uint64_t best = ~0ull;
            for (int l = 0; l < 2; l++)
                for (int r = 0; r < kDepth; r++) best = min(best, me_sad[l][r]);
            for (int l = 0; l < 2; l++)
                for (int r = 1; r < kDepth; r++)
                    if ((me_sad[l][r] - best) * 100ull > (unsigned long long)th * best) do_ref[l][r] = 0;
        }
        __syncthreads();
    }
    uint8_t*  total = out_total + (size_t)b * n_pu;
    uint8_t*  cand  = out_cand + (size_t)b * n_pu * c.max_cand;
    uint32_t* mvs   = out_mv + (size_t)b * n_pu * c.max_refs;
    const bool single = n0 == 1 && n1 == 0, mrp_off = n0 == 1 && n1 == 1;
    if ((single || mrp_off) && t < n_pu) total[t] = 1;  // the memset of the two small variants
    __syncthreads();
    if (t < 85) {
        const int  n = t;
        const int  pu = kZToRaster[n];
        const bool use_pu = c.enable_me_16x16 ? (c.enable_me_8x8 || n < 21) : n < 5;
        uint8_t*   ca = cand + (size_t)pu * c.max_cand;
        if (single) {
            me_distortion[pu] = sad_of(0, 0, n);
            if (do_ref[0][0] && use_pu) {
                ca[0] = cand_byte(0, 0, 0, 0, 0);
                mvs[(size_t)pu * c.max_refs + 0] = mv_of(0, 0, n);
            }
        } else if (mrp_off) {
            int lists = n_list;
            const uint8_t org0 = do_ref[0][0], org1 = (n_list == 1) ? 0 : do_ref[1][0];
            if (lists < 2 || !do_ref[1][0]) lists = 1;
            const uint32_t prune_th = (org0 && org1) ? (uint32_t)c.prune_me_candidates_th : 0u;
            uint8_t  dr[2] = {org0, org1};
            const uint32_t s0 = sad_of(0, 0, n), s1 = n_list > 1 ? sad_of(1, 0, n) : 0u;
            const uint32_t best = (org0 && org1) ? min(s0, s1) : (org0 ? s0 : s1);
            me_distortion[pu] = best;
            int min_list = -1;
            if (c.use_best_unipred_cand_only && dr[0] && dr[1]) min_list = s0 < s1 ? 0 : 1;
            int off = 0;
            for (int l = 0; l < lists && (use_pu || off == 0); l++) {
                if (!dr[l]) continue;
                const uint32_t sl = l ? s1 : s0;
                if (prune_th > 0 && (uint32_t)((sl - best) * 100u) > (uint32_t)(best * prune_th)) { dr[l] = 0; continue; }
                if (min_list != -1 && min_list != l) {
                    if (use_pu) mvs[(size_t)pu * c.max_refs + (l ? c.max_l0 : 0)] = mv_of(l, 0, n);  // kept for an injected bi-prediction
                    continue;
                }
                if (use_pu) {
                    ca[off] = cand_byte(l, 0, 0, 0, l == 1 ? 1 : 0);
                    mvs[(size_t)pu * c.max_refs + (l ? c.max_l0 : 0)] = mv_of(l, 0, n);
                }
                off++;
            }
            if (dr[0] && dr[1] && use_pu) {
                ca[off] = cand_byte(2, 0, 0, 0, 1);
                total[pu] = (uint8_t)(off + 1);
            }
        } else {
            uint8_t  dr[2][kDepth];
            uint32_t best = kMaxU32;
            for (int l = 0; l < n_list; l++)
                for (int r = 0; r < c.n_ref[l]; r++) {
                    dr[l][r] = do_ref[l][r];
                    if (dr[l][r]) best = min(best, sad_of(l, r, n));
                }
            me_distortion[pu] = best;
            const uint32_t prune_th = (uint32_t)c.prune_me_candidates_th;
            int off = 0;
            for (int l = 0; l < n_list && (use_pu || off == 0); l++)
                for (int r = 0; r < c.n_ref[l] && (use_pu || off == 0); r++) {
                    if (!dr[l][r]) continue;
                    if (prune_th > 0 && (uint32_t)((sad_of(l, r, n) - best) * 100u) > (uint32_t)(best * prune_th)) { dr[l][r] = 0; continue; }
                    if (use_pu) {
                        ca[off] = cand_byte(l, r, r, 0, l == 1 ? 1 : 0);
                        mvs[(size_t)pu * c.max_refs + (l ? c.max_l0 : 0) + r] = mv_of(l, r, n);
                    }
                    off++;
                }
            if (n_list == 2 && use_pu) {
                for (int i = 0; i < n0; i++)
                    for (int j = 0; j < n1; j++) {
                        if (c.only_l_bwd && (i > 0 || j > 0)) continue;
                        if (dr[0][i] && dr[1][j]) ca[off++] = cand_byte(2, i, j, 0, 1);
                    }
                if (!c.only_l_bwd) {
                    for (int i = 1; i < n0; i++)
                        if (dr[0][0] && dr[0][i]) ca[off++] = cand_byte(2, 0, i, 0, 0);
                    if (n1 == 3 && dr[1][0] && dr[1][2]) ca[off++] = cand_byte(2, 0, 2, 1, 1);
                }
            }
            if (use_pu) total[pu] = (uint8_t)off;
        }
    }
    __syncthreads();
    // ---- compute_distortion
    const int ox = (b % b64_w) * 64, oy = (b / b64_w) * 64;
    if (t == 0) {
        uint32_t d64 = me_distortion[0], d32 = 0, d16 = 0, d8 = 0;
        for (int i = 0; i < 4; i++) d32 += me_distortion[1 + i];
        for (int i = 0; i < 16; i++) d16 += me_distortion[5 + i];
        for (int i = 0; i < 64; i++) d8 += me_distortion[21 + i];
        const uint64_t mean = d8 / 64;
        uint64_t       sq = 0;
        for (int i = 0; i < 64; i++) {
            const int64_t d = (int64_t)me_distortion[21 + i] - (int64_t)mean;
            sq += (uint64_t)(d * d);
        }
        const uint32_t pix = (uint32_t)(min(64, pic_w - ox) * min(64, pic_h - oy));
        uint32_t* o = out_dist + (size_t)b * 6;
        o[0] = c.resolution_le_480p ? d8 : d16;
        o[1] = (uint32_t)(d64 * 4096u) / pix;
        o[2] = (uint32_t)(d32 * 4096u) / pix;
        o[3] = (uint32_t)(d16 * 4096u) / pix;
        o[4] = (uint32_t)(d8 * 4096u) / pix;
        o[5] = (uint32_t)(sq / 64);
    }
    if (t < 2 * kDepth) out_do_ref[(size_t)b * 8 + t] = (t / kDepth < n_list && t % kDepth < c.n_ref[t / kDepth]) ? do_ref[t / kDepth][t % kDepth] : 0;
    // ---- perform_gm_detection (indices as in the reference: the first candidate of a raster PU, the MV of the same number in ME order)
    if (t == 0) {
        uint8_t stationary = 0, allow_gm = 0;
        if (c.gm_enabled) {
            uint32_t cnt[2][kDepth][2][2];
            for (int i = 0; i < 2 * kDepth * 4; i++) (&cnt[0][0][0][0])[i] = 0;
            uint32_t stat = 0, tot = 0;
            const int count = c.resolution_le_480p ? 64 : 16;
            for (int i = 0; i < count; i++) {
                int n = (c.resolution_le_480p ? 21 : 5) + i;
                if (c.resolution_le_480p && !c.enable_me_8x8) {
                    if (n >= 21) { const int k = n - 21; n = 5 + ((k >> 3) >> 1) * 4 + ((k & 7) >> 1); }
                    if (!c.enable_me_16x16 && n >= 5) { const int k = n - 5; n = 1 + ((k >> 2) >> 1) * 2 + ((k & 3) >> 1); }
                } else if (!c.resolution_le_480p && !c.enable_me_16x16 && n >= 5) {
                    const int k = n - 5;
                    n = 1 + ((k >> 2) >> 1) * 2 + ((k & 3) >> 1);
                }
                const uint8_t cb = cand[(size_t)n * c.max_cand];
                const int dir = cb & 3, i0 = (cb >> 2) & 3, i1 = (cb >> 4) & 3, l0 = (cb >> 6) & 1, l1 = (cb >> 7) & 1;
                const int l = (dir == 0 || dir == 2) ? l0 : l1, r = (dir == 0 || dir == 2) ? i0 : i1;
                const int dist = c.dist[l][r];
                const int active_th = c.resolution_le_480p ? (c.gm_use_distance_based_active_th ? max(dist >> 1, 4) : 4)
                                                           : (c.gm_use_distance_based_active_th ? max(dist * 16, 32) : 32);
                const uint32_t mv = (l < n_list && r < c.n_ref[l]) ? mv_of(l, r, n) : 0u;
                const int mx = (int)(int16_t)(mv & 0xffff) << 2, my = (int)(int16_t)(mv >> 16) << 2;
                if (mx < -active_th) cnt[l][r][0][0]++;
                else if (mx > active_th) cnt[l][r][0][1]++;
                if (my < -active_th) cnt[l][r][1][0]++;
                else if (my > active_th) cnt[l][r][1][1]++;
                const int sth = c.resolution_le_480p ? 0 : 4;
                if (abs(mx) <= sth && abs(my) <= sth) stat++;
                tot++;
            }
            if (stat > (tot * 5) / 100) stationary = 1;
            for (int i = 0; i < 2 * kDepth * 4; i++)
                if ((&cnt[0][0][0][0])[i] > tot / 2) allow_gm = 1;
        }
        out_flags[2 * (size_t)b] = stationary;
        out_flags[2 * (size_t)b + 1] = allow_gm;
    }
}

struct MeB64Workspace {
    size_t cap = 0;  // (reference, block) pairs
    SvtB200FullpelItem* items = nullptr;
    uint32_t* seed = nullptr;
    uint8_t*  do_ref = nullptr;
};
std::map<cudaStream_t, MeB64Workspace> g_ws;
std::mutex g_mu;
ResetHook g_reset([] { std::lock_guard<std::mutex> lk(g_mu); g_ws.clear(); });

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int svt_b200_me_b64_num_pus(const SvtB200MeControls* ctrl) {
    if (!ctrl) return SVT_B200_ERR_BAD_ARG;
    return ctrl->enable_me_16x16 ? (ctrl->enable_me_8x8 ? 85 : 21) : 5;
}

extern "C" int svt_b200_me_b64_picture_dev(const SvtB200MePicture* cur, const SvtB200MePicture* refs, const SvtB200MeControls* ctrl,
                                           const SvtB200MeB64Results* out, void* stream) {
    require_ready();
    if (!cur || !refs || !ctrl || !out) return SVT_B200_ERR_BAD_ARG;
    const SvtB200MeControls& c = *ctrl;
    if (c.n_list < 1 || c.n_list > 2 || c.n_ref[0] < 1 || c.n_ref[0] > kDepth || c.n_ref[1] < 0 || c.n_ref[1] > kDepth) return SVT_B200_ERR_BAD_ARG;
    if (c.n_list == 2 && c.n_ref[1] < 1) return SVT_B200_ERR_BAD_ARG;
    if (c.sr_enable == 2 && !c.me_early_exit_th) return SVT_B200_ERR_BAD_ARG;  // documented: needs another reference's full-pel result mid-block
    if (c.max_cand < 1 || c.max_refs < 1 || c.max_l0 < 1) return SVT_B200_ERR_BAD_ARG;
    if (!out->total_me_candidate_index || !out->me_candidate_array || !out->me_mv_array || !out->distortion || !out->flags || !out->do_ref ||
        !out->hme_centre || !out->zz_sad || !out->best_sad || !out->best_mv)
        return SVT_B200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int W = cur->width[2], H = cur->height[2];
    const int b64_w = (W + 63) >> 6, b64_h = (H + 63) >> 6, n_b64 = b64_w * b64_h;
    const int n1 = c.n_list > 1 ? c.n_ref[1] : 0, n_refs = c.n_ref[0] + n1, pairs = n_refs * n_b64;
    const int n_pu = svt_b200_me_b64_num_pus(ctrl);
    MeB64Table tab;
    memset(&tab, 0, sizeof(tab));
    tab.cur = *cur;
    tab.c = c;
    if (c.n_list < 2) tab.c.n_ref[1] = 0;
    for (int r = 0; r < c.n_ref[0]; r++) tab.ref[0][r] = refs[r];
    for (int r = 0; r < n1; r++) tab.ref[1][r] = refs[c.n_ref[0] + r];
    MeB64Workspace* w;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        w = &g_ws[st];
        if ((size_t)pairs > w->cap) {  // new buffers; the old ones stay alive for graphs captured earlier (freed at shutdown)
            w->cap = (size_t)pairs * 2;
            w->items = (SvtB200FullpelItem*)scratch_alloc(w->cap * sizeof(SvtB200FullpelItem));
            w->seed = (uint32_t*)scratch_alloc(w->cap * 85 * sizeof(uint32_t));
            w->do_ref = (uint8_t*)scratch_alloc(w->cap * 8);
        }
    }
    // the candidate / MV arrays are only partially written by design (me_sb_results_ctor leaves them uninitialised): defined zeros here
    B200_CUDA_CHECK(cudaMemsetAsync(out->total_me_candidate_index, 0, (size_t)n_b64 * n_pu, st));
    B200_CUDA_CHECK(cudaMemsetAsync(out->me_candidate_array, 0, (size_t)n_b64 * n_pu * c.max_cand, st));
    B200_CUDA_CHECK(cudaMemsetAsync(out->me_mv_array, 0, (size_t)n_b64 * n_pu * c.max_refs * 4, st));
    // two references of a block in flight per CTA pays off with many references and costs with few (chosen on the previous target
    // GPU; not re-measured on H100)
    if (n_refs >= 6)
        me_b64_hme_kernel<2><<<n_b64, 256, 0, st>>>(tab, n_b64, b64_w, w->items, w->seed, w->do_ref, out->hme_centre, out->zz_sad);
    else
        me_b64_hme_kernel<1><<<n_b64, 128, 0, st>>>(tab, n_b64, b64_w, w->items, w->seed, w->do_ref, out->hme_centre, out->zz_sad);
    B200_LAUNCH_CHECK();
    if (!launch_fullpel_tma(cur, refs, n_refs, n_b64, w->items, pairs, out->best_sad, out->best_mv, st, w->seed)) {
        fprintf(stderr, "[svt_b200] svt_b200_me_b64_picture_dev: the luma planes do not meet the layout rule (16-byte aligned base and pitch)\n");
        return SVT_B200_ERR_BAD_ARG;
    }
    me_b64_finish_kernel<<<n_b64, 96, 0, st>>>(tab.c, n_b64, b64_w, W, H, n_pu, out->best_sad, out->best_mv, w->do_ref, out->total_me_candidate_index,
                                                out->me_candidate_array, out->me_mv_array, out->distortion, out->flags, out->do_ref);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}
