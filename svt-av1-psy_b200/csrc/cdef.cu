// cdef.cu -- K8 CDEF: direction search, constrained directional filter, distortion, strength search,
// frame apply (sm_90a).
//
// Reference behaviour restated: svt_aom_cdef_find_dir_c (Source/Lib/Codec/cdef.c:150-210),
// constrain/adjust_strength (:85-134), svt_cdef_filter_block_c (:253-305), svt_cdef_filter_fb (:339-430),
// dist_8xn_* / mse_* / svt_aom_compute_cdef_dist{,_8bit}_c (Source/Lib/Codec/enc_cdef.c:23-233),
// svt_search_one_dual_c (:627-690), the tile build of cdef_seg_search (Source/Lib/Codec/cdef_process.c:
// 106-352: CDEF_VERY_LARGE outside the frame, pre-filter neighbours inside).
//
// H100 mapping (T2): a frame-wide kernel finds direction and variance of every non-skip 8x8 (one
// thread per block, the 64 pixels in registers).  Search and apply run one 128-thread CTA per (64x64
// filter block, plane): the padded 16-bit tile of the plane, (fbs + 6) x (fbs + 16) for a filter block of
// fbs x fbs pixels in that plane, is staged in shared memory once, and a thread owns a row segment of one
// block (luma: a processed 8-pixel row of an 8x8, chroma: a 4-pixel row of a 4x4), so the tap offsets of
// the block's direction and the per-strength constants are built once per segment, not per pixel.  A
// pixel's 12 taps are fetched once per direction, as signed differences and magnitudes packed two per
// register, and shared by all candidate strengths; the filter sum is separable into a primary and a
// secondary half, each evaluated once per distinct strength value with native packed 16-bit min/max/add
// and 2-way dot-product instructions.  The search sums a segment's distortion moments in registers (up
// to kGChunk strengths at a time), combines the few segments of a block with shuffles and stores them once
// per (block, strength); the source's moments and those of strength code 0 (the unfiltered block) are not
// recomputed per strength.  The luma distortion's double-precision formula is evaluated with
// round-to-nearest intrinsics in the reference's operand order (FMA contraction is disabled for the whole
// library), which makes it IEEE-identical to the C code.
#include <mutex>

#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

constexpr int kVeryLarge = 0x7f7f;  // CDEF_VERY_LARGE (cdef.h:38)
constexpr int kTP        = 88;      // tile pitch in uint16 (>= 64 + 2*8, keeps rows 16-B aligned)
constexpr int kTileRows  = 64 + 6;

__device__ __forceinline__ int msb32(uint32_t n) { return 31 - __clz(n); }
__device__ __forceinline__ int cdef_adjust_strength(int strength, int var) {
    const int i = (var >> 6) ? min(msb32((uint32_t)(var >> 6)), 12) : 0;
    return var ? (strength * (4 + i) + 8) >> 4 : 0;
}

// Cdef_Directions (AV1 spec 7.15.3) as (dy, dx) pairs for k = 0, 1
__constant__ int8_t c_cdef_dir[8][2][2] = {{{-1, 1}, {-2, 2}}, {{0, 1}, {-1, 2}}, {{0, 1}, {0, 2}}, {{0, 1}, {1, 2}},
                                           {{1, 1}, {2, 2}},   {{1, 0}, {2, 1}},  {{1, 0}, {2, 0}}, {{1, 0}, {2, -1}}};

// direction + variance of one 8x8 (cdef.c:150-210).  The 64 centred pixels sit in registers and the
// eight directions are evaluated one after the other, each with its own (compile-time indexed) line sums.
template <int D>
__device__ __forceinline__ int cdef_dir_bin(int i, int j) {
    return D == 0 ? i + j : D == 1 ? i + j / 2 : D == 2 ? i : D == 3 ? 3 + i - j / 2 : D == 4 ? 7 + i - j : D == 5 ? 3 - i / 2 + j : D == 6 ? j : i / 2 + j;
}
__device__ __forceinline__ constexpr int cdef_div(int n) {  // 840 / n, the weight of a line of n pixels
    return n == 1 ? 840 : n == 2 ? 420 : n == 3 ? 280 : n == 4 ? 210 : n == 5 ? 168 : n == 6 ? 140 : n == 7 ? 120 : 105;
}
template <int D>
__device__ __forceinline__ int cdef_dir_cost(const int (&x)[64]) {
    constexpr int NB = (D == 2 || D == 6) ? 8 : (D & 1) ? 11 : 15;
    int p[NB];
#pragma unroll
    for (int k = 0; k < NB; k++) p[k] = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) p[cdef_dir_bin<D>(i, j)] += x[i * 8 + j];
    int cost = 0;
    if (D == 2 || D == 6) {
#pragma unroll
        for (int i = 0; i < 8; i++) cost += p[i] * p[i];
        cost *= cdef_div(8);
    } else if (D & 1) {
#pragma unroll
        for (int j = 0; j < 5; j++) cost += p[3 + j] * p[3 + j];
        cost *= cdef_div(8);
#pragma unroll
        for (int j = 0; j < 3; j++) cost += (p[j] * p[j] + p[10 - j] * p[10 - j]) * cdef_div(2 * j + 2);
    } else {
#pragma unroll
        for (int i = 0; i < 7; i++) cost += (p[i] * p[i] + p[14 - i] * p[14 - i]) * cdef_div(i + 1);
        cost += p[7] * p[7] * cdef_div(8);
    }
    return cost;
}
template <typename T>
__device__ int cdef_find_dir_dev(const T* img, int stride, int* var, int coeff_shift) {
    int x[64];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) x[i * 8 + j] = ((int)img[i * stride + j] >> coeff_shift) - 128;
    const int cost[8] = {cdef_dir_cost<0>(x), cdef_dir_cost<1>(x), cdef_dir_cost<2>(x), cdef_dir_cost<3>(x),
                         cdef_dir_cost<4>(x), cdef_dir_cost<5>(x), cdef_dir_cost<6>(x), cdef_dir_cost<7>(x)};
    int best_cost = 0, best_dir = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        if (cost[i] > best_cost) {
            best_cost = cost[i];
            best_dir  = i;
        }
    int opp = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) opp = (i == ((best_dir + 4) & 7)) ? cost[i] : opp;
    *var = (best_cost - opp) >> 10;
    return best_dir;
}

// Taps of one pixel along direction `dir` (cdef.c:262-302), reduced to what every candidate strength
// shares, two taps per 32-bit register (16-bit halves; every value fits: pixels <= 4095, CDEF_VERY_LARGE =
// 0x7f7f, |differences| <= 0x7f7f): the signed differences tap - x, their magnitudes, and the min / max over
// the taps that are inside the picture.  Pairs: 0 = primary k=0 (+,-), 1 = primary k=1, 2..3 = secondary
// k=0, 4..5 = secondary k=1.  The packed min/max/add instructions used (VIMNMX.16x2, VIADD.16x2) are native.
struct CdefTaps {
    uint32_t d[6];   // signed differences
    uint32_t ad[6];  // |differences|
    int      mn, mx;
};
// element offsets of the six tap pairs along direction `dir` in a tile of pitch s (pair order as above)
__device__ __forceinline__ void cdef_tap_offsets(int dir, int s, int (&o)[6]) {
    const int d2 = (dir + 2) & 7, d6 = (dir + 6) & 7;
#pragma unroll
    for (int k = 0; k < 2; k++) {
        o[k]         = c_cdef_dir[dir][k][0] * s + c_cdef_dir[dir][k][1];
        o[2 + 2 * k] = c_cdef_dir[d2][k][0] * s + c_cdef_dir[d2][k][1];
        o[3 + 2 * k] = c_cdef_dir[d6][k][0] * s + c_cdef_dir[d6][k][1];
    }
}
__device__ __forceinline__ void cdef_load_taps(const uint16_t* in, const int (&o)[6], int x, CdefTaps& T) {
    // CDEF_VERY_LARGE marks "outside the picture": never the maximum.  The maximum is taken over the halves
    // plus kMxBias (mod 2^16), which maps CDEF_VERY_LARGE to 0 and keeps pixels (<= 4095) in order above it.
    constexpr uint32_t kMxBias = 0x10000u - kVeryLarge;
    const uint32_t xx = (uint32_t)x * 0x10001u, nxx = __vneg2(xx);
    uint32_t       mx2 = __vadd2(xx, kMxBias * 0x10001u), mn2 = xx;
#pragma unroll
    for (int pair = 0; pair < 6; pair++) {
        const uint32_t p = (uint32_t)in[o[pair]] | ((uint32_t)in[-o[pair]] << 16);
        T.d[pair]  = __vadd2(p, nxx);
        T.ad[pair] = __vmaxu2(p, xx) - __vminu2(p, xx);  // halves are >= 0: no borrow between them
        mx2 = __vmaxu2(mx2, __vadd2(p, kMxBias * 0x10001u));
        mn2 = __vminu2(mn2, p);
    }
    T.mn = (int)min(mn2 & 0xffffu, mn2 >> 16);
    T.mx = (int)max(mx2 & 0xffffu, mx2 >> 16) - (int)kMxBias;
}
// What constrain() (cdef.c:85-93) needs of a strength t at a damping: the threshold in both halves, the shift
// max(0, damping - msb(t)), the mask that keeps the shifted high half out of the low one, and the dp2a
// weights of the two primary pairs (byte pair 0-1: k = 0, 2-3: k = 1; cdef_pri_taps[(t >> coeff_shift) & 1]).
// t = 0 gives a zero threshold, which constrains every tap to zero.
__device__ __forceinline__ uint4 cdef_strength_consts(int t, int damping, int coeff_shift) {
    const int sh = max(0, damping - msb32((uint32_t)t));
    return make_uint4((uint32_t)t * 0x10001u, (uint32_t)sh, (0xffffu >> sh) * 0x10001u,
                      ((t >> coeff_shift) & 1) ? 0x03030303u : 0x02020404u);
}
// constrain() of the two taps of a pair: sign(d) * min(|d|, max(0, thr - (|d| >> shift))) = clamp(d, -m, m)
// with m = thr - min(|d| >> shift, thr), as two signed 16-bit halves.
__device__ __forceinline__ uint32_t cdef_constrain2(const CdefTaps& T, int pair, const uint4& c) {
    const uint32_t t1 = (T.ad[pair] >> c.y) & c.z;
    const uint32_t m  = c.x - __vminu2(t1, c.x);
    return __vmins2(__vmaxs2(T.d[pair], __vneg2(m)), m);
}
// The sum splits into a primary part (4 taps, depends on the primary strength only) and a secondary part
// (8 taps, depends on the secondary strength only): candidate strengths that share one of the two share
// that half of the work.  The reference accumulates in int16; |sum| <= 2*(4+2)*240 + 4*(2+1)*64 for 12-bit
// content, so the int32 sum is the same number.  Two constrained secondary taps (|v| <= 64 each) add
// without overflow in a 16-bit half.
__device__ __forceinline__ int cdef_primary_sum(const CdefTaps& T, const uint4& c) {
    return __dp2a_hi((int)cdef_constrain2(T, 1, c), (int)c.w, __dp2a_lo((int)cdef_constrain2(T, 0, c), (int)c.w, 0));
}
__device__ __forceinline__ int cdef_secondary_sum(const CdefTaps& T, const uint4& c) {
    const uint32_t w2 = __vadd2(cdef_constrain2(T, 2, c), cdef_constrain2(T, 3, c));
    const uint32_t w1 = __vadd2(cdef_constrain2(T, 4, c), cdef_constrain2(T, 5, c));
    return __dp2a_lo((int)w2, 0x0202, __dp2a_lo((int)w1, 0x0101, 0));
}
__device__ __forceinline__ int cdef_finish_px(const CdefTaps& T, int x, int sum) {
    const int y = x + ((8 + sum - (sum < 0)) >> 4);
    return y < T.mn ? T.mn : (y > T.mx ? T.mx : y);
}
// one filtered pixel; `in` points at the pixel, s = tile pitch
__device__ __forceinline__ int cdef_filter_px(const uint16_t* in, int s, int pri_strength, int sec_strength, int dir,
                                              int pri_damping, int sec_damping, int coeff_shift) {
    CdefTaps  T;
    int       o[6];
    const int x = in[0];
    cdef_tap_offsets(dir, s, o);
    cdef_load_taps(in, o, x, T);
    return cdef_finish_px(T, x, cdef_primary_sum(T, cdef_strength_consts(pri_strength, pri_damping, coeff_shift)) +
                                    cdef_secondary_sum(T, cdef_strength_consts(sec_strength, sec_damping, coeff_shift)));
}

// luma psy distortion of one 8xN block from its five moments (enc_cdef.c:41-47); exact IEEE sequence
__device__ __forceinline__ unsigned long long cdef_dist_from_sums(unsigned long long sum_s, unsigned long long sum_d,
                                                                  unsigned long long sum_s2, unsigned long long sum_d2,
                                                                  unsigned long long sum_sd, int coeff_shift) {
    const unsigned long long svar = sum_s2 - ((sum_s * sum_s + 32) >> 6);
    const unsigned long long dvar = sum_d2 - ((sum_d * sum_d + 32) >> 6);
    const double num0 = __ull2double_rn(sum_d2 + sum_s2 - 2 * sum_sd);
    const double a    = __dmul_rn(num0, .5);
    const double b    = __ull2double_rn(svar + dvar + (unsigned long long)(400 << 2 * coeff_shift));
    const double num  = __dmul_rn(a, b);
    const double den  = __dsqrt_rn(__dadd_rn((double)(20000 << 4 * coeff_shift), __dmul_rn(__ull2double_rn(svar), __ull2double_rn(dvar))));
    return (unsigned long long)floor(__dadd_rn(.5, __ddiv_rn(num, den)));
}

// ------------------------------------------------------------------------------------------------
// T1 kernels
// ------------------------------------------------------------------------------------------------
__global__ void find_dir_kernel(const uint16_t* img, int stride, int coeff_shift, int n, const int* offs, int* out) {
    const int t = threadIdx.x;
    if (t < n) {
        int var;
        out[2 * t]     = cdef_find_dir_dev(img + offs[t], stride, &var, coeff_shift);
        out[2 * t + 1] = var;
    }
}

// in_c: copy of the caller's tile rows [-2, h+2) x cols [-2, w+2), pitch = w + 4
__global__ void filter_block_kernel(const uint16_t* in_c, int w, int h, int pri, int sec, int dir, int pd, int sd, int cs,
                                    int subs, uint16_t* out) {
    const int p = w + 4;
    for (int idx = threadIdx.x; idx < w * h; idx += blockDim.x) {
        const int i = idx / w, j = idx - i * w;
        if (i % subs) continue;
        out[idx] = (uint16_t)cdef_filter_px(in_c + (i + 2) * p + j + 2, p, pri, sec, dir, pd, sd, cs);
    }
}

template <typename T>
__global__ void cdef_dist_kernel(const T* dst, int dstride, const T* src, const uint8_t* dlist, int count, int bw_log2,
                                 int bh_log2, int coeff_shift, int pli, int subs, unsigned long long* out) {
    __shared__ unsigned long long tot;
    if (threadIdx.x == 0) tot = 0;
    __syncthreads();
    const int bw = 1 << bw_log2, bh = 1 << bh_log2;
    for (int bi = threadIdx.x; bi < count; bi += blockDim.x) {
        const int by = dlist[2 * bi], bx = dlist[2 * bi + 1];
        const T*  s  = src + ((size_t)bi << (bw_log2 + bh_log2));
        const T*  d  = dst + (size_t)(by << bh_log2) * dstride + (bx << bw_log2);
        unsigned long long v;
        if (bw == 8 && bh == 8 && pli == 0) {
            unsigned long long ss = 0, sd_ = 0, s2 = 0, d2 = 0, sdp = 0;
            for (int i = 0; i < 8; i += subs)
                for (int j = 0; j < 8; j++) {
                    const unsigned long long a = s[8 * i + j], b = d[i * dstride + j];
                    ss += a; sd_ += b; s2 += a * a; d2 += b * b; sdp += a * b;
                }
            v = cdef_dist_from_sums(ss, sd_, s2, d2, sdp, coeff_shift);
        } else {
            v = 0;
            for (int i = 0; i < bh; i += subs)
                for (int j = 0; j < bw; j++) {
                    const int e = (int)d[i * dstride + j] - (int)s[bw * i + j];
                    v += (unsigned long long)(long long)(e * e);
                }
        }
        atomicAdd(&tot, v);
    }
    __syncthreads();
    if (threadIdx.x == 0) *out = tot >> (2 * coeff_shift);
}

// svt_search_one_dual: tot[j][k] = sum_i min(best_i, mse0[i][j] + mse1[i][k])
__global__ void search_one_dual_kernel(const unsigned long long* mse0, const unsigned long long* mse1, int sb_count, int ng,
                                       const int* lev0, const int* lev1, int nb, int start_gi, unsigned long long* out) {
    extern __shared__ unsigned long long tot[];  // ng*ng
    for (int p = threadIdx.x; p < ng * ng; p += blockDim.x) {
        const int j = p / ng, k = p - j * ng;
        unsigned long long acc = 0;
        if (j >= start_gi && k >= start_gi)
            for (int i = 0; i < sb_count; i++) {
                unsigned long long best = 1ull << 63;
                for (int g = 0; g < nb; g++) {
                    const unsigned long long c = mse0[(size_t)i * ng + lev0[g]] + mse1[(size_t)i * ng + lev1[g]];
                    best = c < best ? c : best;
                }
                const unsigned long long c = mse0[(size_t)i * ng + j] + mse1[(size_t)i * ng + k];
                acc += c < best ? c : best;
            }
        tot[p] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long bt = 1ull << 63;
        int b0 = 0, b1 = 0;
        for (int j = start_gi; j < ng; j++)
            for (int k = start_gi; k < ng; k++)
                if (tot[j * ng + k] < bt) {
                    bt = tot[j * ng + k];
                    b0 = j;
                    b1 = k;
                }
        out[0] = bt;
        out[1] = (unsigned long long)b0;
        out[2] = (unsigned long long)b1;
    }
}

// ------------------------------------------------------------------------------------------------
// T2: per-filter-block search (all planes, all candidate strengths) and frame apply
// ------------------------------------------------------------------------------------------------
constexpr int kT2Threads = 128;  // threads of a search / apply CTA
constexpr int kGChunk    = 8;    // candidate strengths whose moments a search thread keeps in registers at once

template <typename PIX>
__device__ void stage_cdef_tile(uint16_t* tile, const PIX* plane, int stride, int fbr, int fbc, int nvfb, int nhfb, int fbs,
                                int vsz, int hsz) {
    // tile origin (row 3, col 8) = first pixel of the filter block; everything outside the copied
    // rectangle is CDEF_VERY_LARGE (cdef_process.c:211-230).  Only the (fbs + 6) x (fbs + 16) pixels the
    // filter can read are written.  One pass, two pixels per thread and store.
    const int yoff = 3 * (fbr != 0), xoff = 8 * (fbc != 0);
    const int ysize = vsz + 3 * (fbr + 1 < nvfb) + yoff, xsize = hsz + 8 * (fbc + 1 < nhfb) + xoff;
    const int py0 = fbr * fbs - yoff, px0 = fbc * fbs - xoff;
    const int pairs = (fbs + 16) / 2;
    // a pair starts at an even column: one load per pair when the plane's rows are aligned to it
    const bool pair_load = (((size_t)plane | (size_t)stride * sizeof(PIX)) & (2 * sizeof(PIX) - 1)) == 0;
#pragma unroll 4
    for (int i = threadIdx.x; i < (fbs + 6) * pairs; i += blockDim.x) {
        const int r = i / pairs, c = (i - r * pairs) * 2;
        const int rr = r - (3 - yoff), cc = c - (8 - xoff);  // cc is even, xsize is a multiple of 4: the pair is in or out together
        uint32_t v = (uint32_t)kVeryLarge * 0x10001u;
        if (rr >= 0 && rr < ysize && cc >= 0 && cc < xsize) {
            const PIX* p = plane + (size_t)(py0 + rr) * stride + px0 + cc;
            if (!pair_load) v = (uint32_t)p[0] | ((uint32_t)p[1] << 16);
            else if (sizeof(PIX) == 1) v = __byte_perm(*reinterpret_cast<const uint16_t*>(p), 0, 0x4140);  // 0, p[1], 0, p[0]
            else v = *reinterpret_cast<const uint32_t*>(p);
        }
        *reinterpret_cast<uint32_t*>(tile + r * kTP + c) = v;
    }
    __syncthreads();
}

// Ordered list of the non-skip 8x8s of filter block (fbr, fbc) (svt_sb_compute_cdef_list: by*8+bx, raster
// order) and their directions / variances, into shared memory.  Threads 0..63 (two whole warps) take part;
// the caller synchronises before the list is read.  Returns the count (read from the ballots: CTA-uniform).
__device__ __forceinline__ int cdef_fb_list(const uint8_t* skip8x8, const uint8_t* dir_in, const int* var_in, int fb, int fbr,
                                            int fbc, int w8, int h8, uint8_t* s_list, uint8_t* s_dir, int* s_var, unsigned* s_ballot) {
    if (threadIdx.x < 64) {
        const int  by = threadIdx.x >> 3, bx = threadIdx.x & 7, gy = fbr * 8 + by, gx = fbc * 8 + bx;
        const bool on = gy < h8 && gx < w8 && !skip8x8[gy * w8 + gx];
        const unsigned m = __ballot_sync(0xffffffffu, on);
        s_dir[threadIdx.x] = dir_in[(size_t)fb * 64 + threadIdx.x];
        s_var[threadIdx.x] = var_in[(size_t)fb * 64 + threadIdx.x];
        if ((threadIdx.x & 31) == 0) s_ballot[threadIdx.x >> 5] = m;
    }
    __syncthreads();
    const unsigned m0 = s_ballot[0], m1 = s_ballot[1];
    if (threadIdx.x < 64) {
        const unsigned mine = threadIdx.x < 32 ? m0 : m1, lane = threadIdx.x & 31;
        if ((mine >> lane) & 1) s_list[(threadIdx.x < 32 ? 0 : __popc(m0)) + __popc(mine & ((1u << lane) - 1))] = (uint8_t)threadIdx.x;
    }
    return __popc(m0) + __popc(m1);
}

// direction + variance of every non-skip 8x8 luma block of the frame: one thread per block
template <typename PIX>
__global__ void __launch_bounds__(128)
cdef_dir_kernel(SvtB200CdefFrame f, const uint8_t* __restrict__ skip8x8, uint8_t* __restrict__ dir_out /*[nfb][64]*/,
                int* __restrict__ var_out /*[nfb][64]*/) {
    const int w8 = (f.width + 7) >> 3, h8 = (f.height + 7) >> 3, nhfb = (f.width + 63) >> 6;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= w8 * h8) return;
    const int gy = t / w8, gx = t - gy * w8;
    if (skip8x8[t]) return;
    const int cs = f.bit_depth > 8 ? f.bit_depth - 8 : 0;
    int       var;
    const int dir = cdef_find_dir_dev((const PIX*)f.recon_y + (size_t)gy * 8 * f.recon_stride_y + gx * 8, f.recon_stride_y, &var, cs);
    const size_t o = (size_t)((gy >> 3) * nhfb + (gx >> 3)) * 64 + (gy & 7) * 8 + (gx & 7);
    dir_out[o] = (uint8_t)dir;
    var_out[o] = var;
}

// One chunk of candidate strengths (CTA-uniform description) as the search's threads see it.
struct CdefChunk {
    int      sv[kGChunk];  // strength codes, -1 = not tested (also past the end of the list)
    unsigned todo[2];      // pass 0: taps along the block's direction (a primary part, or code 0); pass 1: along direction 0
    unsigned pri_new;      // pass-0 strengths whose primary code differs from the previous one with a primary part
    unsigned secs[2];      // per pass: bit c set when secondary code c (1..3) occurs
};

// Moments of one row segment (BS pixels at `in`, source at `o_row`) for every strength of `todo`, the
// taps along one direction.  Luma (BS = 8) accumulates sum y, y^2, y*src; chroma (BS = 4) sum (src - y)^2.
// Taps are loaded once per pixel and shared by all strengths; the primary half is recomputed only when the
// primary strength changes and the secondary half once per distinct secondary code.
template <int BS, typename PIX>
__device__ __forceinline__ void cdef_segment_pass(const uint16_t* in, const PIX* o_row, const int (&off)[6], const CdefChunk& C, int pass,
                                                  const int (&tadj)[kGChunk], const uint4* tab, int cs, unsigned (&a0)[kGChunk],
                                                  unsigned (&a1)[kGChunk], unsigned (&a2)[kGChunk]) {
    const unsigned todo = C.todo[pass], pnew = pass ? 0u : C.pri_new, secs = C.secs[pass];
#pragma unroll 1
    for (int j = 0; j < BS; j++) {
        const int      x = in[j];
        const unsigned o = o_row[j];
        CdefTaps       T;
        cdef_load_taps(in + j, off, x, T);
        int s1 = 0, s2 = 0, s3 = 0;  // secondary halves of codes 1, 2, 3 (strengths 1, 2, 4 << cs)
        if (secs & 2) s1 = cdef_secondary_sum(T, tab[1 << cs]);
        if (secs & 4) s2 = cdef_secondary_sum(T, tab[2 << cs]);
        if (secs & 8) s3 = cdef_secondary_sum(T, tab[4 << cs]);
        int psum = 0;
#pragma unroll
        for (int gi = 0; gi < kGChunk; gi++) {
            if (!((todo >> gi) & 1)) continue;  // CTA-uniform
            if ((pnew >> gi) & 1) psum = cdef_primary_sum(T, tab[tadj[gi]]);
            const int sc = C.sv[gi] & 3, ssum = sc == 1 ? s1 : (sc == 2 ? s2 : (sc == 3 ? s3 : 0));
            // code 0 leaves the pixel unchanged (sum = 0, and x lies inside [min, max] of its own neighbourhood)
            const unsigned y = C.sv[gi] == 0 ? (unsigned)x : (unsigned)cdef_finish_px(T, x, psum + ssum);
            if (BS == 8) {
                a0[gi] += y;
                a1[gi] += y * y;
                a2[gi] += y * o;
            } else {
                const int e = (int)o - (int)y;
                a0[gi] += (unsigned)(e * e);
            }
        }
    }
}

// The strength search of one (filter block, plane): every thread owns processed row segments (luma: one
// 8-pixel row of an 8x8, chroma: one 4-pixel row of a 4x4), so tap offsets and strength constants are
// built once per segment, and only the R threads of a block combine their moments, by shuffles.  Their
// sums go to shared memory once per (block, strength); warps then turn them into distortions (luma: the
// psy formula on the five moments) and sum them over the blocks.
template <int BS, typename PIX>
__device__ __forceinline__ void cdef_search_fb(const uint16_t* tile, const uint4* tab, const PIX* src, int sstride, const int* strengths,
                                               int n_strengths, int count, int subs, int cs, int pli, const uint8_t* s_list,
                                               const uint8_t* s_dir, const int* s_var, unsigned (*s_mom)[3][64], unsigned (*s_src)[64],
                                               unsigned long long* mse_fb) {
    const int R = BS / subs, nseg = count * R;  // processed rows per block (a power of two: R divides 32)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int g0 = 0; g0 < n_strengths; g0 += kGChunk) {
        const int ng = min(kGChunk, n_strengths - g0);
        CdefChunk C;
        C.todo[0] = C.todo[1] = C.pri_new = C.secs[0] = C.secs[1] = 0;
        unsigned zero = 0;
        int      last_pri = -1;
#pragma unroll
        for (int gi = 0; gi < kGChunk; gi++) {
            const int sv = gi < ng ? strengths[g0 + gi] : -1;
            C.sv[gi] = sv;
            if (sv < 0) continue;
            const int pri = sv >> 2, sc = sv & 3;
            if (pri) {
                C.todo[0] |= 1u << gi;
                C.secs[0] |= (1u << sc) & ~1u;
                if (pri != last_pri) C.pri_new |= 1u << gi;
                last_pri = pri;
            } else if (sc) {
                C.todo[1] |= 1u << gi;
                C.secs[1] |= 1u << sc;
            } else {
                zero |= 1u << gi;
            }
        }
        // code 0 needs no taps: it joins a pass that runs anyway
        if (C.todo[0] || !C.todo[1]) C.todo[0] |= zero;
        else C.todo[1] |= zero;
        const unsigned tested = C.todo[0] | C.todo[1];
        for (int s = threadIdx.x; s < ((nseg + 31) & ~31); s += kT2Threads) {  // whole warps stay in the loop (shuffles)
            const bool live = s < nseg;
            const int  bi = live ? s / R : 0, r = live ? s - bi * R : 0;
            const int  b = s_list[bi], by = b >> 3, bx = b & 7, row = BS * by + r * subs;
            const uint16_t* in    = tile + (3 + row) * kTP + 8 + BS * bx;
            const PIX*      o_row = src + (size_t)row * sstride + BS * bx;
            unsigned a0[kGChunk], a1[kGChunk], a2[kGChunk];
#pragma unroll
            for (int gi = 0; gi < kGChunk; gi++) a0[gi] = a1[gi] = a2[gi] = 0;
            int tadj[kGChunk];  // the adjusted primary strength of each pass-0 strength that starts a new primary half
            const int var = s_var[b];
#pragma unroll
            for (int gi = 0; gi < kGChunk; gi++) {
                const int pri = (C.sv[gi] >> 2) << cs;
                tadj[gi] = (C.pri_new >> gi) & 1 ? (BS == 4 ? pri : cdef_adjust_strength(pri, var)) : 0;
            }
            int off[6];
            if (C.todo[0]) {
                cdef_tap_offsets(s_dir[b], kTP, off);
                cdef_segment_pass<BS, PIX>(in, o_row, off, C, 0, tadj, tab, cs, a0, a1, a2);
            }
            if (C.todo[1]) {
                cdef_tap_offsets(0, kTP, off);
                cdef_segment_pass<BS, PIX>(in, o_row, off, C, 1, tadj, tab, cs, a0, a1, a2);
            }
            const bool lead = live && r == 0;
#pragma unroll
            for (int gi = 0; gi < kGChunk; gi++) {
                if (!((tested >> gi) & 1)) continue;  // CTA-uniform
                for (int sh = R >> 1; sh > 0; sh >>= 1) {
                    a0[gi] += __shfl_xor_sync(0xffffffffu, a0[gi], sh);
                    if (BS == 8) {
                        a1[gi] += __shfl_xor_sync(0xffffffffu, a1[gi], sh);
                        a2[gi] += __shfl_xor_sync(0xffffffffu, a2[gi], sh);
                    }
                }
                if (lead) {
                    s_mom[gi][0][bi] = a0[gi];
                    if (BS == 8) {
                        s_mom[gi][1][bi] = a1[gi];
                        s_mom[gi][2][bi] = a2[gi];
                    }
                }
            }
            if (BS == 8 && g0 == 0) {  // the source's moments do not depend on the strength
                unsigned so = 0, so2 = 0;
#pragma unroll
                for (int j = 0; j < BS; j++) {
                    const unsigned o = o_row[j];
                    so += o;
                    so2 += o * o;
                }
                for (int sh = R >> 1; sh > 0; sh >>= 1) {
                    so += __shfl_xor_sync(0xffffffffu, so, sh);
                    so2 += __shfl_xor_sync(0xffffffffu, so2, sh);
                }
                if (lead) {
                    s_src[0][bi] = so;
                    s_src[1][bi] = so2;
                }
            }
        }
        __syncthreads();
        // per strength: the blocks' distortions, summed by one warp
        for (int gi = warp; gi < ng; gi += kT2Threads / 32) {
            const int          sv = strengths[g0 + gi];
            unsigned long long acc = 0;
            if (sv >= 0)
                for (int bi = lane; bi < count; bi += 32)
                    acc += BS == 8 ? cdef_dist_from_sums(s_mom[gi][0][bi], s_src[0][bi], s_mom[gi][1][bi], s_src[1][bi], s_mom[gi][2][bi], cs)
                                   : (unsigned long long)s_mom[gi][0][bi];
#pragma unroll
            for (int sh = 16; sh > 0; sh >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sh);
            if (lane == 0) {
                unsigned long long* m = mse_fb + g0 + gi;
                // enc: mse_seg = (sum >> 2*coeff_shift) * subsampling_factor; untested chroma = default_mse_uv*64
                const unsigned long long v = sv >= 0 ? (acc >> (2 * cs)) * (unsigned long long)subs : 0;
                if (pli == 0) *m = v;
                else atomicAdd(m, sv < 0 ? (pli == 1 ? 1040400ull * 64ull : 0ull) : v);
            }
        }
        __syncthreads();  // s_mom is reused by the next chunk
    }
}

// Strength search: one CTA per (filter block, plane).  mse[1] (chroma) must be zero on entry: the two
// chroma planes add into it.
template <typename PIX>
__global__ void __launch_bounds__(kT2Threads, 5)
cdef_search_kernel(SvtB200CdefFrame f, const uint8_t* __restrict__ skip8x8, const int* __restrict__ strengths_y,
                   const int* __restrict__ strengths_uv, int n_strengths, unsigned long long* __restrict__ mse /*[2][nfb][n_strengths]*/,
                   const uint8_t* __restrict__ dir_in /*[nfb][64]*/, const int* __restrict__ var_in /*[nfb][64]*/) {
    __shared__ __align__(16) uint16_t tile[kTileRows * kTP];
    __shared__ uint4    s_tab[2][256];  // cdef_strength_consts of every strength value, luma / chroma damping
    __shared__ uint8_t  s_dir[64];
    __shared__ int      s_var[64];
    __shared__ uint8_t  s_list[64];
    __shared__ unsigned s_ballot[2];
    __shared__ unsigned s_mom[kGChunk][3][64];  // per strength, per listed block: luma sum y, y^2, y*src; chroma [0] = sum (src - y)^2
    __shared__ unsigned s_src[2][64];           // per listed luma block: sum src, src^2
    const int nhfb = (f.width + 63) >> 6, nvfb = (f.height + 63) >> 6, nfb = nhfb * nvfb;
    const int cs = f.bit_depth > 8 ? f.bit_depth - 8 : 0;
    const int w8 = (f.width + 7) >> 3, h8 = (f.height + 7) >> 3;
    // strengths reach (15 << 4) = 240 (primary, 12-bit), adjusted ones no more, secondary 4 << 4
    for (int i = threadIdx.x; i < 2 * 256; i += kT2Threads) s_tab[i >> 8][i & 255] = cdef_strength_consts(i & 255, f.damping + cs - (i >> 8), cs);
    for (int work = blockIdx.x; work < nfb * 3; work += gridDim.x) {
        const int fb = work / 3, pli = work - fb * 3;
        const int fbr = fb / nhfb, fbc = fb - fbr * nhfb;
        __syncthreads();
        const int count = cdef_fb_list(skip8x8, dir_in, var_in, fb, fbr, fbc, w8, h8, s_list, s_dir, s_var, s_ballot);
        if (count == 0) {
            if (pli == 0)
                for (int g = threadIdx.x; g < n_strengths; g += blockDim.x) mse[(size_t)fb * n_strengths + g] = 0;
            continue;
        }
        const int dec = pli ? 1 : 0;
        const PIX* rec = (const PIX*)(pli == 0 ? f.recon_y : (pli == 1 ? f.recon_cb : f.recon_cr));
        const PIX* src = (const PIX*)(pli == 0 ? f.src_y : (pli == 1 ? f.src_cb : f.src_cr));
        const int rstride = pli ? f.recon_stride_c : f.recon_stride_y, sstride = pli ? f.src_stride_c : f.src_stride_y;
        const int pw = f.width >> dec, ph = f.height >> dec, fbs = 64 >> dec;
        const int hsz = min(fbs, pw - fbc * fbs), vsz = min(fbs, ph - fbr * fbs);
        stage_cdef_tile<PIX>(tile, rec, rstride, fbr, fbc, nvfb, nhfb, fbs, vsz, hsz);  // ends with a barrier
        const PIX* src_fb = src + (size_t)fbr * fbs * sstride + fbc * fbs;
        unsigned long long* mse_fb = mse + (size_t)((pli ? 1 : 0) * nfb + fb) * n_strengths;
        const int subs = min(f.subsampling_factor, dec ? 1 : 4);  // cdef_process.c:243-248 (4:2:0 chroma = BLOCK_4X4)
        if (pli == 0)
            cdef_search_fb<8, PIX>(tile, s_tab[0], src_fb, sstride, strengths_y, n_strengths, count, subs, cs, pli, s_list, s_dir, s_var,
                                   s_mom, s_src, mse_fb);
        else
            cdef_search_fb<4, PIX>(tile, s_tab[1], src_fb, sstride, strengths_uv, n_strengths, count, subs, cs, pli, s_list, s_dir, s_var,
                                   s_mom, s_src, mse_fb);
    }
}

// BS filtered pixels to one row of a picture, with one store when the row is aligned to it
template <int BS, typename PIX>
__device__ __forceinline__ void cdef_store_row(PIX* p, const int (&y)[BS], bool wide) {
    constexpr int NW = BS * (int)sizeof(PIX) / 4;  // 32-bit words in the row
    if (wide) {
        uint32_t w[NW];
#pragma unroll
        for (int k = 0; k < NW; k++) {
            if (sizeof(PIX) == 1)
                w[k] = (uint32_t)y[4 * k] | ((uint32_t)y[4 * k + 1] << 8) | ((uint32_t)y[4 * k + 2] << 16) | ((uint32_t)y[4 * k + 3] << 24);
            else
                w[k] = (uint32_t)y[2 * k] | ((uint32_t)y[2 * k + 1] << 16);
        }
        if (NW == 1) *reinterpret_cast<uint32_t*>(p) = w[0];
        else if (NW == 2) *reinterpret_cast<uint2*>(p) = make_uint2(w[0], w[1 % NW]);
        else *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1 % NW], w[2 % NW], w[3 % NW]);
    } else {
#pragma unroll
        for (int j = 0; j < BS; j++) p[j] = (PIX)y[j];
    }
}

// the filter of one (filter block, plane) with one strength: a thread per BS-pixel row of a block
template <int BS, typename PIX>
__device__ __forceinline__ void cdef_apply_fb(const uint16_t* tile, PIX* out_fb, int ostride, bool wide, int count, int pri, int sec,
                                              int damping, int cs, const uint8_t* s_list, const uint8_t* s_dir, const int* s_var) {
    const uint4 csec = cdef_strength_consts(sec, damping, cs);
    for (int s = threadIdx.x; s < count * BS; s += kT2Threads) {
        const int bi = s / BS, r = s - bi * BS;
        const int b = s_list[bi], by = b >> 3, bx = b & 7;
        const uint4 cpri = cdef_strength_consts(BS == 4 ? pri : cdef_adjust_strength(pri, s_var[b]), damping, cs);
        int off[6];
        cdef_tap_offsets(pri ? s_dir[b] : 0, kTP, off);
        const uint16_t* in = tile + (3 + BS * by + r) * kTP + 8 + BS * bx;
        int y[BS];
#pragma unroll
        for (int j = 0; j < BS; j++) {
            CdefTaps  T;
            const int x = in[j];
            cdef_load_taps(in + j, off, x, T);
            y[j] = cdef_finish_px(T, x, (pri ? cdef_primary_sum(T, cpri) : 0) + (sec ? cdef_secondary_sum(T, csec) : 0));
        }
        cdef_store_row<BS, PIX>(out_fb + (size_t)(BS * by + r) * ostride + BS * bx, y, wide);
    }
}

// frame apply (svt_av1_cdef_frame, enc_cdef.c:284-600): per filter block strengths already chosen,
// directions/variances as found by cdef_dir_kernel.  One CTA per (filter block, plane).
template <typename PIX>
__global__ void __launch_bounds__(kT2Threads)
cdef_apply_kernel(SvtB200CdefFrame f, const uint8_t* __restrict__ skip8x8, const int8_t* __restrict__ fb_strength_idx,
                  const int* __restrict__ y_strength, const int* __restrict__ uv_strength, const uint8_t* __restrict__ dir_in,
                  const int* __restrict__ var_in, PIX* out_y, PIX* out_cb, PIX* out_cr, int out_stride_y, int out_stride_c) {
    __shared__ __align__(16) uint16_t tile[kTileRows * kTP];
    __shared__ uint8_t  s_dir[64];
    __shared__ int      s_var[64];
    __shared__ uint8_t  s_list[64];
    __shared__ unsigned s_ballot[2];
    const int nhfb = (f.width + 63) >> 6, nvfb = (f.height + 63) >> 6, nfb = nhfb * nvfb;
    const int cs = f.bit_depth > 8 ? f.bit_depth - 8 : 0;
    const int w8 = (f.width + 7) >> 3, h8 = (f.height + 7) >> 3;
    for (int work = blockIdx.x; work < nfb * 3; work += gridDim.x) {
        const int fb = work / 3, pli = work - fb * 3;
        const int fbr = fb / nhfb, fbc = fb - fbr * nhfb;
        const int sidx = fb_strength_idx[fb];
        if (sidx < 0) continue;  // uniform per CTA
        const int sv = pli ? uv_strength[sidx] : y_strength[sidx];
        const int pri = (sv / 4) << cs;
        int sec = sv % 4;
        sec = (sec + (sec == 3)) << cs;
        if (!(pri || sec)) continue;
        __syncthreads();
        const int count = cdef_fb_list(skip8x8, dir_in, var_in, fb, fbr, fbc, w8, h8, s_list, s_dir, s_var, s_ballot);
        if (count == 0) continue;
        const int dec = pli ? 1 : 0;
        const PIX* rec = (const PIX*)(pli == 0 ? f.recon_y : (pli == 1 ? f.recon_cb : f.recon_cr));
        PIX* out = pli == 0 ? out_y : (pli == 1 ? out_cb : out_cr);
        const int rstride = pli ? f.recon_stride_c : f.recon_stride_y, ostride = pli ? out_stride_c : out_stride_y;
        const int pw = f.width >> dec, ph = f.height >> dec, fbs = 64 >> dec;
        const int hsz = min(fbs, pw - fbc * fbs), vsz = min(fbs, ph - fbr * fbs);
        stage_cdef_tile<PIX>(tile, rec, rstride, fbr, fbc, nvfb, nhfb, fbs, vsz, hsz);  // ends with a barrier
        PIX* out_fb = out + (size_t)fbr * fbs * ostride + fbc * fbs;
        const int damping = f.damping + cs - (pli != 0);
        const size_t row_bytes = (size_t)(8 >> dec) * sizeof(PIX);  // rows start at multiples of it within a picture row
        const bool wide = (((size_t)out | (size_t)ostride * sizeof(PIX)) & (row_bytes - 1)) == 0;
        if (pli == 0) cdef_apply_fb<8, PIX>(tile, out_fb, ostride, wide, count, pri, sec, damping, cs, s_list, s_dir, s_var);
        else cdef_apply_fb<4, PIX>(tile, out_fb, ostride, wide, count, pri, sec, damping, cs, s_list, s_dir, s_var);
    }
}

}  // namespace b200

using namespace b200;

// ---- T1 ------------------------------------------------------------------------------------------
static void find_dir_t1(const uint16_t* const* imgs, int n, int stride, int coeff_shift, int* dirs, int* vars) {
    require_ready();
    LaneGuard l;
    const size_t blk = 7 * (size_t)stride + 8;
    size_t o_img = l->alloc(n * blk * 2), o_off = l->alloc(n * 4);
    size_t in_end = l->used;
    size_t o_out = l->alloc(n * 8);
    for (int i = 0; i < n; i++) {
        memcpy(l->h<uint16_t>(o_img) + i * blk, imgs[i], blk * 2);
        l->h<int>(o_off)[i] = (int)(i * blk);
    }
    l->h2d(0, in_end);
    find_dir_kernel<<<1, 32, 0, l->stream>>>(l->d<uint16_t>(o_img), stride, coeff_shift, n, l->d<int>(o_off), l->d<int>(o_out));
    B200_LAUNCH_CHECK();
    l->d2h(o_out, n * 8);
    l->sync();
    for (int i = 0; i < n; i++) {
        dirs[i] = l->h<int>(o_out)[2 * i];
        vars[i] = l->h<int>(o_out)[2 * i + 1];
    }
}

extern "C" uint8_t svt_b200_aom_cdef_find_dir(const uint16_t* img, int32_t stride, int32_t* var, int32_t coeff_shift) {
    int d, v;
    find_dir_t1(&img, 1, stride, coeff_shift, &d, &v);
    *var = v;
    return (uint8_t)d;
}
extern "C" void svt_b200_aom_cdef_find_dir_dual(const uint16_t* img1, const uint16_t* img2, int stride, int32_t* var1,
                                                int32_t* var2, int32_t coeff_shift, uint8_t* out1, uint8_t* out2) {
    const uint16_t* imgs[2] = {img1, img2};
    int d[2], v[2];
    find_dir_t1(imgs, 2, stride, coeff_shift, d, v);
    *var1 = v[0];
    *var2 = v[1];
    *out1 = (uint8_t)d[0];
    *out2 = (uint8_t)d[1];
}

extern "C" void svt_b200_cdef_filter_block(uint8_t* dst8, uint16_t* dst16, int32_t dstride, const uint16_t* in,
                                           int32_t pri_strength, int32_t sec_strength, int32_t dir, int32_t pri_damping,
                                           int32_t sec_damping, int32_t bsize, int32_t coeff_shift, uint8_t subsampling_factor) {
    require_ready();
    // BlockSize: BLOCK_4X4=0, 4X8=1, 8X4=2, 8X8=3 (definitions.h:765-768)
    const int h = 4 << (bsize == 3 || bsize == 1), w = 4 << (bsize == 3 || bsize == 2);
    const int S = 144;  // CDEF_BSTRIDE (cdef.h:35)
    LaneGuard l;
    const int p = w + 4;
    size_t o_in = l->alloc((size_t)p * (h + 4) * 2);
    size_t in_end = l->used;
    size_t o_out = l->alloc((size_t)w * h * 2);
    for (int r = -2; r < h + 2; r++) memcpy(l->h<uint16_t>(o_in) + (r + 2) * p, in + r * S - 2, p * 2);
    l->h2d(0, in_end);
    filter_block_kernel<<<1, 64, 0, l->stream>>>(l->d<uint16_t>(o_in), w, h, pri_strength, sec_strength, dir, pri_damping, sec_damping,
                                                 coeff_shift, subsampling_factor ? subsampling_factor : 1, l->d<uint16_t>(o_out));
    B200_LAUNCH_CHECK();
    l->d2h(o_out, (size_t)w * h * 2);
    l->sync();
    const uint16_t* o = l->h<uint16_t>(o_out);
    const int subs = subsampling_factor ? subsampling_factor : 1;
    for (int i = 0; i < h; i += subs)
        for (int j = 0; j < w; j++) {
            if (dst8) dst8[i * dstride + j] = (uint8_t)o[i * w + j];
            else dst16[i * dstride + j] = o[i * w + j];
        }
}

extern "C" void svt_b200_aom_copy_rect8_8bit_to_16bit(uint16_t* dst, int32_t dstride, const uint8_t* src, int32_t sstride,
                                                      int32_t v, int32_t h) {
    // A widening host-to-host copy: the T2 path performs this conversion while staging the tile on
    // the device (stage_cdef_tile); the T1 form has no device work to do.
    for (int i = 0; i < v; i++)
        for (int j = 0; j < h; j++) dst[i * dstride + j] = src[i * sstride + j];
}

template <typename T>
static uint64_t cdef_dist_t1(const T* dst, int32_t dstride, const T* src, const uint8_t* dlist, int32_t count, int32_t bsize,
                             int32_t coeff_shift, int32_t pli, uint8_t subs) {
    require_ready();
    if (count <= 0) return 0;
    const int bh_l2 = (bsize == 3 || bsize == 1) ? 3 : 2, bw_l2 = (bsize == 3 || bsize == 2) ? 3 : 2;
    int maxby = 0, maxbx = 0;
    for (int i = 0; i < count; i++) {
        if (dlist[2 * i] > maxby) maxby = dlist[2 * i];
        if (dlist[2 * i + 1] > maxbx) maxbx = dlist[2 * i + 1];
    }
    const size_t rows = ((size_t)maxby + 1) << bh_l2, cols = ((size_t)maxbx + 1) << bw_l2;
    const size_t dbytes = ((rows - 1) * dstride + cols) * sizeof(T), sbytes = ((size_t)count << (bw_l2 + bh_l2)) * sizeof(T);
    LaneGuard l;
    size_t o_d = l->alloc(dbytes), o_s = l->alloc(sbytes), o_l = l->alloc(2 * count);
    size_t in_end = l->used;
    size_t o_o = l->alloc(8);
    memcpy(l->h<uint8_t>(o_d), dst, dbytes);
    memcpy(l->h<uint8_t>(o_s), src, sbytes);
    memcpy(l->h<uint8_t>(o_l), dlist, 2 * count);
    l->h2d(0, in_end);
    cdef_dist_kernel<T><<<1, 64, 0, l->stream>>>(l->d<T>(o_d), dstride, l->d<T>(o_s), l->d<uint8_t>(o_l), count, bw_l2, bh_l2,
                                                 coeff_shift, pli, subs ? subs : 1, l->d<unsigned long long>(o_o));
    B200_LAUNCH_CHECK();
    l->d2h(o_o, 8);
    l->sync();
    return *l->h<uint64_t>(o_o);
}
extern "C" uint64_t svt_b200_compute_cdef_dist_16bit(const uint16_t* dst, int32_t dstride, const uint16_t* src,
                                                     const SvtB200CdefList* dlist, int32_t cdef_count, uint8_t bsize,
                                                     int32_t coeff_shift, int32_t pli, uint8_t subsampling_factor) {
    return cdef_dist_t1<uint16_t>(dst, dstride, src, (const uint8_t*)dlist, cdef_count, bsize, coeff_shift, pli, subsampling_factor);
}
extern "C" uint64_t svt_b200_compute_cdef_dist_8bit(const uint8_t* dst8, int32_t dstride, const uint8_t* src8,
                                                    const SvtB200CdefList* dlist, int32_t cdef_count, uint8_t bsize,
                                                    int32_t coeff_shift, int32_t pli, uint8_t subsampling_factor) {
    return cdef_dist_t1<uint8_t>(dst8, dstride, src8, (const uint8_t*)dlist, cdef_count, bsize, coeff_shift, pli, subsampling_factor);
}

extern "C" uint64_t svt_b200_search_one_dual(int* lev0, int* lev1, int nb_strengths, uint64_t** mse[2], int sb_count,
                                             int start_gi, int end_gi) {
    require_ready();
    const int ng = end_gi;
    LaneGuard l;
    size_t o_m0 = l->alloc((size_t)sb_count * ng * 8), o_m1 = l->alloc((size_t)sb_count * ng * 8), o_lv = l->alloc(2 * 64 * 4);
    size_t in_end = l->used;
    size_t o_o = l->alloc(24);
    for (int i = 0; i < sb_count; i++) {
        memcpy(l->h<uint64_t>(o_m0) + (size_t)i * ng, mse[0][i], (size_t)ng * 8);
        memcpy(l->h<uint64_t>(o_m1) + (size_t)i * ng, mse[1][i], (size_t)ng * 8);
    }
    memcpy(l->h<int>(o_lv), lev0, nb_strengths * 4);
    memcpy(l->h<int>(o_lv) + 64, lev1, nb_strengths * 4);
    l->h2d(0, in_end);
    search_one_dual_kernel<<<1, 256, (size_t)ng * ng * 8, l->stream>>>(l->d<unsigned long long>(o_m0), l->d<unsigned long long>(o_m1),
                                                                     sb_count, ng, l->d<int>(o_lv), l->d<int>(o_lv) + 64, nb_strengths,
                                                                     start_gi, l->d<unsigned long long>(o_o));
    B200_LAUNCH_CHECK();
    l->d2h(o_o, 24);
    l->sync();
    const uint64_t* o = l->h<uint64_t>(o_o);
    lev0[nb_strengths] = (int)o[1];
    lev1[nb_strengths] = (int)o[2];
    return o[0];
}

// ---- T2 ------------------------------------------------------------------------------------------
extern "C" int svt_b200_cdef_search_frame_dev(const SvtB200CdefFrame* frame, const uint8_t* d_skip8x8, const int* d_strengths_y,
                                              const int* d_strengths_uv, int n_strengths, uint64_t* d_mse, uint8_t* d_dir,
                                              int32_t* d_var, void* stream) {
    require_ready();
    if (!frame || n_strengths <= 0 || n_strengths > 64) return SVT_B200_ERR_BAD_ARG;
    const int nfb = ((frame->width + 63) >> 6) * ((frame->height + 63) >> 6);
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = ((frame->width + 7) >> 3) * ((frame->height + 7) >> 3);
    B200_CUDA_CHECK(cudaMemsetAsync(d_mse + (size_t)nfb * n_strengths, 0, (size_t)nfb * n_strengths * sizeof(uint64_t), st));
    if (frame->bit_depth > 8) {
        cdef_dir_kernel<uint16_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, d_dir, d_var);
        B200_LAUNCH_CHECK();
        cdef_search_kernel<uint16_t><<<grid_for((long long)nfb * 3, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_strengths_y, d_strengths_uv, n_strengths,
                                                                                (unsigned long long*)d_mse, d_dir, d_var);
    } else {
        cdef_dir_kernel<uint8_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, d_dir, d_var);
        B200_LAUNCH_CHECK();
        cdef_search_kernel<uint8_t><<<grid_for((long long)nfb * 3, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_strengths_y, d_strengths_uv, n_strengths,
                                                                               (unsigned long long*)d_mse, d_dir, d_var);
    }
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

static uint8_t*   g_cdef_dir = nullptr;  // direction/variance scratch for apply calls that do not bring their own
static int32_t*   g_cdef_var = nullptr;
static size_t     g_cdef_cap = 0;
static std::mutex g_cdef_mu;
static ResetHook  g_cdef_reset([] { std::lock_guard<std::mutex> lk(g_cdef_mu); g_cdef_dir = nullptr; g_cdef_var = nullptr; g_cdef_cap = 0; });

extern "C" int svt_b200_cdef_apply_frame_dev(const SvtB200CdefFrame* frame, const uint8_t* d_skip8x8, const int8_t* d_fb_strength_idx,
                                             const int* d_y_strength, const int* d_uv_strength, const uint8_t* d_dir,
                                             const int32_t* d_var, void* d_out_y, void* d_out_cb, void* d_out_cr, int out_stride_y,
                                             int out_stride_c, void* stream) {
    require_ready();
    if (!frame || ((d_dir == nullptr) != (d_var == nullptr))) return SVT_B200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int nfb = ((frame->width + 63) >> 6) * ((frame->height + 63) >> 6);
    const int nblk = ((frame->width + 7) >> 3) * ((frame->height + 7) >> 3);
    std::unique_lock<std::mutex> lk(g_cdef_mu, std::defer_lock);
    if (!d_dir) {  // calls that share the scratch are serialised on the host (the stream orders the device side)
        lk.lock();
        if ((size_t)nfb > g_cdef_cap) {
            g_cdef_cap = (size_t)nfb * 2;
            g_cdef_dir = (uint8_t*)scratch_alloc(g_cdef_cap * 64);
            g_cdef_var = (int32_t*)scratch_alloc(g_cdef_cap * 64 * 4);
        }
        if (frame->bit_depth > 8) cdef_dir_kernel<uint16_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, g_cdef_dir, g_cdef_var);
        else cdef_dir_kernel<uint8_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, g_cdef_dir, g_cdef_var);
        B200_LAUNCH_CHECK();
        d_dir = g_cdef_dir;
        d_var = g_cdef_var;
    }
    if (frame->bit_depth > 8)
        cdef_apply_kernel<uint16_t><<<grid_for((long long)nfb * 3, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_fb_strength_idx, d_y_strength, d_uv_strength,
                                                                               d_dir, d_var, (uint16_t*)d_out_y, (uint16_t*)d_out_cb,
                                                                               (uint16_t*)d_out_cr, out_stride_y, out_stride_c);
    else
        cdef_apply_kernel<uint8_t><<<grid_for((long long)nfb * 3, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_fb_strength_idx, d_y_strength, d_uv_strength,
                                                                              d_dir, d_var, (uint8_t*)d_out_y, (uint8_t*)d_out_cb,
                                                                              (uint8_t*)d_out_cr, out_stride_y, out_stride_c);
    B200_LAUNCH_CHECK();
    if (lk.owns_lock()) B200_CUDA_CHECK(cudaStreamSynchronize(st));  // the scratch is free again when the call returns
    return SVT_B200_OK;
}
