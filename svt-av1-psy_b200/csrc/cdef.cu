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
// thread per block, the 64 pixels in registers).  Search and apply run one 128-thread CTA per 64x64 filter
// block and luma, and one per filter block and both chroma planes (which share the block list, directions,
// strengths and damping): the padded 16-bit tile of each plane, (fbs + 6) x (fbs + 16) for a filter block of
// fbs x fbs pixels in that plane, is staged in shared memory once, in words of 8 pixels, and a thread owns a row
// segment of one block (luma: a processed 8-pixel row of an 8x8, chroma: a 4-pixel row of a 4x4 in Cb and the
// same row in Cr), so the tap offsets of the block's direction and the per-strength constants are built once per
// segment, not per pixel.  The search evaluates two pixels per step (luma: neighbours, chroma: one per plane).  A
// pixel's 12 taps are fetched once per direction, as magnitudes packed two per register with their signs folded
// into the dot-product weights, and shared by all candidate strengths; the filter sum is separable into a primary and a
// secondary half, each evaluated once per distinct strength value with native packed 16-bit min/max/add
// and 2-way dot-product instructions.  What each candidate strength adds per pixel (rounding, clamp, moments) runs
// on both pixels of a step at once, in packed 16-bit halves, with the clamp bounds and the pixels' part of the
// rounding formed once per pixel; at 8 bit the luma moments are IDP.4A byte products.  The search sums a segment's
// distortion moments in registers (up to kGChunk strengths at a time), combines the few segments of a block with shuffles and stores them once
// per (block, strength); the source's moments and those of strength code 0 (the unfiltered block) are not
// recomputed per strength.  The luma distortion's double-precision formula is evaluated with
// round-to-nearest intrinsics in the reference's operand order (FMA contraction is disabled for the whole
// library), which makes it IEEE-identical to the C code.
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
// 0x7f7f, |differences| <= 0x7f7f): the magnitudes |tap - x|, the dp2a weights of the taps with the sign of
// tap - x folded in, and the min / max over the taps that are inside the picture.  Pairs: 0 = primary k=0 (+,-),
// 1 = primary k=1, 2..3 = secondary k=0, 4..5 = secondary k=1.  The packed min/max/add instructions used
// (VIMNMX.16x2, VIADD.16x2, VIADDMNMX.16x2) are native.
struct CdefTaps {
    uint32_t ad[6];  // |differences|
    uint32_t wp[2];  // signed dp2a weights of pairs 0-1 (bytes 0-1: pair 0, 2-3: pair 1): [0] weights 4, 2; [1] 3, 3
    uint32_t w23;    // signed dp2a weights of pairs 2-3 (2 each)
    uint32_t w45;    // signed dp2a weights of pairs 4-5 (1 each)
    uint32_t mn2;    // min over the pixel and its taps, per half (CDEF_VERY_LARGE never wins)
    uint32_t mx2;    // max over the pixel and its taps, per half, each value plus kMxBias (mod 2^16)
};
// The maximum over the taps is taken over the halves plus kMxBias (mod 2^16), which maps CDEF_VERY_LARGE to 0 and
// keeps pixels (<= 4095) in order above it: the sentinel is never the maximum.
constexpr uint32_t kMxBias = 0x10000u - kVeryLarge;
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
// one byte per 16-bit half of a and b: 0xff where that half is negative (PRMT with sign replication)
__device__ __forceinline__ uint32_t cdef_sign_bytes(uint32_t a, uint32_t b) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, 0xFDB9;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
// weights w (bytes) where the sign byte is 0, -w (bytes nw) where it is 0xff
__device__ __forceinline__ uint32_t cdef_signed_weights(uint32_t sign, uint32_t w, uint32_t nw) { return (w & ~sign) | (nw & sign); }
__device__ __forceinline__ void cdef_load_taps(const uint16_t* in, const int (&o)[6], int x, CdefTaps& T) {
    const uint32_t xx = (uint32_t)x * 0x10001u, nxx = __vneg2(xx);
    uint32_t       mx2 = __vadd2(xx, kMxBias * 0x10001u), mn2 = xx, d[6];
#pragma unroll
    for (int pair = 0; pair < 6; pair++) {
        const uint32_t p = (uint32_t)in[o[pair]] | ((uint32_t)in[-o[pair]] << 16);
        d[pair]    = __vadd2(p, nxx);
        T.ad[pair] = __vmaxu2(p, xx) - __vminu2(p, xx);  // halves are >= 0: no borrow between them
        mx2 = __vmaxu2(mx2, __vadd2(p, kMxBias * 0x10001u));
        mn2 = __vminu2(mn2, p);
    }
    const uint32_t sp = cdef_sign_bytes(d[0], d[1]), s23 = cdef_sign_bytes(d[2], d[3]), s45 = cdef_sign_bytes(d[4], d[5]);
    T.wp[0] = cdef_signed_weights(sp, 0x02020404u, 0xfefefcfcu);
    T.wp[1] = cdef_signed_weights(sp, 0x03030303u, 0xfdfdfdfdu);
    T.w23   = cdef_signed_weights(s23, 0x02020202u, 0xfefefefeu);
    T.w45   = cdef_signed_weights(s45, 0x01010101u, 0xffffffffu);
    T.mn2 = mn2;
    T.mx2 = mx2;
}
// What constrain() (cdef.c:85-93) needs of a strength t at a damping: the threshold plus one in both halves, the
// shift max(0, damping - msb(t)), the mask that keeps the shifted high half out of the low one, and which primary
// weights apply (cdef_pri_taps[(t >> coeff_shift) & 1], CdefTaps::wp).  t = 0 gives a zero threshold, which
// constrains every tap to zero.
__device__ __forceinline__ uint4 cdef_strength_consts(int t, int damping, int coeff_shift) {
    const int sh = max(0, damping - msb32((uint32_t)t));
    return make_uint4((uint32_t)(t + 1) * 0x10001u, (uint32_t)sh, (0xffffu >> sh) * 0x10001u, (uint32_t)((t >> coeff_shift) & 1));
}
// |constrain()| of the two taps of a pair: min(|d|, max(0, thr - (|d| >> shift))) = max(min(thr - t1, |d|), 0) with
// t1 = |d| >> shift, one VIADDMNMX: ~t1 = -t1 - 1 comes with the mask, and c.x = thr + 1.  The sign of d is in the
// weights the magnitude is multiplied by.
__device__ __forceinline__ uint32_t cdef_constrain2(const CdefTaps& T, int pair, const uint4& c) {
    const uint32_t nt1 = ~((T.ad[pair] >> c.y) & c.z);
    return __viaddmin_s16x2_relu(c.x, nt1, T.ad[pair]);
}
// The sum splits into a primary part (4 taps, depends on the primary strength only) and a secondary part
// (8 taps, depends on the secondary strength only): candidate strengths that share one of the two share
// that half of the work.  The reference accumulates in int16; |sum| <= 2*(4+2)*240 + 4*(2+1)*64 for 12-bit
// content, so the int32 sum is the same number.
__device__ __forceinline__ int cdef_primary_sum(const CdefTaps& T, const uint4& c) {
    const int w = (int)(c.w ? T.wp[1] : T.wp[0]);
    return __dp2a_hi((int)cdef_constrain2(T, 1, c), w, __dp2a_lo((int)cdef_constrain2(T, 0, c), w, 0));
}
__device__ __forceinline__ int cdef_secondary_sum(const CdefTaps& T, const uint4& c) {
    const int s = __dp2a_hi((int)cdef_constrain2(T, 3, c), (int)T.w23, __dp2a_lo((int)cdef_constrain2(T, 2, c), (int)T.w23, 0));
    return __dp2a_hi((int)cdef_constrain2(T, 5, c), (int)T.w45, __dp2a_lo((int)cdef_constrain2(T, 4, c), (int)T.w45, s));
}
__device__ __forceinline__ int cdef_finish_px(const CdefTaps& T, int x, int sum) {
    const int mn = (int)min(T.mn2 & 0xffffu, T.mn2 >> 16), mx = (int)max(T.mx2 & 0xffffu, T.mx2 >> 16) - (int)kMxBias;
    const int y = x + ((8 + sum - (sum < 0)) >> 4);
    return y < mn ? mn : (y > mx ? mx : y);
}

// The finish of two pixels at once, pixel A in the low 16-bit halves and pixel B in the high ones.  Every value is
// kept >= 0 in its half by offsets: a filtered pixel is y + kYOff (y + round(sum) may lie below 0 before the clamp),
// and a filter sum arrives as sum + kSumOff.  With u = sum + 0x8007, bit 15 of u is set iff sum >= -7, and
// (u + that bit) >> 4 = ((8 + sum - (sum < 0)) >> 4) + 0x800: the two agree for sum >= 0 and sum < -7, and both
// roundings give 0 for -7 <= sum < 0.  |sum| <= 3648 (cdef_primary_sum), so no half leaves [0, 2^16).
constexpr uint32_t kYOff2   = 0x08000800u;  // 0x800 in both halves
constexpr uint32_t kSumOff2 = 0x80078007u;
struct CdefPx2 {
    uint32_t x;       // the two pixels; at 8 bit 16 x (which fits its half), so it is added before the shift
    uint32_t mn, mx;  // the clamp bounds plus kYOff
};
template <typename PIX>
__device__ __forceinline__ CdefPx2 cdef_px2(const CdefTaps& A, const CdefTaps& B, int xa, int xb) {
    CdefPx2 P;
    const uint32_t x2 = (uint32_t)xa | ((uint32_t)xb << 16);
    P.x  = sizeof(PIX) == 1 ? x2 << 4 : x2;
    P.mn = __vminu2(__byte_perm(A.mn2, B.mn2, 0x5410), __byte_perm(A.mn2, B.mn2, 0x7632)) + kYOff2;
    P.mx = __vadd2(__vmaxu2(__byte_perm(A.mx2, B.mx2, 0x5410), __byte_perm(A.mx2, B.mx2, 0x7632)), ((0x800u - kMxBias) & 0xffffu) * 0x10001u);
    return P;
}
// both halves of one filter sum per pixel (sum_a, sum_b: int32 as cdef_primary_sum / cdef_secondary_sum give them)
__device__ __forceinline__ uint32_t cdef_pack2(int sum_a, int sum_b) { return __byte_perm((uint32_t)sum_a, (uint32_t)sum_b, 0x5410); }
// the two filtered pixels plus kYOff from u = the packed filter sums plus kSumOff2
template <typename PIX>
__device__ __forceinline__ uint32_t cdef_finish2(const CdefPx2& P, uint32_t u) {
    const uint32_t t = (u >> 15) & 0x00010001u;
    const uint32_t w = sizeof(PIX) == 1 ? ((u + t + P.x) >> 4) & 0x0fff0fffu : (((u + t) >> 4) & 0x0fff0fffu) + P.x;
    return __vminu2(__vmaxu2(w, P.mn), P.mx);
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
constexpr int kGChunk    = 6;    // candidate strengths whose moments a search thread keeps in registers at once (every preset lists 6)
constexpr int kTPC       = 48;   // chroma tile pitch in uint16 (32 + 2*8, rows 16-B aligned)
constexpr int kTileC     = (32 + 6) * kTPC;  // one chroma tile; the Cr tile follows the Cb tile
static_assert(2 * kTileC <= kTileRows * kTP, "both chroma tiles fit where the luma tile goes");

// 8 pixels at p as 8 uint16 (p aligned to 8 pixels)
template <typename PIX>
__device__ __forceinline__ uint4 cdef_load_word8(const PIX* p) {
    if (sizeof(PIX) == 1) {
        const uint2 w = *reinterpret_cast<const uint2*>(p);
        return make_uint4(__byte_perm(w.x, 0, 0x4140), __byte_perm(w.x, 0, 0x4342), __byte_perm(w.y, 0, 0x4140), __byte_perm(w.y, 0, 0x4342));
    }
    return *reinterpret_cast<const uint4*>(p);
}

// The padded 16-bit tiles of NP planes of one filter block that share a geometry: luma (NP = 1, 64x64, pitch kTP),
// or Cb and Cr (NP = 2, 32x32 each, pitch kTPC, the Cr tile kTileC elements after the Cb tile).  Tile origin (row 3,
// col 8) = first pixel of the filter block; everything outside the copied rectangle is CDEF_VERY_LARGE
// (cdef_process.c:211-230).  Only the (fbs + 6) x (fbs + 16) pixels the filter can read are written.  A thread moves
// words of 8 pixels (one 8-byte load and PRMT widening at 8 bit, one 16-byte load at 16 bit, one 16-byte store), kLd
// words' loads in flight before the first store.  A word starts at a multiple of 8 pixels in the plane; a plane
// whose origin or pitch is not aligned to that, and a word the copied rectangle cuts, move pixel by pixel.
template <typename PIX, int NP>
__device__ void stage_cdef_tiles(uint16_t* tile, const PIX* plane0, const PIX* plane1, int stride, int fbr, int fbc, int nvfb, int nhfb,
                                 int vsz, int hsz) {
    constexpr int FBS = 64 / NP, TP = NP == 1 ? kTP : kTPC, WPR = (FBS + 16) / 8, PER = (FBS + 6) * WPR, kLd = 4;
    const int yoff = 3 * (fbr != 0), xoff = 8 * (fbc != 0);
    const int ysize = vsz + 3 * (fbr + 1 < nvfb) + yoff, xsize = hsz + 8 * (fbc + 1 < nhfb) + xoff;
    const int py0 = fbr * FBS - yoff, px0 = fbc * FBS - xoff;
    constexpr size_t kAl = 8 * sizeof(PIX) - 1;
    const unsigned word = ((((size_t)plane0 | (size_t)stride * sizeof(PIX)) & kAl) == 0) |
                          (((((size_t)plane1 | (size_t)stride * sizeof(PIX)) & kAl) == 0) << 1);
    constexpr uint32_t kVL2 = (uint32_t)kVeryLarge * 0x10001u;
    for (int i0 = threadIdx.x; i0 < NP * PER; i0 += kLd * kT2Threads) {
        uint4 v[kLd];
#pragma unroll
        for (int k = 0; k < kLd; k++) {
            const int i = i0 + k * kT2Threads, p = NP == 2 && i >= PER, q = i - p * PER;
            const int r = q / WPR, c = (q - r * WPR) * 8;
            const int rr = r - (3 - yoff), cc = c - (8 - xoff);
            v[k] = make_uint4(kVL2, kVL2, kVL2, kVL2);
            if (i < NP * PER && rr >= 0 && rr < ysize && cc + 8 > 0 && cc < xsize) {
                const PIX* row = (p ? plane1 : plane0) + (size_t)(py0 + rr) * stride + px0;
                if (((word >> p) & 1) && cc >= 0 && cc + 8 <= xsize) {
                    v[k] = cdef_load_word8(row + cc);
                } else {
                    uint32_t e[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) e[j] = cc + j >= 0 && cc + j < xsize ? (uint32_t)row[cc + j] : (uint32_t)kVeryLarge;
                    v[k] = make_uint4(e[0] | e[1] << 16, e[2] | e[3] << 16, e[4] | e[5] << 16, e[6] | e[7] << 16);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < kLd; k++) {
            const int i = i0 + k * kT2Threads, p = NP == 2 && i >= PER, q = i - p * PER;
            const int r = q / WPR, c = (q - r * WPR) * 8;
            if (i < NP * PER) *reinterpret_cast<uint4*>(tile + p * kTileC + r * TP + c) = v[k];
        }
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

// Phase split of the search (tools/profile_cdef.py): built with B200_CDEF_PHASES=1, thread 0 of every CTA adds the
// clock64() cycles between consecutive stamps to g_cdef_phase[item][phase] (item 0 = luma, 1 = chroma; phases: table,
// block list, staging, segment pass 0, pass 1, shuffle combine and source moments, wait for the other segments,
// distortion warps), and [item][8] counts the items.  Off in the library as shipped: the stamps compile to nothing.
#ifndef B200_CDEF_PHASES
#define B200_CDEF_PHASES 0
#endif
constexpr int kCdefPhases = 8;
#if B200_CDEF_PHASES
__device__ unsigned long long g_cdef_phase[2][kCdefPhases + 1];
#endif
__device__ __forceinline__ void cdef_phase(int item, int k, long long& t) {
#if B200_CDEF_PHASES
    if (threadIdx.x == 0) {
        const long long now = clock64();
        if (k >= 0) atomicAdd(&g_cdef_phase[item][k], (unsigned long long)(now - t));
        t = now;
    }
#endif
}

// One chunk of candidate strengths (CTA-uniform description) as the search's threads see it.
struct CdefChunk {
    int      sv[kGChunk];  // strength codes, -1 = not tested (also past the end of the list)
    unsigned todo[2];      // pass 0: taps along the block's direction (a primary part, or code 0); pass 1: along direction 0
    unsigned pri_new;      // pass-0 strengths whose primary code differs from the previous one with a primary part
    unsigned secs[2];      // per pass: bit c set when secondary code c (1..3) occurs
    unsigned zero;         // strength code 0 (the unfiltered block)
};

// Moments of one row segment for every strength of `todo`, the taps along one direction.  Luma (BS = 8 pixels at
// `in`, source at `o_row`) accumulates sum y, y^2, y*src into a0, a1, a2; chroma (BS = 4) sum (src - y)^2 of the Cb
// row (`in`, `o_row`) into a0 and of the Cr row (`in2`, `o_row2`) into a1.  Two pixels are evaluated per step (luma:
// two neighbours, chroma: the same pixel of both planes), so that their tap loads and strength chains interleave and
// each strength's constants are read once for both.  Taps are loaded once per pixel and shared by all strengths; the
// primary half is recomputed only when the primary strength changes and the secondary half once per distinct
// secondary code.
template <int BS, typename PIX>
__device__ __forceinline__ void cdef_segment_pass(const uint16_t* in, const uint16_t* in2, const PIX* o_row, const PIX* o_row2,
                                                  const int (&off)[6], const CdefChunk& C, int pass, const int (&tadj)[kGChunk],
                                                  const uint4* tab, int cs, unsigned (&a0)[kGChunk], unsigned (&a1)[kGChunk],
                                                  unsigned (&a2)[kGChunk]) {
    const unsigned todo = C.todo[pass], pnew = pass ? 0u : C.pri_new, secs = C.secs[pass], zero = C.zero;
    constexpr int STEP = BS == 8 ? 2 : 1;
#pragma unroll 1
    for (int j = 0; j < BS; j += STEP) {
        const uint16_t* px[2] = {in + j, BS == 8 ? in + j + 1 : in2 + j};
        int      x[2];
        unsigned o[2];
        CdefTaps T[2];
#pragma unroll
        for (int k = 0; k < 2; k++) {
            x[k] = px[k][0];
            o[k] = BS == 8 ? o_row[j + k] : (k ? o_row2[j] : o_row[j]);
            cdef_load_taps(px[k], off, x[k], T[k]);
        }
        // what depends on the two pixels alone: the clamp bounds, the pixels in the rounding's form, and the source
        // operands of the moments (8-bit luma: both source bytes for IDP.4A; chroma: both sources plus kYOff)
        const CdefPx2  P  = cdef_px2<PIX>(T[0], T[1], x[0], x[1]);
        const uint32_t x0 = ((uint32_t)x[0] | ((uint32_t)x[1] << 16)) + kYOff2;  // code 0: the pixels themselves
        const uint32_t ob = BS == 8 ? (sizeof(PIX) == 1 ? o[0] | (o[1] << 8) : 0u) : (o[0] | (o[1] << 16)) + kYOff2;
        // secondary sums of codes 1, 2, 3 (strengths 1, 2, 4 << cs), packed, plus kSumOff2
        uint32_t s1 = kSumOff2, s2 = kSumOff2, s3 = kSumOff2;
        if (secs & 2) {
            const uint4 c = tab[1 << cs];
            s1 = __vadd2(cdef_pack2(cdef_secondary_sum(T[0], c), cdef_secondary_sum(T[1], c)), kSumOff2);
        }
        if (secs & 4) {
            const uint4 c = tab[2 << cs];
            s2 = __vadd2(cdef_pack2(cdef_secondary_sum(T[0], c), cdef_secondary_sum(T[1], c)), kSumOff2);
        }
        if (secs & 8) {
            const uint4 c = tab[4 << cs];
            s3 = __vadd2(cdef_pack2(cdef_secondary_sum(T[0], c), cdef_secondary_sum(T[1], c)), kSumOff2);
        }
        uint32_t psum = 0;  // packed primary sums of the current primary strength
#pragma unroll
        for (int gi = 0; gi < kGChunk; gi++) {
            if (!((todo >> gi) & 1)) continue;  // CTA-uniform
            if ((pnew >> gi) & 1) {
                const uint4 c = tab[tadj[gi]];
                psum = cdef_pack2(cdef_primary_sum(T[0], c), cdef_primary_sum(T[1], c));
            }
            const int      sc = C.sv[gi] & 3;
            const uint32_t ss = sc & 2 ? (sc & 1 ? s3 : s2) : (sc & 1 ? s1 : kSumOff2);
            // code 0 leaves the pixel unchanged (sum = 0, and x lies inside [min, max] of its own neighbourhood)
            const uint32_t y = (zero >> gi) & 1 ? x0 : cdef_finish2<PIX>(P, __vadd2(psum, ss));  // both pixels plus kYOff
            if (BS == 8 && sizeof(PIX) == 1) {
                // pixels <= 255: the low byte of each half is the pixel (kYOff has none), and every product fits IDP.4A
                const uint32_t yb = __byte_perm(y, 0, 0x4420);
                a0[gi] = __dp4a(yb, 0x01010101u, a0[gi]);
                a1[gi] = __dp4a(yb, yb, a1[gi]);
                a2[gi] = __dp4a(yb, ob, a2[gi]);
            } else if (BS == 8) {
                const uint32_t yy = y - kYOff2, ya = yy & 0xffffu, yb = yy >> 16;
                a0[gi] = __dp2a_lo(yy, 0x0101u, a0[gi]);
                a1[gi] += ya * ya + yb * yb;
                a2[gi] += ya * o[0] + yb * o[1];
            } else {
                const uint32_t e = __vsub2(ob, y);  // Cb and Cr errors, signed halves
                const int      ea = (int)(int16_t)(e & 0xffffu), eb = (int)e >> 16;
                a0[gi] += (unsigned)(ea * ea);
                a1[gi] += (unsigned)(eb * eb);
            }
        }
    }
}

// The strength search of one filter block in luma (BS = 8) or in both chroma planes (BS = 4): every thread owns
// processed row segments (luma: one 8-pixel row of an 8x8, chroma: one 4-pixel row of the 4x4 in Cb and the same
// row in Cr), so tap offsets and strength constants are built once per segment, and only the R threads of a block
// combine their moments, by shuffles.  Their sums go to shared memory once per (block, strength); warps then turn
// them into distortions (luma: the psy formula on the five moments, chroma: Cb + Cr) and sum them over the blocks.
template <int BS, typename PIX>
__device__ __forceinline__ void cdef_search_fb(const uint16_t* tile, const uint4* tab, const PIX* src, const PIX* src2, int sstride,
                                               const int* strengths, int n_strengths, int count, int subs, int cs, const uint8_t* s_list,
                                               const uint8_t* s_dir, const int* s_var, unsigned (*s_mom)[3][64], unsigned (*s_src)[64],
                                               unsigned long long* mse_fb, long long& ph_t) {
    constexpr int TP = BS == 8 ? kTP : kTPC, IT = BS == 8 ? 0 : 1;
    const int R = BS / subs, nseg = count * R;  // processed rows per block (a power of two: R divides 32)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int g0 = 0; g0 < n_strengths; g0 += kGChunk) {
        const int ng = min(kGChunk, n_strengths - g0);
        CdefChunk C;
        C.todo[0] = C.todo[1] = C.pri_new = C.secs[0] = C.secs[1] = C.zero = 0;
        int last_pri = -1;
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
                C.zero |= 1u << gi;
            }
        }
        // code 0 needs no taps: it joins a pass that runs anyway
        if (C.todo[0] || !C.todo[1]) C.todo[0] |= C.zero;
        else C.todo[1] |= C.zero;
        const unsigned tested = C.todo[0] | C.todo[1];
        for (int s = threadIdx.x; s < ((nseg + 31) & ~31); s += kT2Threads) {  // whole warps stay in the loop (shuffles)
            const bool live = s < nseg;
            const int  bi = live ? s / R : 0, r = live ? s - bi * R : 0;
            const int  b = s_list[bi], by = b >> 3, bx = b & 7, row = BS * by + r * subs;
            const uint16_t* in     = tile + (3 + row) * TP + 8 + BS * bx;
            const PIX*      o_row  = src + (size_t)row * sstride + BS * bx;
            const PIX*      o_row2 = BS == 4 ? src2 + (size_t)row * sstride + BS * bx : o_row;
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
                cdef_tap_offsets(s_dir[b], TP, off);
                cdef_segment_pass<BS, PIX>(in, in + kTileC, o_row, o_row2, off, C, 0, tadj, tab, cs, a0, a1, a2);
            }
            cdef_phase(IT, 3, ph_t);
            if (C.todo[1]) {
                cdef_tap_offsets(0, TP, off);
                cdef_segment_pass<BS, PIX>(in, in + kTileC, o_row, o_row2, off, C, 1, tadj, tab, cs, a0, a1, a2);
            }
            cdef_phase(IT, 4, ph_t);
            const bool lead = live && r == 0;
#pragma unroll
            for (int gi = 0; gi < kGChunk; gi++) {
                if (!((tested >> gi) & 1)) continue;  // CTA-uniform
                for (int sh = R >> 1; sh > 0; sh >>= 1) {
                    a0[gi] += __shfl_xor_sync(0xffffffffu, a0[gi], sh);
                    a1[gi] += __shfl_xor_sync(0xffffffffu, a1[gi], sh);
                    if (BS == 8) a2[gi] += __shfl_xor_sync(0xffffffffu, a2[gi], sh);
                }
                if (lead) {
                    s_mom[gi][0][bi] = a0[gi];
                    s_mom[gi][1][bi] = a1[gi];
                    if (BS == 8) s_mom[gi][2][bi] = a2[gi];
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
            cdef_phase(IT, 5, ph_t);
        }
        __syncthreads();
        cdef_phase(IT, 6, ph_t);
        // per strength: the blocks' distortions, summed by one warp
        for (int gi = warp; gi < ng; gi += kT2Threads / 32) {
            const int          sv = strengths[g0 + gi];
            unsigned long long acc = 0, acc2 = 0;  // luma; chroma: Cb, Cr
            if (sv >= 0)
                for (int bi = lane; bi < count; bi += 32) {
                    if (BS == 8) {
                        acc += cdef_dist_from_sums(s_mom[gi][0][bi], s_src[0][bi], s_mom[gi][1][bi], s_src[1][bi], s_mom[gi][2][bi], cs);
                    } else {
                        acc += s_mom[gi][0][bi];
                        acc2 += s_mom[gi][1][bi];
                    }
                }
#pragma unroll
            for (int sh = 16; sh > 0; sh >>= 1) {
                acc += __shfl_xor_sync(0xffffffffu, acc, sh);
                if (BS == 4) acc2 += __shfl_xor_sync(0xffffffffu, acc2, sh);
            }
            if (lane == 0) {
                // enc: mse_seg = (sum >> 2*coeff_shift) * subsampling_factor per plane, Cb and Cr added; an untested
                // chroma strength costs default_mse_uv*64 (once for both planes)
                const unsigned long long v = ((acc >> (2 * cs)) + (BS == 4 ? acc2 >> (2 * cs) : 0ull)) * (unsigned long long)subs;
                mse_fb[g0 + gi] = sv >= 0 ? v : (BS == 4 ? 1040400ull * 64ull : 0ull);
            }
        }
        __syncthreads();  // s_mom is reused by the next chunk
        cdef_phase(IT, 7, ph_t);
    }
}

// Work items of the search and apply grids: the chroma pair (Cb + Cr) of every filter block, then its luma.  A
// chroma item is the longer one in the search, so it is handed out first.
__device__ __forceinline__ bool cdef_item(int work, int nfb, int& fb) {
    const bool chroma = work < nfb;
    fb = chroma ? work : work - nfb;
    return chroma;
}

// Strength search: one CTA per filter block and luma, and one per filter block and both chroma planes.  Every
// mse[plane][fb][g] is written once.  Six CTAs per SM hold the segment loop without a spill (80 registers); the bound
// can be set at build time to measure others (DESIGN §5, §7).
#ifndef CDEF_SEARCH_CTAS
#define CDEF_SEARCH_CTAS 6
#endif
template <typename PIX>
__global__ void __launch_bounds__(kT2Threads, CDEF_SEARCH_CTAS)
cdef_search_kernel(SvtB200CdefFrame f, const uint8_t* __restrict__ skip8x8, const int* __restrict__ strengths_y,
                   const int* __restrict__ strengths_uv, int n_strengths, unsigned long long* __restrict__ mse /*[2][nfb][n_strengths]*/,
                   const uint8_t* __restrict__ dir_in /*[nfb][64]*/, const int* __restrict__ var_in /*[nfb][64]*/) {
    __shared__ __align__(16) uint16_t tile[kTileRows * kTP];  // the luma tile, or the Cb and Cr tiles
    __shared__ uint4    s_tab[256];  // cdef_strength_consts of every strength value at the damping of the item's planes
    __shared__ uint8_t  s_dir[64];
    __shared__ int      s_var[64];
    __shared__ uint8_t  s_list[64];
    __shared__ unsigned s_ballot[2];
    __shared__ unsigned s_mom[kGChunk][3][64];  // per strength, per listed block: luma sum y, y^2, y*src; chroma sum (src - y)^2 of Cb, Cr
    __shared__ unsigned s_src[2][64];           // per listed luma block: sum src, src^2
    const int nhfb = (f.width + 63) >> 6, nvfb = (f.height + 63) >> 6, nfb = nhfb * nvfb;
    const int cs = f.bit_depth > 8 ? f.bit_depth - 8 : 0;
    const int w8 = (f.width + 7) >> 3, h8 = (f.height + 7) >> 3;
    int tab_damping = -1;
    long long ph_t = 0;
    for (int work = blockIdx.x; work < nfb * 2; work += gridDim.x) {
        int        fb;
        const bool chroma = cdef_item(work, nfb, fb);
        const int  fbr = fb / nhfb, fbc = fb - fbr * nhfb;
        const int  damping = f.damping + cs - chroma;
        cdef_phase(chroma, -1, ph_t);
        __syncthreads();
        if (damping != tab_damping) {  // CTA-uniform; cdef_fb_list's barrier publishes the table
            // strengths reach (15 << 4) = 240 (primary, 12-bit), adjusted ones no more, secondary 4 << 4
            for (int i = threadIdx.x; i < 256; i += kT2Threads) s_tab[i] = cdef_strength_consts(i, damping, cs);
            tab_damping = damping;
        }
        cdef_phase(chroma, 0, ph_t);
#if B200_CDEF_PHASES
        if (threadIdx.x == 0) atomicAdd(&g_cdef_phase[chroma][kCdefPhases], 1ull);
#endif
        const int count = cdef_fb_list(skip8x8, dir_in, var_in, fb, fbr, fbc, w8, h8, s_list, s_dir, s_var, s_ballot);
        cdef_phase(chroma, 1, ph_t);
        unsigned long long* mse_fb = mse + (size_t)(chroma * nfb + fb) * n_strengths;
        if (count == 0) {
            for (int g = threadIdx.x; g < n_strengths; g += blockDim.x) mse_fb[g] = 0;
            continue;
        }
        if (!chroma) {
            const int hsz = min(64, f.width - fbc * 64), vsz = min(64, f.height - fbr * 64);
            const PIX* rec = (const PIX*)f.recon_y;
            stage_cdef_tiles<PIX, 1>(tile, rec, rec, f.recon_stride_y, fbr, fbc, nvfb, nhfb, vsz, hsz);  // ends with a barrier
            cdef_phase(0, 2, ph_t);
            const PIX* src_fb = (const PIX*)f.src_y + (size_t)fbr * 64 * f.src_stride_y + fbc * 64;
            const int  subs = min(f.subsampling_factor, 4);  // cdef_process.c:243-248
            cdef_search_fb<8, PIX>(tile, s_tab, src_fb, src_fb, f.src_stride_y, strengths_y, n_strengths, count, subs, cs, s_list, s_dir,
                                   s_var, s_mom, s_src, mse_fb, ph_t);
        } else {
            const int hsz = min(32, (f.width >> 1) - fbc * 32), vsz = min(32, (f.height >> 1) - fbr * 32);
            stage_cdef_tiles<PIX, 2>(tile, (const PIX*)f.recon_cb, (const PIX*)f.recon_cr, f.recon_stride_c, fbr, fbc, nvfb, nhfb, vsz, hsz);
            cdef_phase(1, 2, ph_t);
            const size_t o = (size_t)fbr * 32 * f.src_stride_c + fbc * 32;
            const int subs = min(f.subsampling_factor, 1);  // 4:2:0 chroma = BLOCK_4X4
            cdef_search_fb<4, PIX>(tile, s_tab, (const PIX*)f.src_cb + o, (const PIX*)f.src_cr + o, f.src_stride_c, strengths_uv, n_strengths,
                                   count, subs, cs, s_list, s_dir, s_var, s_mom, s_src, mse_fb, ph_t);
        }
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

// the filter of one filter block with one strength, in luma (BS = 8) or in both chroma planes (BS = 4, the Cr tile
// kTileC elements after the Cb tile): a thread per BS-pixel row of a block, in every plane of the item
template <int BS, typename PIX>
__device__ __forceinline__ void cdef_apply_fb(const uint16_t* tile, PIX* out_fb, PIX* out_fb2, int ostride, unsigned wide, int count,
                                              int pri, int sec, int damping, int cs, const uint8_t* s_list, const uint8_t* s_dir,
                                              const int* s_var) {
    constexpr int TP = BS == 8 ? kTP : kTPC, NP = BS == 8 ? 1 : 2;
    const uint4 csec = cdef_strength_consts(sec, damping, cs);
    for (int s = threadIdx.x; s < count * BS; s += kT2Threads) {
        const int bi = s / BS, r = s - bi * BS;
        const int b = s_list[bi], by = b >> 3, bx = b & 7;
        const uint4 cpri = cdef_strength_consts(BS == 4 ? pri : cdef_adjust_strength(pri, s_var[b]), damping, cs);
        int off[6];
        cdef_tap_offsets(pri ? s_dir[b] : 0, TP, off);
        const uint16_t* in = tile + (3 + BS * by + r) * TP + 8 + BS * bx;
        int y[NP][BS];
#pragma unroll
        for (int j = 0; j < BS; j++)
#pragma unroll
            for (int p = 0; p < NP; p++) {
                CdefTaps  T;
                const int x = in[p * kTileC + j];
                cdef_load_taps(in + p * kTileC + j, off, x, T);
                y[p][j] = cdef_finish_px(T, x, (pri ? cdef_primary_sum(T, cpri) : 0) + (sec ? cdef_secondary_sum(T, csec) : 0));
            }
        const size_t o = (size_t)(BS * by + r) * ostride + BS * bx;
        cdef_store_row<BS, PIX>(out_fb + o, y[0], wide & 1);
        if (NP == 2) cdef_store_row<BS, PIX>(out_fb2 + o, y[NP - 1], wide >> 1);
    }
}

// frame apply (svt_av1_cdef_frame, enc_cdef.c:284-600): per filter block strengths already chosen,
// directions/variances as found by cdef_dir_kernel.  One CTA per filter block and luma, and one per filter block
// and both chroma planes (they share one strength).
template <typename PIX>
__global__ void __launch_bounds__(kT2Threads)
cdef_apply_kernel(SvtB200CdefFrame f, const uint8_t* __restrict__ skip8x8, const int8_t* __restrict__ fb_strength_idx,
                  const int* __restrict__ y_strength, const int* __restrict__ uv_strength, const uint8_t* __restrict__ dir_in,
                  const int* __restrict__ var_in, PIX* out_y, PIX* out_cb, PIX* out_cr, int out_stride_y, int out_stride_c) {
    __shared__ __align__(16) uint16_t tile[kTileRows * kTP];  // the luma tile, or the Cb and Cr tiles
    __shared__ uint8_t  s_dir[64];
    __shared__ int      s_var[64];
    __shared__ uint8_t  s_list[64];
    __shared__ unsigned s_ballot[2];
    const int nhfb = (f.width + 63) >> 6, nvfb = (f.height + 63) >> 6, nfb = nhfb * nvfb;
    const int cs = f.bit_depth > 8 ? f.bit_depth - 8 : 0;
    const int w8 = (f.width + 7) >> 3, h8 = (f.height + 7) >> 3;
    // rows of a block start at multiples of its row within a picture row: one store per row when the plane is aligned to it
    const auto wide_rows = [](const PIX* out, int ostride, size_t row_bytes) {
        return (((size_t)out | (size_t)ostride * sizeof(PIX)) & (row_bytes - 1)) == 0;
    };
    for (int work = blockIdx.x; work < nfb * 2; work += gridDim.x) {
        int        fb;
        const bool chroma = cdef_item(work, nfb, fb);
        const int  fbr = fb / nhfb, fbc = fb - fbr * nhfb;
        const int  sidx = fb_strength_idx[fb];
        if (sidx < 0) continue;  // uniform per CTA
        const int sv = chroma ? uv_strength[sidx] : y_strength[sidx];
        const int pri = (sv / 4) << cs;
        int sec = sv % 4;
        sec = (sec + (sec == 3)) << cs;
        if (!(pri || sec)) continue;
        __syncthreads();
        const int count = cdef_fb_list(skip8x8, dir_in, var_in, fb, fbr, fbc, w8, h8, s_list, s_dir, s_var, s_ballot);
        if (count == 0) continue;
        const int damping = f.damping + cs - chroma;
        if (!chroma) {
            const int hsz = min(64, f.width - fbc * 64), vsz = min(64, f.height - fbr * 64);
            const PIX* rec = (const PIX*)f.recon_y;
            stage_cdef_tiles<PIX, 1>(tile, rec, rec, f.recon_stride_y, fbr, fbc, nvfb, nhfb, vsz, hsz);  // ends with a barrier
            PIX* out_fb = out_y + (size_t)fbr * 64 * out_stride_y + fbc * 64;
            cdef_apply_fb<8, PIX>(tile, out_fb, out_fb, out_stride_y, wide_rows(out_y, out_stride_y, 8 * sizeof(PIX)), count, pri, sec,
                                  damping, cs, s_list, s_dir, s_var);
        } else {
            const int hsz = min(32, (f.width >> 1) - fbc * 32), vsz = min(32, (f.height >> 1) - fbr * 32);
            stage_cdef_tiles<PIX, 2>(tile, (const PIX*)f.recon_cb, (const PIX*)f.recon_cr, f.recon_stride_c, fbr, fbc, nvfb, nhfb, vsz, hsz);
            const size_t o = (size_t)fbr * 32 * out_stride_c + fbc * 32;
            const unsigned wide = wide_rows(out_cb, out_stride_c, 4 * sizeof(PIX)) | (wide_rows(out_cr, out_stride_c, 4 * sizeof(PIX)) << 1);
            cdef_apply_fb<4, PIX>(tile, out_cb + o, out_cr + o, out_stride_c, wide, count, pri, sec, damping, cs, s_list, s_dir, s_var);
        }
    }
}

}  // namespace b200

using namespace b200;

// ---- T1 ------------------------------------------------------------------------------------------
static void find_dir_t1(const uint16_t* const* imgs, int n /* 1 or 2 */, int stride, int coeff_shift, int* dirs, int* vars) {
    require_ready();
    RoundTrip rt;
    const size_t blk = 7 * (size_t)stride + 8;
    const int off[2] = {0, (int)blk};
    auto img = rt.in_row_list(imgs, blk, n);
    auto o = rt.in(off, n);
    auto out = rt.out<int>(nullptr, 2 * n);
    find_dir_kernel<<<1, 32, 0, rt.stream()>>>(rt.dev(img), stride, coeff_shift, n, rt.dev(o), rt.dev(out));
    B200_LAUNCH_CHECK();
    rt.finish();
    for (int i = 0; i < n; i++) {
        dirs[i] = rt.host(out)[2 * i];
        vars[i] = rt.host(out)[2 * i + 1];
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
    RoundTrip rt;
    auto src = rt.in_rows(in - 2 * S - 2, S, w + 4, h + 4);  // the block and its 2-pixel border
    auto out = rt.out<uint16_t>(nullptr, (size_t)w * h);
    filter_block_kernel<<<1, 64, 0, rt.stream()>>>(rt.dev(src), w, h, pri_strength, sec_strength, dir, pri_damping, sec_damping,
                                                   coeff_shift, subsampling_factor ? subsampling_factor : 1, rt.dev(out));
    B200_LAUNCH_CHECK();
    rt.finish();
    // only rows i % subs == 0 are written, into whichever destination the caller passed
    const uint16_t* o = rt.host(out);
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
    // the device (stage_cdef_tiles); the T1 form has no device work to do.
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
    RoundTrip rt;
    auto d = rt.in(dst, (rows - 1) * dstride + cols), s = rt.in(src, (size_t)count << (bw_l2 + bh_l2));
    auto lst = rt.in(dlist, 2 * count);
    auto out = rt.out<unsigned long long>(nullptr, 1);
    cdef_dist_kernel<T><<<1, 64, 0, rt.stream()>>>(rt.dev(d), dstride, rt.dev(s), rt.dev(lst), count, bw_l2, bh_l2, coeff_shift, pli,
                                                   subs ? subs : 1, rt.dev(out));
    B200_LAUNCH_CHECK();
    rt.finish();
    return *rt.host(out);
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
    RoundTrip rt;
    int lev[2 * 64];  // lev0 at 0, lev1 at 64
    memcpy(lev, lev0, nb_strengths * 4);
    memcpy(lev + 64, lev1, nb_strengths * 4);
    auto m0 = rt.in_row_list(mse[0], ng, sb_count), m1 = rt.in_row_list(mse[1], ng, sb_count);
    auto lv = rt.in(lev, 2 * 64);
    auto out = rt.out<uint64_t>(nullptr, 3);
    search_one_dual_kernel<<<1, 256, (size_t)ng * ng * 8, rt.stream()>>>((unsigned long long*)rt.dev(m0), (unsigned long long*)rt.dev(m1),
                                                                       sb_count, ng, rt.dev(lv), rt.dev(lv) + 64, nb_strengths, start_gi,
                                                                       (unsigned long long*)rt.dev(out));
    B200_LAUNCH_CHECK();
    rt.finish();
    const uint64_t* o = rt.host(out);
    lev0[nb_strengths] = (int)o[1];
    lev1[nb_strengths] = (int)o[2];
    return o[0];
}

// ---- T2 ------------------------------------------------------------------------------------------
#if B200_CDEF_PHASES
// the search's phase split since the last read (see cdef_phase), then zeroed; only in a B200_CDEF_PHASES build
extern "C" SVT_B200_API int svt_b200_cdef_phases_read(unsigned long long* out /*[2][kCdefPhases + 1]*/) {
    static const unsigned long long zeros[2][kCdefPhases + 1] = {};
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, g_cdef_phase, sizeof(zeros)) != cudaSuccess ||
        cudaMemcpyToSymbol(g_cdef_phase, zeros, sizeof(zeros)) != cudaSuccess)
        return -1;
    return 0;
}
#endif
extern "C" int svt_b200_cdef_search_frame_dev(const SvtB200CdefFrame* frame, const uint8_t* d_skip8x8, const int* d_strengths_y,
                                              const int* d_strengths_uv, int n_strengths, uint64_t* d_mse, uint8_t* d_dir,
                                              int32_t* d_var, void* stream) {
    require_ready();
    if (!frame || n_strengths <= 0 || n_strengths > 64) return SVT_B200_ERR_BAD_ARG;
    const int nfb = ((frame->width + 63) >> 6) * ((frame->height + 63) >> 6);
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = ((frame->width + 7) >> 3) * ((frame->height + 7) >> 3);
    if (frame->bit_depth > 8) {
        cdef_dir_kernel<uint16_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, d_dir, d_var);
        B200_LAUNCH_CHECK();
        cdef_search_kernel<uint16_t><<<grid_for((long long)nfb * 2, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_strengths_y, d_strengths_uv, n_strengths,
                                                                                (unsigned long long*)d_mse, d_dir, d_var);
    } else {
        cdef_dir_kernel<uint8_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, d_dir, d_var);
        B200_LAUNCH_CHECK();
        cdef_search_kernel<uint8_t><<<grid_for((long long)nfb * 2, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_strengths_y, d_strengths_uv, n_strengths,
                                                                               (unsigned long long*)d_mse, d_dir, d_var);
    }
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_cdef_apply_frame_dev(const SvtB200CdefFrame* frame, const uint8_t* d_skip8x8, const int8_t* d_fb_strength_idx,
                                             const int* d_y_strength, const int* d_uv_strength, const uint8_t* d_dir,
                                             const int32_t* d_var, void* d_out_y, void* d_out_cb, void* d_out_cr, int out_stride_y,
                                             int out_stride_c, void* stream) {
    require_ready();
    if (!frame || ((d_dir == nullptr) != (d_var == nullptr))) return SVT_B200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int nfb = ((frame->width + 63) >> 6) * ((frame->height + 63) >> 6);
    const int nblk = ((frame->width + 7) >> 3) * ((frame->height + 7) >> 3);
    if (!d_dir) {  // the directions and variances the search would have given, in this stream's scratch
        static char key;
        const size_t dir_bytes = align256((size_t)nfb * 64);
        uint8_t* sc = (uint8_t*)stream_scratch(&key, st, dir_bytes + (size_t)nfb * 64 * 4);
        uint8_t* dir = sc;
        int32_t* var = (int32_t*)(sc + dir_bytes);
        if (frame->bit_depth > 8) cdef_dir_kernel<uint16_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, dir, var);
        else cdef_dir_kernel<uint8_t><<<(nblk + 127) / 128, 128, 0, st>>>(*frame, d_skip8x8, dir, var);
        B200_LAUNCH_CHECK();
        d_dir = dir;
        d_var = var;
    }
    if (frame->bit_depth > 8)
        cdef_apply_kernel<uint16_t><<<grid_for((long long)nfb * 2, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_fb_strength_idx, d_y_strength, d_uv_strength,
                                                                               d_dir, d_var, (uint16_t*)d_out_y, (uint16_t*)d_out_cb,
                                                                               (uint16_t*)d_out_cr, out_stride_y, out_stride_c);
    else
        cdef_apply_kernel<uint8_t><<<grid_for((long long)nfb * 2, 16), kT2Threads, 0, st>>>(*frame, d_skip8x8, d_fb_strength_idx, d_y_strength, d_uv_strength,
                                                                              d_dir, d_var, (uint8_t*)d_out_y, (uint8_t*)d_out_cb,
                                                                              (uint8_t*)d_out_cr, out_stride_y, out_stride_c);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}
