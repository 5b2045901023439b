// wiener.cu -- K9 separable Wiener filter, K11 Wiener statistics (M = Y^T x, H = Y^T Y) (sm_90a).
//
// Reference behaviour restated:
//   svt_av1_wiener_convolve_add_src_c / svt_av1_highbd_wiener_convolve_add_src_c
//     (Source/Lib/Codec/convolve.c:100-147, 194-237 and the *_hip helpers :57-98, 149-192):
//     8-tap (7 + zero) horizontal pass with add-src, rounding round_0 and clamp to
//     WIENER_CLAMP_LIMIT, then vertical pass with add-src, rounding round_1 and pixel clip.
//   svt_av1_compute_stats_c / _highbd_c (Source/Lib/Codec/restoration_pick.c:659-745):
//     per pixel the wiener_win^2 window of (dgd - avg) is the vector y (column-major), x = src - avg;
//     M[k] += y[k] x, H[k][l] += y[k] y[l]; high bit depth divides by 4 / 16 at the end (truncating).
//
// H100 mapping of the statistics (the one dense contraction on the path):
//   8-bit pixels -> stats_mma_kernel: exact f16 x f16 -> f32 tensor-core MMA (see the comment above it);
//   10/12-bit    -> the lag-sum kernels of wiener_stats_lag.cuh (H[p][q] depends only on the lag between the two samples).
// The MMA kernel writes per-CTA int64 partials; stats_finalize_kernel adds them, mirrors the triangle and applies
// the bit-depth divider.
#include <cuda_fp16.h>

#include <map>

#include "common.cuh"
#include "wiener_unit.cuh"
#include "../../include/svt_b200.h"
#include "wiener_stats_lag.cuh"

namespace b200 {


// ---------------------------------------------------------------------------------------------
// K9
// ---------------------------------------------------------------------------------------------
template <typename PIX>
__global__ void __launch_bounds__(256)
wiener_convolve_kernel(const PIX* __restrict__ src_base, PIX* __restrict__ dst_base, const SvtB200WienerUnit* __restrict__ units,
                       int n_units, int bd, int round0, int round1, int lbd_rows) {
    __shared__ __align__(16) uint16_t s_src[(64 + 8) * (64 + 8)];
    __shared__ __align__(16) uint16_t s_tmp[(64 + 8) * 64];
    for (int it = blockIdx.x; it < n_units; it += gridDim.x) {
        const SvtB200WienerUnit u = units[it];
        const int w = u.w, h = u.h;
        const PIX* src = src_base + u.src_off;
        PIX*       dst = dst_base + u.dst_off;
        const int sw = w + 8, sh = h + 7;  // rows -3..h+3, cols -3..w+4
#pragma unroll 4
        for (int i = threadIdx.x; i < sw * sh; i += blockDim.x) {
            const int r = i / sw, c = i - r * sw;
            // the 8th tap is read by the reference too (multiplied by its coefficient); the column
            // w+4 it touches on the last pixel is part of the caller's extended border
            s_src[r * 72 + c] = (uint16_t)src[(ptrdiff_t)(r - 3) * u.src_stride + (c - 3)];
        }
        __syncthreads();
        wiener_unit_compute<PIX>(s_src, s_tmp, dst, u.dst_stride, w, h, u.hfilter, u.vfilter, bd, round0, round1, lbd_rows);
    }
}

// ---------------------------------------------------------------------------------------------
// K11
// ---------------------------------------------------------------------------------------------
// Pixel total of every item's region (find_average, restoration_pick.c, divides it by w*h): kSumParts
// CTAs per item, one warp per row, totals combined with one 64-bit atomic per warp.
constexpr int kSumParts = 16;
template <typename PIX>
__global__ void __launch_bounds__(256)
stats_sum_kernel(const PIX* __restrict__ dgd_base, const SvtB200StatsItem* __restrict__ items, unsigned long long* __restrict__ tot_out) {
    const int it = blockIdx.x / kSumParts, part = blockIdx.x % kSumParts;
    const SvtB200StatsItem s = items[it];
    const int w = s.h_end - s.h_start, h = s.v_end - s.v_start;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned int acc = 0;  // <= (rows per warp) * (cols per lane) * 4095: far below 2^32 for any restoration unit
    unsigned long long wide = 0;
    for (int r = part * 8 + warp; r < h; r += kSumParts * 8) {
        const PIX* row = dgd_base + s.dgd_off + (ptrdiff_t)(s.v_start + r) * s.dgd_stride + s.h_start;
        for (int c = lane; c < w; c += 32) acc += row[c];
        if (acc > 0xf0000000u) { wide += acc; acc = 0; }
    }
    wide += acc;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wide += __shfl_xor_sync(0xffffffffu, wide, o);
    if (lane == 0 && wide) atomicAdd(&tot_out[it], wide);
}

__device__ __forceinline__ int stats_average(const unsigned long long* tot, int it, const SvtB200StatsItem& s) {
    return (int)(tot[it] / (unsigned long long)((s.h_end - s.h_start) * (s.v_end - s.v_start)));
}

constexpr int kStatsMaxParts = 32;  // CTAs cooperating on one restoration unit

// partial layout per (item, part): [0, 49*49) = H (upper-triangle tiles only), [2401, 2450) = M
//

// ---------------------------------------------------------------------------------------------
// K11, 8-bit pixels: the contraction on the tensor cores.
//
// H = Y^T Y is a Gram matrix with K = pixels.  |pixel - avg| <= 255 is exact in f16, every product
// (<= 255^2) is exact in f32 and a sum of up to 256 of them stays below 2^24, so an f16 x f16 -> f32
// MMA chain over 256 pixels is EXACT integer arithmetic; the f32 accumulators are then converted and
// added to int32 totals in shared memory (good for 33025 pixels), which fold into the CTA's int64
// partial.  Bit-exact with the reference for any input; tests/test_wiener.py holds the extremes.
//
// Matrix rows are ordered i = 8*kx + ky (window column kx, window row ky < WIN); row 7 is x = src - avg
// (so M = row 7 of the same product) and rows with ky >= WIN are don't-care padding.  One
// mma.m16n8k16 K-step covers a 2-row x 8-column block of pixels, k = 2*column + row: a fragment
// register then holds (d[r][c], d[r+1][c]), which the tile stores pre-paired as one 32-bit word per
// (r, c) -- any window shift is a plain word index, and with a row pitch == 4 (mod 32) words the 8
// window rows x 4 columns a warp fetches per load land in 32 distinct banks.  The B fragment of
// n-tile kx is also one half of the A fragment of m-tile kx/2, so a K-step costs 2*WIN loads for
// all of its MMAs.  Only the tiles of the upper triangle (m-tile m, n-tile n >= 2m) are computed.
constexpr int kMmaWarps = 4;
constexpr int kMmaTW = 64, kMmaTH = 32;
constexpr int kMmaPitch = 100;                                // words per pair-row
constexpr int kMmaPRows = kMmaTH + 8;                         // py <= TH-2, plus window/padding row <= 8
constexpr int kMmaXBase = kMmaPRows * kMmaPitch + 28;         // x rows sit on banks 28..31 like a window row 7
constexpr int kMmaWords = kMmaXBase + kMmaTH * kMmaPitch;
constexpr int kMmaAccMax = 16 * 128;                          // 16 output tiles x 128 accumulators (WIN = 7)
constexpr int kMmaFoldPixels = 33025 - kMmaTW * kMmaTH;       // 2^31 / 255^2, minus the tile about to be added
static_assert(kMmaPitch % 32 == 4 && (kMmaPRows * kMmaPitch) % 32 == 0, "bank layout");
static_assert(kMmaTW + 6 <= kMmaPitch && kMmaAccMax <= 2450, "layout");

__device__ __forceinline__ void mma_16816_f16f32(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                                 uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// (lo, hi), |v| <= 255, as two f16 in one word without integer->float conversions: 0x6400 + n is the
// f16 encoding of 1024 + n for 0 <= n < 1024, and subtracting 1280 from 1024 + (v + 256) is exact.
__device__ __forceinline__ uint32_t pack_pair_f16(int lo, int hi) {
    const uint32_t bits = 0x64006400u + (uint32_t)(lo + 256) + ((uint32_t)(hi + 256) << 16);
    const __half2  h    = __hsub2(*reinterpret_cast<const __half2*>(&bits), __float2half2_rn(1280.f));
    return *reinterpret_cast<const uint32_t*>(&h);
}

__host__ __device__ __forceinline__ int mma_tile_index(int win, int m, int n) { return m * win - m * (m - 1) + n - 2 * m; }
// CTAs of an item that actually get pixel tiles (and so write a partial)
__device__ __forceinline__ int stats_mma_parts(const SvtB200StatsItem& s, int ctas_per_item) {
    const int tiles = ((s.h_end - s.h_start + kMmaTW - 1) / kMmaTW) * ((s.v_end - s.v_start + kMmaTH - 1) / kMmaTH);
    return tiles < ctas_per_item ? tiles : ctas_per_item;
}

template <int WIN>
__device__ __forceinline__ void stats_mma_body(const uint8_t* __restrict__ dgd, const uint8_t* __restrict__ src, const SvtB200StatsItem& s,
                                               const int avg, const int part, const int parts, long long* __restrict__ P,
                                               uint32_t* __restrict__ tile, int* __restrict__ s32) {
    constexpr int NT = WIN, MT = (WIN + 1) / 2, HALF = WIN / 2, OFF = 3 - HALF;
    constexpr int NTILES = MT * WIN - MT * (MT - 1);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    // word offset of this lane's fragment row in n-tile n, relative to the K-step's (py, px) word
    int boff[NT];
#pragma unroll
    for (int n = 0; n < NT; n++) boff[n] = (OFF + g) * kMmaPitch + OFF + n + t;
    if (g == 7) boff[0] = kMmaXBase + t;
    float acc[NTILES][4];
#pragma unroll
    for (int i = 0; i < NTILES; i++) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    for (int i = threadIdx.x; i < NTILES * 128; i += kMmaWarps * 32) s32[i] = 0;
    __syncthreads();
    auto flush_regs = [&]() {
#pragma unroll
        for (int i = 0; i < NTILES; i++)
#pragma unroll
            for (int r = 0; r < 4; r++) {
                atomicAdd(&s32[(i * 4 + r) * 32 + lane], __float2int_rn(acc[i][r]));
                acc[i][r] = 0.f;
            }
    };
    const int W = s.h_end - s.h_start, H = s.v_end - s.v_start;
    const int ntx = (W + kMmaTW - 1) / kMmaTW, nty = (H + kMmaTH - 1) / kMmaTH;
    const int vlo = s.v_start - HALF, vhi = s.v_end + HALF, hlo = s.h_start - HALF, hhi = s.h_end + HALF;
    int  ksteps = 0, pending = 0;
    bool spilled = false;
    // pull the rows a tile needs towards L1 (one 128-byte line per request; every address is inside the
    // region the reference itself reads): issued for tile k+1 right before the MMA loop of tile k
    auto prefetch_tile = [&](int tl) {
        const int ty = tl / ntx, tx = tl - ty * ntx;
        const int r0 = s.v_start + ty * kMmaTH, c0 = s.h_start + tx * kMmaTW;
        for (int w = threadIdx.x; w < 2 * (kMmaPRows + 1) + kMmaTH; w += kMmaWarps * 32) {
            const uint8_t* p;
            if (w < 2 * (kMmaPRows + 1)) {
                const int row = min(max(r0 - 3 + (w >> 1), vlo), vhi - 1);
                const int col = (w & 1) ? min(c0 + kMmaTW + 2, hhi - 1) : max(c0 - 3, hlo);
                p = dgd + (ptrdiff_t)row * s.dgd_stride + col;
            } else {
                const int row = min(r0 + (w - 2 * (kMmaPRows + 1)), s.v_end - 1);
                p = src + (ptrdiff_t)row * s.src_stride + min(c0 + 32, s.h_end - 1);
            }
            asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
        }
    };
    for (int tl = part; tl < ntx * nty; tl += parts) {
        const int ty = tl / ntx, tx = tl - ty * ntx;
        const int r0 = s.v_start + ty * kMmaTH, c0 = s.h_start + tx * kMmaTW;
        const int nrows = min(kMmaTH, s.v_end - r0), ncols = min(kMmaTW, s.h_end - c0);
        if (pending > kMmaFoldPixels) {  // CTA-uniform: fold the int32 totals into the int64 partial
            flush_regs();
            ksteps = 0;
            __syncthreads();
            for (int i = threadIdx.x; i < NTILES * 128; i += kMmaWarps * 32) {
                P[i] = (spilled ? P[i] : 0) + s32[i];
                s32[i] = 0;
            }
            spilled = true;
            pending = 0;
        }
        __syncthreads();
        // pair words of d = dgd - avg for tile rows/cols -3.. (zero outside what the reference reads)
        for (int w = threadIdx.x; w < (kMmaTW + 6) * 4; w += kMmaWarps * 32) {
            const int  seg = w / (kMmaTW + 6), c = w - seg * (kMmaTW + 6);
            const int  col = c0 - 3 + c;
            const bool cv = col >= hlo && col < hhi;
            const int  rbeg = seg * (kMmaPRows / 4);
            auto ld = [&](int rr) {
                const int row = r0 - 3 + rr;
                return (cv && row >= vlo && row < vhi) ? (int)dgd[(ptrdiff_t)row * s.dgd_stride + col] - avg : 0;
            };
            int lo = ld(rbeg);
#pragma unroll
            for (int k = 0; k < kMmaPRows / 4; k++) {
                const int hi = ld(rbeg + k + 1);
                tile[(rbeg + k) * kMmaPitch + c] = pack_pair_f16(lo, hi);
                lo = hi;
            }
        }
        for (int w = threadIdx.x; w < (kMmaTH / 2) * kMmaTW; w += kMmaWarps * 32) {
            const int  r = (w / kMmaTW) * 2, c = w % kMmaTW;
            const bool cv = c < ncols;
            const uint8_t* p = src + (ptrdiff_t)(r0 + r) * s.src_stride + c0 + c;
            const int lo = (cv && r < nrows) ? (int)p[0] - avg : 0;
            const int hi = (cv && r + 1 < nrows) ? (int)p[s.src_stride] - avg : 0;
            tile[kMmaXBase + r * kMmaPitch + c] = pack_pair_f16(lo, hi);
        }
        __syncthreads();
        if (tl + parts < ntx * nty) prefetch_tile(tl + parts);
        const int cgs = (ncols + 7) >> 3, nsteps = cgs * ((nrows + 1) >> 1);
        for (int st = warp; st < nsteps; st += kMmaWarps) {
            const int rp = st / cgs, px = (st - rp * cgs) * 8, py = rp * 2;
            const uint32_t* base = tile + py * kMmaPitch + px;
            // pixels of this K-step outside the region contribute nothing: zero them in the B operand
            const uint32_t rowmask = (py + 1 < nrows) ? 0xffffffffu : 0x0000ffffu;
            const uint32_t m0 = (px + t < ncols) ? rowmask : 0u, m1 = (px + t + 4 < ncols) ? rowmask : 0u;
            uint32_t f0[NT], f1[NT];
#pragma unroll
            for (int n = 0; n < NT; n++) {
                f0[n] = base[boff[n]];
                f1[n] = base[boff[n] + 4];
            }
#pragma unroll
            for (int m = 0; m < MT; m++) {
                constexpr int last = NT - 1;
                const int     lo = 2 * m, hi = 2 * m + 1 <= last ? 2 * m + 1 : last;
#pragma unroll
                for (int n = 2 * m; n < NT; n++)
                    mma_16816_f16f32(acc[m * WIN - m * (m - 1) + n - 2 * m], f0[lo], f0[hi], f1[lo], f1[hi], f0[n] & m0, f1[n] & m1);
            }
            if (++ksteps == 16) {  // 256 pixels: the f32 sums are still exact integers
                flush_regs();
                ksteps = 0;
            }
        }
        pending += nrows * ncols;
    }
    flush_regs();
    __syncthreads();
    for (int i = threadIdx.x; i < NTILES * 128; i += kMmaWarps * 32) P[i] = (spilled ? P[i] : 0) + s32[i];
}

__global__ void __launch_bounds__(kMmaWarps * 32)
stats_mma_kernel(const uint8_t* __restrict__ dgd_base, const uint8_t* __restrict__ src_base, const SvtB200StatsItem* __restrict__ items,
                 const unsigned long long* __restrict__ tot_in, int ctas_per_item, long long* __restrict__ partial) {
    __shared__ uint32_t tile[kMmaWords];
    __shared__ int      s32[kMmaAccMax];
    const int it = blockIdx.x / ctas_per_item, part = blockIdx.x % ctas_per_item;
    const SvtB200StatsItem s = items[it];
    const int avg = stats_average(tot_in, it, s);
    if (part >= stats_mma_parts(s, ctas_per_item)) return;  // more CTAs than tiles: finalize ignores the unused partials
    long long* P = partial + ((size_t)it * ctas_per_item + part) * 2450;
    const uint8_t* dgd = dgd_base + s.dgd_off;
    const uint8_t* src = src_base + s.src_off;
    if (s.wiener_win == 7) stats_mma_body<7>(dgd, src, s, avg, part, ctas_per_item, P, tile, s32);
    else if (s.wiener_win == 5) stats_mma_body<5>(dgd, src, s, avg, part, ctas_per_item, P, tile, s32);
    else stats_mma_body<3>(dgd, src, s, avg, part, ctas_per_item, P, tile, s32);
}

// One thread per output element: it knows where its accumulator sits in a partial, adds that entry of
// every part that was written, applies the bit-depth divider.  grid = (ceil(2450 / 256), n_items).
__global__ void __launch_bounds__(256)
stats_finalize_kernel(const long long* __restrict__ partial, int parts, const SvtB200StatsItem* __restrict__ items, int divider,
                      int mma_layout, long long* __restrict__ M_out, long long* __restrict__ H_out) {
    const int it = blockIdx.y, e = blockIdx.x * blockDim.x + threadIdx.x;
    const int win = items[it].wiener_win, win2 = win * win;
    if (e >= win2 * win2 + win2) return;
    const int used = mma_layout ? stats_mma_parts(items[it], parts) : parts;
    int       src;
    if (e < win2 * win2) {
        const int k = e / win2, l = e - k * win2;
        int ka = k / win, kq = k - ka * win, la = l / win, lq = l - la * win;
        if (mma_layout) {
            // accumulator (row i = 8*kx+ky, column j) of the MMA lives in tile (i/16, j/8), C-fragment
            // register ((i/8)&1)*2 + (j&1) of lane (i&7)*4 + (j&7)/2; only tiles with kx_i <= kx_j exist
            if (ka > la) {
                int x = ka; ka = la; la = x;
                x = kq; kq = lq; lq = x;
            }
            src = (mma_tile_index(win, ka >> 1, la) * 4 + (ka & 1) * 2 + (lq & 1)) * 32 + kq * 4 + (lq >> 1);
        } else {
            // tiles were accumulated for window-column pairs a<=b only: element (k,l) lives in the
            // tile of (k/win, l/win) when k/win <= l/win, else in its mirror
            src = (ka <= la) ? k * win2 + l : l * win2 + k;
        }
    } else {
        const int k = e - win2 * win2, ka = k / win, kq = k - ka * win;
        src = mma_layout ? (mma_tile_index(win, 0, ka) * 4 + (kq & 1)) * 32 + 28 + (kq >> 1) : 2401 + k;  // M = matrix row 7
    }
    long long v = 0;
    for (int p = 0; p < used; p++) v += partial[((size_t)it * parts + p) * 2450 + src];
    if (e < win2 * win2) H_out[(size_t)it * 2401 + e] = v / divider;
    else M_out[(size_t)it * 49 + (e - win2 * win2)] = v / divider;
}

// scratch of the batch call (per-CTA partials, pixel totals), one per stream: calls enqueued on
// different streams may execute concurrently
struct StatsScratch {
    long long*          acc = nullptr;
    unsigned long long* tot = nullptr;
    size_t              cap = 0;
};
static std::map<cudaStream_t, StatsScratch> g_stats;
static std::mutex g_stats_mu;
static ResetHook g_stats_reset([] { std::lock_guard<std::mutex> lk(g_stats_mu); g_stats.clear(); });

template <typename PIX, int WIN>
static void launch_lag_bulk(const PIX* d_dgd, const PIX* d_src, const SvtB200StatsItem* d_items, int n, int cpi, unsigned long long* acc,
                            cudaStream_t st) {
    constexpr size_t smem = lag_bulk_smem<PIX, WIN>();
    static int attr = -1;
    if (attr != epoch()) {
        if (smem > 48 * 1024)
            B200_CUDA_CHECK(cudaFuncSetAttribute(stats_lag_bulk_kernel<PIX, WIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = epoch();
    }
    stats_lag_bulk_kernel<PIX, WIN><<<dim3(cpi, n), 256, smem, st>>>(d_dgd, d_src, d_items, acc);
    B200_LAUNCH_CHECK();
}

template <typename PIX>
static void launch_stats_mma(const PIX* d_dgd, const PIX* d_src, const SvtB200StatsItem* d_items, int n, int bd, long long* d_M,
                             long long* d_H, long long* d_acc, unsigned long long* d_tot, cudaStream_t st);

// Wiener statistics of a batch of units: 8-bit pictures on the tensor cores (stats_mma_kernel), 10 / 12 bit by lag sums
// (wiener_stats_lag.cuh) -- both exact
template <typename PIX>
static void launch_stats(const PIX* d_dgd, const PIX* d_src, const SvtB200StatsItem* d_items, int n, int bd, long long* d_M,
                         long long* d_H, long long* d_acc, unsigned long long* d_tot, cudaStream_t st) {
    if constexpr (sizeof(PIX) == 1) return launch_stats_mma<PIX>(d_dgd, d_src, d_items, n, bd, d_M, d_H, d_acc, d_tot, st);
    const int divider = bd == 12 ? 16 : (bd == 10 ? 4 : 1);
    int cpi = (ctx().sm_count * 8) / (n > 0 ? n : 1);  // CTAs per unit: ~8 resident CTAs per SM over the batch
    if (cpi < 1) cpi = 1;
    if (cpi > 64) cpi = 64;
    unsigned long long* acc = reinterpret_cast<unsigned long long*>(d_acc);
    B200_CUDA_CHECK(cudaMemsetAsync(d_tot, 0, (size_t)n * sizeof(unsigned long long), st));
    B200_CUDA_CHECK(cudaMemsetAsync(acc, 0, (size_t)n * kLagItemWords * sizeof(unsigned long long), st));
    stats_sum_kernel<PIX><<<n * kSumParts, 256, 0, st>>>(d_dgd, d_items, d_tot);
    B200_LAUNCH_CHECK();
    // one launch per window size; units of another size leave at once (a batch mixes 7x7 luma with 5x5 chroma units)
    launch_lag_bulk<PIX, 7>(d_dgd, d_src, d_items, n, cpi, acc, st);
    launch_lag_bulk<PIX, 5>(d_dgd, d_src, d_items, n, cpi, acc, st);
    launch_lag_bulk<PIX, 3>(d_dgd, d_src, d_items, n, cpi, acc, st);
    stats_lag_edges_kernel<PIX><<<dim3(kLagEdge, n), 256, 0, st>>>(d_dgd, d_items, acc);
    B200_LAUNCH_CHECK();
    stats_lag_finalize_kernel<PIX><<<dim3((49 * 50 / 2 + 49 + 127) / 128, n), 128, 0, st>>>(d_dgd, d_items, acc, d_tot, divider, d_M, d_H);
    B200_LAUNCH_CHECK();
}

template <typename PIX>
static void launch_stats_mma(const PIX* d_dgd, const PIX* d_src, const SvtB200StatsItem* d_items, int n, int bd, long long* d_M,
                             long long* d_H, long long* d_acc, unsigned long long* d_tot, cudaStream_t st) {
    const int divider = bd == 12 ? 16 : (bd == 10 ? 4 : 1);
    // CTAs per item: enough for ~6 resident CTAs per SM (the tensor-core kernel gives each of them 1-2 pixel tiles)
    int cpi = (ctx().sm_count * (sizeof(PIX) == 1 ? 6 : 4)) / (n > 0 ? n : 1);
    if (cpi < 1) cpi = 1;
    if (cpi > (sizeof(PIX) == 1 ? kStatsMaxParts : 16)) cpi = sizeof(PIX) == 1 ? kStatsMaxParts : 16;
    B200_CUDA_CHECK(cudaMemsetAsync(d_tot, 0, (size_t)n * sizeof(unsigned long long), st));
    stats_sum_kernel<PIX><<<n * kSumParts, 256, 0, st>>>(d_dgd, d_items, d_tot);
    B200_LAUNCH_CHECK();
    static_assert(sizeof(PIX) == 1, "the tensor-core statistics are the 8-bit path (high bit depth: wiener_stats_lag.cuh)");
    stats_mma_kernel<<<n * cpi, kMmaWarps * 32, 0, st>>>(d_dgd, d_src, d_items, d_tot, cpi, d_acc);
    B200_LAUNCH_CHECK();
    stats_finalize_kernel<<<dim3((2450 + 255) / 256, n), 256, 0, st>>>(d_acc, cpi, d_items, divider, sizeof(PIX) == 1, d_M, d_H);
    B200_LAUNCH_CHECK();
}

template <typename PIX>
static void stats_t1(int wiener_win, const PIX* dgd, const PIX* src, int h_start, int h_end, int v_start, int v_end, int dgd_stride,
                     int src_stride, int64_t* M, int64_t* H, int bd) {
    require_ready();
    const int half = wiener_win >> 1, win2 = wiener_win * wiener_win;
    const int w = h_end - h_start, h = v_end - v_start;
    const int dw = w + 2 * half, dh = h + 2 * half;
    LaneGuard l;
    size_t o_d = l->alloc((size_t)dw * dh * sizeof(PIX)), o_s = l->alloc((size_t)w * h * sizeof(PIX)), o_it = l->alloc(sizeof(SvtB200StatsItem));
    size_t in_end = l->used;
    size_t o_M = l->alloc(49 * 8), o_H = l->alloc(2401 * 8), o_acc = l->alloc((size_t)kStatsMaxParts * 2450 * 8), o_avg = l->alloc(16);
    for (int r = 0; r < dh; r++)
        memcpy(l->h<PIX>(o_d) + (size_t)r * dw, dgd + (ptrdiff_t)(v_start - half + r) * dgd_stride + h_start - half, dw * sizeof(PIX));
    for (int r = 0; r < h; r++) memcpy(l->h<PIX>(o_s) + (size_t)r * w, src + (ptrdiff_t)(v_start + r) * src_stride + h_start, w * sizeof(PIX));
    SvtB200StatsItem* it = l->h<SvtB200StatsItem>(o_it);
    memset(it, 0, sizeof(*it));
    it->dgd_off = (uint64_t)half * dw + half;  // (v_start, h_start) of the packed copy
    it->src_off = 0;
    it->dgd_stride = dw;
    it->src_stride = w;
    it->h_start = 0;
    it->h_end = w;
    it->v_start = 0;
    it->v_end = h;
    it->wiener_win = wiener_win;
    l->h2d(0, in_end);
    launch_stats<PIX>(l->d<PIX>(o_d), l->d<PIX>(o_s), l->d<SvtB200StatsItem>(o_it), 1, bd, l->d<long long>(o_M), l->d<long long>(o_H),
                      l->d<long long>(o_acc), l->d<unsigned long long>(o_avg), l->stream);
    l->d2h(o_M, (o_H + 2401 * 8) - o_M);
    l->sync();
    memcpy(M, l->h<int64_t>(o_M), (size_t)win2 * 8);
    memcpy(H, l->h<int64_t>(o_H), (size_t)win2 * win2 * 8);
}

template <typename PIX>
static void wiener_t1(const PIX* src, ptrdiff_t src_stride, PIX* dst, ptrdiff_t dst_stride, const int16_t* fx, const int16_t* fy, int w,
                      int h, int round0, int round1, int bd, int lbd_rows) {
    require_ready();
    LaneGuard l;
    const int sw = w + 8, sh = h + 7;
    size_t o_s = l->alloc((size_t)sw * sh * sizeof(PIX)), o_u = l->alloc(sizeof(SvtB200WienerUnit));
    size_t in_end = l->used;
    size_t o_d = l->alloc((size_t)w * h * sizeof(PIX));
    for (int r = 0; r < sh; r++) memcpy(l->h<PIX>(o_s) + (size_t)r * sw, src + (ptrdiff_t)(r - 3) * src_stride - 3, sw * sizeof(PIX));
    SvtB200WienerUnit* u = l->h<SvtB200WienerUnit>(o_u);
    memset(u, 0, sizeof(*u));
    u->src_off = (uint64_t)3 * sw + 3;
    u->dst_off = 0;
    u->src_stride = sw;
    u->dst_stride = w;
    u->w = (uint16_t)w;
    u->h = (uint16_t)h;
    memcpy(u->hfilter, fx, 16);
    memcpy(u->vfilter, fy, 16);
    l->h2d(0, in_end);
    wiener_convolve_kernel<PIX><<<1, 256, 0, l->stream>>>(l->d<PIX>(o_s), l->d<PIX>(o_d), l->d<SvtB200WienerUnit>(o_u), 1, bd, round0, round1, lbd_rows);
    B200_LAUNCH_CHECK();
    l->d2h(o_d, (size_t)w * h * sizeof(PIX));
    l->sync();
    for (int r = 0; r < h; r++) memcpy(dst + (ptrdiff_t)r * dst_stride, l->h<PIX>(o_d) + (size_t)r * w, w * sizeof(PIX));
}

}  // namespace b200

using namespace b200;

extern "C" void svt_b200_av1_wiener_convolve_add_src(const uint8_t* src, ptrdiff_t src_stride, uint8_t* dst, ptrdiff_t dst_stride,
                                                     const int16_t* filter_x, const int16_t* filter_y, int32_t w, int32_t h,
                                                     const SvtB200ConvolveParams* conv_params) {
    wiener_t1<uint8_t>(src, src_stride, dst, dst_stride, filter_x, filter_y, w, h, conv_params->round_0, conv_params->round_1, 8, 1);
}
extern "C" void svt_b200_av1_highbd_wiener_convolve_add_src(const uint16_t* src, ptrdiff_t src_stride, uint16_t* dst,
                                                            ptrdiff_t dst_stride, const int16_t* filter_x, const int16_t* filter_y,
                                                            int32_t w, int32_t h, const SvtB200ConvolveParams* conv_params, int32_t bd) {
    wiener_t1<uint16_t>(src, src_stride, dst, dst_stride, filter_x, filter_y, w, h, conv_params->round_0, conv_params->round_1, bd, 0);
}
extern "C" void svt_b200_av1_compute_stats(int32_t wiener_win, const uint8_t* dgd, const uint8_t* src, int32_t h_start, int32_t h_end,
                                           int32_t v_start, int32_t v_end, int32_t dgd_stride, int32_t src_stride, int64_t* M, int64_t* H) {
    stats_t1<uint8_t>(wiener_win, dgd, src, h_start, h_end, v_start, v_end, dgd_stride, src_stride, M, H, 8);
}
extern "C" void svt_b200_av1_compute_stats_highbd(int32_t wiener_win, const uint16_t* dgd, const uint16_t* src, int32_t h_start,
                                                  int32_t h_end, int32_t v_start, int32_t v_end, int32_t dgd_stride, int32_t src_stride,
                                                  int64_t* M, int64_t* H, int32_t bit_depth) {
    stats_t1<uint16_t>(wiener_win, dgd, src, h_start, h_end, v_start, v_end, dgd_stride, src_stride, M, H, bit_depth);
}

extern "C" int svt_b200_wiener_units_dev(const void* d_src, void* d_dst, const SvtB200WienerUnit* d_units, int n_units, int bit_depth,
                                         void* stream) {
    require_ready();
    if (n_units <= 0) return n_units == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    // get_conv_params_wiener (convolve.h): round_0 = 3 (+2 at 12 bit), round_1 = 2*FILTER_BITS - round_0
    const int round0 = bit_depth == 12 ? 5 : 3, round1 = 14 - round0;
    cudaStream_t st = (cudaStream_t)stream;
    if (bit_depth > 8)
        wiener_convolve_kernel<uint16_t><<<grid_for(n_units, 4), 256, 0, st>>>((const uint16_t*)d_src, (uint16_t*)d_dst, d_units, n_units, bit_depth, round0, round1, 0);
    else
        wiener_convolve_kernel<uint8_t><<<grid_for(n_units, 4), 256, 0, st>>>((const uint8_t*)d_src, (uint8_t*)d_dst, d_units, n_units, 8, round0, round1, 1);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_compute_stats_batch_dev(const void* d_dgd, const void* d_src, const SvtB200StatsItem* d_items, int n_items,
                                                int bit_depth, int64_t* d_M, int64_t* d_H, void* stream) {
    require_ready();
    if (n_items <= 0) return n_items == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    std::lock_guard<std::mutex> lk(g_stats_mu);
    StatsScratch& sc = g_stats[(cudaStream_t)stream];
    if ((size_t)n_items > sc.cap) {
        sc.cap = (size_t)n_items * 2;  // new buffers; the old ones live on until shutdown (captured graphs may replay them)
        sc.acc = (long long*)scratch_alloc(sc.cap * kStatsMaxParts * 2450 * 8);
        sc.tot = (unsigned long long*)scratch_alloc(sc.cap * 8);
    }
    if (bit_depth > 8)
        launch_stats<uint16_t>((const uint16_t*)d_dgd, (const uint16_t*)d_src, d_items, n_items, bit_depth, (long long*)d_M, (long long*)d_H,
                               sc.acc, sc.tot, (cudaStream_t)stream);
    else
        launch_stats<uint8_t>((const uint8_t*)d_dgd, (const uint8_t*)d_src, d_items, n_items, 8, (long long*)d_M, (long long*)d_H, sc.acc,
                              sc.tot, (cudaStream_t)stream);
    return SVT_B200_OK;
}
