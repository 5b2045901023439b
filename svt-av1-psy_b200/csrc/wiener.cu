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
//   8-bit pixels -> stats_imma_kernel: raw-pixel moments by exact u8 x u8 -> s32 tensor-core MMA, one launch per call
//                   (see the comment above it);
//   10/12-bit    -> the lag-sum kernels of wiener_stats_lag.cuh (H[p][q] depends only on the lag between the two samples).
#include <cooperative_groups.h>

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

// ---------------------------------------------------------------------------------------------
// K11, 8-bit pixels: raw moments on the tensor cores, one launch per call.
//
// With a = find_average (the truncating mean of the region), y_k = d_k - a and x = s - a, the reference's sums follow
// exactly, in int64, from moments of the RAW pixels:
//     H[k][l] = sum d_k d_l - a (S_k + S_l) + N a^2          M[k] = sum d_k s - a S_k - a S_s + N a^2
// with S_k = sum d_k (window sample k over the region), S_s = sum s and N = w h.  S_k of the centre sample is
// find_average's own total, so nothing needs the mean before the contraction, and the Gram matrix runs on unsigned bytes:
// mma.m16n8k32 u8 x u8 -> s32 (IMMA), exact while a warp has summed at most 33025 pixels (2^31 / 255^2).  Past that bound
// the warps fold their int32 accumulators into the CTA's int64 totals.
//
// Matrix rows are i = 8*kx + ky (window column kx, window row ky < WIN); row 7 is x = src, row 15 (kx = 1, ky = 7) is a
// constant 1, so the tiles (0, n) also give every S_k and S_s; the other rows with ky >= WIN are don't-care padding.  One
// K-step covers a 4-row x 8-column block of pixels, k = 4*column + row: a fragment register then holds (d[r][c], d[r+1][c],
// d[r+2][c], d[r+3][c]), which the tile stores as one quad word per (r, c) -- any window shift is a plain word index, and
// with a row pitch == 4 (mod 32) words the 8 window rows x 4 columns a warp fetches per load land in 32 distinct banks.  The
// B fragment of n-tile kx is also one half of the A fragment of m-tile kx/2, so a K-step costs 2*WIN loads for all of its
// MMAs.  Only the tiles of the upper triangle (m-tile m, n-tile n >= 2m) are computed.  Pixels outside the region are
// zeroed in the B operand only, so halo words may hold anything.
//
// A unit is one cluster of kImCluster CTAs, which share its 64x32 pixel tiles: a 256x256 luma unit gives its 8 CTAs 4
// tiles each, a 128x128 chroma unit 1 (of 9 MMAs per K-step against 16 at 7x7).  Giving a chroma unit only 2 CTAs of 4
// tiles, to even out the work per CTA, measured slower: the 6 idle CTAs of its cluster hold their SM slots until the
// cluster ends, so the batch takes two waves of clusters.  Regions with fewer than 8 tiles leave the remaining CTAs
// idle; they only take part in the cluster barriers.  The raw bytes of the next tile arrive by cp.async in a two-stage
// ring while the current one is contracted.  The working CTAs then share the outputs: each adds the int64 totals it
// needs over the cluster through distributed shared memory, applies the mean correction and writes M and H (both
// triangles) in the reference layout.
constexpr int kImWarps = 4, kImThreads = kImWarps * 32;
constexpr int kImCluster = 8;                                  // CTAs per unit: the portable cluster size
constexpr int kImTW = 64, kImTH = 32;
constexpr int kImPitch = 100;                                  // words per quad-word row
constexpr int kImQRows = kImTH + 6;                            // quad rows py + OFF + g <= TH - 4 + 9
constexpr int kImXPitch = 80;                                  // words per src quad row (== 16 mod 32, like 4 quad rows)
constexpr int kImXRegion = (kImQRows * kImPitch + 31) / 32 * 32;
constexpr int kImQWords = kImXRegion + 32 + (kImTH / 4) * kImXPitch;
constexpr int kImRawRows = kImTH + 9;                          // halo rows 0..TH+5 are loaded, the last 3 only feed padding
constexpr int kImRawPitch = 96;                                // bytes: 70 halo columns behind a <= 15-byte alignment shift
constexpr int kImXRawPitch = 80;                               // bytes: 64 src columns behind the shift
constexpr int kImStage = kImRawRows * kImRawPitch + kImTH * kImXRawPitch;
constexpr int kImAccMax = 16 * 128;                            // 16 output tiles x 128 accumulators (WIN = 7)
constexpr int kImFoldPixels = 33025 - (kImTW * kImTH) / kImWarps;  // 2^31 / 255^2, minus what one more tile adds to a warp
static_assert(kImPitch % 32 == 4 && kImXPitch % 32 == 16 && kImStage % 16 == 0, "bank and cp.async layout");
// the quad builders read two words from byte (shift <= 15) + (first column of their last 4): 68 of the halo, 60 of src
static_assert(kImTW + 8 <= kImPitch && ((15 + kImTW + 4) & ~3) + 8 <= kImRawPitch && ((15 + kImTW - 4) & ~3) + 8 <= kImXRawPitch, "layout");

__device__ __forceinline__ void mma_16832_u8s32(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                                uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}

__host__ __device__ __forceinline__ int mma_tile_index(int win, int m, int n) { return m * win - m * (m - 1) + n - 2 * m; }

// CTAs of the cluster that get pixel tiles of an item
__device__ __forceinline__ int stats_imma_parts(const SvtB200StatsItem& s) {
    const int tiles = ((s.h_end - s.h_start + kImTW - 1) / kImTW) * ((s.v_end - s.v_start + kImTH - 1) / kImTH);
    return min(tiles, kImCluster);
}

// Stage rows [0, nrows) of a tile: row q starts at tile column 0 = row0 + q * stride and lands, behind its alignment
// shift (address & 15), at dst + q * pitch.  Only rows [qlo, qhi) and tile columns [clo, chi) are read -- the rectangle
// the reference reads -- and columns past `need` are not needed: 16-byte chunks that would cross the rectangle fall back
// to 4-byte copies, and those to byte loads.
__device__ __forceinline__ void stats_imma_stage_rows(uint8_t* dst, int pitch, const uint8_t* row0, ptrdiff_t stride, int nrows,
                                                      int nchunks, int qlo, int qhi, int clo, int chi, int need) {
    for (int w = threadIdx.x; w < nrows * nchunks; w += kImThreads) {
        const int q = w / nchunks, ch = w - q * nchunks;
        const uint8_t* rp = row0 + (ptrdiff_t)q * stride;
        const int a = ch * 16 - (int)((uintptr_t)rp & 15);  // tile column of the chunk's first byte
        if (q < qlo || q >= qhi || a >= need || a >= chi || a + 16 <= clo) continue;
        uint8_t*       d = dst + q * pitch + ch * 16;
        const uint8_t* g = rp + a;
        if (a >= clo && a + 16 <= chi) {
            cp_async16(d, g);
            continue;
        }
#pragma unroll
        for (int b4 = 0; b4 < 16; b4 += 4) {
            if (a + b4 >= clo && a + b4 + 4 <= chi) cp_async4(d + b4, g + b4);
            else
                for (int b = b4; b < b4 + 4; b++)
                    if (a + b >= clo && a + b < chi) d[b] = g[b];
        }
    }
}

// 4 bytes of a staged row starting at byte `at` (any alignment; the row and the word after it are in the stage)
__device__ __forceinline__ uint32_t stats_imma_row4(const uint8_t* row, int at) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(row + (at & ~3));
    return __funnelshift_r(w[0], w[1], (at & 3) * 8);
}

template <int WIN>
__device__ __forceinline__ void stats_imma_body(const uint8_t* __restrict__ dgd, const uint8_t* __restrict__ src, const SvtB200StatsItem& s,
                                                const int part, const int parts, uint32_t* __restrict__ quad, uint8_t* __restrict__ ring,
                                                long long* __restrict__ red) {
    constexpr int NT = WIN, MT = (WIN + 1) / 2, HALF = WIN / 2, OFF = 3 - HALF;
    constexpr int NTILES = MT * WIN - MT * (MT - 1);
    constexpr int XB = kImXRegion + ((28 + 5 * OFF) & 31);  // src quad words sit on the banks of a window row 7
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const uint32_t* lane_base = quad + (OFF + g) * kImPitch + OFF + t;  // this lane's fragment row, relative to the K-step
    int acc[NTILES][4];
#pragma unroll
    for (int i = 0; i < NTILES; i++) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0;
    auto fold = [&]() {  // CTA-uniform: the warps add their int32 sums into the int64 totals one after another
#pragma unroll 1
        for (int w = 0; w < kImWarps; w++) {
            if (warp == w)
#pragma unroll
                for (int i = 0; i < NTILES; i++)
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        red[(i * 4 + r) * 32 + lane] += acc[i][r];
                        acc[i][r] = 0;
                    }
            __syncthreads();
        }
    };
    const int W = s.h_end - s.h_start, H = s.v_end - s.v_start;
    const int ntx = (W + kImTW - 1) / kImTW, ntiles = ntx * ((H + kImTH - 1) / kImTH);
    auto stage = [&](int tl, uint8_t* st) {
        const int ty = tl / ntx, tx = tl - ty * ntx;
        const int r0 = s.v_start + ty * kImTH, c0 = s.h_start + tx * kImTW;
        // dgd: halo rows r0-3.., columns c0-3..; the reference reads [v_start-HALF, v_end+HALF) x [h_start-HALF, h_end+HALF)
        stats_imma_stage_rows(st, kImRawPitch, dgd + (ptrdiff_t)(r0 - 3) * s.dgd_stride + (c0 - 3), s.dgd_stride, kImTH + 6,
                              kImRawPitch / 16, s.v_start - HALF - (r0 - 3), s.v_end + HALF - (r0 - 3), s.h_start - HALF - (c0 - 3), s.h_end + HALF - (c0 - 3),
                              kImTW + 6);
        // src: rows r0.., columns c0.. of the region
        stats_imma_stage_rows(st + kImRawRows * kImRawPitch, kImXRawPitch, src + (ptrdiff_t)r0 * s.src_stride + c0, s.src_stride, kImTH,
                              kImXRawPitch / 16, 0, s.v_end - r0, s.h_start - c0, s.h_end - c0, kImTW);
        asm volatile("cp.async.commit_group;\n" ::: "memory");
    };
    int pending = 0;  // pixels any one warp has added to its int32 sums
    if (part < ntiles) stage(part, ring);
    for (int tl = part, k = 0; tl < ntiles; tl += parts, k++) {
        const int ty = tl / ntx, tx = tl - ty * ntx;
        const int r0 = s.v_start + ty * kImTH, c0 = s.h_start + tx * kImTW;
        const int nrows = min(kImTH, s.v_end - r0), ncols = min(kImTW, s.h_end - c0);
        const uint8_t* st = ring + (k & 1) * kImStage;
        if (tl + parts < ntiles) {
            stage(tl + parts, ring + ((k + 1) & 1) * kImStage);  // the build of tile k-1 that read this stage is behind a barrier
            asm volatile("cp.async.wait_group 1;\n" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        }
        __syncthreads();  // the stage is complete, and the MMAs of the previous tile are done with the quad words
        // quad words of the halo: a thread owns 4 columns and a run of 6 quad rows, shifting one raw row in per step
        if (threadIdx.x < 18 * 7) {
            const int cq = (threadIdx.x % 18) * 4, q0 = (threadIdx.x / 18) * 6;
            const uint8_t* rbase = dgd + (ptrdiff_t)(r0 - 3) * s.dgd_stride + (c0 - 3);
            uint32_t v0 = 0, v1 = 0, v2 = 0, v3 = 0;
#pragma unroll
            for (int j = 0; j < 9; j++) {
                const int q = min(q0 + j, kImRawRows - 1);  // rows past the stage only feed quad rows that are not stored
                const uint32_t b = stats_imma_row4(st + q * kImRawPitch, (int)((uintptr_t)(rbase + (ptrdiff_t)q * s.dgd_stride) & 15) + cq);
                v0 = __byte_perm(v0, b, 0x4321);
                v1 = __byte_perm(v1, b, 0x5321);
                v2 = __byte_perm(v2, b, 0x6321);
                v3 = __byte_perm(v3, b, 0x7321);
                if (j >= 3 && q0 + j - 3 < kImQRows)
                    *reinterpret_cast<uint4*>(quad + (q0 + j - 3) * kImPitch + cq) = make_uint4(v0, v1, v2, v3);
            }
        }
        {  // src quad words: rows 4j..4j+3 of 4 columns per thread
            const int cq = (threadIdx.x & 15) * 4, j = threadIdx.x >> 4;
            const uint8_t* xs = st + kImRawRows * kImRawPitch;
            const uint8_t* rbase = src + (ptrdiff_t)r0 * s.src_stride + c0;
            uint32_t rw[4];
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const int q = 4 * j + r;
                rw[r] = stats_imma_row4(xs + q * kImXRawPitch, (int)((uintptr_t)(rbase + (ptrdiff_t)q * s.src_stride) & 15) + cq);
            }
            const uint32_t t0 = __byte_perm(rw[0], rw[1], 0x5140), t1 = __byte_perm(rw[0], rw[1], 0x7362);
            const uint32_t t2 = __byte_perm(rw[2], rw[3], 0x5140), t3 = __byte_perm(rw[2], rw[3], 0x7362);
            uint32_t* xq = quad + XB + j * kImXPitch + cq;
            xq[0] = __byte_perm(t0, t2, 0x5410);
            xq[1] = __byte_perm(t0, t2, 0x7632);
            xq[2] = __byte_perm(t1, t3, 0x5410);
            xq[3] = __byte_perm(t1, t3, 0x7632);
        }
        __syncthreads();
        const int cgs = (ncols + 7) >> 3, nsteps = cgs * ((nrows + 3) >> 2);
        for (int stp = warp; stp < nsteps; stp += kImWarps) {
            const int rp = stp / cgs, px = (stp - rp * cgs) * 8, py = rp * 4;
            const uint32_t* b  = lane_base + py * kImPitch + px;
            const uint32_t* xb = g == 7 ? quad + XB + rp * kImXPitch + px + t : b;
            // pixels of this K-step outside the region contribute nothing: zero them in the B operand
            const int      nr      = nrows - py;
            const uint32_t rowmask = nr >= 4 ? 0xffffffffu : (1u << (8 * nr)) - 1u;
            const uint32_t m0 = (px + t < ncols) ? rowmask : 0u, m1 = (px + t + 4 < ncols) ? rowmask : 0u;
            uint32_t f0[NT], f1[NT];
            f0[0] = xb[0];
            f1[0] = xb[4];
#pragma unroll
            for (int n = 1; n < NT; n++) {
                f0[n] = b[n];
                f1[n] = b[n + 4];
            }
            if (g == 7) f0[1] = f1[1] = 0x01010101u;  // row 15: the window sums
#pragma unroll
            for (int m = 0; m < MT; m++) {
                constexpr int last = NT - 1;
                const int     lo = 2 * m, hi = 2 * m + 1 <= last ? 2 * m + 1 : last;
#pragma unroll
                for (int n = 2 * m; n < NT; n++)
                    mma_16832_u8s32(acc[m * WIN - m * (m - 1) + n - 2 * m], f0[lo], f0[hi], f1[lo], f1[hi], f0[n] & m0, f1[n] & m1);
            }
        }
        pending += ((nsteps + kImWarps - 1) / kImWarps) * 32;
        if (pending > kImFoldPixels && tl + parts < ntiles) {
            fold();
            pending = 0;
        }
    }
    fold();
}

// grid = n_items * kImCluster CTAs, one cluster per item
__global__ void __cluster_dims__(kImCluster, 1, 1) __launch_bounds__(kImThreads, 4)
stats_imma_kernel(const uint8_t* __restrict__ dgd_base, const uint8_t* __restrict__ src_base, const SvtB200StatsItem* __restrict__ items,
                  long long* __restrict__ M_out, long long* __restrict__ H_out) {
    __shared__ __align__(16) uint32_t quad[kImQWords];
    __shared__ __align__(16) uint8_t  ring[2 * kImStage];
    __shared__ long long red[kImAccMax];
    __shared__ long long sums[50];
    namespace cgr = cooperative_groups;
    cgr::cluster_group cluster = cgr::this_cluster();
    const int it = blockIdx.x / kImCluster, part = (int)cluster.block_rank();
    const SvtB200StatsItem s = items[it];
    const int parts = stats_imma_parts(s), win = s.wiener_win;
    if (part < parts) {
        for (int i = threadIdx.x; i < kImAccMax; i += kImThreads) red[i] = 0;
        __syncthreads();
        const uint8_t* dgd = dgd_base + s.dgd_off;
        const uint8_t* src = src_base + s.src_off;
        if (win == 7) stats_imma_body<7>(dgd, src, s, part, parts, quad, ring, red);
        else if (win == 5) stats_imma_body<5>(dgd, src, s, part, parts, quad, ring, red);
        else stats_imma_body<3>(dgd, src, s, part, parts, quad, ring, red);
    }
    cluster.sync();  // every CTA's totals are in its shared memory
    if (part < parts) {
        // the working CTAs share the outputs; each adds the totals it needs over the cluster
        // accumulator (row i = 8*kx+ky, column j) of the MMA lives in tile (i/16, j/8), C-fragment register
        // ((i/8)&1)*2 + (j&1) of lane (i&7)*4 + (j&7)/2; only tiles with kx_i <= kx_j exist
        auto total = [&](int idx) {
            long long v = 0;
#pragma unroll
            for (int p = 0; p < kImCluster; p++)
                if (p < parts) v += cluster.map_shared_rank(red, p)[idx];
            return v;
        };
        const int win2 = win * win, half = win >> 1;
        // row 15 (ones) x column j: S_k of window sample k = (kx, ky), and S_s in column 7
        for (int k = threadIdx.x; k <= win2; k += kImThreads) {
            const int kx = k / win, ky = k - kx * win;
            sums[k] = total(k < win2 ? (mma_tile_index(win, 0, kx) * 4 + 2 + (ky & 1)) * 32 + 28 + (ky >> 1) : 3 * 32 + 31);
        }
        __syncthreads();
        const long long N = (long long)(s.h_end - s.h_start) * (s.v_end - s.v_start);
        const long long a = N ? sums[half * win + half] / N : 0, na2 = N * a * a;  // find_average
        for (int e = part * kImThreads + threadIdx.x; e < win2 * win2 + win2; e += parts * kImThreads) {
            if (e < win2 * win2) {
                const int k = e / win2, l = e - k * win2;
                int ka = k / win, kq = k - ka * win, la = l / win, lq = l - la * win;
                if (ka > la) {
                    int x = ka; ka = la; la = x;
                    x = kq; kq = lq; lq = x;
                }
                const long long raw = total((mma_tile_index(win, ka >> 1, la) * 4 + (ka & 1) * 2 + (lq & 1)) * 32 + kq * 4 + (lq >> 1));
                H_out[(size_t)it * 2401 + e] = raw - a * (sums[k] + sums[l]) + na2;
            } else {
                const int k = e - win2 * win2, ka = k / win, kq = k - ka * win;  // M = matrix row 7 (x)
                const long long raw = total((mma_tile_index(win, 0, ka) * 4 + (kq & 1)) * 32 + 28 + (kq >> 1));
                M_out[(size_t)it * 49 + k] = raw - a * sums[k] - a * sums[win2] + na2;
            }
        }
    }
    cluster.sync();  // no CTA leaves while another may still read its shared memory
}

// scratch of the 10/12-bit batch call (lag sums, pixel totals), one per stream: calls enqueued on
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

// Wiener statistics of a batch of units: 8-bit pictures on the tensor cores (stats_imma_kernel, one launch), 10 / 12 bit
// by lag sums (wiener_stats_lag.cuh, which uses the scratch) -- both exact
template <typename PIX>
static void launch_stats(const PIX* d_dgd, const PIX* d_src, const SvtB200StatsItem* d_items, int n, int bd, long long* d_M,
                         long long* d_H, long long* d_acc, unsigned long long* d_tot, cudaStream_t st) {
    if constexpr (sizeof(PIX) == 1) {
        stats_imma_kernel<<<n * kImCluster, kImThreads, 0, st>>>(d_dgd, d_src, d_items, d_M, d_H);
        B200_LAUNCH_CHECK();
        return;
    }
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
static void stats_t1(int wiener_win, const PIX* dgd, const PIX* src, int h_start, int h_end, int v_start, int v_end, int dgd_stride,
                     int src_stride, int64_t* M, int64_t* H, int bd) {
    require_ready();
    const int half = wiener_win >> 1, win2 = wiener_win * wiener_win;
    const int w = h_end - h_start, h = v_end - v_start;
    const int dw = w + 2 * half, dh = h + 2 * half;
    LaneGuard l;
    size_t o_d = l->alloc((size_t)dw * dh * sizeof(PIX)), o_s = l->alloc((size_t)w * h * sizeof(PIX)), o_it = l->alloc(sizeof(SvtB200StatsItem));
    size_t in_end = l->used;
    size_t o_M = l->alloc(49 * 8), o_H = l->alloc(2401 * 8), o_acc = l->alloc((size_t)kLagItemWords * 8), o_avg = l->alloc(16);
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
    if (bit_depth <= 8) {
        launch_stats<uint8_t>((const uint8_t*)d_dgd, (const uint8_t*)d_src, d_items, n_items, 8, (long long*)d_M, (long long*)d_H, nullptr,
                              nullptr, (cudaStream_t)stream);
        return SVT_B200_OK;
    }
    std::lock_guard<std::mutex> lk(g_stats_mu);
    StatsScratch& sc = g_stats[(cudaStream_t)stream];
    if ((size_t)n_items > sc.cap) {
        sc.cap = (size_t)n_items * 2;  // new buffers; the old ones live on until shutdown (captured graphs may replay them)
        sc.acc = (long long*)scratch_alloc(sc.cap * kLagItemWords * 8);
        sc.tot = (unsigned long long*)scratch_alloc(sc.cap * 8);
    }
    launch_stats<uint16_t>((const uint16_t*)d_dgd, (const uint16_t*)d_src, d_items, n_items, bit_depth, (long long*)d_M, (long long*)d_H,
                           sc.acc, sc.tot, (cudaStream_t)stream);
    return SVT_B200_OK;
}
