// sad_small.cuh -- warp-level full search over a SMALL search area (shared by sad.cu and me_picture.cu).
//
// Small search areas (the 8x3 / 16x4 HME and ME refinements: a few dozen positions, blocks up to
// 64x64): the work is a few hundred VABSDIFF4 per lane, so staging through shared memory and CTA
// barriers would be the whole cost.  One WARP per search, no shared memory: lane = (x mod 8, row slice
// of 4); a lane walks its rows with two sliding funnel-shift windows over aligned words that come
// straight from L1 (the 8 x-lanes of a slice read the same sectors, the source word is a broadcast)
// and evaluates up to four search rows y at once against every source word; the 4 slices are added
// with two shuffles and the raster-order first minimum (compute_sad_c.c:58-101: strict '<') is the
// minimum of the 64-bit key (sad<<32 | y<<16 | x).
#pragma once
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

constexpr int kSmallSearchMaxPos = 256;  // searches with at most this many positions take the warp path

// aligned-word view of `n` bytes at p: word(j) = bytes [4j, 4j+4) of the run; only words holding a valid byte are read
struct ByteRun {
    const uint32_t* w;
    int shift, last;
    __device__ __forceinline__ ByteRun(const uint8_t* p, int n) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(p);
        w     = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
        shift = (int)(a & 3) * 8;
        last  = (int)(((a & 3) + n - 1) >> 2);
    }
    __device__ __forceinline__ uint32_t raw(int j) const { return __ldg(w + (j < last ? j : last)); }
};


__device__ __forceinline__ SvtB200SadSearchResult sad_key_to_result(unsigned long long best) {
    SvtB200SadSearchResult r;
    if (best == ~0ull) {
        r.best_sad = 0xffffffu;
        r.x = r.y = -1;
    } else {
        r.best_sad = (uint32_t)(best >> 32);
        r.y        = (int16_t)((best >> 16) & 0xffff);
        r.x        = (int16_t)(best & 0xffff);
    }
    return r;
}

// ---------------------------------------------------------------------------------------------------
// Blocks whose width is a multiple of 16 (the HME / ME blocks: 16, 32, 64 wide): a lane owns a
// (block row, 16-pixel chunk) UNIT, keeps its 4 source words in registers and, per tile of 8 horizontally
// adjacent search positions, fetches the 7 aligned reference words that cover the 23 bytes those
// positions touch, normalises them once to the row's byte alignment and evaluates the 8 positions with
// compile-time funnel shifts: 4 x (SHF + VABSDIFF4) per position, no loads inside.  Units of one search
// spread over the lanes (several per lane when the block has more than 32); when the block has fewer
// than 32 units the lanes split into groups that take different position tiles.  Partial sums are added
// across the lanes of a group with shuffles.
// ---------------------------------------------------------------------------------------------------
template <int NB>  // NB = bytes that are certainly needed (their words are read without an index clamp)
__device__ __forceinline__ void sad_load_run(const uint8_t* p, int nbytes, uint32_t (&out)[6]) {
    // out[j] = bytes [4j, 4j+4) counted from p, for the first 24 bytes; only aligned words holding one of
    // the first `nbytes` bytes are read (others repeat the last valid word: their bytes are never used)
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* w0 = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    const int       shift = (int)(a & 3) * 8, last = (int)(((a & 3) + nbytes - 1) >> 2);
    uint32_t w[7];
#pragma unroll
    for (int j = 0; j < 7; j++) w[j] = __ldg(w0 + (j <= (NB - 1) / 4 ? j : min(j, last)));
#pragma unroll
    for (int j = 0; j < 6; j++) out[j] = __funnelshift_r(w[j], w[j + 1], shift);
}

__device__ __forceinline__ unsigned long long sad_search_warp_w16(const uint8_t* __restrict__ src0, const uint8_t* __restrict__ ref0,
                                                                  const SvtB200SadSearchItem& item, int lane) {
    const int bw = item.block_w, bh = item.block_h, sa_w = item.sa_w, sa_h = item.sa_h;
    const bool skip = (bw == 16 && bh <= 16 && item.skip_search_line);
    const int  lgc = bw == 64 ? 2 : (bw == 32 ? 1 : 0), chunks = 1 << lgc, units = bh << lgc;
    // lanes per group: the smallest power of two >= min(units, 32) (>= chunks, so a lane keeps its chunk)
    int gl = 1;
    while (gl < 32 && gl < units) gl <<= 1;
    const int groups = 32 / gl, grp = lane / gl, ul = lane - grp * gl;
    // with line skipping only the odd search rows are evaluated (compute_sad_c.c:74-79): the tile walk visits just those
    const int ny = skip ? (sa_h >> 1) : sa_h;
    const int xtiles = (sa_w + 7) >> 3, tiles = xtiles * ny;
    const int c = ul & (chunks - 1), r_first = ul >> lgc, r_step = gl >> lgc;
    const uint8_t* src_u = src0 + (size_t)r_first * item.src_stride + 16 * c;  // this lane's first unit
    const uint8_t* ref_u = ref0 + (size_t)r_first * item.ref_stride + 16 * c;
    const size_t   src_adv = (size_t)r_step * item.src_stride, ref_adv = (size_t)r_step * item.ref_stride;
    unsigned long long best = ~0ull;
    int y = 0, xt = grp;  // this group's tile, advanced by `groups` tiles per round
    while (xt >= xtiles) { xt -= xtiles; y++; }
    for (int t0 = 0; t0 < tiles; t0 += groups) {
        const bool tile_on = y < ny;
        const int  yk = tile_on ? y : ny - 1, yy = skip ? 2 * yk + 1 : yk;  // idle groups shadow a valid tile and drop the result
        const int  x0 = (tile_on ? xt : 0) * 8;
        const int  npos = min(8, sa_w - x0);
        const bool line_on = true;
        uint32_t   acc[8];
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = 0;
        if (line_on) {
            const uint8_t* ps = src_u;
            const uint8_t* pr = ref_u + (size_t)yy * item.ref_step + x0;
            for (int r = r_first; r < bh; r += r_step, ps += src_adv, pr += ref_adv) {
                uint32_t sw[6], rw[6];
                sad_load_run<16>(ps, 16, sw);
                sad_load_run<16>(pr, 16 + npos - 1, rw);
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const int ws = i >> 2, sh = (i & 3) * 8;
#pragma unroll
                    for (int k = 0; k < 4; k++)
                        acc[i] = __vsadu4(sw[k], sh ? __funnelshift_r(rw[k + ws], rw[k + ws + 1], sh) : rw[k + ws]) + acc[i];
                }
            }
        }
        // Sum the 8 position accumulators over the lanes of the group.  Shuffle trees, not REDUX (__reduce_add_sync): chosen by
        // kernel times taken on the previous target GPU (not re-measured on H100).
        // Lane distances >= 8 are plain butterflies; the last three steps halve the number of live accumulators each time
        // (a lane keeps the half selected by its own lane bit and hands the other half over), so lane L ends up with the total of
        // position L & 7: 7 shuffles instead of 24.
#pragma unroll
        for (int o = 16; o >= 8; o >>= 1) {
            if (o < gl) {
#pragma unroll
                for (int i = 0; i < 8; i++) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
            }
        }
        if (gl < 8) {  // blocks of fewer than 8 units (picture-edge slivers): groups of 1, 2 or 4 lanes, every lane ranks all 8 positions
#pragma unroll
            for (int o = 2; o >= 1; o >>= 1) {
                if (o < gl) {
#pragma unroll
                    for (int i = 0; i < 8; i++) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
                }
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
                if (tile_on && i < npos && acc[i] < 0xffffffu) {
                    const unsigned long long key = ((unsigned long long)acc[i] << 32) | ((unsigned long long)(uint32_t)yy << 16) | (unsigned long long)(uint32_t)(x0 + i);
                    best = key < best ? key : best;
                }
            }
        } else {
            const bool b2 = lane & 4, b1 = lane & 2, b0 = lane & 1;
            uint32_t   k4[4], k2[2];
#pragma unroll
            for (int i = 0; i < 4; i++) k4[i] = (b2 ? acc[i + 4] : acc[i]) + __shfl_xor_sync(0xffffffffu, b2 ? acc[i] : acc[i + 4], 4);
#pragma unroll
            for (int i = 0; i < 2; i++) k2[i] = (b1 ? k4[i + 2] : k4[i]) + __shfl_xor_sync(0xffffffffu, b1 ? k4[i] : k4[i + 2], 2);
            const uint32_t a = (b0 ? k2[1] : k2[0]) + __shfl_xor_sync(0xffffffffu, b0 ? k2[0] : k2[1], 1);
            const int      i = lane & 7;
            if (tile_on && i < npos && a < 0xffffffu) {
                const unsigned long long key = ((unsigned long long)a << 32) | ((unsigned long long)(uint32_t)yy << 16) | (unsigned long long)(uint32_t)(x0 + i);
                best = key < best ? key : best;
            }
        }
        xt += groups;
        while (xt >= xtiles) { xt -= xtiles; y++; }
    }
    for (int o = 16; o > 0; o >>= 1) {  // every lane holds the best of its own position column / group: the minimum over the warp
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other < best ? other : best;
    }
    return best;
}

// all 32 lanes call; every lane returns the winning key (~0ull when no position qualifies)
__device__ __forceinline__ unsigned long long sad_search_warp(const uint8_t* __restrict__ src0, const uint8_t* __restrict__ ref0,
                                                              const SvtB200SadSearchItem& item, int lane) {
    const int bw = item.block_w, bh = item.block_h, sa_w = item.sa_w, sa_h = item.sa_h;
    unsigned long long best = ~0ull;
    if (sa_w <= 0 || sa_h <= 0 || bw <= 0 || bh <= 0) return best;
    if (bw == 16 || bw == 32 || bw == 64) return sad_search_warp_w16(src0, ref0, item, lane);
    const bool     skip = (bw == 16 && bh <= 16 && item.skip_search_line);
    const int      xs = lane & 7, slice = lane >> 3;
    const int      nw = (bw + 3) >> 2, tail = bw & 3;
    const uint32_t tailmask = tail ? ((1u << (tail * 8)) - 1u) : 0xffffffffu;
    constexpr int  YG = 4;  // search rows evaluated per pass over the source block (the loop body below is written for 4)
    for (int y0 = 0; y0 < sa_h; y0 += YG) {
        for (int x0 = 0; x0 < sa_w; x0 += 8) {
            const bool valid = x0 + xs < sa_w;
            const int  x = valid ? x0 + xs : sa_w - 1;  // idle lanes shadow the last column (stays inside the window)
            uint32_t   acc[YG];
#pragma unroll
            for (int k = 0; k < YG; k++) acc[k] = 0;
            for (int r = slice; r < bh; r += 4) {
                const ByteRun  S(src0 + (size_t)r * item.src_stride, bw);
                const uint8_t* rrow = ref0 + (size_t)r * item.ref_stride + x;
                // rows past the area repeat the last one; their sums are dropped below
                const ByteRun R0(rrow + (size_t)min(y0 + 0, sa_h - 1) * item.ref_step, bw), R1(rrow + (size_t)min(y0 + 1, sa_h - 1) * item.ref_step, bw),
                    R2(rrow + (size_t)min(y0 + 2, sa_h - 1) * item.ref_step, bw), R3(rrow + (size_t)min(y0 + 3, sa_h - 1) * item.ref_step, bw);
                uint32_t slo = S.raw(0), r0 = R0.raw(0), r1 = R1.raw(0), r2 = R2.raw(0), r3 = R3.raw(0);
                // all words but the last: the next aligned word always holds valid bytes, nothing to mask
#pragma unroll 4
                for (int j = 0; j < nw - 1; j++) {
                    const uint32_t shi = __ldg(S.w + j + 1), h0 = __ldg(R0.w + j + 1), h1 = __ldg(R1.w + j + 1), h2 = __ldg(R2.w + j + 1),
                                   h3 = __ldg(R3.w + j + 1);
                    const uint32_t sv = __funnelshift_r(slo, shi, S.shift);  // one source word against four search rows
                    acc[0] = __vsadu4(sv, __funnelshift_r(r0, h0, R0.shift)) + acc[0];
                    acc[1] = __vsadu4(sv, __funnelshift_r(r1, h1, R1.shift)) + acc[1];
                    acc[2] = __vsadu4(sv, __funnelshift_r(r2, h2, R2.shift)) + acc[2];
                    acc[3] = __vsadu4(sv, __funnelshift_r(r3, h3, R3.shift)) + acc[3];
                    slo = shi;
                    r0  = h0;
                    r1  = h1;
                    r2  = h2;
                    r3  = h3;
                }
                {  // last word: the following aligned word may lie past the row (clamped index), bytes past bw are masked
                    const uint32_t shi = S.raw(nw), h0 = R0.raw(nw), h1 = R1.raw(nw), h2 = R2.raw(nw), h3 = R3.raw(nw);
                    const uint32_t sv = __funnelshift_r(slo, shi, S.shift) & tailmask;
                    acc[0] = __vsadu4(sv, __funnelshift_r(r0, h0, R0.shift) & tailmask) + acc[0];
                    acc[1] = __vsadu4(sv, __funnelshift_r(r1, h1, R1.shift) & tailmask) + acc[1];
                    acc[2] = __vsadu4(sv, __funnelshift_r(r2, h2, R2.shift) & tailmask) + acc[2];
                    acc[3] = __vsadu4(sv, __funnelshift_r(r3, h3, R3.shift) & tailmask) + acc[3];
                }
            }
#pragma unroll
            for (int k = 0; k < YG; k++) {
                uint32_t a = acc[k];
                a += __shfl_xor_sync(0xffffffffu, a, 8);
                a += __shfl_xor_sync(0xffffffffu, a, 16);
                const int y = y0 + k;
                if (valid && y < sa_h && !(skip && ((y & 1) == 0)) && a < 0xffffffu) {
                    const unsigned long long key = ((unsigned long long)a << 32) | ((unsigned long long)(uint32_t)y << 16) | (unsigned long long)(uint32_t)x;
                    best = key < best ? key : best;
                }
            }
        }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {  // the 4 slices hold identical keys; reduce over the 8 x-lanes
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other < best ? other : best;
    }
    return best;
}

}  // namespace b200
