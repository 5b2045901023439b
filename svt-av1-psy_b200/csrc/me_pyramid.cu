// me_pyramid.cu -- K2 SAD pyramid (8x8 -> 16x16 -> 32x32 -> 64x64) and the T2 full-pel search that
// is built from it (sm_90a).
//
// Reference behaviour restated:
//   svt_ext_all_sad_calculation_8x8_16x16_c   Source/Lib/Codec/motion_estimation.c:335-363 (+:210-333)
//   svt_ext_eight_sad_calculation_32x32_64x64_c                                   :369-427
//   svt_ext_sad_calculation_8x8_16x16_c / _32x32_64x64_c (1-point variants)        :98-205
//   open_loop_me_fullpel_search_sblock                                            :781-817
// Block numbering: 16x16 blocks are indexed in 32x32-quadrant order (offsets[] table at :341), the
// four 8x8 of 16x16 p are 4p..4p+3 in raster order.  Every best-SAD update is a strict '<' in search
// order (y outer, x inner), i.e. "first minimum in raster order" per PU -- reproduced here as the
// minimum of the 64-bit key (sad << 32 | raster index).  Result layout = me_context.h:54-75
// (64x64 at 0, 32x32 at 1..4, 16x16 at 5..20, 8x8 at 21..84).
#include <cuda.h>
#include <mutex>
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

__device__ __forceinline__ int z16_of(int y16, int x16) { return 4 * (2 * (y16 >> 1) + (x16 >> 1)) + 2 * (y16 & 1) + (x16 & 1); }
__device__ __forceinline__ uint32_t pack_mv(int x, int y) { return ((uint32_t)(y & 0xffff) << 16) | (uint32_t)(x & 0xffff); }

// ---------------------------------------------------------------------------------------------
// T1 kernels (caller state in/out, one launch per reference call)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sad8x8_global(const uint8_t* s, uint32_t ss, const uint8_t* r, uint32_t rs, bool sub) {
    uint32_t acc = 0;
    const int step = sub ? 2 : 1;
    for (int y = 0; y < 8; y += step)
        for (int x = 0; x < 8; x++) {
            int d = (int)s[y * ss + x] - (int)r[y * rs + x];
            acc += (uint32_t)(d < 0 ? -d : d);
        }
    return sub ? acc << 1 : acc;
}

// 64 threads: thread = (16x16 raster index, 8x8 k)
__global__ void ext_all_sad_kernel(const uint8_t* src, uint32_t ss, const uint8_t* ref, uint32_t rs, uint32_t mv,
                                   uint32_t* best8, uint32_t* best16, uint32_t* mv8, uint32_t* mv16, uint32_t* eight16,
                                   int sub) {
    __shared__ uint32_t s8[64][8];
    const int t = threadIdx.x, b16 = t >> 2, k = t & 3;
    const int y16 = b16 >> 2, x16 = b16 & 3, p16 = z16_of(y16, x16);
    const uint8_t* s = src + (16 * y16 + 8 * (k >> 1)) * ss + 16 * x16 + 8 * (k & 1);
    const uint8_t* r = ref + (16 * y16 + 8 * (k >> 1)) * rs + 16 * x16 + 8 * (k & 1);
    const int xmv = (int16_t)(mv & 0xffff), ymv = (int16_t)(mv >> 16);
    uint32_t b = best8[4 * p16 + k], bm = mv8[4 * p16 + k];
    for (int i = 0; i < 8; i++) {
        const uint32_t v = sad8x8_global(s, ss, r + i, rs, sub);
        s8[4 * p16 + k][i] = v;
        if (v < b) {
            b  = v;
            bm = pack_mv((int16_t)(xmv + i), ymv);
        }
    }
    best8[4 * p16 + k] = b;
    mv8[4 * p16 + k]   = bm;
    __syncthreads();
    if (t < 16) {
        uint32_t bb = best16[t], bbm = mv16[t];
        for (int i = 0; i < 8; i++) {
            const uint32_t v = s8[4 * t][i] + s8[4 * t + 1][i] + s8[4 * t + 2][i] + s8[4 * t + 3][i];
            eight16[t * 8 + i] = v;
            if (v < bb) {
                bb  = v;
                bbm = pack_mv((int16_t)(xmv + i), ymv);
            }
        }
        best16[t] = bb;
        mv16[t]   = bbm;
    }
}

// n_idx = 8 (eight-point form, sad16 is [16][8]) or 1 (one-point form, sad16 is [16])
__global__ void ext_sad_32_64_kernel(const uint32_t* sad16, uint32_t* best32, uint32_t* best64, uint32_t* mv32,
                                     uint32_t* mv64, uint32_t mv, uint32_t* sad32, int n_idx) {
    if (threadIdx.x != 0) return;
    const int xmv = (int16_t)(mv & 0xffff), ymv = (int16_t)(mv >> 16);
    for (int i = 0; i < n_idx; i++) {
        uint32_t tot = 0;
        const uint32_t m = n_idx == 8 ? pack_mv((int16_t)(xmv + i), ymv) : mv;
        for (int q = 0; q < 4; q++) {
            const uint32_t v = sad16[(4 * q + 0) * n_idx + i] + sad16[(4 * q + 1) * n_idx + i] + sad16[(4 * q + 2) * n_idx + i] +
                               sad16[(4 * q + 3) * n_idx + i];
            sad32[q * n_idx + i] = v;
            if (v < best32[q]) {
                best32[q] = v;
                mv32[q]   = m;
            }
            tot += v;
        }
        if (tot < best64[0]) {
            best64[0] = tot;
            mv64[0]   = m;
        }
    }
}

// one 16x16: 4 threads
__global__ void ext_sad_8_16_kernel(const uint8_t* src, uint32_t ss, const uint8_t* ref, uint32_t rs, uint32_t* best8,
                                    uint32_t* best16, uint32_t* mv8, uint32_t* mv16, uint32_t mv, uint32_t* sad16,
                                    uint32_t* sad8, int sub) {
    __shared__ uint32_t v4[4];
    const int k = threadIdx.x;
    const uint32_t v = sad8x8_global(src + 8 * (k >> 1) * ss + 8 * (k & 1), ss, ref + 8 * (k >> 1) * rs + 8 * (k & 1), rs, sub);
    v4[k]   = v;
    sad8[k] = v;
    if (v < best8[k]) {
        best8[k] = v;
        mv8[k]   = mv;
    }
    __syncthreads();
    if (k == 0) {
        const uint32_t t = v4[0] + v4[1] + v4[2] + v4[3];
        if (t < best16[0]) {
            best16[0] = t;
            mv16[0]   = mv;
        }
        *sad16 = t;
    }
}

// ---------------------------------------------------------------------------------------------
// T2: full-pel search of one 64x64 block over sa_w x sa_h positions, all 85 square PUs at once
// ---------------------------------------------------------------------------------------------
constexpr int kFpThreads = 256;
constexpr int kFpTW = 16, kFpTH = 4;              // positions per chunk
constexpr int kFpLW = (kFpTW + 64 + 3) / 4 + 3;   // words per staged window line (odd-ish pitch)
constexpr int kFpLines = kFpTH + 63;

__device__ __forceinline__ void stage_words(uint32_t* dst, int nwords, const uint8_t* g, int nbytes, int lane, int nlanes) {
    const uintptr_t ga = reinterpret_cast<uintptr_t>(g);
    const int       shift = (int)(ga & 3) * 8;
    const uint32_t* gw = reinterpret_cast<const uint32_t*>(ga & ~uintptr_t(3));
    const int       valid = (nbytes + 3) >> 2, last_src = (int)(((ga & 3) + nbytes - 1) >> 2);
    for (int w = lane; w < nwords; w += nlanes) {
        uint32_t v = 0;
        if (w < valid) {
            const uint32_t lo = __ldg(gw + w);
            const uint32_t hi = (shift && (w + 1) <= last_src) ? __ldg(gw + w + 1) : 0u;
            v = __funnelshift_r(lo, hi, shift);
            const int rem = nbytes - (w << 2);
            if (rem < 4) v &= (1u << (rem * 8)) - 1u;
        }
        dst[w] = v;
    }
}

// rows x nwords words of `nbytes`-byte rows at any alignment, all threads of the CTA, one word per step
__device__ __forceinline__ void stage_rows(uint32_t* dst, int nwords, int rows, const uint8_t* g, size_t pitch, int nbytes) {
    const int valid = (nbytes + 3) >> 2;
#pragma unroll 4
    for (int i = threadIdx.x; i < rows * nwords; i += kFpThreads) {
        const int r = i / nwords, w = i - r * nwords;
        const uintptr_t ga = reinterpret_cast<uintptr_t>(g + (size_t)r * pitch);
        const int       shift = (int)(ga & 3) * 8, last_src = (int)(((ga & 3) + nbytes - 1) >> 2);
        const uint32_t* gw = reinterpret_cast<const uint32_t*>(ga & ~uintptr_t(3));
        uint32_t v = 0;
        if (w < valid) {
            const uint32_t lo = __ldg(gw + w);
            const uint32_t hi = (shift && (w + 1) <= last_src) ? __ldg(gw + w + 1) : 0u;
            v = __funnelshift_r(lo, hi, shift);
            const int rem = nbytes - (w << 2);
            if (rem < 4) v &= (1u << (rem * 8)) - 1u;
        }
        dst[r * nwords + w] = v;
    }
}

// ---- TMA plumbing (sm_90a): one elected thread arms an mbarrier with the byte count and issues cp.async.bulk.tensor;
// the box lands in shared memory with no per-thread address arithmetic, alignment fix-up or funnel shifts --------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

constexpr int kFpTmaRefs = 8;                     // reference pictures per launch that can be addressed through tensor maps
// Design rule: every box of a 1-byte tensor starts on a 16-byte aligned innermost coordinate.  A search window starts anywhere,
// so its box is taken from the aligned address below it, 16 bytes wider, and the positions are addressed with the residual
// byte offset.
constexpr int kFpBoxW = 96, kFpBoxH = kFpLines;   // bytes x rows of one window box (15 + kFpTW + 63 = 94 bytes used)
constexpr int kFpSrcBoxW = 80;                    // source block: 64 bytes + up to 12 of alignment slack (word-aligned origins only)
struct FpTma {
    CUtensorMap cur, ref[kFpTmaRefs];             // 2-D byte tensors over the padded full-resolution luma planes
    const uint8_t* cur_base;
    const uint8_t* ref_base[kFpTmaRefs];
    int32_t cur_pitch, ref_pitch[kFpTmaRefs];
    int32_t n_b64;                                // items are ordered (reference, b64)
};

// TMA = true (open-loop ME of a picture, svt_b200_me_b64_picture_dev): source block and search-window boxes arrive by TMA,
// double-buffered -- the box of the next (item, chunk) is in flight while the current one is searched.
// TMA = false (svt_b200_fullpel_search_batch_dev on caller planes of unknown extent): staged by the threads.
template <bool TMA>
__global__ void __launch_bounds__(kFpThreads)
fullpel_search_kernel(const uint8_t* __restrict__ src_plane, const uint8_t* __restrict__ ref_plane,
                      const SvtB200FullpelItem* __restrict__ items, int n_items, uint32_t* __restrict__ best_sad,
                      uint32_t* __restrict__ best_mv, const uint32_t* __restrict__ seed_sad /* [n_items][85] or null */,
                      const __grid_constant__ FpTma tm) {
    constexpr int LW = TMA ? kFpBoxW / 4 : kFpLW;  // words per staged window line
    constexpr int SW = TMA ? kFpSrcBoxW / 4 : 16;  // words per staged source line
    __shared__ __align__(128) uint32_t Sbuf[TMA ? 2 : 1][64 * (TMA ? kFpSrcBoxW / 4 : 16)];
    __shared__ __align__(128) uint32_t Wbuf[TMA ? 2 : 1][TMA ? (((kFpBoxW / 4) * kFpBoxH + 31) & ~31) : kFpLines * kFpLW];  // every TMA buffer starts 128-byte aligned
    __shared__ uint32_t sad8[kFpTW * kFpTH][65];
    __shared__ uint32_t sadpu[kFpTW * kFpTH][21];  // 64x64, 4 x 32x32, 16 x 16x16 of every position
    __shared__ unsigned long long best[85];
    __shared__ uint64_t bars[2];

    // issue the boxes of chunk (y0, x0) of item `it` into buffer `b` (one thread)
    auto issue = [&](int it, int y0, int x0, int b, int sbuf, bool with_src) {
        const SvtB200FullpelItem& item = items[it];
        const int r = it / tm.n_b64;
        const size_t roff = (size_t)(item.ref_off - (uint64_t)(uintptr_t)tm.ref_base[r]);
        const int ry = (int)(roff / (size_t)tm.ref_pitch[r]), rx = (int)(roff - (size_t)ry * tm.ref_pitch[r]);
        mbar_expect_tx(&bars[b], (uint32_t)(kFpBoxW * kFpBoxH + (with_src ? kFpSrcBoxW * 64 : 0)));
        tma_load_2d(Wbuf[b], &tm.ref[r], (rx + x0) & ~15, ry + y0, &bars[b]);
        if (with_src) {
            const size_t soff = (size_t)(item.src_off - (uint64_t)(uintptr_t)tm.cur_base);
            const int sy = (int)(soff / (size_t)tm.cur_pitch), sx = (int)(soff - (size_t)sy * tm.cur_pitch);
            tma_load_2d(Sbuf[sbuf], &tm.cur, sx & ~15, sy, &bars[b]);
        }
    };
    if (TMA) {
        if (threadIdx.x == 0) {
            mbar_init(&bars[0], 1);
            mbar_init(&bars[1], 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0 && (int)blockIdx.x < n_items) issue(blockIdx.x, 0, 0, 0, 0, true);
    }
    int n = 0, k = 0;  // n: boxes consumed so far (buffer n & 1, phase (n >> 1) & 1); k: items processed by this CTA

    for (int it = blockIdx.x; it < n_items; it += gridDim.x, k++) {
        const SvtB200FullpelItem item = items[it];
        const int sa_w = item.sa_w, sa_h = item.sa_h, sub = item.sub_sad;
        // key = sad << 32 | (scan index + 1); index 0 is the seed position (evaluated before the scan, so it wins ties)
        if (threadIdx.x < 85)
            best[threadIdx.x] = (item.seeded && seed_sad) ? ((unsigned long long)seed_sad[(size_t)it * 85 + threadIdx.x] << 32)
                                                          : (((unsigned long long)(128u * 128u * 255u) << 32) | 0xffffffffull);
        int rx0 = 0;  // column of the window origin / word offset of the source block inside their aligned boxes
        const uint32_t* S = Sbuf[TMA ? (k & 1) : 0];
        if (TMA) {
            const int r = it / tm.n_b64;
            const size_t roff = (size_t)(item.ref_off - (uint64_t)(uintptr_t)tm.ref_base[r]);
            rx0 = (int)(roff % (size_t)tm.ref_pitch[r]);
            const size_t soff = (size_t)(item.src_off - (uint64_t)(uintptr_t)tm.cur_base);
            S += ((int)(soff % (size_t)tm.cur_pitch) & 15) >> 2;
        }
        // flat staging: every thread's words are independent loads, so one global round trip covers the block
        if (!TMA) stage_rows(Sbuf[0], 16, 64, src_plane + item.src_off, item.src_stride, 64);
        for (int y0 = 0; y0 < sa_h; y0 += kFpTH) {
            const int th = min(kFpTH, sa_h - y0);
            for (int x0 = 0; x0 < sa_w; x0 += kFpTW) {
                const int tw = min(kFpTW, sa_w - x0);
                __syncthreads();
                const uint32_t* W = Wbuf[TMA ? (n & 1) : 0];
                if (TMA) {
                    if (threadIdx.x == 0) {  // prefetch the next box: next chunk of this item, else the first chunk of the CTA's next item
                        int nx = x0 + kFpTW, ny = y0, nit = it;
                        bool src = false;
                        if (nx >= sa_w) { nx = 0; ny = y0 + kFpTH; }
                        if (ny >= sa_h) { ny = 0; nit = it + gridDim.x; src = true; }
                        if (nit < n_items) issue(nit, ny, nx, (n + 1) & 1, (k + 1) & 1, src);
                    }
                    while (!mbar_try_wait(&bars[n & 1], (uint32_t)((n >> 1) & 1))) {}
                    n++;
                } else {
                    stage_rows(Wbuf[0], kFpLW, th + 63, ref_plane + item.ref_off + (size_t)y0 * item.ref_stride + x0, item.ref_stride, tw + 63);
                    __syncthreads();
                }
                // 8x8 SADs: unit = (position, 8x8 block).  A warp takes one block row `by`, the 8 block columns and 4 consecutive
                // positions: lanes that differ in position read the same window words (broadcast), lanes that differ in column read
                // words 2 apart -- conflict free at any line pitch.  Results are stored in z-order so that the four 8x8 of a 16x16
                // (and the four 16x16 of a 32x32) are neighbours.
                const int npos = tw * th, ngrp = (npos + 3) >> 2;
                const int dx = TMA ? ((rx0 + x0) & 15) : 0;
                for (int u = threadIdx.x; u < ngrp * 256; u += kFpThreads) {
                    const int lane = u & 31, wi = u >> 5;
                    const int bx = lane & 7, by = wi & 7, pos = (wi >> 3) * 4 + (lane >> 3);
                    if (pos >= npos) continue;
                    const int py = pos / tw, px = pos - py * tw;
                    const int a8 = ((px + dx) & 3) * 8, wb = ((px + dx) >> 2) + 2 * bx;
                    uint32_t  acc = 0;
#pragma unroll
                    for (int r = 0; r < 8; r++) {
                        if (sub && (r & 1)) continue;
                        const uint32_t* L = W + (py + 8 * by + r) * LW + wb;
                        const uint32_t* Sr = S + (8 * by + r) * SW + 2 * bx;
                        const uint32_t w0 = L[0], w1 = L[1], w2 = L[2];
                        acc = __vsadu4(Sr[0], __funnelshift_r(w0, w1, a8)) + acc;
                        acc = __vsadu4(Sr[1], __funnelshift_r(w1, w2, a8)) + acc;
                    }
                    if (sub) acc <<= 1;
                    const int y16 = by >> 1, x16 = bx >> 1;
                    sad8[pos][4 * z16_of(y16, x16) + 2 * (by & 1) + (bx & 1)] = acc;
                }
                __syncthreads();
                // 16x16 / 32x32 / 64x64 sums: 16 lanes per position, lane = 16x16 z-index; two shuffle
                // steps give the 32x32 of each quad, two more the 64x64
                for (int u = threadIdx.x; u < ((npos * 16 + 31) & ~31); u += kFpThreads) {
                    const int  pos = u >> 4, z = u & 15;
                    const bool on = pos < npos;
                    uint32_t   v16 = 0;
                    if (on) v16 = sad8[pos][4 * z] + sad8[pos][4 * z + 1] + sad8[pos][4 * z + 2] + sad8[pos][4 * z + 3];
                    uint32_t v32 = v16 + __shfl_xor_sync(0xffffffffu, v16, 1);
                    v32 += __shfl_xor_sync(0xffffffffu, v32, 2);
                    uint32_t v64 = v32 + __shfl_xor_sync(0xffffffffu, v32, 4);
                    v64 += __shfl_xor_sync(0xffffffffu, v64, 8);
                    if (on) {
                        sadpu[pos][5 + z] = v16;
                        if ((z & 3) == 0) sadpu[pos][1 + (z >> 2)] = v32;
                        if (z == 0) sadpu[pos][0] = v64;
                    }
                }
                __syncthreads();
                // per-PU scan of this chunk's positions; key = sad<<32 | raster index
                if (threadIdx.x < 85) {
                    const int pu = threadIdx.x;
                    unsigned long long b = best[pu];
                    for (int pos = 0; pos < npos; pos++) {
                        const uint32_t v = pu < 21 ? sadpu[pos][pu] : sad8[pos][pu - 21];
                        const int py = pos / tw, px = pos - py * tw;
                        const unsigned long long key =
                            ((unsigned long long)v << 32) | (unsigned long long)(uint32_t)((y0 + py) * sa_w + (x0 + px) + 1);
                        b = key < b ? key : b;
                    }
                    best[pu] = b;
                }
            }
        }
        __syncthreads();
        if (threadIdx.x < 85) {
            const unsigned long long b = best[threadIdx.x];
            const uint32_t idx = (uint32_t)(b & 0xffffffffull);
            best_sad[(size_t)it * 85 + threadIdx.x] = (uint32_t)(b >> 32);
            if (idx == 0xffffffffu)
                best_mv[(size_t)it * 85 + threadIdx.x] = 0;
            else if (idx == 0)
                best_mv[(size_t)it * 85 + threadIdx.x] = pack_mv(item.seed_x, item.seed_y);
            else {
                const int y = (int)((idx - 1) / (uint32_t)sa_w), x = (int)((idx - 1) - (uint32_t)y * sa_w);
                best_mv[(size_t)it * 85 + threadIdx.x] = pack_mv(item.org_x + x, item.org_y + y);
            }
        }
        __syncthreads();
    }
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        B200_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        if (q != cudaDriverEntryPointSuccess || !p) {
            fprintf(stderr, "[svt_b200] FATAL: cuTensorMapEncodeTiled is not available from this driver\n");
            abort();
        }
        fn = (EncodeTiledFn)p;
    });
    return fn;
}
// 2-D byte tensor over a padded 8-bit plane (base 16-byte aligned, pitch a multiple of 16: the layout rule of every plane of
// this library, DESIGN.md section 4), box = box_w x box_h bytes, no swizzle; elements outside the plane read as zero
static bool make_plane_map(CUtensorMap* m, const uint8_t* base, int pitch, int rows, int box_w, int box_h) {
    if ((reinterpret_cast<uintptr_t>(base) & 15) || (pitch & 15) || pitch <= 0 || rows <= 0) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)pitch, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)pitch};
    const cuuint32_t box[2] = {(cuuint32_t)box_w, (cuuint32_t)box_h};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode_tiled_fn()(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(base), dims, strides, box, estr,
                                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// full-pel search of a picture's (reference, b64) items through TMA; false = geometry not expressible (the caller fails)
bool launch_fullpel_tma(const SvtB200MePicture* cur, const SvtB200MePicture* refs, int n_refs, int n_b64, const SvtB200FullpelItem* d_items,
                        int n_items, uint32_t* d_best_sad, uint32_t* d_best_mv, cudaStream_t st, const uint32_t* d_seed_sad) {
    if (n_refs > kFpTmaRefs) return false;
    FpTma tm;
    memset(&tm, 0, sizeof(tm));
    auto rows_of = [](const SvtB200MePicture& p) { return p.height[2] + 2 * p.org_y[2]; };
    if (cur->org_x[2] & 3) return false;  // the source block must start on a word of its aligned box
    if (!make_plane_map(&tm.cur, cur->plane[2], cur->stride[2], rows_of(*cur), kFpSrcBoxW, 64)) return false;
    tm.cur_base = cur->plane[2];
    tm.cur_pitch = cur->stride[2];
    for (int r = 0; r < n_refs; r++) {
        if (!make_plane_map(&tm.ref[r], refs[r].plane[2], refs[r].stride[2], rows_of(refs[r]), kFpBoxW, kFpBoxH)) return false;
        tm.ref_base[r] = refs[r].plane[2];
        tm.ref_pitch[r] = refs[r].stride[2];
    }
    tm.n_b64 = n_b64;
    fullpel_search_kernel<true><<<grid_for(n_items, 4), kFpThreads, 0, st>>>(nullptr, nullptr, d_items, n_items, d_best_sad, d_best_mv, d_seed_sad, tm);
    B200_LAUNCH_CHECK();
    return true;
}

}  // namespace b200

using namespace b200;

extern "C" void svt_b200_ext_all_sad_calculation_8x8_16x16(uint8_t* src, uint32_t src_stride, uint8_t* ref, uint32_t ref_stride,
                                                           uint32_t mv, uint32_t* p_best_sad_8x8, uint32_t* p_best_sad_16x16,
                                                           uint32_t* p_best_mv8x8, uint32_t* p_best_mv16x16,
                                                           uint32_t p_eight_sad16x16[16][8], uint32_t p_eight_sad8x8[64][8],
                                                           uint8_t sub_sad) {
    (void)p_eight_sad8x8;  // not written by the reference C kernel either (motion_estimation.c:221)
    require_ready();
    LaneGuard l;
    const size_t sb = 63 * (size_t)src_stride + 64, rb = 63 * (size_t)ref_stride + 64 + 7;
    size_t o_src = l->alloc(sb), o_ref = l->alloc(rb);
    size_t o_st = l->alloc((64 + 16 + 64 + 16) * 4);  // best8, best16, mv8, mv16
    size_t in_end = l->used;
    size_t o_e16 = l->alloc(16 * 8 * 4);
    memcpy(l->h<uint8_t>(o_src), src, sb);
    memcpy(l->h<uint8_t>(o_ref), ref, rb);
    uint32_t* st = l->h<uint32_t>(o_st);
    memcpy(st, p_best_sad_8x8, 64 * 4);
    memcpy(st + 64, p_best_sad_16x16, 16 * 4);
    memcpy(st + 80, p_best_mv8x8, 64 * 4);
    memcpy(st + 144, p_best_mv16x16, 16 * 4);
    l->h2d(0, in_end);
    uint32_t* d = l->d<uint32_t>(o_st);
    ext_all_sad_kernel<<<1, 64, 0, l->stream>>>(l->d<uint8_t>(o_src), src_stride, l->d<uint8_t>(o_ref), ref_stride, mv, d, d + 64,
                                                d + 80, d + 144, l->d<uint32_t>(o_e16), sub_sad ? 1 : 0);
    B200_LAUNCH_CHECK();
    l->d2h(o_st, (o_e16 + 16 * 8 * 4) - o_st);
    l->sync();
    memcpy(p_best_sad_8x8, st, 64 * 4);
    memcpy(p_best_sad_16x16, st + 64, 16 * 4);
    memcpy(p_best_mv8x8, st + 80, 64 * 4);
    memcpy(p_best_mv16x16, st + 144, 16 * 4);
    memcpy(p_eight_sad16x16, l->h<uint32_t>(o_e16), 16 * 8 * 4);
}

static void ext_32_64_t1(const uint32_t* sad16, uint32_t* b32, uint32_t* b64, uint32_t* m32, uint32_t* m64, uint32_t mv,
                         uint32_t* sad32, int n_idx) {
    require_ready();
    LaneGuard l;
    size_t o_in = l->alloc(16 * 8 * 4), o_st = l->alloc(10 * 4);
    size_t in_end = l->used;
    size_t o_s32 = l->alloc(4 * 8 * 4);
    memcpy(l->h<uint32_t>(o_in), sad16, (size_t)16 * n_idx * 4);
    uint32_t* st = l->h<uint32_t>(o_st);
    memcpy(st, b32, 16);
    st[4] = b64[0];
    memcpy(st + 5, m32, 16);
    st[9] = m64[0];
    l->h2d(0, in_end);
    uint32_t* d = l->d<uint32_t>(o_st);
    ext_sad_32_64_kernel<<<1, 32, 0, l->stream>>>(l->d<uint32_t>(o_in), d, d + 4, d + 5, d + 9, mv, l->d<uint32_t>(o_s32), n_idx);
    B200_LAUNCH_CHECK();
    l->d2h(o_st, (o_s32 + 4 * 8 * 4) - o_st);
    l->sync();
    memcpy(b32, st, 16);
    b64[0] = st[4];
    memcpy(m32, st + 5, 16);
    m64[0] = st[9];
    memcpy(sad32, l->h<uint32_t>(o_s32), (size_t)4 * n_idx * 4);
}

extern "C" void svt_b200_ext_eight_sad_calculation_32x32_64x64(uint32_t p_sad16x16[16][8], uint32_t* p_best_sad_32x32,
                                                               uint32_t* p_best_sad_64x64, uint32_t* p_best_mv32x32,
                                                               uint32_t* p_best_mv64x64, uint32_t mv, uint32_t p_sad32x32[4][8]) {
    ext_32_64_t1(&p_sad16x16[0][0], p_best_sad_32x32, p_best_sad_64x64, p_best_mv32x32, p_best_mv64x64, mv, &p_sad32x32[0][0], 8);
}
extern "C" void svt_b200_ext_sad_calculation_32x32_64x64(uint32_t* p_sad16x16, uint32_t* p_best_sad_32x32,
                                                         uint32_t* p_best_sad_64x64, uint32_t* p_best_mv32x32,
                                                         uint32_t* p_best_mv64x64, uint32_t mv, uint32_t* p_sad32x32) {
    ext_32_64_t1(p_sad16x16, p_best_sad_32x32, p_best_sad_64x64, p_best_mv32x32, p_best_mv64x64, mv, p_sad32x32, 1);
}

extern "C" void svt_b200_ext_sad_calculation_8x8_16x16(uint8_t* src, uint32_t src_stride, uint8_t* ref, uint32_t ref_stride,
                                                       uint32_t* p_best_sad_8x8, uint32_t* p_best_sad_16x16, uint32_t* p_best_mv8x8,
                                                       uint32_t* p_best_mv16x16, uint32_t mv, uint32_t* p_sad16x16,
                                                       uint32_t* p_sad8x8, uint8_t sub_sad) {
    require_ready();
    LaneGuard l;
    const size_t sb = 15 * (size_t)src_stride + 16, rb = 15 * (size_t)ref_stride + 16;
    size_t o_src = l->alloc(sb), o_ref = l->alloc(rb), o_st = l->alloc(10 * 4);
    size_t in_end = l->used;
    size_t o_out = l->alloc(5 * 4);
    memcpy(l->h<uint8_t>(o_src), src, sb);
    memcpy(l->h<uint8_t>(o_ref), ref, rb);
    uint32_t* st = l->h<uint32_t>(o_st);
    memcpy(st, p_best_sad_8x8, 16);
    st[4] = p_best_sad_16x16[0];
    memcpy(st + 5, p_best_mv8x8, 16);
    st[9] = p_best_mv16x16[0];
    l->h2d(0, in_end);
    uint32_t* d = l->d<uint32_t>(o_st);
    uint32_t* o = l->d<uint32_t>(o_out);
    ext_sad_8_16_kernel<<<1, 4, 0, l->stream>>>(l->d<uint8_t>(o_src), src_stride, l->d<uint8_t>(o_ref), ref_stride, d, d + 4, d + 5,
                                                d + 9, mv, o + 4, o, sub_sad ? 1 : 0);
    B200_LAUNCH_CHECK();
    l->d2h(o_st, (o_out + 20) - o_st);
    l->sync();
    memcpy(p_best_sad_8x8, st, 16);
    p_best_sad_16x16[0] = st[4];
    memcpy(p_best_mv8x8, st + 5, 16);
    p_best_mv16x16[0] = st[9];
    memcpy(p_sad8x8, l->h<uint32_t>(o_out), 16);
    *p_sad16x16 = l->h<uint32_t>(o_out)[4];
}

// svt_initialize_buffer_32bits (aom_dsp_rtcd.h:855): pure host-memory fill; there is nothing for a
// device to do here, so the H100 tier keeps it as the trivial host loop it is.
extern "C" void svt_b200_initialize_buffer_32bits(uint32_t* pointer, uint32_t count128, uint32_t count32, uint32_t value) {
    const uint32_t n = count128 * 4 + count32;
    for (uint32_t i = 0; i < n; i++) pointer[i] = value;
}

extern "C" int svt_b200_fullpel_search_batch_dev(const uint8_t* d_src_plane, const uint8_t* d_ref_plane,
                                                 const SvtB200FullpelItem* d_items, int n_items, uint32_t* d_best_sad,
                                                 uint32_t* d_best_mv, void* stream) {
    require_ready();
    if (n_items <= 0) return n_items == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    FpTma none;
    memset(&none, 0, sizeof(none));
    none.n_b64 = 1;
    fullpel_search_kernel<false><<<grid_for(n_items, 4), kFpThreads, 0, (cudaStream_t)stream>>>(d_src_plane, d_ref_plane, d_items, n_items,
                                                                                              d_best_sad, d_best_mv, nullptr, none);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_fullpel_search_batch_host(const uint8_t* src_plane, size_t src_bytes, const uint8_t* ref_plane,
                                                  size_t ref_bytes, const SvtB200FullpelItem* items, int n_items,
                                                  uint32_t* best_sad, uint32_t* best_mv) {
    require_ready();
    if (n_items <= 0) return n_items == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    LaneGuard l;
    size_t o_src = l->alloc(src_bytes + 8), o_ref = l->alloc(ref_bytes + 8), o_it = l->alloc(sizeof(SvtB200FullpelItem) * n_items);
    size_t in_end = l->used;
    size_t o_sad = l->alloc((size_t)n_items * 85 * 4), o_mv = l->alloc((size_t)n_items * 85 * 4);
    memcpy(l->h<uint8_t>(o_src), src_plane, src_bytes);
    memcpy(l->h<uint8_t>(o_ref), ref_plane, ref_bytes);
    memcpy(l->h<uint8_t>(o_it), items, sizeof(SvtB200FullpelItem) * n_items);
    l->h2d(0, in_end);
    svt_b200_fullpel_search_batch_dev(l->d<uint8_t>(o_src), l->d<uint8_t>(o_ref), l->d<SvtB200FullpelItem>(o_it), n_items,
                                      l->d<uint32_t>(o_sad), l->d<uint32_t>(o_mv), l->stream);
    l->d2h(o_sad, (o_mv + (size_t)n_items * 85 * 4) - o_sad);
    l->sync();
    memcpy(best_sad, l->h<uint32_t>(o_sad), (size_t)n_items * 85 * 4);
    memcpy(best_mv, l->h<uint32_t>(o_mv), (size_t)n_items * 85 * 4);
    return SVT_B200_OK;
}
