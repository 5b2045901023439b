// sad.cu -- K1 full-search SAD (svt_sad_loop_kernel) and K3 single SAD, sm_90a.
//
// Reference behaviour restated (not translated): Source/Lib/C_DEFAULT/compute_sad_c.c:58-101.
//   for y in [0,sa_h): (optionally skip even y when bw==16 && bh<=16 && skip_search_line)
//     for x in [0,sa_w):  sad(x,y) = sum |src[r*src_stride+c] - ref[y*ref_step + x + r*ref_stride + c]|
//     strict '<' update  => the FIRST minimum in raster order wins.
//
// H100 design.  Searches of at most 256 positions (every HME / ME refinement of the presets in scope) take
// the warp-per-search path of sad_small.cuh; larger areas the tiled kernel below: one CTA per work item
// (grid-stride over the list, so one launch serves a whole picture's searches).  The block and a tile of the search window are staged in shared memory as
// 32-bit words; a thread owns M search positions x, x+4, ... x+4(M-1) of one search row so that the
// window words it assembles with a funnel shift are re-used M times against each source word
// (the same sliding trick mpsadbw gives AVX2, but on VABSDIFF4.U8.ACC).  Block rows are split
// across threads when the search area is small (the 8x3 HME refinements), partial sums are merged
// with shared-memory atomics and the winner is the minimum of the 64-bit key (sad<<32 | y<<16 | x),
// which reproduces the raster-order first-minimum rule exactly.
#include "common.cuh"
#include "sad_small.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

constexpr int kSadThreads = 256;
constexpr int kMaxTilePos = 2048;  // search positions per tile (sad buffer 8 KB)

struct TilePlan {
    int tw, th;      // tile size in search positions
    int lw;          // words per staged window line
    int lines;       // staged window lines
    int sw;          // words per staged source row
    int k;           // block-row pitch in units of window lines
    int line_pitch;  // bytes between staged lines in global memory
    int divisible;
};

__host__ __device__ inline TilePlan plan_tile(int bw, int bh, int sa_w, int sa_h, uint32_t ref_stride,
                                              uint32_t ref_step, int smem_bytes) {
    TilePlan p;
    p.sw        = ((bw + 15) >> 4) << 2;
    p.divisible = (ref_step != 0 && (ref_stride % ref_step) == 0) ? 1 : 0;
    p.k         = p.divisible ? (int)(ref_stride / ref_step) : 1;
    p.line_pitch = p.divisible ? (int)ref_step : (int)ref_stride;
    p.tw        = sa_w < 128 ? sa_w : 128;
    if (p.tw < 1) p.tw = 1;
    p.lw   = ((p.tw + bw + 3) >> 2) + 10;
    int avail = smem_bytes - p.sw * 4 * bh - kMaxTilePos * 4 - 64;
    int max_lines = avail / (p.lw * 4);
    if (p.divisible && max_lines < p.k * (bh - 1) + 1) {  // block-row pitch too large to share lines between rows
        p.divisible  = 0;
        p.k          = 1;
        p.line_pitch = (int)ref_stride;
    }
    int th = p.divisible ? (max_lines - p.k * (bh - 1)) : 1;
    if (th > sa_h) th = sa_h;
    if (th > kMaxTilePos / p.tw) th = kMaxTilePos / p.tw;
    if (th < 1) th = 1;
    p.th    = th;
    p.lines = (th - 1) + p.k * (bh - 1) + 1;
    return p;
}

__host__ inline size_t smem_needed(int bw, int bh, int sa_w, int sa_h, int k) {
    int    sw  = ((bw + 15) >> 4) << 2;
    int    tw  = sa_w < 128 ? sa_w : 128;
    int    lw  = ((tw + bw + 3) >> 2) + 10;
    int    th  = sa_h < (kMaxTilePos / (tw > 0 ? tw : 1)) ? sa_h : (kMaxTilePos / (tw > 0 ? tw : 1));
    if (th < 1) th = 1;
    size_t lines = (size_t)(th - 1) + (size_t)k * (bh - 1) + 1;
    return (size_t)sw * 4 * bh + (size_t)kMaxTilePos * 4 + 64 + lines * lw * 4;
}

// Stage `nbytes` starting at global address g (any alignment) into word-aligned shared memory,
// zero-filling up to `nwords` words.  Reads only aligned words that contain at least one valid byte.
__device__ __forceinline__ void stage_line(uint32_t* dst, int nwords, const uint8_t* g, int nbytes, int lane, int nlanes) {
    const uintptr_t ga    = reinterpret_cast<uintptr_t>(g);
    const int       shift = (int)(ga & 3) * 8;
    const uint32_t* gw    = reinterpret_cast<const uint32_t*>(ga & ~uintptr_t(3));
    const int       valid_words = (nbytes + 3) >> 2;
    const int       last_src    = (int)(((ga & 3) + nbytes - 1) >> 2);  // last aligned word holding valid bytes
    for (int w = lane; w < nwords; w += nlanes) {
        uint32_t v = 0;
        if (w < valid_words) {
            uint32_t lo = __ldg(gw + w);
            uint32_t hi = (shift && (w + 1) <= last_src) ? __ldg(gw + w + 1) : 0u;
            v           = __funnelshift_r(lo, hi, shift);
            int rem     = nbytes - (w << 2);
            if (rem < 4) v &= (1u << (rem * 8)) - 1u;
        }
        dst[w] = v;
    }
}

template <int M>
__device__ __forceinline__ void sad_unit(const uint32_t* __restrict__ S, int sw, const uint32_t* __restrict__ W0,
                                         int lw, int k, int xbyte, int nw, uint32_t tailmask, int bh, int s,
                                         int splits, uint32_t (&acc)[M]) {
    const int a8    = (xbyte & 3) * 8;
    const int wbase = xbyte >> 2;
#pragma unroll
    for (int m = 0; m < M; m++) acc[m] = 0;
    for (int r = s; r < bh; r += splits) {
        const uint32_t* Lr = W0 + (size_t)r * k * lw + wbase;
        const uint32_t* Sr = S + r * sw;
        uint32_t        lo = Lr[0];
        uint32_t        w[M];
#pragma unroll
        for (int m = 0; m < M - 1; m++) {
            uint32_t hi = Lr[m + 1];
            w[m]        = __funnelshift_r(lo, hi, a8);
            lo          = hi;
        }
#pragma unroll 4
        for (int j = 0; j < nw - 1; j++) {
            uint32_t hi = Lr[j + M];
            w[M - 1]    = __funnelshift_r(lo, hi, a8);
            lo          = hi;
            uint32_t sv = Sr[j];
#pragma unroll
            for (int m = 0; m < M; m++) acc[m] = __vsadu4(sv, w[m]) + acc[m];
#pragma unroll
            for (int m = 0; m < M - 1; m++) w[m] = w[m + 1];
        }
        {
            const int j  = nw - 1;
            uint32_t  hi = Lr[j + M];
            w[M - 1]     = __funnelshift_r(lo, hi, a8);
            uint32_t sv  = Sr[j];  // bytes beyond bw are zero in the staged block
#pragma unroll
            for (int m = 0; m < M; m++) acc[m] = __vsadu4(sv, w[m] & tailmask) + acc[m];
        }
    }
}

template <int M>
__device__ __forceinline__ void sad_tile(const uint32_t* S, int sw, const uint32_t* W, int lw, int k, int tw, int th,
                                         int bw, int bh, uint32_t* sadbuf, bool skip, int y0) {
    const int      nw       = (bw + 3) >> 2;
    const int      tail     = bw & 3;
    const uint32_t tailmask = tail ? ((1u << (tail * 8)) - 1u) : 0xffffffffu;
    const int      xgroups  = (tw + 4 * M - 1) / (4 * M);
    const int      base_units = xgroups * 4 * th;
    int            splits   = kSadThreads / base_units;
    if (splits < 1) splits = 1;
    if (splits > bh) splits = bh;
    const int nunits = base_units * splits;
    for (int u = threadIdx.x; u < nunits; u += kSadThreads) {
        const int a   = u & 3;
        int       rest = u >> 2;
        const int xg  = rest % xgroups;
        rest /= xgroups;
        const int s  = rest % splits;
        const int yl = rest / splits;
        if (skip && (((y0 + yl) & 1) == 0)) continue;
        const int xbyte = 4 * (xg * M) + a;
        uint32_t  acc[M];
        sad_unit<M>(S, sw, W + (size_t)yl * lw, lw, k, xbyte, nw, tailmask, bh, s, splits, acc);
#pragma unroll
        for (int m = 0; m < M; m++) {
            const int x = xbyte + 4 * m;
            if (x < tw) atomicAdd(&sadbuf[yl * tw + x], acc[m]);
        }
    }
}

__global__ void __launch_bounds__(kSadThreads)
sad_search_kernel(const uint8_t* __restrict__ src_plane, const uint8_t* __restrict__ ref_plane,
                  const SvtB200SadSearchItem* __restrict__ items, int n_items, SvtB200SadSearchResult* __restrict__ results,
                  int smem_bytes) {
    extern __shared__ __align__(16) uint32_t smem[];
    __shared__ unsigned long long             best_key;

    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const SvtB200SadSearchItem item = items[it];
        const int bw = item.block_w, bh = item.block_h;
        const int sa_w = item.sa_w, sa_h = item.sa_h;
        const bool skip = (bw == 16 && bh <= 16 && item.skip_search_line);
        if (threadIdx.x == 0) best_key = ~0ull;
        if (sa_w <= 0 || sa_h <= 0 || bw <= 0 || bh <= 0) {
            __syncthreads();
            if (threadIdx.x == 0) results[it] = SvtB200SadSearchResult{0xffffffu, (int16_t)-1, (int16_t)-1};
            __syncthreads();
            continue;
        }
        const TilePlan p = plan_tile(bw, bh, sa_w, sa_h, item.ref_stride, item.ref_step, smem_bytes);
        uint32_t* S      = smem;
        uint32_t* sadbuf = S + p.sw * bh;
        uint32_t* W      = sadbuf + kMaxTilePos;

        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = kSadThreads >> 5;
        // stage the source block once per item
        for (int r = warp; r < bh; r += nwarps)
            stage_line(S + r * p.sw, p.sw, src_plane + item.src_off + (size_t)r * item.src_stride, bw, lane, 32);

        const uint8_t* ref0 = ref_plane + item.ref_off;
        for (int y0 = 0; y0 < sa_h; y0 += p.th) {
            const int th = min(p.th, sa_h - y0);
            for (int x0 = 0; x0 < sa_w; x0 += p.tw) {
                const int tw = min(p.tw, sa_w - x0);
                __syncthreads();  // previous tile fully consumed (also orders S staging / best_key init)
                const int lines = p.divisible ? ((th - 1) + p.k * (bh - 1) + 1) : bh;
                const uint8_t* lbase = ref0 + (size_t)y0 * item.ref_step + x0;
                for (int l = warp; l < lines; l += nwarps)
                    stage_line(W + (size_t)l * p.lw, p.lw, lbase + (size_t)l * p.line_pitch, tw + bw - 1, lane, 32);
                for (int i = threadIdx.x; i < tw * th; i += kSadThreads) sadbuf[i] = 0;
                __syncthreads();
                if (tw >= 32)
                    sad_tile<4>(S, p.sw, W, p.lw, p.k, tw, th, bw, bh, sadbuf, skip, y0);
                else if (tw >= 8)
                    sad_tile<2>(S, p.sw, W, p.lw, p.k, tw, th, bw, bh, sadbuf, skip, y0);
                else
                    sad_tile<1>(S, p.sw, W, p.lw, p.k, tw, th, bw, bh, sadbuf, skip, y0);
                __syncthreads();
                unsigned long long key = ~0ull;
                for (int i = threadIdx.x; i < tw * th; i += kSadThreads) {
                    const int yl = i / tw, xl = i - yl * tw;
                    const int y = y0 + yl, x = x0 + xl;
                    if (skip && ((y & 1) == 0)) continue;
                    const uint32_t sad = sadbuf[i];
                    if (sad < 0xffffffu) {
                        unsigned long long kk = ((unsigned long long)sad << 32) | ((unsigned long long)(uint32_t)y << 16) |
                                                (unsigned long long)(uint32_t)x;
                        key = kk < key ? kk : key;
                    }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
                    key                      = other < key ? other : key;
                }
                if (lane == 0 && key != ~0ull) atomicMin(&best_key, key);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            SvtB200SadSearchResult r;
            if (best_key == ~0ull) {
                r.best_sad = 0xffffffu;
                r.x = r.y = -1;
            } else {
                r.best_sad = (uint32_t)(best_key >> 32);
                r.y        = (int16_t)((best_key >> 16) & 0xffff);
                r.x        = (int16_t)(best_key & 0xffff);
            }
            results[it] = r;
        }
        __syncthreads();
    }
}

constexpr int kSmallWarps = 4;

__global__ void __launch_bounds__(kSmallWarps * 32)
sad_search_small_kernel(const uint8_t* __restrict__ src_plane, const uint8_t* __restrict__ ref_plane,
                        const SvtB200SadSearchItem* __restrict__ items, int n_items, SvtB200SadSearchResult* __restrict__ results) {
    const int it = blockIdx.x * kSmallWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (it >= n_items) return;
    const SvtB200SadSearchItem item = items[it];
    const unsigned long long best = sad_search_warp(src_plane + item.src_off, ref_plane + item.ref_off, item, lane);
    if (lane == 0) results[it] = sad_key_to_result(best);
}

// K3: one CTA (one warp) per single-SAD item is overkill; T1 callers ask for one block at a time.
__global__ void nxm_sad_kernel(const uint8_t* __restrict__ src, uint32_t src_stride, const uint8_t* __restrict__ ref,
                               uint32_t ref_stride, uint32_t height, uint32_t width, uint32_t* out) {
    uint32_t acc = 0;
    for (uint32_t i = threadIdx.x; i < height * width; i += blockDim.x) {
        uint32_t r = i / width, c = i - r * width;
        int      d = (int)src[(size_t)r * src_stride + c] - (int)ref[(size_t)r * ref_stride + c];
        acc += (uint32_t)(d < 0 ? -d : d);
    }
    __shared__ uint32_t tot;
    if (threadIdx.x == 0) tot = 0;
    __syncthreads();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&tot, acc);
    __syncthreads();
    if (threadIdx.x == 0) *out = tot;
}

void launch_sad_search(const uint8_t* d_src, const uint8_t* d_ref, const SvtB200SadSearchItem* d_items, int n,
                              SvtB200SadSearchResult* d_results, size_t smem, int max_positions, cudaStream_t st) {
    if (n <= 0) return;
    if (max_positions <= kSmallSearchMaxPos) {  // every item of the batch searches at most this many positions
        sad_search_small_kernel<<<(n + kSmallWarps - 1) / kSmallWarps, kSmallWarps * 32, 0, st>>>(d_src, d_ref, d_items, n, d_results);
        B200_LAUNCH_CHECK();
        return;
    }
    Context& c = ctx();
    const size_t dyn_max = (size_t)c.max_smem - 2048;  // opt-in limit minus this kernel's static shared memory
    if (smem > dyn_max) smem = dyn_max;
    if (smem < 32 * 1024) smem = 32 * 1024;
    allow_dynamic_smem(sad_search_kernel, dyn_max);
    int ctas_per_sm = (int)(dyn_max / (smem + 1024));
    if (ctas_per_sm < 1) ctas_per_sm = 1;
    if (ctas_per_sm > 8) ctas_per_sm = 8;
    int grid = grid_for(n, ctas_per_sm);
    sad_search_kernel<<<grid, kSadThreads, smem, st>>>(d_src, d_ref, d_items, n, d_results, (int)smem);
    B200_LAUNCH_CHECK();
}

}  // namespace b200

using namespace b200;

extern "C" int svt_b200_sad_search_batch_dev(const uint8_t* d_src_plane, const uint8_t* d_ref_plane,
                                             const SvtB200SadSearchItem* d_items, int n_items,
                                             SvtB200SadSearchResult* d_results, int max_block_w, int max_block_h,
                                             int max_sa_w, int max_sa_h, int max_row_mult, void* stream) {
    require_ready();
    if (n_items < 0) return SVT_B200_ERR_BAD_ARG;
    size_t smem = smem_needed(max_block_w, max_block_h, max_sa_w, max_sa_h, max_row_mult < 1 ? 1 : max_row_mult);
    launch_sad_search(d_src_plane, d_ref_plane, d_items, n_items, d_results, smem, max_sa_w * max_sa_h, (cudaStream_t)stream);
    return SVT_B200_OK;
}

extern "C" int svt_b200_sad_search_batch_host(const uint8_t* src_plane, size_t src_bytes, const uint8_t* ref_plane,
                                              size_t ref_bytes, const SvtB200SadSearchItem* items, int n_items,
                                              SvtB200SadSearchResult* results) {
    require_ready();
    if (n_items <= 0) return n_items == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    RoundTrip rt;
    auto src = rt.in(src_plane, src_bytes, src_bytes + 8), ref = rt.in(ref_plane, ref_bytes, ref_bytes + 8);
    auto it = rt.in(items, n_items);
    auto res = rt.out(results, n_items);
    size_t smem = 0;
    int max_pos = 0;
    for (int i = 0; i < n_items; i++) {
        const SvtB200SadSearchItem& it = items[i];
        int k = (it.ref_step && it.ref_stride % it.ref_step == 0) ? (int)(it.ref_stride / it.ref_step) : 1;
        size_t s = smem_needed(it.block_w, it.block_h, it.sa_w, it.sa_h, k);
        if (s > smem) smem = s;
        if ((int)it.sa_w * it.sa_h > max_pos) max_pos = (int)it.sa_w * it.sa_h;
    }
    launch_sad_search(rt.dev(src), rt.dev(ref), rt.dev(it), n_items, rt.dev(res), smem, max_pos, rt.stream());
    rt.finish();
    return SVT_B200_OK;
}

extern "C" void svt_b200_sad_loop_kernel(uint8_t* src, uint32_t src_stride, uint8_t* ref, uint32_t ref_stride,
                                         uint32_t block_height, uint32_t block_width, uint64_t* best_sad,
                                         int16_t* x_search_center, int16_t* y_search_center, uint32_t src_stride_raw,
                                         uint8_t skip_search_line, int16_t search_area_width,
                                         int16_t search_area_height) {
    require_ready();
    *best_sad = 0xffffff;
    if (search_area_width <= 0 || search_area_height <= 0 || block_width == 0 || block_height == 0) return;
    RoundTrip rt;
    // the caller's regions as they lie: block rows at src_stride, window at its own pitch
    const size_t src_bytes = (size_t)(block_height - 1) * src_stride + block_width;
    const size_t ref_bytes = (size_t)(search_area_height - 1) * src_stride_raw + (size_t)(block_height - 1) * ref_stride +
                             (size_t)search_area_width + block_width - 1;
    SvtB200SadSearchItem item{};
    item.src_stride = src_stride;
    item.ref_stride = ref_stride;
    item.ref_step = src_stride_raw;
    item.block_w = (uint16_t)block_width;
    item.block_h = (uint16_t)block_height;
    item.sa_w = search_area_width;
    item.sa_h = search_area_height;
    item.skip_search_line = skip_search_line;
    auto s = rt.in(src, src_bytes, src_bytes + 8), win = rt.in(ref, ref_bytes, ref_bytes + 8);
    auto it = rt.in(&item, 1);
    auto res = rt.out<SvtB200SadSearchResult>(nullptr, 1);
    int k = (src_stride_raw && ref_stride % src_stride_raw == 0) ? (int)(ref_stride / src_stride_raw) : 1;
    size_t smem = smem_needed((int)block_width, (int)block_height, search_area_width, search_area_height, k);
    launch_sad_search(rt.dev(s), rt.dev(win), rt.dev(it), 1, rt.dev(res), smem, (int)search_area_width * search_area_height, rt.stream());
    rt.finish();
    const SvtB200SadSearchResult* r = rt.host(res);
    if (r->x >= 0) {
        *best_sad        = r->best_sad;
        *x_search_center = r->x;
        *y_search_center = r->y;
    }
}

extern "C" uint32_t svt_b200_nxm_sad_kernel(const uint8_t* src, uint32_t src_stride, const uint8_t* ref,
                                            uint32_t ref_stride, uint32_t height, uint32_t width) {
    require_ready();
    if (!height || !width) return 0;
    RoundTrip rt;
    const size_t sb = (size_t)(height - 1) * src_stride + width, rb = (size_t)(height - 1) * ref_stride + width;
    auto s = rt.in(src, sb), r = rt.in(ref, rb);
    auto out = rt.out<uint32_t>(nullptr, 1);
    nxm_sad_kernel<<<1, 256, 0, rt.stream()>>>(rt.dev(s), src_stride, rt.dev(r), ref_stride, height, width, rt.dev(out));
    B200_LAUNCH_CHECK();
    rt.finish();
    return *rt.host(out);
}

// ---- T1: svt_aom_sadMxN / svt_aom_sadMxNx4d (aom_dsp_rtcd.h:275-403; C: compute_sad_c.c:104-215) ----
#define B200_SAD_MXN(M, N)                                                                                          \
    extern "C" uint32_t svt_b200_aom_sad##M##x##N(const uint8_t* src, int src_stride, const uint8_t* ref, int ref_stride) { \
        return svt_b200_nxm_sad_kernel(src, (uint32_t)src_stride, ref, (uint32_t)ref_stride, N, M);                \
    }                                                                                                               \
    extern "C" void svt_b200_aom_sad##M##x##N##x4d(const uint8_t* src, int src_stride, const uint8_t* const ref_array[], \
                                                   int ref_stride, uint32_t* sad_array) {                           \
        for (int i = 0; i < 4; i++)                                                                                 \
            sad_array[i] = svt_b200_nxm_sad_kernel(src, (uint32_t)src_stride, ref_array[i], (uint32_t)ref_stride, N, M); \
    }
B200_SAD_MXN(128, 128)
B200_SAD_MXN(128, 64)
B200_SAD_MXN(64, 128)
B200_SAD_MXN(64, 64)
B200_SAD_MXN(64, 32)
B200_SAD_MXN(64, 16)
B200_SAD_MXN(32, 64)
B200_SAD_MXN(32, 32)
B200_SAD_MXN(32, 16)
B200_SAD_MXN(32, 8)
B200_SAD_MXN(16, 64)
B200_SAD_MXN(16, 32)
B200_SAD_MXN(16, 16)
B200_SAD_MXN(16, 8)
B200_SAD_MXN(16, 4)
B200_SAD_MXN(8, 32)
B200_SAD_MXN(8, 16)
B200_SAD_MXN(8, 8)
B200_SAD_MXN(8, 4)
B200_SAD_MXN(4, 16)
B200_SAD_MXN(4, 8)
B200_SAD_MXN(4, 4)
#undef B200_SAD_MXN
