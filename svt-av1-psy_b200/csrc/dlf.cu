// dlf.cu -- K14, the AV1 deblocking loop filter (reference: deblocking_common.c:242-866, deblocking_filter.c:144-654).
//
// T1: the 16 dispatched lpf functions.  A call stages exactly the pixels the reference reads (4 lines of 2 x 2/3/4/7),
// launches one 4-thread kernel and copies back the pixels it may write (2 x 2/2/3/6 per line).
//
// T2: svt_b200_loop_filter_frame_dev, two launches.  The first filters every vertical edge of the three planes, the
// second every horizontal edge; one thread per 4-pixel edge segment evaluates set_lpf_parameters
// (deblocking_filter.c:163) from the mode-info records and filters the segment's 4 lines.  Within one direction the
// segments are independent: the 14-tap filter needs 16-point transforms on both sides, the 8- and 6-tap filters
// 8-point ones, and the 4-tap filter writes only p1..q1, so no segment reads a pixel another segment of its direction
// writes.  The reference's superblock order (vertical edges of SB n, horizontal edges of SB n - 1) applies every
// vertical edge touching a pixel before any horizontal one, so the two passes give its result exactly.
//
// T2: svt_b200_dlf_level_sse_dev, one launch (after a memset of the sums): the trial SSEs of the filter-level search,
// filtered tile by tile in shared memory (see dlf_level_sse_kernel).
#include "svt_b200.h"
#include "common.cuh"
#include "dlf.cuh"
#include "dlf_tables.h"

namespace b200 {
namespace dlf {

__constant__ uint8_t c_tx_depth[3][B200_DLF_N_BSIZE] = B200_DLF_TX_DEPTH_TO_TX_SIZE;
__constant__ uint8_t c_uv_tx[B200_DLF_N_BSIZE]       = B200_DLF_UV_TX_SIZE_420;
__constant__ uint8_t c_horz[B200_DLF_N_TXSIZE]       = B200_DLF_TXSIZE_HORZ_MAP;
__constant__ uint8_t c_vert[B200_DLF_N_TXSIZE]       = B200_DLF_TXSIZE_VERT_MAP;
__constant__ uint8_t c_plane_bsize[B200_DLF_N_BSIZE] = B200_DLF_PLANE_BSIZE_420;
__constant__ uint8_t c_block_w[B200_DLF_N_BSIZE]     = B200_DLF_BLOCK_W;
__constant__ uint8_t c_block_h[B200_DLF_N_BSIZE]     = B200_DLF_BLOCK_H;
__constant__ uint8_t c_mode_lf[B200_DLF_N_MODES]     = B200_DLF_MODE_LF_LUT;

// ---- T1 --------------------------------------------------------------------------------------------------------------
template <int TAPS> struct Depth;
template <> struct Depth<4>  { static constexpr int read = 2, write = 2; };
template <> struct Depth<6>  { static constexpr int read = 3, write = 2; };
template <> struct Depth<8>  { static constexpr int read = 4, write = 3; };
template <> struct Depth<14> { static constexpr int read = 7, write = 6; };

// buf: 4 packed lines of 2 * read pixels, the edge between index read - 1 and read of each line
template <int TAPS, typename T>
__global__ void __launch_bounds__(32) lpf_t1_kernel(T* buf, int blimit, int limit, int thresh, int shift) {
    const int i = threadIdx.x;
    if (i >= 4) return;
    constexpr int D = Depth<TAPS>::read;
    filter_line<TAPS, T>(buf + i * 2 * D + D, 1, make_thr(blimit, limit, thresh, shift));
}

// ---- T2 --------------------------------------------------------------------------------------------------------------
// tx size (square TxSize 0..4 = 4..64 points) of a block across an edge of direction dir (0: vertical edge)
__device__ __forceinline__ int tx_across(const SvtB200DlfMi& m, int dir, int plane, int skipped) {
    const int tx = plane ? c_uv_tx[m.bsize] : c_tx_depth[skipped ? 0 : m.tx_depth][m.bsize];
    return dir == 0 ? c_horz[tx] : c_vert[tx];
}

// set_lpf_parameters (deblocking_filter.c:163) for the edge segment at plane pixel (x, y), both inside the plane:
// returns the filter length (0 = not filtered) and the level.  lvl: the plane's level table, [segment][dir][ref_frame0]
// [mode delta index] as in SvtB200DlfFrame.lvl[plane].
__device__ __forceinline__ int edge_params(const SvtB200DlfFrame& f, const uint8_t* __restrict__ lvl, const SvtB200DlfMi* __restrict__ mi,
                                           int plane, int dir, int x, int y, int& level) {
    const int ss = plane ? 1 : 0;
    const int mi_row = ss | ((y << ss) >> 2), mi_col = ss | ((x << ss) >> 2);
    const SvtB200DlfMi* cp = mi + (size_t)mi_row * f.mi_stride + mi_col;
    const SvtB200DlfMi cur = *cp;
    const int coord = dir == 0 ? x : y;
    const int c_skip = cur.skip && cur.ref_frame0 > 0;
    const int ts = tx_across(cur, dir, plane, c_skip);
    if (coord == 0 || (coord & ((4 << ts) - 1))) return 0;  // picture edge, or inside a transform block
    const SvtB200DlfMi prv = *(cp - (dir == 0 ? (ptrdiff_t)(1 << ss) : ((ptrdiff_t)f.mi_stride << ss)));
    const int c_lvl = lvl[((cur.segment_id * 2 + dir) * 8 + cur.ref_frame0) * 2 + c_mode_lf[cur.mode]];
    const int p_lvl = lvl[((prv.segment_id * 2 + dir) * 8 + prv.ref_frame0) * 2 + c_mode_lf[prv.mode]];
    const int p_skip = prv.skip && prv.ref_frame0 > 0;
    const int p_ts = tx_across(prv, dir, plane, p_skip);
    const int pb = plane ? c_plane_bsize[cur.bsize] : cur.bsize;
    const int pu_edge = !(coord & ((dir == 0 ? c_block_w[pb] : c_block_h[pb]) - 1));
    if (!(c_lvl || p_lvl) || (p_skip && c_skip && !pu_edge)) return 0;
    level = c_lvl ? c_lvl : p_lvl;
    const int min_ts = ts < p_ts ? ts : p_ts;
    return min_ts == 0 ? 4 : plane ? 6 : min_ts == 1 ? 8 : 14;
}

__device__ __forceinline__ Thr edge_thr(const SvtB200DlfFrame& f, int level) {
    return make_thr(f.lfthr[level][0], f.lfthr[level][1], f.lfthr[level][2], f.pixel_bytes == 2 ? f.bit_depth - 8 : 0);
}

// lines i0 <= i < i1 of the 4-line edge segment at p with the filter of length len; step: across the edge, next: along it
template <typename T>
__device__ __forceinline__ void filter_segment(T* p, ptrdiff_t step, ptrdiff_t next, int len, const Thr& t, int i0, int i1) {
    switch (len) {
    case 4:  for (int i = i0; i < i1; i++) filter_line<4, T>(p + i * next, step, t); break;
    case 6:  for (int i = i0; i < i1; i++) filter_line<6, T>(p + i * next, step, t); break;
    case 8:  for (int i = i0; i < i1; i++) filter_line<8, T>(p + i * next, step, t); break;
    default: for (int i = i0; i < i1; i++) filter_line<14, T>(p + i * next, step, t); break;
    }
}

struct PassShape {
    int n[3];     // segments per plane (0: plane not filtered)
    int cols[3];  // segments per plane row
};

// DIR 0: every vertical edge segment of the three planes; DIR 1: every horizontal one.  Segment (r, c) of a plane is the
// edge at plane pixel (4c, 4r); consecutive threads take consecutive columns.
template <int DIR, typename T>
__global__ void __launch_bounds__(128) dlf_pass_kernel(const __grid_constant__ SvtB200DlfFrame f, const SvtB200DlfMi* __restrict__ mi,
                                                       const PassShape s) {
    const int total = s.n[0] + s.n[1] + s.n[2];
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < total; u += gridDim.x * blockDim.x) {
        int plane = 0, k = u;
        if (k >= s.n[0]) { k -= s.n[0]; plane = 1; if (k >= s.n[1]) { k -= s.n[1]; plane = 2; } }
        const int r = k / s.cols[plane], c = k - r * s.cols[plane];
        const int x = c << 2, y = r << 2;
        int level = 0;
        const int len = edge_params(f, &f.lvl[plane][0][0][0][0], mi, plane, DIR, x, y, level);
        if (!len) continue;
        const ptrdiff_t pitch = f.stride[plane];
        T* p = (T*)f.plane[plane] + (ptrdiff_t)y * pitch + x;
        filter_segment(p, DIR == 0 ? 1 : pitch, DIR == 0 ? pitch : 1, len, edge_thr(f, level), 0, 4);
    }
}

// ---- T2: per-level SSE of the filter-level search ----------------------------------------------------------------------
// One CTA takes a kSseTile x kSseTile core of one plane and up to kSseLevels levels.  It stages the recon core with a
// 7-pixel halo (rows top-7 .. bottom+6, columns left-7 .. right+6, right / bottom = the first row / column past the core)
// in shared memory once, then for each level filters a copy of it -- vertical edges, then horizontal edges -- and sums
// the squared differences against the source over the core clipped to the SSE region.  Nothing is written to HBM but
// the sums.  Why the halo is enough, with tile corners on multiples of 16:
//   - An edge writes at most 6 pixels on each side and reads at most 7 (14-tap: x-6 .. x+5 written, x-7 .. x+6 read;
//     8-tap x-3 .. x+2 / x-4 .. x+3; 4- and 6-tap x-2 .. x+1 / x-3 .. x+2).  14-tap edges lie on multiples of 16 and
//     8-tap ones on multiples of 8, so the vertical edges that write a core column are those at x in [left, right]:
//     the one at left - 4 (4-tap at most) writes up to left - 3, the one at right + 4 starts at right + 2.
//   - Those edges read columns left-7 .. right+6, and, as in the picture call, what they read no other vertical edge
//     writes: the staged values are the right input (test_two_pass_equals_superblock_order checks that claim).
//   - The horizontal edges that write a core row are those at y in [top, bottom] by the same argument; in a core column
//     they read rows top-7 .. bottom+6, which the vertical pass above has fully filtered in the core columns.
//   - Staged pixels the picture call would not read (left of or above (0, 0), 7 or more past the plane's width or
//     height) are not loaded: no edge reads them, and the SSE region ends before them.
// Shared memory: (kSseTile + 14)^2 pixels staged + as many filtered + kSseTile^2 source pixels, 32.5 KB for 16-bit.
constexpr int kSseTile = 64, kSseHalo = 7, kSseSpan = kSseTile + 2 * kSseHalo, kSseLevels = 4;
constexpr int kSseVEdges = kSseTile / 4 + 1, kSseVSegs = (kSseTile + 16) / 4, kSseHSegs = kSseTile / 4;

struct SseShape {
    int n[3];        // tiles per plane (0: plane not evaluated)
    int cols[3];     // tiles per plane row
    int w[3], h[3];  // SSE region per plane
};

template <typename T>
__global__ void __launch_bounds__(256) dlf_level_sse_kernel(const __grid_constant__ SvtB200DlfFrame f, const __grid_constant__ SvtB200DlfLevelSse s,
                                                            const SseShape g, const SvtB200DlfMi* __restrict__ mi,
                                                            unsigned long long* __restrict__ d_sse) {
    __shared__ T orig[kSseSpan * kSseSpan], work[kSseSpan * kSseSpan], src[kSseTile * kSseTile];
    int plane = 0, k = blockIdx.x;
    if (k >= g.n[0]) { k -= g.n[0]; plane = 1; if (k >= g.n[1]) { k -= g.n[1]; plane = 2; } }
    const int ty = k / g.cols[plane], tx = k - ty * g.cols[plane];
    const int left = tx * kSseTile, top = ty * kSseTile;
    const int pw = plane ? f.width >> 1 : f.width, ph = plane ? f.height >> 1 : f.height;
    const int cw = min(kSseTile, g.w[plane] - left), ch = min(kSseTile, g.h[plane] - top);  // core within the SSE region
    const T* rec = (const T*)f.plane[plane];
    const ptrdiff_t rp = f.stride[plane], sp = s.src_stride[plane];
    for (int i = threadIdx.x; i < kSseSpan * kSseSpan; i += blockDim.x) {
        const int r = i / kSseSpan, c = i - r * kSseSpan, y = top - kSseHalo + r, x = left - kSseHalo + c;
        orig[i] = (x >= 0 && y >= 0 && x < pw + kSseHalo && y < ph + kSseHalo) ? rec[(ptrdiff_t)y * rp + x] : (T)0;
    }
    const T* srcp = (const T*)s.src[plane] + (ptrdiff_t)top * sp + left;
    for (int i = threadIdx.x; i < kSseTile * kSseTile; i += blockDim.x) {
        const int r = i / kSseTile, c = i - r * kSseTile;
        src[i] = (r < ch && c < cw) ? srcp[(ptrdiff_t)r * sp + c] : (T)0;
    }
    __syncthreads();
    const int l0 = blockIdx.y * kSseLevels, l1 = min(l0 + kSseLevels, s.n_levels);
    for (int li = l0; li < l1; li++) {
        const T* out = orig;
        if (s.level[li]) {  // level 0: the plane unfiltered (its table is stale in the reference: not read)
            const uint8_t* lvl = s.d_lvl + ((size_t)plane * s.n_levels + li) * sizeof(f.lvl[0]);
            for (int i = threadIdx.x; i < kSseSpan * kSseSpan; i += blockDim.x) work[i] = orig[i];
            __syncthreads();
            // vertical edges x = left .. right; 4-row segments from top - 8, of which only the staged rows are filtered
            for (int u = threadIdx.x; u < kSseVEdges * kSseVSegs; u += blockDim.x) {
                const int sr = u / kSseVEdges, x = left + 4 * (u - sr * kSseVEdges), y = top - 8 + 4 * sr;
                if (x >= pw || y < 0 || y >= ph) continue;
                int level = 0;
                const int len = edge_params(f, lvl, mi, plane, 0, x, y, level);
                if (!len) continue;
                filter_segment(work + (y - top + kSseHalo) * kSseSpan + x - left + kSseHalo, 1, kSseSpan, len, edge_thr(f, level),
                               sr == 0 ? 1 : 0, sr == kSseVSegs - 1 ? 3 : 4);
            }
            __syncthreads();
            // horizontal edges y = top .. bottom, core columns only
            for (int u = threadIdx.x; u < kSseVEdges * kSseHSegs; u += blockDim.x) {
                const int e = u / kSseHSegs, x = left + 4 * (u - e * kSseHSegs), y = top + 4 * e;
                if (x >= pw || y >= ph) continue;
                int level = 0;
                const int len = edge_params(f, lvl, mi, plane, 1, x, y, level);
                if (!len) continue;
                filter_segment(work + (y - top + kSseHalo) * kSseSpan + x - left + kSseHalo, kSseSpan, 1, len, edge_thr(f, level), 0, 4);
            }
            __syncthreads();
            out = work;
        }
        unsigned acc = 0;  // at most 16 pixels per thread: < 2^32 at 12 bits
        for (int i = threadIdx.x; i < kSseTile * kSseTile; i += blockDim.x) {
            const int r = i / kSseTile, c = i - r * kSseTile;
            if (r < ch && c < cw) {
                const int d = (int)out[(r + kSseHalo) * kSseSpan + c + kSseHalo] - (int)src[i];
                acc += (unsigned)(d * d);
            }
        }
        unsigned long long sum = acc;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if ((threadIdx.x & 31) == 0 && sum) atomicAdd(&d_sse[plane * s.n_levels + li], sum);
        __syncthreads();  // `work` is refilled for the next level
    }
}

}  // namespace dlf
}  // namespace b200

using namespace b200;
using namespace b200::dlf;

template <int TAPS, typename T>
static void lpf_t1(T* s, int32_t pitch, const uint8_t* blimit, const uint8_t* limit, const uint8_t* thresh, int bd, bool vertical) {
    require_ready();
    constexpr int D = Depth<TAPS>::read, W = Depth<TAPS>::write;
    RoundTrip rt;
    T px[4 * 2 * D];  // D pixels either side of the edge on each of the 4 lines; W of them are written back
    const ptrdiff_t across = vertical ? 1 : pitch, along = vertical ? pitch : 1;
    for (int i = 0; i < 4; i++)
        for (int k = -D; k < D; k++) px[i * 2 * D + D + k] = s[i * along + k * across];
    auto b = rt.inout(px, 4 * 2 * D);
    lpf_t1_kernel<TAPS, T><<<1, 32, 0, rt.stream()>>>(rt.dev(b), *blimit, *limit, *thresh, bd - 8);
    B200_LAUNCH_CHECK();
    rt.finish();
    for (int i = 0; i < 4; i++)
        for (int k = -W; k < W; k++) s[i * along + k * across] = px[i * 2 * D + D + k];
}

#define B200_DEF_LPF(DIR, N, VERT)                                                                                            \
    extern "C" void svt_b200_aom_lpf_##DIR##_##N(uint8_t* s, int32_t pitch, const uint8_t* blimit, const uint8_t* limit,     \
                                                 const uint8_t* thresh) {                                                    \
        lpf_t1<N, uint8_t>(s, pitch, blimit, limit, thresh, 8, VERT);                                                        \
    }                                                                                                                        \
    extern "C" void svt_b200_aom_highbd_lpf_##DIR##_##N(uint16_t* s, int32_t pitch, const uint8_t* blimit,                   \
                                                        const uint8_t* limit, const uint8_t* thresh, int32_t bd) {           \
        lpf_t1<N, uint16_t>(s, pitch, blimit, limit, thresh, bd, VERT);                                                      \
    }
B200_DEF_LPF(horizontal, 4, false) B200_DEF_LPF(horizontal, 6, false) B200_DEF_LPF(horizontal, 8, false) B200_DEF_LPF(horizontal, 14, false)
B200_DEF_LPF(vertical, 4, true) B200_DEF_LPF(vertical, 6, true) B200_DEF_LPF(vertical, 8, true) B200_DEF_LPF(vertical, 14, true)
#undef B200_DEF_LPF

// the geometry, pixel format and record grid of a frame are consistent
static bool frame_ok(const SvtB200DlfFrame& f) {
    const bool bd_ok = f.pixel_bytes == 1 ? f.bit_depth == 8 : (f.pixel_bytes == 2 && (f.bit_depth == 8 || f.bit_depth == 10 || f.bit_depth == 12));
    return bd_ok && f.width > 0 && f.height > 0 && f.mi_rows * 4 >= ((f.height + 7) & ~7) && f.mi_cols * 4 >= ((f.width + 7) & ~7) &&
           f.mi_stride >= f.mi_cols;
}

extern "C" int svt_b200_loop_filter_frame_dev(const SvtB200DlfFrame* frame, const SvtB200DlfMi* d_mi, void* stream) {
    require_ready();
    if (!frame || !d_mi) return SVT_B200_ERR_BAD_ARG;
    const SvtB200DlfFrame& f = *frame;
    if (!frame_ok(f)) return SVT_B200_ERR_BAD_ARG;
    if (!f.filter_level[0] && !f.filter_level[1]) return SVT_B200_OK;  // deblocking_filter.c:573-575: chroma is skipped too
    PassShape s;
    const int on[3] = {1, f.filter_level_u != 0, f.filter_level_v != 0};
    for (int p = 0; p < 3; p++) {
        const int pw = p ? f.width >> 1 : f.width, ph = p ? f.height >> 1 : f.height;
        if (!f.plane[p] && on[p]) return SVT_B200_ERR_BAD_ARG;
        s.cols[p] = (pw + 3) >> 2;
        s.n[p] = on[p] ? s.cols[p] * ((ph + 3) >> 2) : 0;
        if (!s.cols[p]) s.cols[p] = 1;
    }
    const long long total = (long long)s.n[0] + s.n[1] + s.n[2];
    if (!total) return SVT_B200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = grid_for((total + 127) / 128, 16);
    if (f.pixel_bytes == 2) {
        dlf_pass_kernel<0, uint16_t><<<grid, 128, 0, st>>>(f, d_mi, s);
        B200_LAUNCH_CHECK();
        dlf_pass_kernel<1, uint16_t><<<grid, 128, 0, st>>>(f, d_mi, s);
    } else {
        dlf_pass_kernel<0, uint8_t><<<grid, 128, 0, st>>>(f, d_mi, s);
        B200_LAUNCH_CHECK();
        dlf_pass_kernel<1, uint8_t><<<grid, 128, 0, st>>>(f, d_mi, s);
    }
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_dlf_level_sse_dev(const SvtB200DlfFrame* frame, const SvtB200DlfLevelSse* sse, const SvtB200DlfMi* d_mi,
                                          int64_t* d_sse, void* stream) {
    require_ready();
    if (!frame || !sse || !d_mi || !d_sse) return SVT_B200_ERR_BAD_ARG;
    const SvtB200DlfFrame& f = *frame;
    const SvtB200DlfLevelSse& s = *sse;
    if (!frame_ok(f) || s.n_levels < 1 || s.n_levels > 64 || !s.d_lvl || (s.plane_mask & 7) == 0 || (s.plane_mask & ~7) ||
        s.sse_width <= 0 || s.sse_height <= 0 || s.sse_width > ((f.width + 7) & ~7) || s.sse_height > ((f.height + 7) & ~7))
        return SVT_B200_ERR_BAD_ARG;
    for (int i = 0; i < s.n_levels; i++)
        if (s.level[i] > 63) return SVT_B200_ERR_BAD_ARG;
    SseShape g;
    long long tiles = 0;
    for (int p = 0; p < 3; p++) {
        g.w[p] = p ? s.sse_width >> 1 : s.sse_width;
        g.h[p] = p ? s.sse_height >> 1 : s.sse_height;
        g.cols[p] = (g.w[p] + kSseTile - 1) / kSseTile;
        g.n[p] = 0;
        if (!((s.plane_mask >> p) & 1)) continue;
        if (!f.plane[p] || !s.src[p] || f.stride[p] < g.w[p] || s.src_stride[p] < g.w[p]) return SVT_B200_ERR_BAD_ARG;
        g.n[p] = g.cols[p] * ((g.h[p] + kSseTile - 1) / kSseTile);
        tiles += g.n[p];
    }
    cudaStream_t st = (cudaStream_t)stream;
    for (int p = 0; p < 3; p++)
        if ((s.plane_mask >> p) & 1) B200_CUDA_CHECK(cudaMemsetAsync(d_sse + (size_t)p * s.n_levels, 0, sizeof(int64_t) * s.n_levels, st));
    if (!tiles) return SVT_B200_OK;  // a chroma plane of a 1-pixel-wide picture
    const dim3 grid((unsigned)tiles, (s.n_levels + kSseLevels - 1) / kSseLevels);
    if (f.pixel_bytes == 2) dlf_level_sse_kernel<uint16_t><<<grid, 256, 0, st>>>(f, s, g, d_mi, (unsigned long long*)d_sse);
    else dlf_level_sse_kernel<uint8_t><<<grid, 256, 0, st>>>(f, s, g, d_mi, (unsigned long long*)d_sse);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}
