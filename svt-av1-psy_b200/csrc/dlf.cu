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
// returns the filter length (0 = not filtered) and the level
__device__ __forceinline__ int edge_params(const SvtB200DlfFrame& f, const SvtB200DlfMi* __restrict__ mi, int plane, int dir, int x,
                                           int y, int& level) {
    const int ss = plane ? 1 : 0;
    const int mi_row = ss | ((y << ss) >> 2), mi_col = ss | ((x << ss) >> 2);
    const SvtB200DlfMi* cp = mi + (size_t)mi_row * f.mi_stride + mi_col;
    const SvtB200DlfMi cur = *cp;
    const int coord = dir == 0 ? x : y;
    const int c_skip = cur.skip && cur.ref_frame0 > 0;
    const int ts = tx_across(cur, dir, plane, c_skip);
    if (coord == 0 || (coord & ((4 << ts) - 1))) return 0;  // picture edge, or inside a transform block
    const SvtB200DlfMi prv = *(cp - (dir == 0 ? (ptrdiff_t)(1 << ss) : ((ptrdiff_t)f.mi_stride << ss)));
    const int c_lvl = f.lvl[plane][cur.segment_id][dir][cur.ref_frame0][c_mode_lf[cur.mode]];
    const int p_lvl = f.lvl[plane][prv.segment_id][dir][prv.ref_frame0][c_mode_lf[prv.mode]];
    const int p_skip = prv.skip && prv.ref_frame0 > 0;
    const int p_ts = tx_across(prv, dir, plane, p_skip);
    const int pb = plane ? c_plane_bsize[cur.bsize] : cur.bsize;
    const int pu_edge = !(coord & ((dir == 0 ? c_block_w[pb] : c_block_h[pb]) - 1));
    if (!(c_lvl || p_lvl) || (p_skip && c_skip && !pu_edge)) return 0;
    level = c_lvl ? c_lvl : p_lvl;
    const int min_ts = ts < p_ts ? ts : p_ts;
    return min_ts == 0 ? 4 : plane ? 6 : min_ts == 1 ? 8 : 14;
}

struct PassShape {
    int n[3];     // segments per plane (0: plane not filtered)
    int cols[3];  // segments per plane row
};

// DIR 0: every vertical edge segment of the three planes; DIR 1: every horizontal one.  Segment (r, c) of a plane is the
// edge at plane pixel (4c, 4r); consecutive threads take consecutive columns.
template <int DIR, typename T>
__global__ void __launch_bounds__(128) dlf_pass_kernel(const SvtB200DlfFrame f, const SvtB200DlfMi* __restrict__ mi, const PassShape s) {
    const int total = s.n[0] + s.n[1] + s.n[2];
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < total; u += gridDim.x * blockDim.x) {
        int plane = 0, k = u;
        if (k >= s.n[0]) { k -= s.n[0]; plane = 1; if (k >= s.n[1]) { k -= s.n[1]; plane = 2; } }
        const int r = k / s.cols[plane], c = k - r * s.cols[plane];
        const int x = c << 2, y = r << 2;
        int level = 0;
        const int len = edge_params(f, mi, plane, DIR, x, y, level);
        if (!len) continue;
        const Thr t = make_thr(f.lfthr[level][0], f.lfthr[level][1], f.lfthr[level][2], f.pixel_bytes == 2 ? f.bit_depth - 8 : 0);
        const ptrdiff_t pitch = f.stride[plane];
        T* p = (T*)f.plane[plane] + (ptrdiff_t)y * pitch + x;
        const ptrdiff_t step = DIR == 0 ? 1 : pitch, next = DIR == 0 ? pitch : 1;  // across the edge / along it
        switch (len) {
        case 4:  for (int i = 0; i < 4; i++) filter_line<4, T>(p + i * next, step, t); break;
        case 6:  for (int i = 0; i < 4; i++) filter_line<6, T>(p + i * next, step, t); break;
        case 8:  for (int i = 0; i < 4; i++) filter_line<8, T>(p + i * next, step, t); break;
        default: for (int i = 0; i < 4; i++) filter_line<14, T>(p + i * next, step, t); break;
        }
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
    const size_t bytes = 4 * 2 * D * sizeof(T);
    LaneGuard l;
    const size_t o = l->alloc(bytes);
    T* h = l->h<T>(o);
    const ptrdiff_t across = vertical ? 1 : pitch, along = vertical ? pitch : 1;
    for (int i = 0; i < 4; i++)
        for (int k = -D; k < D; k++) h[i * 2 * D + D + k] = s[i * along + k * across];
    l->h2d(o, bytes);
    lpf_t1_kernel<TAPS, T><<<1, 32, 0, l->stream>>>(l->d<T>(o), *blimit, *limit, *thresh, bd - 8);
    B200_LAUNCH_CHECK();
    l->d2h(o, bytes);
    l->sync();
    for (int i = 0; i < 4; i++)
        for (int k = -W; k < W; k++) s[i * along + k * across] = h[i * 2 * D + D + k];
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

extern "C" int svt_b200_loop_filter_frame_dev(const SvtB200DlfFrame* frame, const SvtB200DlfMi* d_mi, void* stream) {
    require_ready();
    if (!frame || !d_mi) return SVT_B200_ERR_BAD_ARG;
    const SvtB200DlfFrame& f = *frame;
    const bool bd_ok = f.pixel_bytes == 1 ? f.bit_depth == 8 : (f.pixel_bytes == 2 && (f.bit_depth == 8 || f.bit_depth == 10 || f.bit_depth == 12));
    if (!bd_ok || f.width <= 0 || f.height <= 0 || f.mi_rows * 4 < ((f.height + 7) & ~7) || f.mi_cols * 4 < ((f.width + 7) & ~7) ||
        f.mi_stride < f.mi_cols)
        return SVT_B200_ERR_BAD_ARG;
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
