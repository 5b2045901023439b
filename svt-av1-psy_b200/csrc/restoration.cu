// restoration.cu -- a13: loop-restoration drivers on the device (sm_90a).
//
// Reference behaviour restated (Source/Lib/Codec/restoration.c):
//   svt_av1_loop_restoration_save_boundary_lines (:1682) / svt_aom_save_tile_row_boundary_lines (:1606) /
//   svt_aom_save_deblock_boundary_lines (:1518) / svt_aom_save_cdef_boundary_lines (:1576) / svt_aom_extend_lines (:1506):
//     per 64-row processing stripe (offset upwards by 8 luma rows), two context lines above and two below, taken from
//     the DEBLOCKED picture at interior stripe boundaries and from the CDEF output at the top / bottom of the picture;
//   svt_av1_loop_restoration_filter_frame (:1179) -> svt_aom_foreach_rest_unit_in_frame (:1296) ->
//   svt_av1_loop_restoration_filter_unit (:1067): every restoration unit is filtered stripe by stripe; the 3 rows above /
//   below a stripe are replaced by the saved lines (svt_aom_setup_processing_stripe_boundary :289-371, both the normal and
//   the optimized_lr form), then svt_aom_wiener_filter_stripe (:437) / svt_aom_sgrproj_filter_stripe (:994) run on
//   <= 64-wide column chunks; RESTORE_NONE units are copied;
//   sse_restoration_unit (restoration_pick.c:103): squared error of a unit against the source (the trial cost of the RU search).
//
// H100 mapping.  The reference patches the picture rows in place around every stripe and restores them afterwards -- a
// serial save / overwrite / filter / restore dance.  Here one CTA owns one (stripe, 64-column chunk) of a plane: it
// stages the (h + 7) x (w + 8) input tile into shared memory, fetching each halo row from wherever the reference would
// have found it (picture, saved above / below line, or the neighbouring picture row in optimized_lr mode), looks up the
// restoration unit that covers the chunk in a device-resident unit table and runs that unit's filter on the tile
// (wiener_unit.cuh / sgr_unit.cuh: the same arithmetic as the unit-list kernels).  Nothing is modified in place, all
// chunks of all stripes of all planes run concurrently (blockIdx.z = plane), and the call is CUDA-graph capturable.
#include "common.cuh"
#include "wiener_unit.cuh"
#include "sgr_unit.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

struct LrGeom {
    int W, H, full, off, procw, us, hunits, vunits, n_stripes, n_chunks;
};
__host__ __device__ inline int lr_count_units(int size, int us) {  // svt_av1_lr_count_units_in_tile
    const int n = (size + (us >> 1)) / us;
    return n > 1 ? n : 1;
}
__host__ __device__ inline LrGeom lr_geom(const SvtB200LrPlane& p) {
    LrGeom g;
    g.W = p.width; g.H = p.height;
    g.full = 64 >> p.ss_y; g.off = 8 >> p.ss_y; g.procw = 64 >> p.ss_x;
    g.us = p.unit_size;
    g.hunits = lr_count_units(g.W, g.us); g.vunits = lr_count_units(g.H, g.us);
    g.n_stripes = (g.H + g.off + g.full - 1) / g.full;
    g.n_chunks = (g.W + g.procw - 1) / g.procw;
    return g;
}
__host__ __device__ inline void lr_stripe(const LrGeom& g, int s, int& y0, int& y1) {
    y0 = s * g.full - g.off; if (y0 < 0) y0 = 0;
    y1 = (s + 1) * g.full - g.off; if (y1 > g.H) y1 = g.H;
}

struct LrPlanes { SvtB200LrPlane p[3]; };

// ---- boundary lines -------------------------------------------------------------------------------------------------
template <typename PIX>
__global__ void __launch_bounds__(256) lr_save_boundary_kernel(const __grid_constant__ LrPlanes pl, int after_cdef) {
    const SvtB200LrPlane& p = pl.p[blockIdx.z];
    const LrGeom g = lr_geom(p);
    const int s = blockIdx.y >> 1, is_above = !(blockIdx.y & 1);
    if (s >= g.n_stripes) return;
    int y0, y1;
    lr_stripe(g, s, y0, y1);
    const int use_deblock = is_above ? (s > 0) : (y1 < g.H);
    if (after_cdef == use_deblock) return;  // deblocked lines are saved in the first pass, CDEF lines (picture top / bottom) in the second
    const PIX* src = reinterpret_cast<const PIX*>(after_cdef ? p.cdef : p.deblocked);
    const int  stride = after_cdef ? p.stride_cdef : p.stride_deblocked;
    PIX*       buf = reinterpret_cast<PIX*>(is_above ? p.boundary_above : p.boundary_below);
    int row[2];
    if (!after_cdef) {
        const int r = is_above ? y0 - 2 : y1;
        const int lines = (g.H - r) < 2 ? (g.H - r) : 2;  // a stripe may end 1 row above the crop border: that row is duplicated
        row[0] = r; row[1] = lines == 1 ? r : r + 1;
    } else {
        row[0] = row[1] = is_above ? y0 : y1 - 1;          // the outermost CDEF row of the picture, twice
    }
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < 2 * (g.W + 8); t += gridDim.x * blockDim.x) {
        const int i = t / (g.W + 8), x = t - i * (g.W + 8) - 4;  // logical column -4 .. W+3 (svt_aom_extend_lines)
        const int xc = x < 0 ? 0 : (x >= g.W ? g.W - 1 : x);
        buf[(size_t)(2 * s + i) * p.boundary_stride + (x + 4)] = src[(size_t)row[i] * stride + xc];
    }
}

// ---- filter ---------------------------------------------------------------------------------------------------------
constexpr int kLrTilePitch = 72;
constexpr size_t kLrSmem = (size_t)kLrTilePitch * (64 + 8) * 2                 // staged tile
                           + (size_t)2 * 66 * 66 * 4                            // A / B planes (also the Wiener intermediate)
                           + (size_t)2 * 64 * 64 * 4;                           // flt0 / flt1
constexpr size_t kLrSmemWiener = (size_t)kLrTilePitch * (64 + 8) * 2 + (size_t)(64 + 8) * 64 * 2;  // tile + horizontal-pass intermediate

template <typename PIX>
__global__ void __launch_bounds__(256) lr_filter_kernel(const __grid_constant__ LrPlanes pl, const SvtB200LrUnitInfo* __restrict__ units0,
                                                        const SvtB200LrUnitInfo* __restrict__ units1, const SvtB200LrUnitInfo* __restrict__ units2,
                                                        int optimized_lr, int bd) {
    extern __shared__ __align__(16) unsigned char lsm[];
    const SvtB200LrPlane& p = pl.p[blockIdx.z];
    const LrGeom g = lr_geom(p);
    const int s = blockIdx.y, j = blockIdx.x;
    if (s >= g.n_stripes || j >= g.n_chunks) return;
    int y0, y1;
    lr_stripe(g, s, y0, y1);
    const int h = y1 - y0, x0 = j * g.procw, w = min(g.procw, g.W - x0);
    // svt_aom_get_stripe_boundary_info: no substitution above the first / below the last stripe of the picture
    const bool copy_above = s > 0;
    const bool copy_below = !(y0 + (g.full - (s == 0 ? g.off : 0)) >= g.H);
    const SvtB200LrUnitInfo* units = blockIdx.z == 0 ? units0 : (blockIdx.z == 1 ? units1 : units2);
    const int ucol = min(x0 / g.us, g.hunits - 1), urow = min((y0 + g.off) / g.us, g.vunits - 1);
    const SvtB200LrUnitInfo info = units[urow * g.hunits + ucol];

    const PIX* data = reinterpret_cast<const PIX*>(p.cdef);
    PIX*       dst = reinterpret_cast<PIX*>(p.dst) + (size_t)y0 * p.stride_dst + x0;
    if (info.restoration_type == 0) {  // RESTORE_NONE: svt_aom_copy_tile
        for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
            const int r = i / w, c = i - r * w;
            dst[(size_t)r * p.stride_dst + c] = data[(size_t)(y0 + r) * p.stride_cdef + x0 + c];
        }
        return;
    }
    uint16_t* tile = reinterpret_cast<uint16_t*>(lsm);
    const PIX* above = reinterpret_cast<const PIX*>(p.boundary_above);
    const PIX* below = reinterpret_cast<const PIX*>(p.boundary_below);
    const int sw = w + 8, sh = h + 7;  // rows -3 .. h+3, columns -3 .. w+4
    // one warp per tile row: where the row comes from (picture, saved above / below line, neighbouring row) is decided once
    // per row, the copy itself is a coalesced run
    for (int tr = threadIdx.x >> 5; tr < sh; tr += blockDim.x >> 5) {
        const int r = tr - 3;
        const PIX* rowp;
        bool from_lines = false;
        if (r < 0 && copy_above && !optimized_lr) {
            rowp = above + (size_t)(2 * s + (r + 2 > 0 ? r + 2 : 0)) * p.boundary_stride + 4;   // rows -3,-2,-1 <- saved lines 0,0,1
            from_lines = true;
        } else if (r >= h && copy_below && !optimized_lr) {
            const int k = r - h;
            rowp = below + (size_t)(2 * s + (k < 1 ? k : 1)) * p.boundary_stride + 4;           // rows h,h+1,h+2 <- saved lines 0,1,1
            from_lines = true;
        } else {
            int yy = y0 + r;
            if (optimized_lr) {  // only the outermost context row is replaced, by its inner neighbour (:339-359)
                if (r == -3 && copy_above) yy = y0 - 2;
                if (r == h + 2 && copy_below) yy = y1 + 1;
            }
            // the picture is extended by RESTORATION_BORDER pixels of edge replication before filtering (svt_extend_frame, :1223)
            yy = yy < 0 ? 0 : (yy >= g.H ? g.H - 1 : yy);
            rowp = data + (size_t)yy * p.stride_cdef;
        }
        const int lo = from_lines ? -4 : 0, hi = from_lines ? g.W + 3 : g.W - 1;  // the saved lines carry 4 extended columns each side
        for (int tc = threadIdx.x & 31; tc < sw; tc += 32) {
            int xx = x0 + tc - 3;
            xx = xx < lo ? lo : (xx > hi ? hi : xx);
            tile[tr * kLrTilePitch + tc] = (uint16_t)rowp[xx];
        }
    }
    __syncthreads();
    int32_t* AB = reinterpret_cast<int32_t*>(lsm + (size_t)kLrTilePitch * (64 + 8) * 2);
    if (info.restoration_type == 1) {  // RESTORE_WIENER: svt_aom_wiener_filter_stripe -> svt_av1_(highbd_)wiener_convolve_add_src
        int round0 = 3, round1 = 11;    // get_conv_params_wiener (convolve.h:70-85)
        if (bd == 12) { round0 = 5; round1 = 9; }
        wiener_unit_compute<PIX>(tile, reinterpret_cast<uint16_t*>(AB), dst, p.stride_dst, w, h, info.hfilter, info.vfilter, bd, round0, round1,
                                 sizeof(PIX) == 1);
        return;
    }
    // RESTORE_SGRPROJ: svt_aom_sgrproj_filter_stripe -> svt_apply_selfguided_restoration (:957-992)
    if (p.frame_restoration_type == 1) __trap();  // the caller declared a Wiener-only plane: the launch has no room for this filter
    int32_t* A = AB;
    int32_t* B = A + 66 * 66;
    int32_t* f0 = B + 66 * 66;
    int32_t* f1 = f0 + 64 * 64;
    const int* prm = c_sgr_params + 4 * info.sgr_ep;
    if (prm[0] > 0) sgr_pass(tile, kLrTilePitch, w, h, A, B, w + 2, prm[0], (uint32_t)prm[2], bd, 1, f0, w);
    if (prm[1] > 0) sgr_pass(tile, kLrTilePitch, w, h, A, B, w + 2, prm[1], (uint32_t)prm[3], bd, 0, f1, w);
    int xq0, xq1;  // svt_decode_xq (:634-645)
    if (prm[0] == 0) { xq0 = 0; xq1 = 128 - info.sgr_xqd[1]; }
    else if (prm[1] == 0) { xq0 = info.sgr_xqd[0]; xq1 = 0; }
    else { xq0 = info.sgr_xqd[0]; xq1 = 128 - xq0 - info.sgr_xqd[1]; }
    const int pmax = (1 << bd) - 1;
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        const int32_t u = (int32_t)tile[(r + 3) * kLrTilePitch + c + 3] << 4;
        int32_t v = u << 7;
        if (prm[0] > 0) v += xq0 * (f0[i] - u);
        if (prm[1] > 0) v += xq1 * (f1[i] - u);
        const int16_t wv = (int16_t)rp2s(v, 11);
        dst[(size_t)r * p.stride_dst + c] = (PIX)(wv < 0 ? 0 : (wv > pmax ? pmax : wv));
    }
}

// ---- squared error of every restoration unit against the source (sse_restoration_unit) --------------------------------------
template <typename PIX>
__global__ void __launch_bounds__(256) lr_unit_sse_kernel(const __grid_constant__ LrPlanes pl, unsigned long long* __restrict__ sse0,
                                                          unsigned long long* __restrict__ sse1, unsigned long long* __restrict__ sse2) {
    const SvtB200LrPlane& p = pl.p[blockIdx.z];
    const LrGeom g = lr_geom(p);
    const int unit = blockIdx.x;
    if (unit >= g.hunits * g.vunits) return;
    const int ur = unit / g.hunits, uc = unit - ur * g.hunits;
    // foreach_rest_unit_in_tile (:1247-1294): units of `us`, the last one absorbs a remainder below us/2, rows shifted up by `off`
    const int hs = uc * g.us, he = uc == g.hunits - 1 ? g.W : hs + g.us;
    int vs = ur * g.us - g.off, ve = ur == g.vunits - 1 ? g.H : (ur + 1) * g.us - g.off;
    if (vs < 0) vs = 0;
    const PIX* a = reinterpret_cast<const PIX*>(p.dst);
    const PIX* b = reinterpret_cast<const PIX*>(p.src);
    const int w = he - hs, rows = ve - vs;
    const int parts = gridDim.y, part = blockIdx.y;
    unsigned long long acc = 0;
    for (int r = part; r < rows; r += parts)
        for (int c = threadIdx.x; c < w; c += blockDim.x) {
            const int d = (int)a[(size_t)(vs + r) * p.stride_dst + hs + c] - (int)b[(size_t)(vs + r) * p.stride_src + hs + c];
            acc += (unsigned long long)(d * d);
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    unsigned long long* out = blockIdx.z == 0 ? sse0 : (blockIdx.z == 1 ? sse1 : sse2);
    if ((threadIdx.x & 31) == 0 && acc) atomicAdd(&out[unit], acc);
}

static int lr_check(const SvtB200LrPlane* planes, int n_planes, int bit_depth) {
    if (!planes || n_planes < 1 || n_planes > 3 || (bit_depth != 8 && bit_depth != 10 && bit_depth != 12)) return SVT_B200_ERR_BAD_ARG;
    for (int i = 0; i < n_planes; i++) {
        const SvtB200LrPlane& p = planes[i];
        if (p.width <= 0 || p.height <= 0 || p.unit_size < (64 >> p.ss_x) || (p.unit_size & (p.unit_size - 1)) || p.ss_x < 0 || p.ss_x > 1 ||
            p.ss_y < 0 || p.ss_y > 1)
            return SVT_B200_ERR_BAD_ARG;
    }
    return SVT_B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int svt_b200_lr_num_stripes(int plane_height, int ss_y) {
    return (plane_height + (8 >> ss_y) + (64 >> ss_y) - 1) / (64 >> ss_y);
}
extern "C" int svt_b200_lr_boundary_stride(int plane_width) { return (plane_width + 8 + 31) & ~31; }  // svt_av1_alloc_restoration_buffers (:1738-1741)
extern "C" int svt_b200_lr_units_per_dim(int size, int unit_size) { return lr_count_units(size, unit_size); }

extern "C" int svt_b200_lr_save_boundary_lines_dev(const SvtB200LrPlane* planes, int n_planes, int after_cdef, int bit_depth, void* stream) {
    require_ready();
    int rc = lr_check(planes, n_planes, bit_depth);
    if (rc) return rc;
    LrPlanes pl;
    memset(&pl, 0, sizeof(pl));
    int max_stripes = 0, max_w = 0;
    for (int i = 0; i < n_planes; i++) {
        pl.p[i] = planes[i];
        if (!planes[i].boundary_above || !planes[i].boundary_below || !(after_cdef ? planes[i].cdef : planes[i].deblocked)) return SVT_B200_ERR_BAD_ARG;
        const LrGeom g = lr_geom(planes[i]);
        max_stripes = g.n_stripes > max_stripes ? g.n_stripes : max_stripes;
        max_w = g.W > max_w ? g.W : max_w;
    }
    const dim3 grid((2 * (max_w + 8) + 255) / 256, 2 * max_stripes, n_planes);
    if (bit_depth == 8) lr_save_boundary_kernel<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>(pl, after_cdef ? 1 : 0);
    else lr_save_boundary_kernel<uint16_t><<<grid, 256, 0, (cudaStream_t)stream>>>(pl, after_cdef ? 1 : 0);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_lr_filter_frame_dev(const SvtB200LrPlane* planes, int n_planes, const SvtB200LrUnitInfo* const d_units[3], int optimized_lr,
                                            int bit_depth, void* stream) {
    require_ready();
    int rc = lr_check(planes, n_planes, bit_depth);
    if (rc) return rc;
    if (!d_units) return SVT_B200_ERR_BAD_ARG;
    LrPlanes pl;
    memset(&pl, 0, sizeof(pl));
    int max_stripes = 0, max_chunks = 0;
    for (int i = 0; i < n_planes; i++) {
        pl.p[i] = planes[i];
        if (!planes[i].cdef || !planes[i].dst || !d_units[i] || (!optimized_lr && (!planes[i].boundary_above || !planes[i].boundary_below)))
            return SVT_B200_ERR_BAD_ARG;
        const LrGeom g = lr_geom(planes[i]);
        max_stripes = g.n_stripes > max_stripes ? g.n_stripes : max_stripes;
        max_chunks = g.n_chunks > max_chunks ? g.n_chunks : max_chunks;
    }
    static std::mutex mu;
    static bool attr8 = false, attr16 = false;
    static int  attr_epoch = -1;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (attr_epoch != epoch()) { attr8 = attr16 = false; attr_epoch = epoch(); }
        bool& a = bit_depth == 8 ? attr8 : attr16;
        if (!a) {
            if (bit_depth == 8) B200_CUDA_CHECK(cudaFuncSetAttribute(lr_filter_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLrSmem));
            else B200_CUDA_CHECK(cudaFuncSetAttribute(lr_filter_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLrSmem));
            a = true;
        }
    }
    // planes whose frame_restoration_type rules the self-guided filter out need only the Wiener footprint (more CTAs per SM)
    bool sgr_possible = false;
    for (int i = 0; i < n_planes; i++) sgr_possible |= planes[i].frame_restoration_type != 1;
    const size_t smem = sgr_possible ? kLrSmem : kLrSmemWiener;
    const dim3 grid(max_chunks, max_stripes, n_planes);
    const SvtB200LrUnitInfo *u0 = d_units[0], *u1 = n_planes > 1 ? d_units[1] : nullptr, *u2 = n_planes > 2 ? d_units[2] : nullptr;
    if (bit_depth == 8) lr_filter_kernel<uint8_t><<<grid, 256, smem, (cudaStream_t)stream>>>(pl, u0, u1, u2, optimized_lr ? 1 : 0, 8);
    else lr_filter_kernel<uint16_t><<<grid, 256, smem, (cudaStream_t)stream>>>(pl, u0, u1, u2, optimized_lr ? 1 : 0, bit_depth);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_lr_unit_sse_dev(const SvtB200LrPlane* planes, int n_planes, int64_t* const d_sse[3], int bit_depth, void* stream) {
    require_ready();
    int rc = lr_check(planes, n_planes, bit_depth);
    if (rc) return rc;
    if (!d_sse) return SVT_B200_ERR_BAD_ARG;
    LrPlanes pl;
    memset(&pl, 0, sizeof(pl));
    int max_units = 0;
    for (int i = 0; i < n_planes; i++) {
        pl.p[i] = planes[i];
        if (!planes[i].dst || !planes[i].src || !d_sse[i]) return SVT_B200_ERR_BAD_ARG;
        const LrGeom g = lr_geom(planes[i]);
        const int n = g.hunits * g.vunits;
        max_units = n > max_units ? n : max_units;
        B200_CUDA_CHECK(cudaMemsetAsync(d_sse[i], 0, sizeof(int64_t) * n, (cudaStream_t)stream));
    }
    const dim3 grid(max_units, 16, n_planes);
    unsigned long long *s0 = (unsigned long long*)d_sse[0], *s1 = n_planes > 1 ? (unsigned long long*)d_sse[1] : nullptr,
                       *s2 = n_planes > 2 ? (unsigned long long*)d_sse[2] : nullptr;
    if (bit_depth == 8) lr_unit_sse_kernel<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>(pl, s0, s1, s2);
    else lr_unit_sse_kernel<uint16_t><<<grid, 256, 0, (cudaStream_t)stream>>>(pl, s0, s1, s2);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}
