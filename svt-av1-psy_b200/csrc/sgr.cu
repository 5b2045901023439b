// sgr.cu -- K10 self-guided restoration filter, K12 projection error / projection subspace (sm_90a).
//
// Reference behaviour restated:
//   svt_av1_selfguided_restoration_c (Source/Lib/Codec/restoration.c:923-955) with
//   selfguided_restoration_fast_internal (:669-801, r=2, coefficients only on odd rows) and
//   selfguided_restoration_internal (:803-921, r=1); svt_apply_selfguided_restoration_c (:957-992);
//   svt_av1_{lowbd,highbd}_pixel_proj_error_c (Source/Lib/Codec/restoration_pick.c:167-318);
//   svt_get_proj_subspace_c (:413-498).
// The box sums are plain (2r+1)^2 window sums (the reference's boxsum1/boxsum2 only differ at the
// border of the extended area, which the filter never reads); all intermediate arithmetic is done in
// the reference's types (uint32 wrap for p*s, int32 for the weighted combine).
//
// get_proj_subspace accumulates products of integer-valued doubles; every partial sum is an integer
// below 2^53, so the sums are exact in any order -- they are accumulated here in int64 and converted
// once, then the 2x2 solve runs in IEEE double with the reference's operation order (no FMA).
//
// Mapping: one CTA per processing unit (<= 96x96): the extended tile, the A/B coefficient planes of
// the current radius live in dynamic shared memory; outputs are written once.
#include "common.cuh"
#include "../../include/svt_b200.h"
#include "sgr_unit.cuh"

namespace b200 {

template <typename PIX>
__global__ void __launch_bounds__(256)
sgr_filter_kernel(const PIX* __restrict__ dgd_base, const SvtB200SgrUnit* __restrict__ units, int n_units, int32_t* __restrict__ flt0_base,
                  int32_t* __restrict__ flt1_base, int bd) {
    extern __shared__ __align__(16) unsigned char sm[];
    for (int it = blockIdx.x; it < n_units; it += gridDim.x) {
        const SvtB200SgrUnit u = units[it];
        const int w = u.w, h = u.h, tp = w + 6, ap = w + 2;
        uint16_t* tile = reinterpret_cast<uint16_t*>(sm);
        int32_t*  A    = reinterpret_cast<int32_t*>(sm + (((size_t)tp * (h + 6) * 2 + 15) & ~size_t(15)));
        int32_t*  B    = A + (size_t)ap * (h + 2);
        for (int i = threadIdx.x; i < tp * (h + 6); i += blockDim.x) {
            const int r = i / tp, c = i - r * tp;
            tile[i] = (uint16_t)dgd_base[u.dgd_off + (ptrdiff_t)(r - 3) * u.dgd_stride + (c - 3)];
        }
        __syncthreads();
        const int* prm = c_sgr_params + 4 * u.params_idx;
        if (prm[0] > 0) sgr_pass(tile, tp, w, h, A, B, ap, prm[0], (uint32_t)prm[2], bd, 1, flt0_base + u.flt0_off, u.flt_stride);
        if (prm[1] > 0) sgr_pass(tile, tp, w, h, A, B, ap, prm[1], (uint32_t)prm[3], bd, 0, flt1_base + u.flt1_off, u.flt_stride);
    }
}

// dst = clip(round((u << 7) + xq0 (flt0 - u) + xq1 (flt1 - u)))  (restoration.c:968-990)
template <typename PIX>
__global__ void sgr_project_kernel(const PIX* dat, int w, int h, int stride, const int32_t* flt0, const int32_t* flt1, int xq0, int xq1,
                                   int r0, int r1, PIX* dst, int dst_stride, int bd) {
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < w * h; idx += gridDim.x * blockDim.x) {
        const int i = idx / w, j = idx - i * w;
        const int32_t u = (int32_t)dat[(size_t)i * stride + j] << 4;
        int32_t v = u << 7;
        if (r0 > 0) v += xq0 * (flt0[idx] - u);
        if (r1 > 0) v += xq1 * (flt1[idx] - u);
        const int16_t wv = (int16_t)rp2s(v, 11);
        int o = wv < 0 ? 0 : (wv > (1 << bd) - 1 ? (1 << bd) - 1 : wv);
        dst[(size_t)i * dst_stride + j] = (PIX)o;
    }
}

template <typename PIX, bool HBD_FORM>
__global__ void proj_error_kernel(const PIX* src, int w, int h, int ss, const PIX* dat, int ds, const int32_t* flt0, int f0s,
                                  const int32_t* flt1, int f1s, int xq0, int xq1, int r0, int r1, long long* out) {
    long long acc = 0;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < w * h; idx += gridDim.x * blockDim.x) {
        const int i = idx / w, j = idx - i * w;
        const int32_t d = dat[(size_t)i * ds + j], s = src[(size_t)i * ss + j];
        int32_t e;
        if (r0 > 0 || r1 > 0) {
            const int32_t u = d << 4;
            if (HBD_FORM) {
                int32_t v = 1 << 10;
                if (r0 > 0) v += xq0 * (flt0[(size_t)i * f0s + j] - u);
                if (r1 > 0) v += xq1 * (flt1[(size_t)i * f1s + j] - u);
                e = (v >> 11) + d - s;
            } else {
                int32_t v = u << 7;
                if (r0 > 0) v += xq0 * (flt0[(size_t)i * f0s + j] - u);
                if (r1 > 0) v += xq1 * (flt1[(size_t)i * f1s + j] - u);
                e = rp2s(v, 11) - s;
            }
        } else
            e = d - s;
        acc += (long long)(e * e);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd((unsigned long long*)out, (unsigned long long)acc);
}

template <typename PIX>
__global__ void proj_subspace_sums_kernel(const PIX* src, int w, int h, int ss, const PIX* dat, int ds, const int32_t* flt0, int f0s,
                                          const int32_t* flt1, int f1s, int r0, int r1, long long* sums /*5*/) {
    long long h00 = 0, h11 = 0, h01 = 0, c0 = 0, c1 = 0;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < w * h; idx += gridDim.x * blockDim.x) {
        const int i = idx / w, j = idx - i * w;
        const long long u = (long long)((int32_t)dat[(size_t)i * ds + j] << 4);
        const long long s = (long long)((int32_t)src[(size_t)i * ss + j] << 4) - u;
        const long long f1 = r0 > 0 ? (long long)flt0[(size_t)i * f0s + j] - u : 0;
        const long long f2 = r1 > 0 ? (long long)flt1[(size_t)i * f1s + j] - u : 0;
        h00 += f1 * f1; h11 += f2 * f2; h01 += f1 * f2; c0 += f1 * s; c1 += f2 * s;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        h00 += __shfl_xor_sync(0xffffffffu, h00, o);
        h11 += __shfl_xor_sync(0xffffffffu, h11, o);
        h01 += __shfl_xor_sync(0xffffffffu, h01, o);
        c0 += __shfl_xor_sync(0xffffffffu, c0, o);
        c1 += __shfl_xor_sync(0xffffffffu, c1, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd((unsigned long long*)&sums[0], (unsigned long long)h00);
        atomicAdd((unsigned long long*)&sums[1], (unsigned long long)h11);
        atomicAdd((unsigned long long*)&sums[2], (unsigned long long)h01);
        atomicAdd((unsigned long long*)&sums[3], (unsigned long long)c0);
        atomicAdd((unsigned long long*)&sums[4], (unsigned long long)c1);
    }
}

__global__ void proj_subspace_solve_kernel(const long long* sums, int size, int r0, int r1, int* xq) {
    double H00 = __ddiv_rn((double)sums[0], (double)size), H11 = __ddiv_rn((double)sums[1], (double)size);
    double H01 = __ddiv_rn((double)sums[2], (double)size), C0 = __ddiv_rn((double)sums[3], (double)size);
    double C1 = __ddiv_rn((double)sums[4], (double)size);
    const double H10 = H01;
    xq[0] = 0;
    xq[1] = 0;
    if (r0 == 0) {
        const double det = H11;
        if (det < 1e-8) return;
        xq[1] = (int)rint(__dmul_rn(__ddiv_rn(C1, det), 128.0));
    } else if (r1 == 0) {
        const double det = H00;
        if (det < 1e-8) return;
        xq[0] = (int)rint(__dmul_rn(__ddiv_rn(C0, det), 128.0));
    } else {
        const double det = __dsub_rn(__dmul_rn(H00, H11), __dmul_rn(H01, H10));
        if (det < 1e-8) return;
        const double x0 = __ddiv_rn(__dsub_rn(__dmul_rn(H11, C0), __dmul_rn(H01, C1)), det);
        const double x1 = __ddiv_rn(__dsub_rn(__dmul_rn(H00, C1), __dmul_rn(H10, C0)), det);
        xq[0] = (int)rint(__dmul_rn(x0, 128.0));
        xq[1] = (int)rint(__dmul_rn(x1, 128.0));
    }
}

static size_t sgr_smem(int w, int h) {
    return (((size_t)(w + 6) * (h + 6) * 2 + 15) & ~size_t(15)) + (size_t)2 * (w + 2) * (h + 2) * 4;
}

template <typename PIX>
static void launch_sgr(const PIX* d_dgd, const SvtB200SgrUnit* d_units, int n, int32_t* d_f0, int32_t* d_f1, int bd, int max_w, int max_h,
                       cudaStream_t st) {
    const size_t smem = sgr_smem(max_w, max_h);
    static std::mutex mu;
    static size_t set8 = 0, set16 = 0;
    static int    set_epoch = -1;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (set_epoch != epoch()) { set8 = set16 = 0; set_epoch = epoch(); }
        size_t& s = sizeof(PIX) == 1 ? set8 : set16;
        if (smem > 48 * 1024 && smem > s) {
            B200_CUDA_CHECK(cudaFuncSetAttribute(sgr_filter_kernel<PIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(ctx().max_smem - 1024)));
            s = ctx().max_smem;
        }
    }
    sgr_filter_kernel<PIX><<<grid_for(n, 2), 256, smem, st>>>(d_dgd, d_units, n, d_f0, d_f1, bd);
    B200_LAUNCH_CHECK();
}

// stage (w+6)x(h+6) pixels around dat into the lane; returns offset of pixel (0,0)
template <typename PIX>
static size_t stage_ext(Lane* l, const PIX* dgd, int w, int h, int stride, int border, size_t* pitch) {
    const int tw = w + 2 * border, th = h + 2 * border;
    size_t o = l->alloc((size_t)tw * th * sizeof(PIX));
    for (int r = 0; r < th; r++) memcpy(l->h<PIX>(o) + (size_t)r * tw, dgd + (ptrdiff_t)(r - border) * stride - border, tw * sizeof(PIX));
    *pitch = tw;
    return o;
}

template <typename PIX>
static void sgr_t1(const PIX* dgd, int w, int h, int stride, int32_t* flt0, int32_t* flt1, int flt_stride, int idx, int bd) {
    require_ready();
    LaneGuard l;
    size_t pitch;
    size_t o_d = stage_ext<PIX>(l.l, dgd, w, h, stride, 3, &pitch), o_u = l->alloc(sizeof(SvtB200SgrUnit));
    size_t in_end = l->used;
    size_t o_f0 = l->alloc((size_t)w * h * 4), o_f1 = l->alloc((size_t)w * h * 4);
    SvtB200SgrUnit* u = l->h<SvtB200SgrUnit>(o_u);
    memset(u, 0, sizeof(*u));
    u->dgd_off = 3 * pitch + 3;
    u->dgd_stride = (int32_t)pitch;
    u->flt_stride = w;
    u->w = (uint16_t)w;
    u->h = (uint16_t)h;
    u->params_idx = (uint16_t)idx;
    l->h2d(0, in_end);
    launch_sgr<PIX>(l->d<PIX>(o_d), l->d<SvtB200SgrUnit>(o_u), 1, l->d<int32_t>(o_f0), l->d<int32_t>(o_f1), bd, w, h, l->stream);
    l->d2h(o_f0, (o_f1 + (size_t)w * h * 4) - o_f0);
    l->sync();
    const int* prm = h_sgr_params + 4 * idx;
    for (int r = 0; r < h; r++) {
        if (prm[0] > 0) memcpy(flt0 + (size_t)r * flt_stride, l->h<int32_t>(o_f0) + (size_t)r * w, w * 4);
        if (prm[1] > 0) memcpy(flt1 + (size_t)r * flt_stride, l->h<int32_t>(o_f1) + (size_t)r * w, w * 4);
    }
}

template <typename PIX>
static void sgr_apply_t1(const PIX* dat, int w, int h, int stride, int eps, const int32_t* xqd, PIX* dst, int dst_stride, int bd) {
    require_ready();
    const int* prm = h_sgr_params + 4 * eps;
    int xq[2];  // svt_decode_xq (restoration.c:634-645)
    if (prm[0] == 0) { xq[0] = 0; xq[1] = 128 - xqd[1]; }
    else if (prm[1] == 0) { xq[0] = xqd[0]; xq[1] = 0; }
    else { xq[0] = xqd[0]; xq[1] = 128 - xq[0] - xqd[1]; }
    LaneGuard l;
    size_t pitch;
    size_t o_d = stage_ext<PIX>(l.l, dat, w, h, stride, 3, &pitch), o_u = l->alloc(sizeof(SvtB200SgrUnit));
    size_t in_end = l->used;
    size_t o_f0 = l->alloc((size_t)w * h * 4), o_f1 = l->alloc((size_t)w * h * 4), o_o = l->alloc((size_t)w * h * sizeof(PIX));
    SvtB200SgrUnit* u = l->h<SvtB200SgrUnit>(o_u);
    memset(u, 0, sizeof(*u));
    u->dgd_off = 3 * pitch + 3;
    u->dgd_stride = (int32_t)pitch;
    u->flt_stride = w;
    u->w = (uint16_t)w;
    u->h = (uint16_t)h;
    u->params_idx = (uint16_t)eps;
    l->h2d(0, in_end);
    launch_sgr<PIX>(l->d<PIX>(o_d), l->d<SvtB200SgrUnit>(o_u), 1, l->d<int32_t>(o_f0), l->d<int32_t>(o_f1), bd, w, h, l->stream);
    sgr_project_kernel<PIX><<<grid_for((w * h + 255) / 256, 8), 256, 0, l->stream>>>(l->d<PIX>(o_d) + 3 * pitch + 3, w, h, (int)pitch, l->d<int32_t>(o_f0),
                                                                                  l->d<int32_t>(o_f1), xq[0], xq[1], prm[0], prm[1], l->d<PIX>(o_o), w, bd);
    B200_LAUNCH_CHECK();
    l->d2h(o_o, (size_t)w * h * sizeof(PIX));
    l->sync();
    for (int r = 0; r < h; r++) memcpy(dst + (size_t)r * dst_stride, l->h<PIX>(o_o) + (size_t)r * w, w * sizeof(PIX));
}

struct ProjStage { size_t o_src, o_dat, o_f0, o_f1; };
template <typename PIX>
static ProjStage stage_proj(Lane* l, const PIX* src, int w, int h, int ss, const PIX* dat, int ds, const int32_t* flt0, int f0s,
                            const int32_t* flt1, int f1s, int r0, int r1) {
    ProjStage p;
    p.o_src = l->alloc((size_t)w * h * sizeof(PIX));
    p.o_dat = l->alloc((size_t)w * h * sizeof(PIX));
    p.o_f0 = l->alloc((size_t)w * h * 4);
    p.o_f1 = l->alloc((size_t)w * h * 4);
    for (int r = 0; r < h; r++) {
        memcpy(l->h<PIX>(p.o_src) + (size_t)r * w, src + (size_t)r * ss, w * sizeof(PIX));
        memcpy(l->h<PIX>(p.o_dat) + (size_t)r * w, dat + (size_t)r * ds, w * sizeof(PIX));
        if (r0 > 0) memcpy(l->h<int32_t>(p.o_f0) + (size_t)r * w, flt0 + (size_t)r * f0s, w * 4);
        if (r1 > 0) memcpy(l->h<int32_t>(p.o_f1) + (size_t)r * w, flt1 + (size_t)r * f1s, w * 4);
    }
    return p;
}

template <typename PIX, bool HBD_FORM>
static int64_t proj_error_t1(const PIX* src, int w, int h, int ss, const PIX* dat, int ds, int32_t* flt0, int f0s, int32_t* flt1, int f1s,
                             int32_t xq[2], const int32_t* params) {
    require_ready();
    LaneGuard l;
    ProjStage p = stage_proj<PIX>(l.l, src, w, h, ss, dat, ds, flt0, f0s, flt1, f1s, params[0], params[1]);
    size_t o_out = l->alloc(8);
    *l->h<int64_t>(o_out) = 0;
    l->h2d(0, l->used);
    proj_error_kernel<PIX, HBD_FORM><<<grid_for((w * h + 255) / 256, 8), 256, 0, l->stream>>>(
        l->d<PIX>(p.o_src), w, h, w, l->d<PIX>(p.o_dat), w, l->d<int32_t>(p.o_f0), w, l->d<int32_t>(p.o_f1), w, xq[0], xq[1], params[0], params[1],
        l->d<long long>(o_out));
    B200_LAUNCH_CHECK();
    l->d2h(o_out, 8);
    l->sync();
    return *l->h<int64_t>(o_out);
}

template <typename PIX>
static void proj_subspace_t1(const PIX* src, int w, int h, int ss, const PIX* dat, int ds, int32_t* flt0, int f0s, int32_t* flt1, int f1s,
                             int* xq, const int32_t* params) {
    require_ready();
    LaneGuard l;
    ProjStage p = stage_proj<PIX>(l.l, src, w, h, ss, dat, ds, flt0, f0s, flt1, f1s, params[0], params[1]);
    size_t o_s = l->alloc(48);
    memset(l->h<uint8_t>(o_s), 0, 48);
    l->h2d(0, l->used);
    proj_subspace_sums_kernel<PIX><<<grid_for((w * h + 255) / 256, 8), 256, 0, l->stream>>>(l->d<PIX>(p.o_src), w, h, w, l->d<PIX>(p.o_dat), w,
                                                                                          l->d<int32_t>(p.o_f0), w, l->d<int32_t>(p.o_f1), w,
                                                                                          params[0], params[1], l->d<long long>(o_s));
    B200_LAUNCH_CHECK();
    proj_subspace_solve_kernel<<<1, 1, 0, l->stream>>>(l->d<long long>(o_s), w * h, params[0], params[1], (int*)(l->d<long long>(o_s) + 5));
    B200_LAUNCH_CHECK();
    l->d2h(o_s, 48);
    l->sync();
    const int* r = (const int*)(l->h<long long>(o_s) + 5);
    xq[0] = r[0];
    xq[1] = r[1];
}

}  // namespace b200

using namespace b200;

extern "C" void svt_b200_av1_selfguided_restoration(const uint8_t* dgd8, int32_t width, int32_t height, int32_t dgd_stride, int32_t* flt0,
                                                    int32_t* flt1, int32_t flt_stride, int32_t sgr_params_idx, int32_t bit_depth,
                                                    int32_t highbd) {
    if (highbd) sgr_t1<uint16_t>((const uint16_t*)dgd8, width, height, dgd_stride, flt0, flt1, flt_stride, sgr_params_idx, bit_depth);
    else sgr_t1<uint8_t>(dgd8, width, height, dgd_stride, flt0, flt1, flt_stride, sgr_params_idx, bit_depth);
}
extern "C" void svt_b200_apply_selfguided_restoration(const uint8_t* dat8, int32_t width, int32_t height, int32_t stride, int32_t eps,
                                                      const int32_t* xqd, uint8_t* dst8, int32_t dst_stride, int32_t* tmpbuf,
                                                      int32_t bit_depth, int32_t highbd) {
    (void)tmpbuf;
    if (highbd) sgr_apply_t1<uint16_t>((const uint16_t*)dat8, width, height, stride, eps, xqd, (uint16_t*)dst8, dst_stride, bit_depth);
    else sgr_apply_t1<uint8_t>(dat8, width, height, stride, eps, xqd, dst8, dst_stride, bit_depth);
}
extern "C" int64_t svt_b200_av1_lowbd_pixel_proj_error(const uint8_t* src8, int32_t width, int32_t height, int32_t src_stride,
                                                       const uint8_t* dat8, int32_t dat_stride, int32_t* flt0, int32_t flt0_stride,
                                                       int32_t* flt1, int32_t flt1_stride, int32_t xq[2], const int32_t* params) {
    return proj_error_t1<uint8_t, false>(src8, width, height, src_stride, dat8, dat_stride, flt0, flt0_stride, flt1, flt1_stride, xq, params);
}
extern "C" int64_t svt_b200_av1_highbd_pixel_proj_error(const uint16_t* src, int32_t width, int32_t height, int32_t src_stride,
                                                        const uint16_t* dat, int32_t dat_stride, int32_t* flt0, int32_t flt0_stride,
                                                        int32_t* flt1, int32_t flt1_stride, int32_t xq[2], const int32_t* params) {
    return proj_error_t1<uint16_t, true>(src, width, height, src_stride, dat, dat_stride, flt0, flt0_stride, flt1, flt1_stride, xq, params);
}
extern "C" void svt_b200_get_proj_subspace(const uint8_t* src8, int width, int height, int src_stride, const uint8_t* dat8, int dat_stride,
                                           int use_highbitdepth, int32_t* flt0, int flt0_stride, int32_t* flt1, int flt1_stride, int* xq,
                                           const int32_t* params) {
    if (use_highbitdepth)
        proj_subspace_t1<uint16_t>((const uint16_t*)src8, width, height, src_stride, (const uint16_t*)dat8, dat_stride, flt0, flt0_stride, flt1,
                                   flt1_stride, xq, params);
    else
        proj_subspace_t1<uint8_t>(src8, width, height, src_stride, dat8, dat_stride, flt0, flt0_stride, flt1, flt1_stride, xq, params);
}

extern "C" int svt_b200_sgr_units_dev(const void* d_dgd, const SvtB200SgrUnit* d_units, int n_units, int32_t* d_flt0, int32_t* d_flt1,
                                      int bit_depth, int max_w, int max_h, void* stream) {
    require_ready();
    if (n_units <= 0) return n_units == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    if (max_w > 128 || max_h > 128) return SVT_B200_ERR_BAD_ARG;
    if (bit_depth > 8) launch_sgr<uint16_t>((const uint16_t*)d_dgd, d_units, n_units, d_flt0, d_flt1, bit_depth, max_w, max_h, (cudaStream_t)stream);
    else launch_sgr<uint8_t>((const uint8_t*)d_dgd, d_units, n_units, d_flt0, d_flt1, 8, max_w, max_h, (cudaStream_t)stream);
    return SVT_B200_OK;
}
