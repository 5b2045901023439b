// pa_stats.cu -- K15 picture-analysis statistics (sm_90a): the per-64x64 block variances and the scene-change
// histograms of svt_aom_gathering_picture_statistics, and the four block-mean dispatch pointers.
//
// Reference behaviour restated:
//   compute_block_mean_compute_variance   Source/Lib/Codec/pic_analysis_process.c:306-1290
//   svt_compute_mean_c / svt_compute_mean_squared_values_c / svt_compute_sub_mean_8x8_c /
//   svt_aom_compute_sub_mean_squared_values_c / svt_compute_interm_var_four8x8_c               :190-300
//   sub_sample_luma_generate_pixel_intensity_histogram_bins + calculate_histogram              :1461-1525, :166
//   compute_picture_spatial_statistics, svt_aom_gathering_picture_statistics                    :1531-1576
// Everything is integer: the 8x8 means / mean squares are exact (FULL: (S << 8) / 64, (SS << 16) / 64; SUB: S << 3,
// SS << 11 over rows 0, 2, 4, 6), the 16x16 / 32x32 / 64x64 values are the reference's u64 ">> 2 of four" tree, and a
// variance is (uint16_t)((meansq - mean * mean) >> VARIANCE_PRECISION) with the u64 wrap the reference has.
//
// The T2 call is two launches on the caller's stream:
//   pa_stats_kernel     one grid: a CTA per histogram region (first, the longer jobs), then a CTA per 64x64 block
//   pa_finalize_kernel  one CTA: pic_avg_variance from the 64x64 variances and avg_luma from the final histograms
// A last-CTA-done reduction would fold the second launch into the first, but it needs a ticket counter in device memory
// that concurrent calls on other streams must not share (per-stream scratch, a lock, a self-resetting counter); the
// second launch needs no state at all and reads only what the first one wrote.  Its cost is reported by
// tools/profile_pa_stats.py (the call with both parts off runs only this kernel).
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

constexpr int kPaThreads = 256;
constexpr int kVarPrec   = 16;   // VARIANCE_PRECISION (me_context.h:25)
constexpr unsigned long long kInvalidLuma = 256;  // INVALID_LUMA (definitions.h:78)

__device__ __forceinline__ uint16_t variance_of(unsigned long long msq, unsigned long long m) {
    return (uint16_t)((msq - m * m) >> kVarPrec);
}

// 16 bytes at any alignment as four words, reading only words that hold one of the 16 bytes
__device__ __forceinline__ void load16(const uint8_t* p, uint32_t w[4]) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* g = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    const int sh = (int)(a & 3) * 8;
    uint32_t v[5];
#pragma unroll
    for (int i = 0; i < 4; i++) v[i] = __ldg(g + i);
    v[4] = sh ? __ldg(g + 4) : 0u;
#pragma unroll
    for (int i = 0; i < 4; i++) w[i] = __funnelshift_r(v[i], v[i + 1], sh);
}

__device__ __forceinline__ uint32_t sum8(uint32_t a, uint32_t b) { return __vsadu4(a, 0u) + __vsadu4(b, 0u); }
__device__ __forceinline__ uint32_t sumsq8(uint32_t a, uint32_t b) { return __dp4a(a, a, 0u) + __dp4a(b, b, 0u); }

// ---- one 64x64 block: compute_block_mean_compute_variance ----------------------------------------------------------------
// Warp w takes 8x8 block row w; lane = (row in the block row) * 4 + q, q = 16-byte quarter of the 64 columns = 8x8 block
// columns 2q and 2q + 1.  Three xor-shuffles over the row bits leave each 8x8 block's sums in lanes 0..3.
__device__ void block_variance(const uint8_t* blk, int stride, int sub, int var8, uint16_t* out) {
    __shared__ unsigned long long m8[64], q8[64], m16[16], q16[16], m32[4], q32[4];
    const int t = threadIdx.x, lane = t & 31, by = t >> 5, r = lane >> 2, q = lane & 3;
    uint32_t s0 = 0, s1 = 0, ss0 = 0, ss1 = 0;
    if (!sub || !(r & 1)) {  // BLOCK_MEAN_PREC_SUB reads rows 0, 2, 4, 6 of every 8x8
        uint32_t w[4];
        load16(blk + (size_t)(8 * by + r) * stride + 16 * q, w);
        s0 = sum8(w[0], w[1]);
        s1 = sum8(w[2], w[3]);
        ss0 = sumsq8(w[0], w[1]);
        ss1 = sumsq8(w[2], w[3]);
    }
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        ss0 += __shfl_xor_sync(0xffffffffu, ss0, o);
        ss1 += __shfl_xor_sync(0xffffffffu, ss1, o);
    }
    if (lane < 4) {
        const int k = 8 * by + 2 * q;
        if (sub) {  // svt_compute_sub_mean_8x8_c, svt_aom_compute_sub_mean_squared_values_c
            m8[k] = (unsigned long long)s0 << 3;
            m8[k + 1] = (unsigned long long)s1 << 3;
            q8[k] = (unsigned long long)ss0 << 11;
            q8[k + 1] = (unsigned long long)ss1 << 11;
        } else {    // svt_compute_mean_c / svt_compute_mean_squared_values_c at 8x8
            m8[k] = ((unsigned long long)s0 << (kVarPrec >> 1)) / 64;
            m8[k + 1] = ((unsigned long long)s1 << (kVarPrec >> 1)) / 64;
            q8[k] = ((unsigned long long)ss0 << kVarPrec) / 64;
            q8[k + 1] = ((unsigned long long)ss1 << kVarPrec) / 64;
        }
    }
    __syncthreads();
    if (t < 16) {  // 16x16 i = t: 8x8 rows 2(i/4), 2(i/4)+1, columns 2(i%4), 2(i%4)+1
        const int a = 16 * (t >> 2) + 2 * (t & 3);
        m16[t] = (m8[a] + m8[a + 1] + m8[a + 8] + m8[a + 9]) >> 2;
        q16[t] = (q8[a] + q8[a + 1] + q8[a + 8] + q8[a + 9]) >> 2;
    }
    __syncthreads();
    if (t < 4) {
        const int a = 8 * (t >> 1) + 2 * (t & 1);
        m32[t] = (m16[a] + m16[a + 1] + m16[a + 4] + m16[a + 5]) >> 2;
        q32[t] = (q16[a] + q16[a + 1] + q16[a + 4] + q16[a + 5]) >> 2;
    }
    __syncthreads();
    if (t < 64) out[21 + t] = var8 ? variance_of(q8[t], m8[t]) : 0;
    if (t < 16) out[5 + t] = var8 ? variance_of(q16[t], m16[t]) : 0;
    if (t < 4) out[1 + t] = var8 ? variance_of(q32[t], m32[t]) : 0;
    if (t == 0) {
        const unsigned long long m64 = (m32[0] + m32[1] + m32[2] + m32[3]) >> 2;
        const unsigned long long q64 = (q32[0] + q32[1] + q32[2] + q32[3]) >> 2;
        out[0] = variance_of(q64, m64);
    }
}

// ---- one region of the 1/16 plane: calculate_histogram + the bin scaling and average of :1479-1518 ------------------------
// Lanes that see the same value are merged (__match_any_sync) before the shared atomic, so flat content costs one atomic
// per warp and step rather than 32 on one address.
__device__ void region_histogram(const uint8_t* p, int stride, int w, int h, int d, uint32_t* hist, uint8_t* avg) {
    __shared__ uint32_t bins[256];
    __shared__ unsigned long long part[kPaThreads / 32];
    const int t = threadIdx.x, lane = t & 31;
    bins[t] = 0;
    __syncthreads();
    const int cols = (w + d - 1) / d, rows = (h + d - 1) / d, n = cols * rows;
    uint32_t sum = 0;
    for (int base = 0; base < n; base += kPaThreads) {
        const int i = base + t;
        uint32_t v = 256;  // no sample
        if (i < n) {
            const int y = i / cols, x = i - y * cols;
            v = p[(size_t)y * d * stride + x * d];
            sum += v;
        }
        const uint32_t grp = __match_any_sync(0xffffffffu, v);
        if (v < 256 && lane == __ffs(grp) - 1) atomicAdd(&bins[v], (uint32_t)__popc(grp));
    }
    // svt_initialize_buffer_32bits(..., 1), then each bin * 4 * 4 * decim_step * decim_step
    __syncthreads();
    hist[t] = (1u + bins[t]) * 4u * 4u * (uint32_t)d * (uint32_t)d;
    unsigned long long s = sum;
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) part[t >> 5] = s;
    __syncthreads();
    if (t == 0) {
        unsigned long long tot = 0;
        for (int i = 0; i < kPaThreads / 32; i++) tot += part[i];
        tot *= (unsigned long long)d * d;
        const uint32_t area = (uint32_t)w * (uint32_t)h;
        *avg = (uint8_t)((tot + (area >> 1)) / area);
    }
}

struct PaArgs {
    const uint8_t* full;      // plane[2] at the visible origin
    int            full_stride, b64_w, n_b64, sub, var8;
    const uint8_t* sixteenth; // plane[0] at the visible origin
    int            s_stride, s_w, s_h, d, rw, rh, n_hist;
    uint16_t*      variance;
    uint32_t*      histogram;
    uint8_t*       average_intensity;
};

__global__ void __launch_bounds__(kPaThreads) pa_stats_kernel(const __grid_constant__ PaArgs a) {
    const int c = blockIdx.x;
    if (c < a.n_hist) {  // region (iw, ih) of sub_sample_luma_generate_pixel_intensity_histogram_bins, histogram[iw][ih]
        const int iw = c / a.rh, ih = c - iw * a.rh;
        const int rw = a.s_w / a.rw, rh = a.s_h / a.rh;
        const int w = rw + (iw == a.rw - 1 ? a.s_w - a.rw * rw : 0);  // the last region takes the remainder
        const int h = rh + (ih == a.rh - 1 ? a.s_h - a.rh * rh : 0);
        region_histogram(a.sixteenth + (size_t)ih * rh * a.s_stride + iw * rw, a.s_stride, w, h, a.d, a.histogram + (size_t)c * 256,
                         a.average_intensity + c);
        return;
    }
    const int b = c - a.n_hist, bx = b % a.b64_w, by = b / a.b64_w;
    block_variance(a.full + (size_t)by * 64 * a.full_stride + bx * 64, a.full_stride, a.sub, a.var8, a.variance + (size_t)b * 85);
}

// pic_avg_variance = (uint16_t)(sum of the 64x64 variances / b64_total_count) (:1531-1550) and avg_luma = the sum of every
// region's decim_step^2-weighted pixel sum over the plane area (:1519-1524).  A region's sum is read back from its final
// histogram: bin v holds (1 + count_v) * 16 * d^2, so sum = d^2 * sum_v v * count_v exactly.
__global__ void __launch_bounds__(kPaThreads) pa_finalize_kernel(const uint16_t* variance, int n_b64, uint16_t* pic_avg_variance,
                                                                 const uint32_t* histogram, int n_regions, int d, uint32_t area,
                                                                 uint64_t* avg_luma) {
    __shared__ unsigned long long pv[kPaThreads / 32], pl[kPaThreads / 32];
    const int t = threadIdx.x, lane = t & 31;
    unsigned long long v = 0, l = 0;
    if (variance)
        for (int b = t; b < n_b64; b += kPaThreads) v += variance[(size_t)b * 85];
    if (histogram) {
        const uint32_t unit = 16u * (uint32_t)d * (uint32_t)d;
        for (int r = 0; r < n_regions; r++) l += (unsigned long long)t * (histogram[(size_t)r * 256 + t] / unit - 1u);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        v += __shfl_xor_sync(0xffffffffu, v, o);
        l += __shfl_xor_sync(0xffffffffu, l, o);
    }
    if (lane == 0) {
        pv[t >> 5] = v;
        pl[t >> 5] = l;
    }
    __syncthreads();
    if (t == 0) {
        unsigned long long sv = 0, sl = 0;
        for (int i = 0; i < kPaThreads / 32; i++) {
            sv += pv[i];
            sl += pl[i];
        }
        *pic_avg_variance = variance ? (uint16_t)(sv / (unsigned long long)n_b64) : 0;
        *avg_luma = histogram ? sl * (unsigned long long)d * d / area : kInvalidLuma;
    }
}

// ---- T1: one warp over the packed rows (pitch w) of one call ---------------------------------------------------------------
// mode 0: svt_compute_mean_c, 1: svt_compute_mean_squared_values_c (any w x h); 2: svt_compute_sub_mean_8x8_c (8 x 4 packed
// rows); 3: svt_compute_interm_var_four8x8_c (32 x 4 packed rows: four 8-column groups, means then mean squares)
__global__ void pa_t1_kernel(const uint8_t* px, uint32_t w, uint32_t h, int mode, uint64_t* out) {
    const int lane = threadIdx.x;
    unsigned long long s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};  // u64 like the reference's accumulators (any w x h)
    const uint32_t n = w * h;
    for (uint32_t i = lane; i < n; i += 32) {
        const uint32_t v = px[i], g = mode == 3 ? (i % w) >> 3 : 0;
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (g == (uint32_t)k) {
                s[k] += v;
                ss[k] += v * v;
            }
    }
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
            ss[k] += __shfl_xor_sync(0xffffffffu, ss[k], o);
        }
    if (lane != 0) return;
    switch (mode) {
        case 0: out[0] = (s[0] << (kVarPrec >> 1)) / n; break;
        case 1: out[0] = (ss[0] << kVarPrec) / n; break;
        case 2: out[0] = s[0] << 3; break;
        default:
            for (int k = 0; k < 4; k++) {
                out[k] = s[k] << 3;
                out[4 + k] = ss[k] << 11;
            }
    }
}

// rows at `pitch` of `w` bytes each, packed and sent; returns the results the kernel wrote
static void pa_t1(const uint8_t* p, size_t pitch, uint32_t w, uint32_t rows, int mode, uint64_t* out, int n_out) {
    require_ready();
    RoundTrip rt;
    auto in = rt.in_rows(p, pitch, w, rows);
    auto o = rt.out(out, (size_t)n_out);
    pa_t1_kernel<<<1, 32, 0, rt.stream()>>>(rt.dev(in), w, rows, mode, rt.dev(o));
    B200_LAUNCH_CHECK();
    rt.finish();
}

}  // namespace b200

using namespace b200;

extern "C" uint64_t svt_b200_compute_mean_8x8(uint8_t* input_samples, uint32_t input_stride, uint32_t input_area_width,
                                              uint32_t input_area_height) {
    uint64_t r = 0;
    if (input_area_width && input_area_height) pa_t1(input_samples, input_stride, input_area_width, input_area_height, 0, &r, 1);
    return r;
}

extern "C" uint64_t svt_b200_compute_mean_square_values_8x8(uint8_t* input_samples, uint32_t input_stride, uint32_t input_area_width,
                                                            uint32_t input_area_height) {
    uint64_t r = 0;
    if (input_area_width && input_area_height) pa_t1(input_samples, input_stride, input_area_width, input_area_height, 1, &r, 1);
    return r;
}

extern "C" uint64_t svt_b200_compute_sub_mean_8x8(uint8_t* input_samples, uint16_t input_stride) {
    uint64_t r = 0;
    pa_t1(input_samples, 2 * (size_t)input_stride, 8, 4, 2, &r, 1);
    return r;
}

extern "C" void svt_b200_compute_interm_var_four8x8(uint8_t* input_samples, uint16_t input_stride, uint64_t* mean_of8x8_blocks,
                                                    uint64_t* mean_of_squared8x8_blocks) {
    uint64_t r[8];
    pa_t1(input_samples, 2 * (size_t)input_stride, 32, 4, 3, r, 8);
    memcpy(mean_of8x8_blocks, r, 4 * sizeof(uint64_t));
    memcpy(mean_of_squared8x8_blocks, r + 4, 4 * sizeof(uint64_t));
}

extern "C" int svt_b200_picture_statistics_dev(const SvtB200MePicture* pic, const SvtB200PaStatsControls* ctl,
                                               const SvtB200PaStatsResults* out, void* stream) {
    require_ready();
    if (!pic || !ctl || !out || !out->pic_avg_variance || !out->avg_luma) return SVT_B200_ERR_BAD_ARG;
    PaArgs a;
    memset(&a, 0, sizeof(a));
    const bool var = ctl->calculate_variance != 0, hist = ctl->calc_hist != 0;
    if (var) {
        const int W = pic->width[2], H = pic->height[2], W64 = (W + 63) & ~63, H64 = (H + 63) & ~63;
        if (!pic->plane[2] || !out->variance || W <= 0 || H <= 0 || pic->org_x[2] < 0 || pic->org_y[2] < H64 - H ||
            pic->stride[2] < pic->org_x[2] + W64)
            return SVT_B200_ERR_BAD_ARG;
        if (ctl->block_mean_calc_prec != 0 && ctl->block_mean_calc_prec != 1) return SVT_B200_ERR_BAD_ARG;
        a.full = pic->plane[2] + (size_t)pic->org_y[2] * pic->stride[2] + pic->org_x[2];
        a.full_stride = pic->stride[2];
        a.b64_w = W64 / 64;
        a.n_b64 = a.b64_w * (H64 / 64);
        a.sub = ctl->block_mean_calc_prec;
        a.var8 = ctl->var_8x8 != 0;
        a.variance = out->variance;
    }
    if (hist) {
        const int w = pic->width[0], h = pic->height[0];
        if (!pic->plane[0] || !out->histogram || !out->average_intensity) return SVT_B200_ERR_BAD_ARG;
        if (ctl->regions_w < 1 || ctl->regions_w > SVT_B200_PA_MAX_REGIONS || ctl->regions_h < 1 || ctl->regions_h > SVT_B200_PA_MAX_REGIONS)
            return SVT_B200_ERR_BAD_ARG;
        if (ctl->decim_step != 1 && ctl->decim_step != 4) return SVT_B200_ERR_BAD_ARG;
        if (w < ctl->regions_w || h < ctl->regions_h || (long long)w * h >= (1ll << 26) || pic->org_x[0] < 0 || pic->org_y[0] < 0 ||
            pic->stride[0] < pic->org_x[0] + w)
            return SVT_B200_ERR_BAD_ARG;
        a.sixteenth = pic->plane[0] + (size_t)pic->org_y[0] * pic->stride[0] + pic->org_x[0];
        a.s_stride = pic->stride[0];
        a.s_w = w;
        a.s_h = h;
        a.d = ctl->decim_step;
        a.rw = ctl->regions_w;
        a.rh = ctl->regions_h;
        a.n_hist = a.rw * a.rh;
        a.histogram = out->histogram;
        a.average_intensity = out->average_intensity;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (a.n_hist + a.n_b64 > 0) {
        pa_stats_kernel<<<a.n_hist + a.n_b64, kPaThreads, 0, st>>>(a);
        B200_LAUNCH_CHECK();
    }
    pa_finalize_kernel<<<1, kPaThreads, 0, st>>>(var ? out->variance : nullptr, a.n_b64, out->pic_avg_variance, hist ? out->histogram : nullptr,
                                                 a.n_hist, a.d, (uint32_t)a.s_w * (uint32_t)a.s_h, out->avg_luma);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}
