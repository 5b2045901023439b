// me_picture.cu -- K13, the HME pyramid and plane padding (sm_90a): the padded 1/4 and 1/16 luma planes built from the full
// plane, and the replicated padding of 8- and 16-bit picture planes.
//
// Reference behaviour restated:
//   svt_aom_downsample_2d_c + svt_aom_generate_padding   Source/Lib/Codec/pic_analysis_process.c:130-160, 2138-2190
// The motion estimation itself is me_b64.cu (HME, full-pel item derivation) and me_pyramid.cu (full-pel search).
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

// ---- K13 ----------------------------------------------------------------------------------------
__global__ void downsample_2d_kernel(const uint8_t* __restrict__ in, int in_stride, int in_w, int in_h, uint8_t* __restrict__ out,
                                     int out_stride, int step) {
    const int half = step >> 1;
    const int ow = (in_w - half + step - 1) / step, oh = (in_h - half + step - 1) / step;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < ow * oh; idx += gridDim.x * blockDim.x) {
        const int oy = idx / ow, ox = idx - oy * ow;
        const int y = half + oy * step, x = half + ox * step;
        const uint32_t s = (uint32_t)in[(size_t)(y - 1) * in_stride + x - 1] + in[(size_t)(y - 1) * in_stride + x] +
                           in[(size_t)y * in_stride + x - 1] + in[(size_t)y * in_stride + x];
        out[(size_t)oy * out_stride + ox] = (uint8_t)((s + 2) >> 2);
    }
}
// replicate the w x h interior (at (org_x, org_y)) into the surrounding padding (svt_aom_generate_padding);
// only the border elements are visited: top band, bottom band, then the left/right strips of the interior rows
template <typename PIX>
__device__ __forceinline__ void pad_border_element(PIX* buf, int stride, int w, int h, int org_x, int org_y, int idx) {
    const int tw = w + 2 * org_x, band = org_y * tw;
    int x, y;
    if (idx < 2 * band) {
        const int j = idx < band ? idx : idx - band;
        y = j / tw + (idx < band ? 0 : org_y + h);
        x = j % tw;
    } else {
        const int j = idx - 2 * band, xx = j % (2 * org_x);
        y = org_y + j / (2 * org_x);
        x = xx < org_x ? xx : w + xx;
    }
    const int sx = min(max(x, org_x), org_x + w - 1), sy = min(max(y, org_y), org_y + h - 1);
    buf[(size_t)y * stride + x] = buf[(size_t)sy * stride + sx];
}
__host__ __device__ __forceinline__ int pad_border_count(int w, int h, int org_x, int org_y) {
    return 2 * org_y * (w + 2 * org_x) + 2 * org_x * h;
}
__global__ void pad_plane_kernel(uint8_t* buf, int stride, int w, int h, int org_x, int org_y) {
    const int n = pad_border_count(w, h, org_x, org_y);
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x)
        pad_border_element(buf, stride, w, h, org_x, org_y, idx);
}

}  // namespace b200

using namespace b200;

// T1: downsample_2d (aom_dsp_rtcd.h:841)
extern "C" void svt_b200_downsample_2d(uint8_t* input_samples, uint32_t input_stride, uint32_t input_area_width, uint32_t input_area_height,
                                       uint8_t* decim_samples, uint32_t decim_stride, uint32_t decim_step) {
    require_ready();
    const uint32_t half = decim_step >> 1;
    if (input_area_width <= half || input_area_height <= half) return;
    const uint32_t ow = (input_area_width - half + decim_step - 1) / decim_step, oh = (input_area_height - half + decim_step - 1) / decim_step;
    RoundTrip rt;
    auto in = rt.in_rows(input_samples, input_stride, input_area_width, input_area_height);
    auto out = rt.out_rows(decim_samples, decim_stride, ow, oh);
    downsample_2d_kernel<<<grid_for((ow * oh + 255) / 256, 8), 256, 0, rt.stream()>>>(rt.dev(in), (int)input_area_width, (int)input_area_width,
                                                                                   (int)input_area_height, rt.dev(out), (int)ow, (int)decim_step);
    B200_LAUNCH_CHECK();
    rt.finish();
}

struct PadPlanes {
    SvtB200PlaneExtent p[4];
};
// several planes in one launch: blockIdx.y = plane
__global__ void pad_planes_kernel(const __grid_constant__ PadPlanes pl) {
    const SvtB200PlaneExtent& e = pl.p[blockIdx.y];
    const int n = pad_border_count(e.w, e.h, e.org_x, e.org_y);
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x)
        if (e.pixel_bytes == 2) pad_border_element(reinterpret_cast<uint16_t*>(e.buf), e.stride, e.w, e.h, e.org_x, e.org_y, idx);
        else pad_border_element(e.buf, e.stride, e.w, e.h, e.org_x, e.org_y, idx);
}

extern "C" int svt_b200_extend_planes_dev(const SvtB200PlaneExtent* planes, int n_planes, void* stream) {
    require_ready();
    if (!planes || n_planes <= 0 || n_planes > 4) return SVT_B200_ERR_BAD_ARG;
    PadPlanes pl;
    memset(&pl, 0, sizeof(pl));
    int tn = 0;
    for (int i = 0; i < n_planes; i++) {
        if (!planes[i].buf || planes[i].w <= 0 || planes[i].h <= 0) return SVT_B200_ERR_BAD_ARG;
        pl.p[i] = planes[i];
        const int t = pad_border_count(planes[i].w, planes[i].h, planes[i].org_x, planes[i].org_y);
        tn = t > tn ? t : tn;
    }
    pad_planes_kernel<<<dim3(grid_for((tn + 255) / 256, 4), n_planes), 256, 0, (cudaStream_t)stream>>>(pl);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

extern "C" int svt_b200_extend_plane_dev(uint8_t* d_buf, int stride, int w, int h, int org_x, int org_y, void* stream) {
    require_ready();
    if (!d_buf || w <= 0 || h <= 0) return SVT_B200_ERR_BAD_ARG;
    const int tn = pad_border_count(w, h, org_x, org_y);
    if (tn <= 0) return SVT_B200_OK;
    pad_plane_kernel<<<grid_for((tn + 255) / 256, 8), 256, 0, (cudaStream_t)stream>>>(d_buf, stride, w, h, org_x, org_y);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

// T2: build the padded 1/4 and 1/16 luma planes of one picture on the device
extern "C" int svt_b200_build_hme_pyramid_dev(const SvtB200MePicture* pic, void* stream) {
    require_ready();
    if (!pic) return SVT_B200_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    for (int lvl = 1; lvl >= 0; lvl--) {  // quarter from full, sixteenth from quarter
        const int s = lvl + 1;
        const uint8_t* in = pic->plane[s] + (size_t)pic->org_y[s] * pic->stride[s] + pic->org_x[s];
        uint8_t* out = const_cast<uint8_t*>(pic->plane[lvl]) + (size_t)pic->org_y[lvl] * pic->stride[lvl] + pic->org_x[lvl];
        const int n = pic->width[lvl] * pic->height[lvl];
        downsample_2d_kernel<<<grid_for((n + 255) / 256, 8), 256, 0, st>>>(in, pic->stride[s], pic->width[s], pic->height[s], out, pic->stride[lvl], 2);
        B200_LAUNCH_CHECK();
        const int tn = pad_border_count(pic->width[lvl], pic->height[lvl], pic->org_x[lvl], pic->org_y[lvl]);
        pad_plane_kernel<<<grid_for((tn + 255) / 256, 8), 256, 0, st>>>(const_cast<uint8_t*>(pic->plane[lvl]), pic->stride[lvl], pic->width[lvl],
                                                                      pic->height[lvl], pic->org_x[lvl], pic->org_y[lvl]);
        B200_LAUNCH_CHECK();
    }
    return SVT_B200_OK;
}
