/* svt_b200_rtcd.c -- see svt_b200_rtcd.h.  Compiled INSIDE the reference tree (it includes the reference's own
 * rtcd headers), linked against libsvtav1_b200.so.  Plain assignments only: the C compiler checks every prototype
 * of include/svt_b200.h against the reference's pointer type (build with -Werror=incompatible-pointer-types). */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include "definitions.h"
#include "aom_dsp_rtcd.h"
#include "common_dsp_rtcd.h"
#include "inv_transforms.h"
#include "svt_b200.h"
#include "svt_b200_rtcd.h"

/* ---- adaptors where the reference's calling convention is not a plain pointer list ---------------------------------- */
/* svt_av1_inv_txfm_add (common_dsp_rtcd.h:144): the 8-bit inverse takes its transform type / size in a TxfmParam.
 * Lossless blocks use the Walsh-Hadamard transform, which is not on the H100 path: they stay on the C function. */
static void b200_av1_inv_txfm_add(const TranLow* dqcoeff, uint8_t* dst_r, int32_t stride_r, uint8_t* dst_w, int32_t stride_w,
                                  const TxfmParam* p) {
    if (p->lossless) {
        svt_av1_inv_txfm_add_c(dqcoeff, dst_r, stride_r, dst_w, stride_w, p);
        return;
    }
    svt_b200_inv_txfm_add_8bit(dqcoeff, dst_r, stride_r, dst_w, stride_w, (int)p->tx_type, (int)p->tx_size);
}
/* High-bit-depth pixel pointers travel through uint8_t* arguments as CONVERT_TO_BYTEPTR disguises (address >> 1:
 * full_loop.c:1843-1846, restoration.c:933); the H100 entry points take the real uint16_t address. */
#define B200_U16(p) ((const uint16_t*)CONVERT_TO_SHORTPTR(p))
static void b200_highbd_wiener_convolve_add_src(const uint8_t* const src, const ptrdiff_t src_stride, uint8_t* const dst,
                                                const ptrdiff_t dst_stride, const int16_t* const filter_x, const int16_t* const filter_y,
                                                const int32_t w, const int32_t h, const ConvolveParams* const cp, const int32_t bd) {
    svt_b200_av1_highbd_wiener_convolve_add_src(B200_U16(src), src_stride, (uint16_t*)CONVERT_TO_SHORTPTR(dst), dst_stride, filter_x, filter_y, w, h,
                                                (const SvtB200ConvolveParams*)cp, bd);
}
static void b200_wiener_convolve_add_src(const uint8_t* const src, const ptrdiff_t src_stride, uint8_t* const dst, const ptrdiff_t dst_stride,
                                         const int16_t* const filter_x, const int16_t* const filter_y, const int32_t w, const int32_t h,
                                         const ConvolveParams* const cp) {
    svt_b200_av1_wiener_convolve_add_src(src, src_stride, dst, dst_stride, filter_x, filter_y, w, h, (const SvtB200ConvolveParams*)cp);
}
static void b200_compute_stats_highbd(int32_t wiener_win, const uint8_t* dgd8, const uint8_t* src8, int32_t h_start, int32_t h_end,
                                      int32_t v_start, int32_t v_end, int32_t dgd_stride, int32_t src_stride, int64_t* M, int64_t* H,
                                      EbBitDepth bit_depth) {
    svt_b200_av1_compute_stats_highbd(wiener_win, B200_U16(dgd8), B200_U16(src8), h_start, h_end, v_start, v_end, dgd_stride, src_stride, M, H,
                                      (int32_t)bit_depth);
}
static void b200_selfguided_restoration(const uint8_t* dgd8, int32_t width, int32_t height, int32_t dgd_stride, int32_t* flt0, int32_t* flt1,
                                        int32_t flt_stride, int32_t sgr_params_idx, int32_t bit_depth, int32_t highbd) {
    svt_b200_av1_selfguided_restoration(highbd ? (const uint8_t*)B200_U16(dgd8) : dgd8, width, height, dgd_stride, flt0, flt1, flt_stride,
                                        sgr_params_idx, bit_depth, highbd);
}
static void b200_apply_selfguided_restoration(const uint8_t* dat, int32_t width, int32_t height, int32_t stride, int32_t eps, const int32_t* xqd,
                                              uint8_t* dst, int32_t dst_stride, int32_t* tmpbuf, int32_t bit_depth, int32_t highbd) {
    svt_b200_apply_selfguided_restoration(highbd ? (const uint8_t*)B200_U16(dat) : dat, width, height, stride, eps, xqd,
                                          highbd ? (uint8_t*)CONVERT_TO_SHORTPTR(dst) : dst, dst_stride, tmpbuf, bit_depth, highbd);
}
static int64_t b200_lowbd_pixel_proj_error(const uint8_t* src8, int32_t width, int32_t height, int32_t src_stride, const uint8_t* dat8,
                                           int32_t dat_stride, int32_t* flt0, int32_t flt0_stride, int32_t* flt1, int32_t flt1_stride,
                                           int32_t xq[2], const SgrParamsType* params) {
    return svt_b200_av1_lowbd_pixel_proj_error(src8, width, height, src_stride, dat8, dat_stride, flt0, flt0_stride, flt1, flt1_stride, xq,
                                               (const int32_t*)params);
}
static int64_t b200_highbd_pixel_proj_error(const uint8_t* src8, int32_t width, int32_t height, int32_t src_stride, const uint8_t* dat8,
                                            int32_t dat_stride, int32_t* flt0, int32_t flt0_stride, int32_t* flt1, int32_t flt1_stride,
                                            int32_t xq[2], const SgrParamsType* params) {
    return svt_b200_av1_highbd_pixel_proj_error(B200_U16(src8), width, height, src_stride, B200_U16(dat8), dat_stride, flt0, flt0_stride, flt1,
                                                flt1_stride, xq, (const int32_t*)params);
}
static void b200_get_proj_subspace(const uint8_t* src8, int width, int height, int src_stride, const uint8_t* dat8, int dat_stride,
                                   int use_highbitdepth, int32_t* flt0, int flt0_stride, int32_t* flt1, int flt1_stride, int* xq,
                                   const SgrParamsType* params) {
    svt_b200_get_proj_subspace(use_highbitdepth ? (const uint8_t*)B200_U16(src8) : src8, width, height, src_stride,
                               use_highbitdepth ? (const uint8_t*)B200_U16(dat8) : dat8, dat_stride, use_highbitdepth, flt0, flt0_stride, flt1,
                               flt1_stride, xq, (const int32_t*)params);
}
static void b200_ext_all_sad_calculation_8x8_16x16(uint8_t* src, uint32_t src_stride, uint8_t* ref, uint32_t ref_stride, uint32_t mv,
                                                   uint32_t* p_best_sad_8x8, uint32_t* p_best_sad_16x16, uint32_t* p_best_mv8x8,
                                                   uint32_t* p_best_mv16x16, uint32_t p_eight_sad16x16[16][8], uint32_t p_eight_sad8x8[64][8],
                                                   bool sub_sad) {
    svt_b200_ext_all_sad_calculation_8x8_16x16(src, src_stride, ref, ref_stride, mv, p_best_sad_8x8, p_best_sad_16x16, p_best_mv8x8,
                                               p_best_mv16x16, p_eight_sad16x16, p_eight_sad8x8, (uint8_t)sub_sad);
}
static void b200_ext_sad_calculation_8x8_16x16(uint8_t* src, uint32_t src_stride, uint8_t* ref, uint32_t ref_stride, uint32_t* p_best_sad_8x8,
                                               uint32_t* p_best_sad_16x16, uint32_t* p_best_mv8x8, uint32_t* p_best_mv16x16, uint32_t mv,
                                               uint32_t* p_sad16x16, uint32_t* p_sad8x8, bool sub_sad) {
    svt_b200_ext_sad_calculation_8x8_16x16(src, src_stride, ref, ref_stride, p_best_sad_8x8, p_best_sad_16x16, p_best_mv8x8, p_best_mv16x16, mv,
                                           p_sad16x16, p_sad8x8, (uint8_t)sub_sad);
}
static uint64_t b200_cdef_dist_16bit(const uint16_t* dst, int32_t dstride, const uint16_t* src, const CdefList* dlist, int32_t cdef_count,
                                     BlockSize bsize, int32_t coeff_shift, int32_t pli, uint8_t subsampling_factor) {
    return svt_b200_compute_cdef_dist_16bit(dst, dstride, src, (const SvtB200CdefList*)dlist, cdef_count, (uint8_t)bsize, coeff_shift, pli,
                                            subsampling_factor);
}
static uint64_t b200_cdef_dist_8bit(const uint8_t* dst8, int32_t dstride, const uint8_t* src8, const CdefList* dlist, int32_t cdef_count,
                                    BlockSize bsize, int32_t coeff_shift, int32_t pli, uint8_t subsampling_factor) {
    return svt_b200_compute_cdef_dist_8bit(dst8, dstride, src8, (const SvtB200CdefList*)dlist, cdef_count, (uint8_t)bsize, coeff_shift, pli,
                                           subsampling_factor);
}

static uint32_t b200_hadamard_path(Buf2D residual, Buf2D coeff, Buf2D input, Buf2D pred, BlockSize bsize) {
    SvtB200Buf2D r = {residual.buf, residual.buf0, residual.width, residual.height, residual.stride};
    SvtB200Buf2D c = {coeff.buf, coeff.buf0, coeff.width, coeff.height, coeff.stride};
    SvtB200Buf2D i = {input.buf, input.buf0, input.width, input.height, input.stride};
    SvtB200Buf2D p = {pred.buf, pred.buf0, pred.width, pred.height, pred.stride};
    return svt_b200_hadamard_path(r, c, i, p, (uint8_t)bsize);
}

static int g_count = 0;
static unsigned g_groups = ~0u, g_cur = 0; /* SVT_B200_RTCD_GROUPS (debug): bit mask of the kernel groups to install, default all */
#define GROUP(bit) g_cur = (bit)
#define BIND(ptr, fn) do { if (g_groups & g_cur) { (ptr) = (fn); g_count++; } } while (0)
#define BIND_FWD(WxH)                                                    \
    BIND(svt_av1_fwd_txfm2d_##WxH, svt_b200_av1_fwd_txfm2d_##WxH);        \
    BIND(svt_av1_fwd_txfm2d_##WxH##_N2, svt_b200_av1_fwd_txfm2d_##WxH##_N2); \
    BIND(svt_av1_fwd_txfm2d_##WxH##_N4, svt_b200_av1_fwd_txfm2d_##WxH##_N4); \
    g_cur = 8u;                                                           \
    BIND(svt_av1_inv_txfm2d_add_##WxH, svt_b200_av1_inv_txfm2d_add_##WxH); \
    g_cur = 4u
#define BIND_SAD(MxN)                                        \
    BIND(svt_aom_sad##MxN, svt_b200_aom_sad##MxN);            \
    BIND(svt_aom_sad##MxN##x4d, svt_b200_aom_sad##MxN##x4d)
#define BIND_HANDLE(WxH)                                                        \
    BIND(svt_handle_transform##WxH, svt_b200_handle_transform##WxH);             \
    BIND(svt_handle_transform##WxH##_N2_N4, svt_b200_handle_transform##WxH##_N2_N4)

int svt_b200_rtcd_count(void) { return g_count; }

int svt_b200_install_rtcd(int device) {
    const int rc = svt_b200_init(device);
    if (rc != SVT_B200_OK && rc != SVT_B200_ERR_ALREADY_INIT) return rc;
    g_count = 0;
    {
        const char* m = getenv("SVT_B200_RTCD_GROUPS");
        g_groups = (m && *m) ? (unsigned)strtoul(m, NULL, 0) : ~0u;
    }
    GROUP(1u);
    /* K1 / K2 / K3: SAD search, SAD pyramid, single SADs (aom_dsp_rtcd.h:779,842-856,275-403) */
    BIND(svt_sad_loop_kernel, svt_b200_sad_loop_kernel);
    BIND(svt_nxm_sad_kernel, svt_b200_nxm_sad_kernel);
    BIND(svt_ext_all_sad_calculation_8x8_16x16, b200_ext_all_sad_calculation_8x8_16x16);
    BIND(svt_ext_eight_sad_calculation_32x32_64x64, svt_b200_ext_eight_sad_calculation_32x32_64x64);
    BIND(svt_ext_sad_calculation_8x8_16x16, b200_ext_sad_calculation_8x8_16x16);
    BIND(svt_ext_sad_calculation_32x32_64x64, svt_b200_ext_sad_calculation_32x32_64x64);
    BIND(svt_initialize_buffer_32bits, svt_b200_initialize_buffer_32bits);
    BIND(downsample_2d, svt_b200_downsample_2d);
    BIND_SAD(128x128); BIND_SAD(128x64); BIND_SAD(64x128); BIND_SAD(64x64); BIND_SAD(64x32); BIND_SAD(64x16); BIND_SAD(32x64); BIND_SAD(32x32);
    BIND_SAD(32x16); BIND_SAD(32x8); BIND_SAD(16x64); BIND_SAD(16x32); BIND_SAD(16x16); BIND_SAD(16x8); BIND_SAD(16x4); BIND_SAD(8x32);
    BIND_SAD(8x16); BIND_SAD(8x8); BIND_SAD(8x4); BIND_SAD(4x16); BIND_SAD(4x8); BIND_SAD(4x4);
    GROUP(2u);
    /* K4: Hadamard / SATD (svt_aom_hadamard_4x4 is a #define to the C function in the reference, not a pointer) */
    BIND(svt_aom_hadamard_8x8, svt_b200_aom_hadamard_8x8);
    BIND(svt_aom_hadamard_16x16, svt_b200_aom_hadamard_16x16);
    BIND(svt_aom_hadamard_32x32, svt_b200_aom_hadamard_32x32);
    BIND(svt_aom_satd, svt_b200_aom_satd);
    BIND(hadamard_path, b200_hadamard_path);
    GROUP(4u);
    /* K5 / K6: forward (full, N2, N4) and inverse transforms, 19 sizes */
    BIND_FWD(4x4); BIND_FWD(8x8); BIND_FWD(16x16); BIND_FWD(32x32); BIND_FWD(64x64); BIND_FWD(4x8); BIND_FWD(8x4); BIND_FWD(8x16);
    BIND_FWD(16x8); BIND_FWD(16x32); BIND_FWD(32x16); BIND_FWD(32x64); BIND_FWD(64x32); BIND_FWD(4x16); BIND_FWD(16x4); BIND_FWD(8x32);
    BIND_FWD(32x8); BIND_FWD(16x64); BIND_FWD(64x16);
    BIND_HANDLE(16x64); BIND_HANDLE(32x64); BIND_HANDLE(64x16); BIND_HANDLE(64x32); BIND_HANDLE(64x64);
    GROUP(8u);
    BIND(svt_av1_inv_txfm_add, b200_av1_inv_txfm_add);
    GROUP(4u);
    BIND(svt_av1_fwht4x4, svt_b200_av1_fwht4x4);
    GROUP(16u);
    /* K7: quantizers */
    BIND(svt_aom_quantize_b, svt_b200_aom_quantize_b);
    BIND(svt_aom_highbd_quantize_b, svt_b200_aom_highbd_quantize_b);
    BIND(svt_av1_quantize_b_qm, svt_b200_av1_quantize_b_qm);
    BIND(svt_av1_highbd_quantize_b_qm, svt_b200_av1_highbd_quantize_b_qm);
    BIND(svt_av1_quantize_fp, svt_b200_av1_quantize_fp);
    BIND(svt_av1_quantize_fp_32x32, svt_b200_av1_quantize_fp_32x32);
    BIND(svt_av1_quantize_fp_64x64, svt_b200_av1_quantize_fp_64x64);
    BIND(svt_av1_quantize_fp_qm, svt_b200_av1_quantize_fp_qm);
    BIND(svt_av1_highbd_quantize_fp, svt_b200_av1_highbd_quantize_fp);
    BIND(svt_av1_highbd_quantize_fp_qm, svt_b200_av1_highbd_quantize_fp_qm);
    BIND(svt_av1_compute_cul_level, svt_b200_av1_compute_cul_level);
    GROUP(32u);
    /* K8: CDEF */
    BIND(svt_aom_cdef_find_dir, svt_b200_aom_cdef_find_dir);
    BIND(svt_aom_cdef_find_dir_dual, svt_b200_aom_cdef_find_dir_dual);
    BIND(svt_cdef_filter_block, svt_b200_cdef_filter_block);
    BIND(svt_aom_copy_rect8_8bit_to_16bit, svt_b200_aom_copy_rect8_8bit_to_16bit);
    BIND(svt_compute_cdef_dist_16bit, b200_cdef_dist_16bit);
    BIND(svt_compute_cdef_dist_8bit, b200_cdef_dist_8bit);
    BIND(svt_search_one_dual, svt_b200_search_one_dual);
    GROUP(64u);
    /* K9 / K11: Wiener filter + statistics */
    BIND(svt_av1_wiener_convolve_add_src, b200_wiener_convolve_add_src);
    BIND(svt_av1_highbd_wiener_convolve_add_src, b200_highbd_wiener_convolve_add_src);
    BIND(svt_av1_compute_stats, svt_b200_av1_compute_stats);
    BIND(svt_av1_compute_stats_highbd, b200_compute_stats_highbd);
    GROUP(128u);
    /* K10 / K12: self-guided restoration */
    BIND(svt_av1_selfguided_restoration, b200_selfguided_restoration);
    BIND(svt_apply_selfguided_restoration, b200_apply_selfguided_restoration);
    BIND(svt_av1_lowbd_pixel_proj_error, b200_lowbd_pixel_proj_error);
    BIND(svt_av1_highbd_pixel_proj_error, b200_highbd_pixel_proj_error);
    BIND(svt_get_proj_subspace, b200_get_proj_subspace);
    return SVT_B200_OK;
}

void svt_b200_setup_rtcd_then_install(uint64_t flags) {
    svt_aom_setup_rtcd_internal((EbCpuFlags)flags);
    const char* dev = getenv("SVT_B200_DEVICE");
    if ((flags & EB_CPU_FLAGS_B200) || (dev && *dev)) {
        const int rc = svt_b200_install_rtcd(dev && *dev ? atoi(dev) : 0);
        if (rc != 0) { /* no CPU fallback: an encoder asked to run on the H100 tier must not silently run on the host */
            fprintf(stderr, "[svt_b200] FATAL: svt_b200_install_rtcd failed (%d): an sm_90 device is required\n", rc);
            abort();
        }
    }
}
