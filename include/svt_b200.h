/*
 * svt_b200.h -- C ABI of libsvtav1_b200.so: the H100 (sm_90a) tier of SVT-AV1-PSY's inner-loop DSP.
 *
 * Two layers (SURVEY.md F12):
 *
 *  T1  "pointer" entry points.  Same argument list, argument meaning and output contract as the
 *      reference's run-time dispatched function pointers (declared RTCD_EXTERN in
 *      Source/Lib/Codec/aom_dsp_rtcd.h and common_dsp_rtcd.h, bound in
 *      svt_aom_setup_rtcd_internal, aom_dsp_rtcd.c:188, and svt_aom_setup_common_rtcd_internal,
 *      common_dsp_rtcd.c:466).  Every pointer argument is caller-owned HOST memory; outputs are
 *      fully written on return; the functions are re-entrant and thread safe.  A reference build
 *      installs them by assigning   svt_sad_loop_kernel = svt_b200_sad_loop_kernel;   etc. right
 *      after the two stock rtcd calls (Source/Lib/Globals/enc_handle.c:1444-1445); see
 *      INTEGRATION.md.  They are the parity surface.
 *
 *  T2  batch entry points (new): one call carries a whole picture / segment worth of work items.
 *      "_host" variants take host buffers (copies are part of the call); "_dev" variants take
 *      device pointers + a CUDA stream (passed as void*) and only enqueue work.
 *
 * No CPU fallback exists: svt_b200_init() fails unless an sm_90 device is present and every other
 * entry point aborts if it has not succeeded.
 *
 * Types are plain C (stdint); no CUDA or torch types appear in any signature.
 */
#ifndef SVT_B200_H
#define SVT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SVT_B200_API __attribute__((visibility("default")))
#else
#define SVT_B200_API
#endif

/* ------------------------------------------------------------------------------------------ */
/* lifecycle                                                                                  */
/* ------------------------------------------------------------------------------------------ */
enum {
    SVT_B200_OK               = 0,
    SVT_B200_ERR_NO_DEVICE    = -1, /* maps to EB_ErrorInsufficientResources at svt_av1_enc_init time */
    SVT_B200_ERR_BAD_ARCH     = -2, /* device is not sm_90 */
    SVT_B200_ERR_ALREADY_INIT = -3,
    SVT_B200_ERR_BAD_ARG      = -4
};

/* Bind the library to CUDA device `device` (<0: device 0).  Replaces the CPU-flag probing of
 * svt_aom_get_cpu_flags_to_use (Source/Lib/Codec/common_dsp_rtcd.c:97). */
SVT_B200_API int                svt_b200_init(int device);
SVT_B200_API void               svt_b200_shutdown(void);
SVT_B200_API int                svt_b200_sm_count(void);
SVT_B200_API unsigned long long svt_b200_launch_count(void); /* kernels launched so far by this library */
SVT_B200_API const char*        svt_b200_version(void);
/* Asynchronous copies on a caller stream -- the host-buffer half of a T2 call (kind 0: pinned host -> device, 1: device ->
 * pinned host, 2: device -> device).  The caller keeps the buffers alive until the stream has passed the copy. */
SVT_B200_API int svt_b200_copy_async(void* dst, const void* src, size_t bytes, int kind, void* stream);
SVT_B200_API int svt_b200_copy2d_async(void* dst, size_t dst_pitch, const void* src, size_t src_pitch, size_t width_bytes, size_t rows,
                                       int kind, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* K1/K3  SAD search + single SADs  (reference: Source/Lib/C_DEFAULT/compute_sad_c.c)           */
/* ------------------------------------------------------------------------------------------ */

/* T1: svt_sad_loop_kernel (aom_dsp_rtcd.h:779; C: compute_sad_c.c:58-101).  Full search of a
 * block_width x block_height 8-bit block over search_area_width x search_area_height positions;
 * first minimum in raster order wins (strict '<', best initialised to 0xffffff);
 * x/y_search_center are left untouched when nothing beats 0xffffff. */
SVT_B200_API void svt_b200_sad_loop_kernel(uint8_t* src, uint32_t src_stride, uint8_t* ref, uint32_t ref_stride,
                                           uint32_t block_height, uint32_t block_width, uint64_t* best_sad,
                                           int16_t* x_search_center, int16_t* y_search_center,
                                           uint32_t src_stride_raw, uint8_t skip_search_line,
                                           int16_t search_area_width, int16_t search_area_height);

/* T1: svt_nxm_sad_kernel (aom_dsp_rtcd.h:856; C: svt_nxm_sad_kernel_helper_c / compute_sad_c.c:20-37). */
SVT_B200_API uint32_t svt_b200_nxm_sad_kernel(const uint8_t* src, uint32_t src_stride, const uint8_t* ref,
                                              uint32_t ref_stride, uint32_t height, uint32_t width);

/* T1: svt_aom_sadMxN and svt_aom_sadMxNx4d (aom_dsp_rtcd.h:275-403; C: compute_sad_c.c:104-215): the single-block
 * SADs of mode decision, M = width, N = height; x4d = the same source block against four references. */
#define SVT_B200_DECL_SAD(M, N)                                                                                      \
    SVT_B200_API uint32_t svt_b200_aom_sad##M##x##N(const uint8_t* src, int src_stride, const uint8_t* ref, int ref_stride); \
    SVT_B200_API void svt_b200_aom_sad##M##x##N##x4d(const uint8_t* src, int src_stride, const uint8_t* const ref_array[], \
                                                     int ref_stride, uint32_t* sad_array);
SVT_B200_DECL_SAD(128, 128) SVT_B200_DECL_SAD(128, 64) SVT_B200_DECL_SAD(64, 128) SVT_B200_DECL_SAD(64, 64) SVT_B200_DECL_SAD(64, 32) SVT_B200_DECL_SAD(64, 16) SVT_B200_DECL_SAD(32, 64) SVT_B200_DECL_SAD(32, 32)
SVT_B200_DECL_SAD(32, 16) SVT_B200_DECL_SAD(32, 8) SVT_B200_DECL_SAD(16, 64) SVT_B200_DECL_SAD(16, 32) SVT_B200_DECL_SAD(16, 16) SVT_B200_DECL_SAD(16, 8) SVT_B200_DECL_SAD(16, 4) SVT_B200_DECL_SAD(8, 32)
SVT_B200_DECL_SAD(8, 16) SVT_B200_DECL_SAD(8, 8) SVT_B200_DECL_SAD(8, 4) SVT_B200_DECL_SAD(4, 16) SVT_B200_DECL_SAD(4, 8) SVT_B200_DECL_SAD(4, 4)
#undef SVT_B200_DECL_SAD

/* T2 work item: one full search.  Offsets are in bytes from the plane base pointers given to the
 * batch call.  src_stride/ref_stride are the row pitches used for BLOCK rows (2x the plane pitch in
 * SUB_SAD mode, motion_estimation.c:463-481); ref_step is the pitch between SEARCH rows (the
 * reference's `src_stride_raw`). */
typedef struct SvtB200SadSearchItem {
    uint64_t src_off;
    uint64_t ref_off;
    uint32_t src_stride;
    uint32_t ref_stride;
    uint32_t ref_step;
    uint16_t block_w;
    uint16_t block_h;
    int16_t  sa_w;
    int16_t  sa_h;
    uint16_t skip_search_line;
    uint16_t reserved;
} SvtB200SadSearchItem;

typedef struct SvtB200SadSearchResult {
    uint32_t best_sad; /* 0xffffff when no position was evaluated */
    int16_t  x;        /* search-area-relative, -1 when none       */
    int16_t  y;
} SvtB200SadSearchResult;

SVT_B200_API int svt_b200_sad_search_batch_host(const uint8_t* src_plane, size_t src_bytes, const uint8_t* ref_plane,
                                                size_t ref_bytes, const SvtB200SadSearchItem* items, int n_items,
                                                SvtB200SadSearchResult* results);
/* device-resident planes/items/results; `max_*` bound the items' geometry (for shared-memory sizing) */
SVT_B200_API int svt_b200_sad_search_batch_dev(const uint8_t* d_src_plane, const uint8_t* d_ref_plane,
                                               const SvtB200SadSearchItem* d_items, int n_items,
                                               SvtB200SadSearchResult* d_results, int max_block_w, int max_block_h,
                                               int max_sa_w, int max_sa_h, int max_row_mult, void* stream);


/* ------------------------------------------------------------------------------------------ */
/* K5/K6  2-D transforms  (reference: Source/Lib/Codec/transforms.c, inv_transforms.c)          */
/* ------------------------------------------------------------------------------------------ */
/* tx_size / tx_type use the reference's TxSize / TxType enumerators (Source/Lib/Codec/definitions.h):
 * TX_4X4=0, 8X8, 16X16, 32X32, 64X64, 4X8, 8X4, 8X16, 16X8, 16X32, 32X16, 32X64, 64X32, 4X16, 16X4,
 * 8X32, 32X8, 16X64, 64X16=18;  DCT_DCT=0, ADST_DCT, DCT_ADST, ADST_ADST, FLIPADST_DCT, DCT_FLIPADST,
 * FLIPADST_FLIPADST, ADST_FLIPADST, FLIPADST_ADST, IDTX, V_DCT, H_DCT, V_ADST, H_ADST, V_FLIPADST,
 * H_FLIPADST=15. */
SVT_B200_API int svt_b200_txfm_valid(int tx_size, int tx_type);

/* T1 generic forms.  svt_av1_fwd_txfm2d_WxH (aom_dsp_rtcd.h:121-197; C: av1_tranform_two_d_core_c,
 * transforms.c:2259) and svt_av1_inv_txfm2d_add_WxH (common_dsp_rtcd.h:106-142; C: inv_txfm2d_add_c,
 * inv_transforms.c:2459).  Output of the forward transform is W*H int32, row-major, stride W.
 * Input of the inverse is min(W,32) x min(H,32) packed coefficients (inv_transforms.c:2567-2686). */
SVT_B200_API void svt_b200_fwd_txfm2d(int16_t* input, int32_t* output, uint32_t input_stride, int tx_type,
                                      int tx_size, uint8_t bit_depth);
/* level 0 = full, 1 = N2, 2 = N4 (see the _N2 / _N4 named forms below) */
SVT_B200_API void svt_b200_fwd_txfm2d_partial(int16_t* input, int32_t* output, uint32_t input_stride, int tx_type,
                                              int tx_size, uint8_t bit_depth, int level);
SVT_B200_API void svt_b200_inv_txfm2d_add(const int32_t* input, uint16_t* output_r, int32_t stride_r,
                                          uint16_t* output_w, int32_t stride_w, int tx_type, int tx_size, int32_t bd);
/* svt_av1_inv_txfm_add (common_dsp_rtcd.h:144; C: inv_transforms.c:3177): 8-bit pixels. */
SVT_B200_API void svt_b200_inv_txfm_add_8bit(const int32_t* dqcoeff, uint8_t* dst_r, int32_t stride_r, uint8_t* dst_w,
                                             int32_t stride_w, int tx_type, int tx_size);

/* T1 named forms, one per reference pointer, identical argument lists.  TxType / TxSize / BlockSize are
 * ATTRIBUTE_PACKED one-byte enums in the reference (Source/Lib/Codec/definitions.h:849-878,972-995): they are
 * uint8_t here, so the prototypes are assignment-compatible with the rtcd pointers without casts. */
#define SVT_B200_DECL_FWD(WxH)                                                                              \
    SVT_B200_API void svt_b200_av1_fwd_txfm2d_##WxH(int16_t* input, int32_t* output, uint32_t input_stride, \
                                                    uint8_t transform_type /* TxType: 1-byte packed enum */, uint8_t bit_depth);
SVT_B200_DECL_FWD(4x4) SVT_B200_DECL_FWD(8x8) SVT_B200_DECL_FWD(16x16) SVT_B200_DECL_FWD(32x32) SVT_B200_DECL_FWD(64x64)
SVT_B200_DECL_FWD(4x8) SVT_B200_DECL_FWD(8x4) SVT_B200_DECL_FWD(8x16) SVT_B200_DECL_FWD(16x8) SVT_B200_DECL_FWD(16x32)
SVT_B200_DECL_FWD(32x16) SVT_B200_DECL_FWD(32x64) SVT_B200_DECL_FWD(64x32) SVT_B200_DECL_FWD(4x16) SVT_B200_DECL_FWD(16x4)
SVT_B200_DECL_FWD(8x32) SVT_B200_DECL_FWD(32x8) SVT_B200_DECL_FWD(16x64) SVT_B200_DECL_FWD(64x16)
/* svt_av1_fwd_txfm2d_WxH_N2 / _N4 (aom_dsp_rtcd.h:131-245; C: av1_tranform_two_d_core_N2_c / _N4_c,
 * transforms.c:5202, 6769): only the top-left (W/2 x H/2) / (W/4 x H/4) coefficients, the rest zero. */
SVT_B200_DECL_FWD(4x4_N2) SVT_B200_DECL_FWD(8x8_N2) SVT_B200_DECL_FWD(16x16_N2) SVT_B200_DECL_FWD(32x32_N2) SVT_B200_DECL_FWD(64x64_N2)
SVT_B200_DECL_FWD(4x8_N2) SVT_B200_DECL_FWD(8x4_N2) SVT_B200_DECL_FWD(8x16_N2) SVT_B200_DECL_FWD(16x8_N2) SVT_B200_DECL_FWD(16x32_N2)
SVT_B200_DECL_FWD(32x16_N2) SVT_B200_DECL_FWD(32x64_N2) SVT_B200_DECL_FWD(64x32_N2) SVT_B200_DECL_FWD(4x16_N2) SVT_B200_DECL_FWD(16x4_N2)
SVT_B200_DECL_FWD(8x32_N2) SVT_B200_DECL_FWD(32x8_N2) SVT_B200_DECL_FWD(16x64_N2) SVT_B200_DECL_FWD(64x16_N2)
SVT_B200_DECL_FWD(4x4_N4) SVT_B200_DECL_FWD(8x8_N4) SVT_B200_DECL_FWD(16x16_N4) SVT_B200_DECL_FWD(32x32_N4) SVT_B200_DECL_FWD(64x64_N4)
SVT_B200_DECL_FWD(4x8_N4) SVT_B200_DECL_FWD(8x4_N4) SVT_B200_DECL_FWD(8x16_N4) SVT_B200_DECL_FWD(16x8_N4) SVT_B200_DECL_FWD(16x32_N4)
SVT_B200_DECL_FWD(32x16_N4) SVT_B200_DECL_FWD(32x64_N4) SVT_B200_DECL_FWD(64x32_N4) SVT_B200_DECL_FWD(4x16_N4) SVT_B200_DECL_FWD(16x4_N4)
SVT_B200_DECL_FWD(8x32_N4) SVT_B200_DECL_FWD(32x8_N4) SVT_B200_DECL_FWD(16x64_N4) SVT_B200_DECL_FWD(64x16_N4)
#undef SVT_B200_DECL_FWD
#define SVT_B200_DECL_INV_A(WxH)                                                                                \
    SVT_B200_API void svt_b200_av1_inv_txfm2d_add_##WxH(const int32_t* input, uint16_t* output_r, int32_t stride_r, \
                                                        uint16_t* output_w, int32_t stride_w, uint8_t tx_type, int32_t bd);
#define SVT_B200_DECL_INV_B(WxH)                                                                                \
    SVT_B200_API void svt_b200_av1_inv_txfm2d_add_##WxH(const int32_t* input, uint16_t* output_r, int32_t stride_r, \
                                                        uint16_t* output_w, int32_t stride_w, uint8_t tx_type,   \
                                                        uint8_t tx_size, int32_t bd);
#define SVT_B200_DECL_INV_C(WxH)                                                                                \
    SVT_B200_API void svt_b200_av1_inv_txfm2d_add_##WxH(const int32_t* input, uint16_t* output_r, int32_t stride_r, \
                                                        uint16_t* output_w, int32_t stride_w, uint8_t tx_type,   \
                                                        uint8_t tx_size, int32_t eob, int32_t bd);
SVT_B200_DECL_INV_A(4x4) SVT_B200_DECL_INV_A(8x8) SVT_B200_DECL_INV_A(16x16) SVT_B200_DECL_INV_A(32x32) SVT_B200_DECL_INV_A(64x64)
SVT_B200_DECL_INV_B(4x8) SVT_B200_DECL_INV_B(8x4) SVT_B200_DECL_INV_B(4x16) SVT_B200_DECL_INV_B(16x4)
SVT_B200_DECL_INV_C(8x16) SVT_B200_DECL_INV_C(16x8) SVT_B200_DECL_INV_C(16x32) SVT_B200_DECL_INV_C(32x16) SVT_B200_DECL_INV_C(32x8)
SVT_B200_DECL_INV_C(8x32) SVT_B200_DECL_INV_C(32x64) SVT_B200_DECL_INV_C(64x32) SVT_B200_DECL_INV_C(16x64) SVT_B200_DECL_INV_C(64x16)
#undef SVT_B200_DECL_INV_A
#undef SVT_B200_DECL_INV_B
#undef SVT_B200_DECL_INV_C

/* T2 work items.  Offsets are in ELEMENTS of the respective plane (int16 residual, int32 coeff,
 * pixels). */
typedef struct SvtB200FwdTxfmItem {
    uint64_t src_off;    /* residual block origin */
    uint64_t dst_off;    /* W*H contiguous int32 */
    uint32_t src_stride;
    uint8_t  tx_size;
    uint8_t  tx_type;
    uint16_t reserved;   /* bits 1-2: 1 = N2, 2 = N4 partial transform (coefficients outside the top-left half /
                            quarter of each dimension are written as zero);
                            bit 0: packed output -- only the top-left min(W,32) x min(H,32) coefficients are
                            written, at stride min(W,32) (the re-pack half of svt_handle_transform64x64 etc.,
                            transforms.c:2374-2542); dst must then hold min(W,32)*min(H,32) int32 */
} SvtB200FwdTxfmItem;

typedef struct SvtB200InvTxfmItem {
    uint64_t coef_off;   /* min(W,32)*min(H,32) packed int32 */
    uint64_t pred_off;   /* prediction read  (output_r) */
    uint64_t recon_off;  /* reconstruction written (output_w) */
    uint32_t pred_stride;
    uint32_t recon_stride;
    uint8_t  tx_size;
    uint8_t  tx_type;
    uint8_t  bd;
    uint8_t  reserved;
    uint32_t reserved2;
} SvtB200InvTxfmItem;

/* T1: svt_handle_transform{16x64,32x64,64x16,64x32,64x64}{,_N2_N4} (aom_dsp_rtcd.h:216-240; C: transforms.c:2374-2543):
 * returns the energy of the coefficients outside the kept top-left min(W,32) x min(H,32) and re-packs the
 * kept rows of a 64-wide block to stride 32, in place. */
#define SVT_B200_DECL_HANDLE(WxH)                                         \
    SVT_B200_API uint64_t svt_b200_handle_transform##WxH(int32_t* output); \
    SVT_B200_API uint64_t svt_b200_handle_transform##WxH##_N2_N4(int32_t* output);
SVT_B200_DECL_HANDLE(16x64) SVT_B200_DECL_HANDLE(32x64) SVT_B200_DECL_HANDLE(64x16) SVT_B200_DECL_HANDLE(64x32) SVT_B200_DECL_HANDLE(64x64)
#undef SVT_B200_DECL_HANDLE

/* A transform block is processed by a team of threads chosen by its "team class",
 * log2(max(W,H)) - 2 (0: 4x4 .. 4: the 64-point sizes).  Items must be ordered by class: the
 * n_per_class[0] class-0 items first, then class 1, ...; within a class, keeping equal (tx_size,
 * tx_type) together lets the teams that share a warp run in lock step. */
#define SVT_B200_TXFM_CLASSES 5
SVT_B200_API int svt_b200_txfm_team_class(int tx_size);
SVT_B200_API int svt_b200_fwd_txfm_batch_dev(const int16_t* d_residual, int32_t* d_coeff,
                                             const SvtB200FwdTxfmItem* d_items,
                                             const int n_per_class[SVT_B200_TXFM_CLASSES], void* stream);
SVT_B200_API int svt_b200_inv_txfm_batch_dev(const int32_t* d_coeff, const void* d_pred, void* d_recon,
                                             const SvtB200InvTxfmItem* d_items,
                                             const int n_per_class[SVT_B200_TXFM_CLASSES], int pixel_bytes,
                                             void* stream);
/* any order; the library groups the items itself */
SVT_B200_API int svt_b200_fwd_txfm_batch_host(const int16_t* residual, size_t residual_elems, int32_t* coeff,
                                              size_t coeff_elems, const SvtB200FwdTxfmItem* items, int n_items);

/* ------------------------------------------------------------------------------------------ */
/* K7  quantize / dequantize  (reference: Source/Lib/Codec/full_loop.c:29-516)                  */
/* ------------------------------------------------------------------------------------------ */
/* T1: identical argument lists to svt_aom_quantize_b / svt_aom_highbd_quantize_b /
 * svt_av1_quantize_b_qm / svt_av1_highbd_quantize_b_qm / svt_av1_quantize_fp{,_32x32,_64x64,_qm} /
 * svt_av1_highbd_quantize_fp{,_qm} (aom_dsp_rtcd.h:247-263).  TranLow = int32_t, QmVal = uint8_t. */
#define SVT_B200_QARGS                                                                                         \
    const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr, const int16_t *round_ptr,            \
        const int16_t *quant_ptr, const int16_t *quant_shift_ptr, int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr,   \
        const int16_t *dequant_ptr, uint16_t *eob_ptr, const int16_t *scan, const int16_t *iscan
SVT_B200_API void svt_b200_aom_quantize_b(SVT_B200_QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale);
SVT_B200_API void svt_b200_aom_highbd_quantize_b(SVT_B200_QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale);
SVT_B200_API void svt_b200_av1_quantize_b_qm(SVT_B200_QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale);
SVT_B200_API void svt_b200_av1_highbd_quantize_b_qm(SVT_B200_QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale);
SVT_B200_API void svt_b200_av1_quantize_fp(SVT_B200_QARGS);
SVT_B200_API void svt_b200_av1_quantize_fp_32x32(SVT_B200_QARGS);
SVT_B200_API void svt_b200_av1_quantize_fp_64x64(SVT_B200_QARGS);
SVT_B200_API void svt_b200_av1_quantize_fp_qm(SVT_B200_QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int16_t log_scale);
SVT_B200_API void svt_b200_av1_highbd_quantize_fp(SVT_B200_QARGS, int16_t log_scale);
SVT_B200_API void svt_b200_av1_highbd_quantize_fp_qm(SVT_B200_QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int16_t log_scale);
#undef SVT_B200_QARGS

enum { SVT_B200_QUANT_B_LBD = 0, SVT_B200_QUANT_B_HBD = 1, SVT_B200_QUANT_FP_LBD = 2, SVT_B200_QUANT_FP_HBD = 3 };
#define SVT_B200_NO_QM 0xffffffffu

/* T2 work item: one coefficient block.  Offsets in elements of the respective base array. */
typedef struct SvtB200QuantItem {
    uint64_t coeff_off;
    uint64_t q_off;
    uint64_t dq_off;
    uint32_t scan_off;   /* into the int16 scan-table (and inverse-scan-table) buffer */
    uint32_t qm_off;     /* into the uint8 QM buffer, SVT_B200_NO_QM = no matrix */
    uint32_t iqm_off;
    uint32_t n_coeffs;
    int16_t  zbin[2], round[2], quant[2], quant_shift[2], dequant[2]; /* [0]=DC, [1]=AC (MacroblockPlane *_qtx) */
    uint8_t  mode;       /* SVT_B200_QUANT_* */
    uint8_t  log_scale;
    uint16_t reserved;
} SvtB200QuantItem;

/* d_scan / d_iscan: the scan tables and their inverses (the `scan` and `iscan` arguments of the reference
 * quantizers), same layout, addressed by SvtB200QuantItem.scan_off.  With d_iscan the blocks are walked in
 * raster order (coalesced); d_iscan == NULL falls back to scan order through d_scan. */
SVT_B200_API int svt_b200_quant_batch_dev(const int32_t* d_coeff, int32_t* d_qcoeff, int32_t* d_dqcoeff,
                                          const int16_t* d_scan, const int16_t* d_iscan, const uint8_t* d_qm,
                                          const SvtB200QuantItem* d_items, int n_items, uint16_t* d_eobs, void* stream);

/* Fused per-block chain of the final encode pass (coding_loop.c:405-658): forward transform -> quantise
 * -> inverse transform + reconstruction, one call, intermediates kept on chip.  Item = the three items
 * the separate calls take (fwd.dst_off, quant.coeff_off and inv.coef_off are ignored; the forward output
 * is always the packed min(W,32) x min(H,32) block).  Same ordering rule (team classes) as the transform
 * batches; d_eobs[i] belongs to item i; d_dqcoeff may be NULL.  Results are bit-identical to
 * svt_b200_fwd_txfm_batch_dev + svt_b200_quant_batch_dev + svt_b200_inv_txfm_batch_dev. */
typedef struct SvtB200TrioItem {
    SvtB200FwdTxfmItem fwd;
    SvtB200QuantItem   quant;
    SvtB200InvTxfmItem inv;
} SvtB200TrioItem;
SVT_B200_API int svt_b200_txfm_trio_batch_dev(const int16_t* d_residual, const void* d_pred, void* d_recon, int32_t* d_qcoeff,
                                              int32_t* d_dqcoeff, const int16_t* d_iscan, const uint8_t* d_qm,
                                              const SvtB200TrioItem* d_items, const int n_per_class[SVT_B200_TXFM_CLASSES],
                                              uint16_t* d_eobs, int pixel_bytes, void* stream);

/* The same chain with the residual formed on the fly: residual = source - prediction (svt_aom_residual_kernel,
 * pic_operators.c; rtcd svt_residual_kernel8bit / svt_residual_kernel16bit) for the block at fwd.src_off / fwd.src_stride
 * of the SOURCE picture plane and inv.pred_off / inv.pred_stride of the prediction; no int16 residual plane exists. */
SVT_B200_API int svt_b200_residual_txfm_trio_batch_dev(const void* d_source, const void* d_pred, void* d_recon, int32_t* d_qcoeff,
                                                       int32_t* d_dqcoeff, const int16_t* d_iscan, const uint8_t* d_qm,
                                                       const SvtB200TrioItem* d_items, const int n_per_class[SVT_B200_TXFM_CLASSES],
                                                       uint16_t* d_eobs, int pixel_bytes, void* stream);

/* T2: svt_aom_residual_kernel over up to 3 planes in one launch (offsets / strides in elements). */
typedef struct SvtB200ResidualPlane {
    uint64_t src_off, pred_off, res_off;
    int32_t  src_stride, pred_stride, res_stride;
    int32_t  w, h;
    int32_t  reserved;
} SvtB200ResidualPlane;
typedef struct SvtB200ResidualPlanes { SvtB200ResidualPlane p[3]; } SvtB200ResidualPlanes;
SVT_B200_API int svt_b200_residual_planes_dev(const void* d_source, const void* d_pred, int16_t* d_residual,
                                              const SvtB200ResidualPlanes* planes, int n_planes, int pixel_bytes, void* stream);

/* T2: eob-bounded scan-order packing of a batch's quantised levels -- what the entropy coder consumes.  d_offsets[i]
 * (n_items + 2 entries: exclusive prefix sum of d_eobs; d_offsets[n_items] = total; d_offsets[n_items + 1] = number of
 * levels that did not fit level_bytes) locates block i's first level in d_levels; block i contributes d_eobs[i] levels,
 * qcoeff[scan[0..eob)] of its coefficient block.  level_bytes = 2 (int16: the levels of 8-bit pictures fit, as the
 * reference's 16-bit-lane low-bit-depth quantizers rely on) or 4 (int32, high bit depth).  Levels beyond `capacity` are
 * dropped (the caller sees total > capacity and re-issues with a larger buffer).  d_iscan is the INVERSE scan table
 * (the `iscan` argument of the reference quantizers) addressed by quant.scan_off: blocks are read in raster order. */
SVT_B200_API int svt_b200_pack_levels_dev(const int32_t* d_qcoeff, const int16_t* d_iscan, const SvtB200TrioItem* d_items,
                                          const uint16_t* d_eobs, int n_items, uint32_t* d_offsets, void* d_levels,
                                          int level_bytes, uint32_t capacity, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* K4  Hadamard / SATD  (reference: Source/Lib/C_DEFAULT/picture_operators_c.c:188-330)        */
/* ------------------------------------------------------------------------------------------ */
/* T1: svt_aom_hadamard_{4x4,8x8,16x16,32x32} (common_dsp_rtcd.h:1075-1083), svt_aom_satd (:210). */
SVT_B200_API void svt_b200_aom_hadamard_4x4(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff);
SVT_B200_API void svt_b200_aom_hadamard_8x8(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff);
SVT_B200_API void svt_b200_aom_hadamard_16x16(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff);
SVT_B200_API void svt_b200_aom_hadamard_32x32(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff);
SVT_B200_API int  svt_b200_aom_satd(const int32_t* coeff, int length);
/* T1: hadamard_path (aom_dsp_rtcd.h:582; C: enc_mode_config.c:2147-2212): SATD cost of a prediction block, transform block by
 * transform block (8-bit input / prediction).  SvtB200Buf2D has the layout of the reference's Buf2D (definitions.h:243-249);
 * `bsize` is the reference's 1-byte BlockSize.  Like the reference's loop, the call leaves the last transform block's residual
 * (int16, residual.stride) in residual.buf and its coefficients in coeff.buf. */
typedef struct SvtB200Buf2D { uint8_t* buf; uint8_t* buf0; int width; int height; int stride; } SvtB200Buf2D;
SVT_B200_API uint32_t svt_b200_hadamard_path(SvtB200Buf2D residual, SvtB200Buf2D coeff, SvtB200Buf2D input, SvtB200Buf2D pred, uint8_t bsize);
/* T1: svt_av1_fwht4x4 (aom_dsp_rtcd.h:208; C: transforms.c:3099): the Walsh-Hadamard transform of lossless 4x4 blocks */
SVT_B200_API void svt_b200_av1_fwht4x4(int16_t* input, int32_t* output, uint32_t stride);
/* T1: svt_av1_compute_cul_level (aom_dsp_rtcd.h:904; C: full_loop.c:1449) */
SVT_B200_API uint8_t svt_b200_av1_compute_cul_level(const int16_t* const scan, const int32_t* const quant_coeff, uint16_t* eob);

typedef struct SvtB200HadamardItem {
    uint64_t src_off;    /* int16 residual elements */
    uint64_t coeff_off;  /* int32 elements (ignored when no coefficient plane is given) */
    uint32_t src_stride;
    uint32_t size;       /* 4, 8, 16 or 32 */
} SvtB200HadamardItem;
/* T2: fused Hadamard + sum|coeff| per item; d_coeff_or_null may be NULL (SATD only).  An item whose size is not
 * 4, 8, 16 or 32 gets d_satd[i] = -1 and writes no coefficients. */
SVT_B200_API int svt_b200_hadamard_satd_batch_dev(const int16_t* d_residual, const SvtB200HadamardItem* d_items,
                                                  int n_items, int32_t* d_coeff_or_null, int32_t* d_satd, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* K2  SAD pyramid + full-pel search  (reference: Source/Lib/Codec/motion_estimation.c:98-817) */
/* ------------------------------------------------------------------------------------------ */
/* T1: identical argument lists to aom_dsp_rtcd.h:842-855 (bool passed as uint8_t). */
SVT_B200_API void svt_b200_ext_all_sad_calculation_8x8_16x16(uint8_t* src, uint32_t src_stride, uint8_t* ref,
                                                             uint32_t ref_stride, uint32_t mv, uint32_t* p_best_sad_8x8,
                                                             uint32_t* p_best_sad_16x16, uint32_t* p_best_mv8x8,
                                                             uint32_t* p_best_mv16x16, uint32_t p_eight_sad16x16[16][8],
                                                             uint32_t p_eight_sad8x8[64][8], uint8_t sub_sad);
SVT_B200_API void svt_b200_ext_eight_sad_calculation_32x32_64x64(uint32_t p_sad16x16[16][8], uint32_t* p_best_sad_32x32,
                                                                 uint32_t* p_best_sad_64x64, uint32_t* p_best_mv32x32,
                                                                 uint32_t* p_best_mv64x64, uint32_t mv,
                                                                 uint32_t p_sad32x32[4][8]);
SVT_B200_API void svt_b200_ext_sad_calculation_8x8_16x16(uint8_t* src, uint32_t src_stride, uint8_t* ref,
                                                         uint32_t ref_stride, uint32_t* p_best_sad_8x8,
                                                         uint32_t* p_best_sad_16x16, uint32_t* p_best_mv8x8,
                                                         uint32_t* p_best_mv16x16, uint32_t mv, uint32_t* p_sad16x16,
                                                         uint32_t* p_sad8x8, uint8_t sub_sad);
SVT_B200_API void svt_b200_ext_sad_calculation_32x32_64x64(uint32_t* p_sad16x16, uint32_t* p_best_sad_32x32,
                                                           uint32_t* p_best_sad_64x64, uint32_t* p_best_mv32x32,
                                                           uint32_t* p_best_mv64x64, uint32_t mv, uint32_t* p_sad32x32);
SVT_B200_API void svt_b200_initialize_buffer_32bits(uint32_t* pointer, uint32_t count128, uint32_t count32, uint32_t value);

/* T2: open_loop_me_fullpel_search_sblock (motion_estimation.c:781) for one 64x64 block and one
 * reference: all sa_w x sa_h integer positions, best SAD + MV for the 85 square PUs
 * (me_context.h:54-75 order).  MV = ((org_y + y) << 16) | ((org_x + x) & 0xffff). */
typedef struct SvtB200FullpelItem {
    uint64_t src_off;    /* 64x64 source block origin (bytes) */
    uint64_t ref_off;    /* reference sample of search position (0,0) (bytes) */
    uint32_t src_stride;
    uint32_t ref_stride;
    int16_t  sa_w, sa_h;
    int16_t  org_x, org_y; /* x/y_search_area_origin */
    uint8_t  sub_sad;      /* me_search_method == SUB_SAD_SEARCH */
    uint8_t  seeded;       /* 1: the best arrays start from the SADs of one probe position (d_seed_sad of the seeded call), which
                              wins ties -- integer_search_b64 evaluates the search centre first when the 8x8-variance control is
                              on and does not reset p_sb_best_sad afterwards (motion_estimation.c:1358-1412) */
    int16_t  seed_x, seed_y; /* MV of the probe position */
    uint8_t  reserved[2];
} SvtB200FullpelItem;
SVT_B200_API int svt_b200_fullpel_search_batch_dev(const uint8_t* d_src_plane, const uint8_t* d_ref_plane,
                                                   const SvtB200FullpelItem* d_items, int n_items, uint32_t* d_best_sad,
                                                   uint32_t* d_best_mv, void* stream);
SVT_B200_API int svt_b200_fullpel_search_batch_host(const uint8_t* src_plane, size_t src_bytes, const uint8_t* ref_plane,
                                                    size_t ref_bytes, const SvtB200FullpelItem* items, int n_items,
                                                    uint32_t* best_sad, uint32_t* best_mv);

/* ------------------------------------------------------------------------------------------ */
/* K8  CDEF  (reference: Source/Lib/Codec/cdef.c, enc_cdef.c, cdef_process.c)                   */
/* ------------------------------------------------------------------------------------------ */
typedef struct SvtB200CdefList { uint8_t by, bx; } SvtB200CdefList; /* == CdefList, definitions.h:256-259 */

/* T1: common_dsp_rtcd.h:1015-1029, aom_dsp_rtcd.h:62-64,242.  `bsize` is the reference BlockSize
 * enumerator (BLOCK_4X4=0, BLOCK_4X8=1, BLOCK_8X4=2, BLOCK_8X8=3); `in` points into a tile of pitch
 * CDEF_BSTRIDE (144) with at least 2 valid rows/columns around the block. */
SVT_B200_API uint8_t  svt_b200_aom_cdef_find_dir(const uint16_t* img, int32_t stride, int32_t* var, int32_t coeff_shift);
SVT_B200_API void     svt_b200_aom_cdef_find_dir_dual(const uint16_t* img1, const uint16_t* img2, int stride, int32_t* var1,
                                                      int32_t* var2, int32_t coeff_shift, uint8_t* out1, uint8_t* out2);
SVT_B200_API void     svt_b200_cdef_filter_block(uint8_t* dst8, uint16_t* dst16, int32_t dstride, const uint16_t* in,
                                                 int32_t pri_strength, int32_t sec_strength, int32_t dir,
                                                 int32_t pri_damping, int32_t sec_damping, int32_t bsize,
                                                 int32_t coeff_shift, uint8_t subsampling_factor);
SVT_B200_API void     svt_b200_aom_copy_rect8_8bit_to_16bit(uint16_t* dst, int32_t dstride, const uint8_t* src,
                                                            int32_t sstride, int32_t v, int32_t h);
SVT_B200_API uint64_t svt_b200_compute_cdef_dist_16bit(const uint16_t* dst, int32_t dstride, const uint16_t* src,
                                                       const SvtB200CdefList* dlist, int32_t cdef_count, uint8_t bsize /* BlockSize */,
                                                       int32_t coeff_shift, int32_t pli, uint8_t subsampling_factor);
SVT_B200_API uint64_t svt_b200_compute_cdef_dist_8bit(const uint8_t* dst8, int32_t dstride, const uint8_t* src8,
                                                      const SvtB200CdefList* dlist, int32_t cdef_count, uint8_t bsize /* BlockSize */,
                                                      int32_t coeff_shift, int32_t pli, uint8_t subsampling_factor);
SVT_B200_API uint64_t svt_b200_search_one_dual(int* lev0, int* lev1, int nb_strengths, uint64_t** mse[2], int sb_count,
                                               int start_gi, int end_gi);

/* T2: whole-picture CDEF strength search (cdef_seg_search, cdef_process.c:106-352) and apply
 * (svt_av1_cdef_frame, enc_cdef.c:284).  4:2:0, width/height multiples of 8, all pointers DEVICE
 * memory pointing at the first visible pixel of each plane.  recon_* = deblocked reconstruction
 * (filter input), src_* = source picture.  Pixels are uint8 (bit_depth 8) or uint16.  Like the
 * reference, both calls read recon_cb / recon_cr rows up to 4 pixels past the chroma width when the last
 * filter block column is 8 luma pixels wide (the 8-pixel right border of its neighbour's tile): those
 * pixels never change the result, but they must be readable memory. */
typedef struct SvtB200CdefFrame {
    const void* recon_y; const void* recon_cb; const void* recon_cr;
    const void* src_y;   const void* src_cb;   const void* src_cr;
    int32_t recon_stride_y, recon_stride_c, src_stride_y, src_stride_c; /* in pixels */
    int32_t width, height;       /* luma */
    int32_t bit_depth;
    int32_t damping;             /* 3 + (base_q_idx >> 6) */
    int32_t subsampling_factor;  /* CdefSearchControls.subsampling_factor */
    int32_t reserved;
} SvtB200CdefFrame;
/* d_skip8x8: one byte per luma 8x8 (raster, (width/8) per row), non-zero = skip (not in the cdef
 * list).  strengths: candidate (pri*4+sec) codes per gi, -1 = not tested for chroma.
 * d_mse: [2][nfb][n_strengths] uint64 laid out like pcs->mse_seg; d_dir/d_var: [nfb][64]. */
SVT_B200_API int svt_b200_cdef_search_frame_dev(const SvtB200CdefFrame* frame, const uint8_t* d_skip8x8,
                                                const int* d_strengths_y, const int* d_strengths_uv, int n_strengths,
                                                uint64_t* d_mse, uint8_t* d_dir, int32_t* d_var, void* stream);
/* d_fb_strength_idx: per filter block index into the frame's strength tables (-1 = leave untouched);
 * output planes receive the filtered pixels of non-skip blocks only (copy the input first).
 * d_dir/d_var: the [nfb][64] arrays svt_b200_cdef_search_frame_dev wrote for this reconstruction (the
 * reference keeps them in pcs->cdef_dir_data between search and apply); both NULL = recompute. */
SVT_B200_API int svt_b200_cdef_apply_frame_dev(const SvtB200CdefFrame* frame, const uint8_t* d_skip8x8,
                                               const int8_t* d_fb_strength_idx, const int* d_y_strength,
                                               const int* d_uv_strength, const uint8_t* d_dir, const int32_t* d_var,
                                               void* d_out_y, void* d_out_cb, void* d_out_cr, int out_stride_y,
                                               int out_stride_c, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* K14  deblocking loop filter  (reference: deblocking_common.c:242-866, deblocking_filter.c:144-654) */
/* ------------------------------------------------------------------------------------------ */
/* T1: common_dsp_rtcd.h:1036-1067.  Each call filters 4 pixels along one edge at `s` (the first pixel on the q side):
 * _4 / _6 / _8 / _14 read 2 / 3 / 4 / 7 pixels on each side of the edge and write 2 / 2 / 3 / 6.  Only blimit[0],
 * limit[0] and thresh[0] are read.  High-bit-depth pixels are plain uint16_t*. */
#define SVT_B200_DECL_LPF(DIR, N)                                                                                          \
    SVT_B200_API void svt_b200_aom_lpf_##DIR##_##N(uint8_t* s, int32_t pitch, const uint8_t* blimit, const uint8_t* limit, \
                                                   const uint8_t* thresh);                                                 \
    SVT_B200_API void svt_b200_aom_highbd_lpf_##DIR##_##N(uint16_t* s, int32_t pitch, const uint8_t* blimit,               \
                                                          const uint8_t* limit, const uint8_t* thresh, int32_t bd);
SVT_B200_DECL_LPF(horizontal, 4) SVT_B200_DECL_LPF(horizontal, 6) SVT_B200_DECL_LPF(horizontal, 8) SVT_B200_DECL_LPF(horizontal, 14)
SVT_B200_DECL_LPF(vertical, 4) SVT_B200_DECL_LPF(vertical, 6) SVT_B200_DECL_LPF(vertical, 8) SVT_B200_DECL_LPF(vertical, 14)
#undef SVT_B200_DECL_LPF

/* One record per 4x4 luma position of the picture's mode-info grid (ModeInfo.mbmi.block_mi, block_structures.h:108):
 * the fields the edge derivation reads.  bsize = BlockSize, mode = PredictionMode, ref_frame0 = MvReferenceFrame
 * (0 = INTRA_FRAME, 1..7 = LAST..ALTREF). */
typedef struct SvtB200DlfMi {
    uint8_t bsize;
    uint8_t tx_depth;
    uint8_t skip;
    int8_t  ref_frame0;
    uint8_t mode;
    uint8_t segment_id;
    uint8_t reserved[2];
} SvtB200DlfMi;

/* The picture and the frame's loop-filter state.  Pixels are uint8 (pixel_bytes 1: the 8-bit filters) or uint16
 * (pixel_bytes 2: the high-bit-depth filters at bit_depth, 8 included).  4:2:0 only.  lvl and lfthr are the
 * LoopFilterInfoN (definitions.h:1913-1922) that svt_av1_loop_filter_frame_init derives from the frame header on the host;
 * lfthr[level] = {mblim, lim, hev_thr}. */
typedef struct SvtB200DlfFrame {
    void*   plane[3];       /* DEVICE pointers to pixel (0, 0) of Y, Cb, Cr */
    int32_t stride[3];      /* in pixels */
    int32_t width, height;  /* luma, unpadded: edges at x >= width (chroma: width >> 1) or y >= height are not filtered */
    int32_t mi_rows, mi_cols, mi_stride; /* the record grid: at least ((height + 7) & ~7) / 4 rows, ((width + 7) & ~7) / 4 columns */
    int32_t bit_depth;
    int32_t pixel_bytes;
    int32_t filter_level[2]; /* luma vertical / horizontal edges: both 0 = nothing is filtered, chroma included */
    int32_t filter_level_u, filter_level_v; /* 0 = that plane is not filtered */
    int32_t reserved;
    uint8_t lvl[3][8][2][8][2]; /* [plane][segment][dir: 0 vertical edges, 1 horizontal][ref_frame0][mode delta index] */
    uint8_t lfthr[64][3];
    uint8_t reserved2[4];
} SvtB200DlfFrame;

/* T2: svt_av1_loop_filter_frame (deblocking_filter.c:625) over all three planes, in place: one pass over every vertical
 * edge, then one over every horizontal edge (no edge reads a pixel another edge of its direction writes, so this equals
 * the reference's superblock order).  d_mi: DEVICE array of mi_rows x mi_stride records.  Filtering reads and writes up
 * to 7 pixels past the plane's width and height at edges that start inside it: the planes need that much readable and
 * writable padding (the reference's recon pictures have it).  Returns SVT_B200_ERR_BAD_ARG for an inconsistent frame. */
SVT_B200_API int svt_b200_loop_filter_frame_dev(const SvtB200DlfFrame* frame, const SvtB200DlfMi* d_mi, void* stream);

/* The trial costs of the filter-level search (search_filter_level, deblocking_filter.c:886): for each listed base level, the
 * SSE against the source of one plane filtered at that level alone, as try_filter_frame (:840) measures it.  The host keeps
 * the search itself and looks the costs up instead of filtering. */
typedef struct SvtB200DlfLevelSse {
    const void*    src[3];        /* DEVICE: source planes at pixel (0, 0), same pixel type as the recon planes */
    int32_t        src_stride[3]; /* in pixels */
    int32_t        sse_width, sse_height; /* luma SSE region (ppcs->aligned_width x aligned_height, at most
                                             ((width + 7) & ~7) x ((height + 7) & ~7)); chroma: >> 1 */
    int32_t        plane_mask;    /* bit p: evaluate plane p */
    int32_t        n_levels;      /* 1..64 */
    uint8_t        level[64];     /* base level of entry i (0..63); 0 = the plane unfiltered */
    uint8_t        reserved[4];
    const uint8_t* d_lvl;         /* DEVICE [3][n_levels][8][2][8][2]: lf_info.lvl[plane] as svt_av1_loop_filter_frame_init
                                     derives it for level[i] (luma: both directions at level[i]); not read for level 0 */
} SvtB200DlfLevelSse;

/* T2: d_sse[p * n_levels + i] = try_filter_frame(level[i], plane p) for every plane p in the mask (other entries are not
 * written).  From `frame` the call uses the recon planes, the geometry, bit_depth, pixel_bytes and lfthr (which must
 * reflect the sharpness the search runs at), not filter_level* or lvl.  A chroma entry filters its plane whatever the
 * frame's luma levels are, as the search does.  The recon planes are read, never written; no pixel left of or above
 * (0, 0) or more than 7 past the plane's width or height is read.  d_mi: as for svt_b200_loop_filter_frame_dev.
 * Returns SVT_B200_ERR_BAD_ARG for an inconsistent frame or level list, an empty mask or a missing plane. */
SVT_B200_API int svt_b200_dlf_level_sse_dev(const SvtB200DlfFrame* frame, const SvtB200DlfLevelSse* s, const SvtB200DlfMi* d_mi,
                                           int64_t* d_sse, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* K9/K11  Wiener filter + statistics  (reference: convolve.c:100-237, restoration_pick.c:659) */
/* ------------------------------------------------------------------------------------------ */
typedef struct SvtB200ConvolveParams { /* layout of ConvolveParams, Source/Lib/Codec/definitions.h:572-585 */
    int32_t   ref;
    int32_t   do_average;
    uint16_t* dst;
    int32_t   dst_stride;
    int32_t   round_0;
    int32_t   round_1;
    int32_t   plane;
    int32_t   is_compound;
    int32_t   use_jnt_comp_avg;
    int32_t   fwd_offset;
    int32_t   bck_offset;
    int32_t   use_dist_wtd_comp_avg;
} SvtB200ConvolveParams;

/* T1: common_dsp_rtcd.h:173-175 (w, h <= 64; the caller's buffer must be readable 3 rows/columns
 * before and 4 after the unit, as for the reference); aom_dsp_rtcd.h:66-68.  High-bit-depth pixel
 * pointers are plain uint16_t* here (the reference passes CONVERT_TO_BYTEPTR disguises). */
SVT_B200_API void svt_b200_av1_wiener_convolve_add_src(const uint8_t* src, ptrdiff_t src_stride, uint8_t* dst,
                                                       ptrdiff_t dst_stride, const int16_t* filter_x,
                                                       const int16_t* filter_y, int32_t w, int32_t h,
                                                       const SvtB200ConvolveParams* conv_params);
SVT_B200_API void svt_b200_av1_highbd_wiener_convolve_add_src(const uint16_t* src, ptrdiff_t src_stride, uint16_t* dst,
                                                              ptrdiff_t dst_stride, const int16_t* filter_x,
                                                              const int16_t* filter_y, int32_t w, int32_t h,
                                                              const SvtB200ConvolveParams* conv_params, int32_t bd);
SVT_B200_API void svt_b200_av1_compute_stats(int32_t wiener_win, const uint8_t* dgd, const uint8_t* src, int32_t h_start,
                                             int32_t h_end, int32_t v_start, int32_t v_end, int32_t dgd_stride,
                                             int32_t src_stride, int64_t* M, int64_t* H);
SVT_B200_API void svt_b200_av1_compute_stats_highbd(int32_t wiener_win, const uint16_t* dgd, const uint16_t* src,
                                                    int32_t h_start, int32_t h_end, int32_t v_start, int32_t v_end,
                                                    int32_t dgd_stride, int32_t src_stride, int64_t* M, int64_t* H,
                                                    int32_t bit_depth);

/* T2.  Offsets/strides in pixels of the device planes. */
typedef struct SvtB200WienerUnit {
    uint64_t src_off;
    uint64_t dst_off;
    int32_t  src_stride;
    int32_t  dst_stride;
    uint16_t w, h;         /* <= 64 */
    uint32_t reserved;
    int16_t  hfilter[8];   /* WienerInfo.hfilter / vfilter: 7 taps + 0 */
    int16_t  vfilter[8];
} SvtB200WienerUnit;
SVT_B200_API int svt_b200_wiener_units_dev(const void* d_src, void* d_dst, const SvtB200WienerUnit* d_units, int n_units,
                                           int bit_depth, void* stream);

typedef struct SvtB200StatsItem {
    uint64_t dgd_off;      /* plane origin of this item (the h/v limits are relative to it) */
    uint64_t src_off;
    int32_t  dgd_stride;
    int32_t  src_stride;
    int32_t  h_start, h_end, v_start, v_end;
    int32_t  wiener_win;   /* 7, 5 or 3 */
    int32_t  reserved;
} SvtB200StatsItem;
/* d_M: [n_items][49], d_H: [n_items][49*49] (first win^2 resp. win^4 entries used, reference layout) */
SVT_B200_API int svt_b200_compute_stats_batch_dev(const void* d_dgd, const void* d_src, const SvtB200StatsItem* d_items,
                                                  int n_items, int bit_depth, int64_t* d_M, int64_t* d_H, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* K10/K12  self-guided restoration  (reference: restoration.c:634-992, restoration_pick.c:167-498) */
/* ------------------------------------------------------------------------------------------ */
/* T1: common_dsp_rtcd.h:177-181, aom_dsp_rtcd.h:79-81,215.  `params` is the reference's
 * SgrParamsType {int32 r[2]; int32 s[2]} passed as 4 ints.  High-bit-depth pixel pointers are plain
 * uint16_t* carried in the uint8_t* arguments (no CONVERT_TO_BYTEPTR shift). */
SVT_B200_API void    svt_b200_av1_selfguided_restoration(const uint8_t* dgd8, int32_t width, int32_t height, int32_t dgd_stride,
                                                         int32_t* flt0, int32_t* flt1, int32_t flt_stride,
                                                         int32_t sgr_params_idx, int32_t bit_depth, int32_t highbd);
SVT_B200_API void    svt_b200_apply_selfguided_restoration(const uint8_t* dat8, int32_t width, int32_t height, int32_t stride,
                                                           int32_t eps, const int32_t* xqd, uint8_t* dst8, int32_t dst_stride,
                                                           int32_t* tmpbuf, int32_t bit_depth, int32_t highbd);
SVT_B200_API int64_t svt_b200_av1_lowbd_pixel_proj_error(const uint8_t* src8, int32_t width, int32_t height, int32_t src_stride,
                                                         const uint8_t* dat8, int32_t dat_stride, int32_t* flt0,
                                                         int32_t flt0_stride, int32_t* flt1, int32_t flt1_stride, int32_t xq[2],
                                                         const int32_t* params);
SVT_B200_API int64_t svt_b200_av1_highbd_pixel_proj_error(const uint16_t* src, int32_t width, int32_t height, int32_t src_stride,
                                                          const uint16_t* dat, int32_t dat_stride, int32_t* flt0,
                                                          int32_t flt0_stride, int32_t* flt1, int32_t flt1_stride, int32_t xq[2],
                                                          const int32_t* params);
SVT_B200_API void    svt_b200_get_proj_subspace(const uint8_t* src8, int width, int height, int src_stride, const uint8_t* dat8,
                                                int dat_stride, int use_highbitdepth, int32_t* flt0, int flt0_stride,
                                                int32_t* flt1, int flt1_stride, int* xq, const int32_t* params);

/* T2: batch of processing units (<= 128 x 128) over a device plane that is readable 3 pixels
 * around every unit. */
typedef struct SvtB200SgrUnit {
    uint64_t dgd_off;   /* pixels */
    uint64_t flt0_off;  /* int32 elements */
    uint64_t flt1_off;
    int32_t  dgd_stride;
    int32_t  flt_stride;
    uint16_t w, h;
    uint16_t params_idx; /* 0..15, svt_aom_eb_sgr_params */
    uint16_t reserved;
} SvtB200SgrUnit;
SVT_B200_API int svt_b200_sgr_units_dev(const void* d_dgd, const SvtB200SgrUnit* d_units, int n_units, int32_t* d_flt0,
                                        int32_t* d_flt1, int bit_depth, int max_w, int max_h, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* a13  loop-restoration drivers  (reference: Source/Lib/Codec/restoration.c:257-435,1067-1294,  */
/*      1506-1700; restoration_pick.c:103)                                                      */
/* ------------------------------------------------------------------------------------------ */
/* One plane of a picture for the restoration stage.  All pointers are DEVICE memory addressing pixel (0,0); strides
 * in pixels; pixels are uint8 (bit_depth 8) or uint16.  boundary_above / boundary_below use the layout of the
 * reference's RestorationStripeBoundaries (restoration.h): row 2 * stripe + i (i = 0, 1), boundary_stride pixels per
 * row, logical column x stored at index x + 4 (RESTORATION_EXTRA_HORZ), columns -4 .. width + 3 filled. */
typedef struct SvtB200LrPlane {
    const void* deblocked;   /* loop-filtered picture BEFORE CDEF: source of the interior stripe-boundary lines */
    const void* cdef;        /* CDEF output: the restoration input; source of the picture-top / -bottom lines */
    void*       dst;         /* restored output (cm->rst_frame) */
    const void* src;         /* source picture, only for svt_b200_lr_unit_sse_dev */
    void*       boundary_above;
    void*       boundary_below;
    int32_t     stride_deblocked, stride_cdef, stride_dst, stride_src;
    int32_t     boundary_stride; /* svt_b200_lr_boundary_stride(width) */
    int32_t     width, height;   /* crop size of this plane */
    int32_t     ss_x, ss_y;      /* 1 for the chroma planes of 4:2:0 */
    int32_t     unit_size;       /* rst_info[plane].restoration_unit_size (power of two, >= 64 >> ss_x) */
    int32_t     frame_restoration_type; /* rst_info[plane].frame_restoration_type: 1 = RESTORE_WIENER promises that no unit of the
                                           plane is RESTORE_SGRPROJ (smaller shared-memory footprint); anything else = any unit type */
} SvtB200LrPlane;

/* RestorationUnitInfo (restoration.h) flattened: restoration_type 0 = RESTORE_NONE, 1 = RESTORE_WIENER, 2 = RESTORE_SGRPROJ */
typedef struct SvtB200LrUnitInfo {
    int32_t restoration_type;
    int32_t sgr_ep;       /* SgrprojInfo.ep */
    int32_t sgr_xqd[2];   /* SgrprojInfo.xqd */
    int16_t hfilter[8];   /* WienerInfo.hfilter (7 taps + 0) */
    int16_t vfilter[8];
} SvtB200LrUnitInfo;

SVT_B200_API int svt_b200_lr_num_stripes(int plane_height, int ss_y);   /* rows of 2 lines in each boundary buffer */
SVT_B200_API int svt_b200_lr_boundary_stride(int plane_width);
SVT_B200_API int svt_b200_lr_units_per_dim(int size, int unit_size);    /* svt_av1_lr_count_units_in_tile */
/* svt_av1_loop_restoration_save_boundary_lines (restoration.c:1682): after_cdef = 0 saves the deblocked lines of the
 * interior stripe boundaries (read from `deblocked`), after_cdef = 1 the CDEF lines at the top / bottom of the picture
 * (read from `cdef`); call once each, as the reference does around CDEF. */
SVT_B200_API int svt_b200_lr_save_boundary_lines_dev(const SvtB200LrPlane* planes, int n_planes, int after_cdef, int bit_depth, void* stream);
/* svt_av1_loop_restoration_filter_frame (restoration.c:1179): every unit of every plane, stripe by stripe with the saved
 * boundary lines, into `dst`.  d_units[p]: DEVICE array of the plane's units in raster order
 * (svt_b200_lr_units_per_dim(height) rows x svt_b200_lr_units_per_dim(width) columns).  The picture itself is not
 * modified (the reference's in-place save / restore of the rows around a stripe is not needed) and needs no border. */
SVT_B200_API int svt_b200_lr_filter_frame_dev(const SvtB200LrPlane* planes, int n_planes, const SvtB200LrUnitInfo* const d_units[3],
                                              int optimized_lr, int bit_depth, void* stream);
/* sse_restoration_unit (restoration_pick.c:103) for every unit: d_sse[p][unit] = sum (dst - src)^2 over the unit's limits */
SVT_B200_API int svt_b200_lr_unit_sse_dev(const SvtB200LrPlane* planes, int n_planes, int64_t* const d_sse[3], int bit_depth, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* K13 HME pyramid + plane padding (pic_analysis_process.c:130-160, 2138-2190) and the T2     */
/*      open-loop ME driver of a picture (motion_estimation.c:781-3076; me_process.c:97-291)  */
/* ------------------------------------------------------------------------------------------ */
/* T1: downsample_2d (aom_dsp_rtcd.h:841). */
SVT_B200_API void svt_b200_downsample_2d(uint8_t* input_samples, uint32_t input_stride, uint32_t input_area_width,
                                         uint32_t input_area_height, uint8_t* decim_samples, uint32_t decim_stride,
                                         uint32_t decim_step);

/* One 8-bit luma pyramid (EbPaReferenceObject, reference_object.c:257-290).  Index 0 = 1/16
 * resolution, 1 = 1/4, 2 = full.  plane[] are DEVICE pointers to the start of each padded buffer;
 * the visible picture starts at (org_x, org_y).  The full plane needs >= 64+8 pixels of padding,
 * the 1/4 and 1/16 planes the reference's 32 / 16. */
typedef struct SvtB200MePicture {
    const uint8_t* plane[3];
    int32_t stride[3];
    int32_t org_x[3];
    int32_t org_y[3];
    int32_t width[3];
    int32_t height[3];
    int32_t reserved[2];
} SvtB200MePicture;

/* replicate the w x h interior at (org_x, org_y) of an 8-bit device plane into its padding
 * (svt_aom_generate_padding / svt_extend_frame) */
SVT_B200_API int svt_b200_extend_plane_dev(uint8_t* d_buf, int stride, int w, int h, int org_x, int org_y, void* stream);
/* the same for up to 4 planes (a picture's Y, Cb, Cr) in one launch */
typedef struct SvtB200PlaneExtent {
    uint8_t* buf;     /* first byte of the padded plane */
    int32_t  stride;  /* in pixels */
    int32_t  w, h;    /* interior size */
    int32_t  org_x, org_y; /* interior origin = padding widths */
    int32_t  pixel_bytes;  /* 0 or 1: 8-bit samples; 2: 16-bit samples (high-bit-depth planes) */
} SvtB200PlaneExtent;
SVT_B200_API int svt_b200_extend_planes_dev(const SvtB200PlaneExtent* planes, int n_planes, void* stream);
/* fills the 1/4 and 1/16 planes (interior + replicated padding) from the full plane */
SVT_B200_API int svt_b200_build_hme_pyramid_dev(const SvtB200MePicture* pic, void* stream);

/* ---- T2, the complete driver: svt_aom_motion_estimation_b64 (motion_estimation.c:3076) for every 64x64 block of a picture ----
 * zz-SAD reference pruning (init_zz_sad :2391), pre-HME (prehme_b64 :1722), HME level 0/1/2 with the early exits and the
 * pre-HME quadrant replacement (:1906-2180), final search centre (:2182), HME-based reference pruning and search-area divisors
 * (hme_prune_ref_and_adjust_sr :2477), the integer-search area derivation incl. the 8x8-SAD-variance probe
 * (integer_search_b64 :1249-1520), the 85-PU full-pel search, ME-based reference pruning (me_prune_ref :1522), candidate
 * construction (construct_me_candidate_array* :2532-2840), per-size distortions (compute_distortion :2964) and the
 * global-motion detection flags (perform_gm_detection :2842).
 *
 * SvtB200MeControls is the MeContext (me_context.h:366-509) control state AFTER svt_aom_sig_deriv_me (enc_mode_config.c:681),
 * flattened, plus the few picture-level fields the driver reads.  The host derives it exactly as the encoder does and passes
 * the result; tests obtain it from the reference's own derivation (oracle/ref_me_b64.c).  Not supported (the call returns
 * SVT_B200_ERR_BAD_ARG): me_sr_adjustment level 2 (screen-content presets: its rule reads the full-pel result of another
 * reference of the same block), ME_MCTF (temporal-filter ME, SURVEY 8 f3). */
typedef struct SvtB200MeControls {
    int32_t n_list, n_ref[2];        /* num_of_list_to_search, num_of_ref_pic_to_search[] */
    int32_t temporal_layer_index, is_ref, hierarchical_levels;
    int32_t dist[2][4];              /* |picture_number - reference picture_number| */
    int32_t enable_hme, enable_l0, enable_l1, enable_l2, hme_sub_sad, me_sub_sad;
    int32_t hme_l0_min_w, hme_l0_min_h, hme_l0_max_w, hme_l0_max_h, hme_l1_w, hme_l1_h, hme_l2_w, hme_l2_h;
    int32_t me_min_w, me_min_h, me_max_w, me_max_h;
    int32_t prehme_enable, prehme_sa[2][4] /* [region]{min w, min h, max w, max h} */, prehme_skip_search_line, prehme_l1_early_exit;
    int32_t prune_enable, prune_hme_th, prune_me_th, zz_sad_th, zz_sad_pct, phme_sad_th, phme_sad_pct;   /* MeHmeRefPruneCtrls */
    int32_t sr_enable, sr_mv_length_th, sr_stationary_hme_sad_abs_th, sr_stationary_divisor, sr_hme_sad_abs_th, sr_low_hme_sad_divisor,
        sr_distance_based_hme_resizing;                                                                /* MeSrCtrls */
    int32_t var_enable, var_div4_th, var_div2_th, var_mult2_th;                                          /* Me8x8VarCtrls (uint32 values) */
    int32_t mvsa_enable, mvsa_nearest_ref_only, mvsa_mv_size_th, mvsa_multiplier;                        /* MvBasedSearchAdj */
    int32_t reduce_hme_l0_sr_th_min, reduce_hme_l0_sr_th_max;
    int32_t me_early_exit_th, me_safe_limit_zz_th, prev_me_stage_based_exit_th, prune_me_candidates_th, use_best_unipred_cand_only;
    int32_t similar_brightness_refs, only_l_bwd, enable_me_8x8, enable_me_16x16;
    int32_t max_cand, max_refs, max_l0; /* MotionEstimationData: strides of me_candidate_array / me_mv_array (pcs.h:500-502) */
    int32_t gm_enabled, gm_use_distance_based_active_th, resolution_le_480p;
    int32_t reserved[5];
} SvtB200MeControls;

/* device buffers the call fills (all of them are overwritten completely).  n_pu = svt_b200_me_b64_num_pus(). */
typedef struct SvtB200MeB64Results {
    uint8_t*  total_me_candidate_index; /* [n_b64][n_pu]              MeSbResults (me_sb_results.h:44-52), raster PU order */
    uint8_t*  me_candidate_array;       /* [n_b64][n_pu * max_cand]   MeCandidate bytes: direction | ref_idx_l0<<2 | ref_idx_l1<<4 | ref0_list<<6 | ref1_list<<7 */
    uint32_t* me_mv_array;              /* [n_b64][n_pu * max_refs]   (y << 16) | (x & 0xffff), full-pel */
    uint32_t* distortion;               /* [n_b64][6]: rc_me_distortion, me_64x64/32x32/16x16/8x8_distortion, me_8x8_cost_variance */
    uint8_t*  flags;                    /* [n_b64][2]: stationary_block_present_sb, rc_me_allow_gm */
    uint8_t*  do_ref;                   /* [n_b64][2][4]   references still alive after all pruning */
    int16_t*  hme_centre;               /* [n_b64][2][4][2] search_results[].hme_sc_x / hme_sc_y */
    uint32_t* zz_sad;                   /* [n_b64][2][4] */
    uint32_t* best_sad;                 /* [n_refs][n_b64][85] p_sb_best_sad of every reference (list 0 first), ME z-order; pruned references: undefined */
    uint32_t* best_mv;                  /* [n_refs][n_b64][85] */
} SvtB200MeB64Results;
/* 85, 21 or 5: the square PUs that carry candidates (me_sb_results_ctor, pcs.c:107-112) */
SVT_B200_API int svt_b200_me_b64_num_pus(const SvtB200MeControls* ctrl);
/* cur / refs / ctrl / out are HOST structs holding device pointers; refs = n_ref[0] list-0 pictures, then n_ref[1] list-1 pictures */
SVT_B200_API int svt_b200_me_b64_picture_dev(const SvtB200MePicture* cur, const SvtB200MePicture* refs, const SvtB200MeControls* ctrl,
                                             const SvtB200MeB64Results* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVT_B200_H */
