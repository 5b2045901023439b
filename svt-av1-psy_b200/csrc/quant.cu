// quant.cu -- K7 quantize / dequantize (sm_90a).
//
// Reference behaviour restated: svt_aom_quantize_b_c_ii (Source/Lib/Codec/full_loop.c:29-79),
// svt_aom_highbd_quantize_b_c (:149-198), quantize_fp_helper_c (:282-342), highbd_quantize_fp_helper_c
// (:387-453).  All four are element-wise in scan order (the reference's end-of-block pre-scan is an
// early-out, not a dependency: a coefficient the pre-scan drops also fails the dead-zone test of the
// quantisation pass), so a team of threads walks the scan, every thread quantises the coefficient at
// scan[i], and eob is a max-reduction over the scan indices that produced a non-zero level.
//
// Layout: coefficients int32 (TranLow), scan int16, QM weights uint8 (AOM_QM_BITS = 5); the 2-entry
// (DC, AC) zbin/round/quant/quant_shift/dequant tables travel inside the work item.
#include "common.cuh"
#include "../../include/svt_b200.h"
#include "quant_one.cuh"

namespace b200 {

// One warp per item, 8 items per CTA: n_coeffs is 16..1024, i.e. 0.5..32 coefficients per lane.
// Every coefficient is quantised on its own; only the end-of-block position depends on the scan order
// (eob = 1 + the last scan position with a non-zero level).  With the inverse scan table (the `iscan`
// argument the reference passes to the same functions) the warp walks the block in RASTER order -- the
// coefficient, level, dequantised and matrix accesses are all coalesced and independent -- and takes
// eob = max(iscan[rc] + 1).  Without it the block is walked in scan order (gathered accesses).
__global__ void __launch_bounds__(256)
quant_kernel(const int32_t* __restrict__ coeff_base, int32_t* __restrict__ q_base, int32_t* __restrict__ dq_base,
             const int16_t* __restrict__ scan_base, const int16_t* __restrict__ iscan_base, const uint8_t* __restrict__ qm_base,
             const SvtB200QuantItem* __restrict__ items, int n_items, uint16_t* __restrict__ eobs) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int idx = blockIdx.x * 8 + warp; idx < n_items; idx += gridDim.x * 8) {
        const SvtB200QuantItem it = items[idx];
        const int32_t* coeff = coeff_base + it.coeff_off;
        int32_t*       qc    = q_base + it.q_off;
        int32_t*       dqc   = dq_base + it.dq_off;
        const uint8_t* qm    = it.qm_off == SVT_B200_NO_QM ? nullptr : qm_base + it.qm_off;
        const uint8_t* iqm   = it.iqm_off == SVT_B200_NO_QM ? nullptr : qm_base + it.iqm_off;
        int            eob   = 0;
        if (iscan_base) {
            const int16_t* iscan = iscan_base + it.scan_off;
#pragma unroll 4
            for (int rc = lane; rc < (int)it.n_coeffs; rc += 32) {
                const int pos = iscan[rc];
                int32_t   q, dq;
                quant_one(it, coeff[rc], rc, qm, iqm, q, dq);
                qc[rc]  = q;
                dqc[rc] = dq;
                if (q) eob = max(eob, pos + 1);
            }
        } else {
            const int16_t* scan = scan_base + it.scan_off;
            for (int i = lane; i < (int)it.n_coeffs; i += 32) {
                const int rc = scan[i];
                int32_t   q, dq;
                quant_one(it, coeff[rc], rc, qm, iqm, q, dq);
                qc[rc]  = q;
                dqc[rc] = dq;
                if (q) eob = i + 1;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) eob = max(eob, __shfl_xor_sync(0xffffffffu, eob, o));
        if (lane == 0) eobs[idx] = (uint16_t)eob;
    }
}

void launch_quant(const int32_t* d_coeff, int32_t* d_q, int32_t* d_dq, const int16_t* d_scan, const int16_t* d_iscan,
                  const uint8_t* d_qm, const SvtB200QuantItem* d_items, int n, uint16_t* d_eobs, cudaStream_t st) {
    if (n <= 0) return;
    quant_kernel<<<grid_for((n + 7) / 8, 8), 256, 0, st>>>(d_coeff, d_q, d_dq, d_scan, d_iscan, d_qm, d_items, n, d_eobs);
    B200_LAUNCH_CHECK();
}

// shared T1 body: stage one block, run, copy q/dq/eob back
static void quant_t1(int mode, const int32_t* coeff_ptr, intptr_t n_coeffs, const int16_t* zbin_ptr, const int16_t* round_ptr,
                     const int16_t* quant_ptr, const int16_t* quant_shift_ptr, int32_t* qcoeff_ptr, int32_t* dqcoeff_ptr,
                     const int16_t* dequant_ptr, uint16_t* eob_ptr, const int16_t* scan, const uint8_t* qm_ptr,
                     const uint8_t* iqm_ptr, int log_scale) {
    require_ready();
    const size_t n = (size_t)n_coeffs;
    LaneGuard    l;
    size_t o_c = l->alloc(n * 4), o_scan = l->alloc(n * 2), o_qm = l->alloc(2 * n + 16), o_it = l->alloc(sizeof(SvtB200QuantItem));
    size_t in_end = l->used;
    size_t o_q = l->alloc(n * 4), o_dq = l->alloc(n * 4), o_eob = l->alloc(16);
    memcpy(l->h<int32_t>(o_c), coeff_ptr, n * 4);
    memcpy(l->h<int16_t>(o_scan), scan, n * 2);
    SvtB200QuantItem* it = l->h<SvtB200QuantItem>(o_it);
    memset(it, 0, sizeof(*it));
    it->n_coeffs = (uint32_t)n;
    it->mode = (uint8_t)mode;
    it->log_scale = (uint8_t)log_scale;
    it->qm_off = it->iqm_off = SVT_B200_NO_QM;
    if (qm_ptr) {
        memcpy(l->h<uint8_t>(o_qm), qm_ptr, n);
        it->qm_off = 0;
    }
    if (iqm_ptr) {
        memcpy(l->h<uint8_t>(o_qm) + n, iqm_ptr, n);
        it->iqm_off = (uint32_t)n;
    }
    for (int k = 0; k < 2; k++) {
        it->zbin[k] = zbin_ptr ? zbin_ptr[k] : 0;
        it->round[k] = round_ptr[k];
        it->quant[k] = quant_ptr[k];
        it->quant_shift[k] = quant_shift_ptr ? quant_shift_ptr[k] : 0;
        it->dequant[k] = dequant_ptr[k];
    }
    l->h2d(0, in_end);
    launch_quant(l->d<int32_t>(o_c), l->d<int32_t>(o_q), l->d<int32_t>(o_dq), l->d<int16_t>(o_scan), nullptr, l->d<uint8_t>(o_qm),
                 l->d<SvtB200QuantItem>(o_it), 1, l->d<uint16_t>(o_eob), l->stream);
    l->d2h(o_q, (o_eob + 16) - o_q);
    l->sync();
    memcpy(qcoeff_ptr, l->h<int32_t>(o_q), n * 4);
    memcpy(dqcoeff_ptr, l->h<int32_t>(o_dq), n * 4);
    *eob_ptr = *l->h<uint16_t>(o_eob);
}

}  // namespace b200

using namespace b200;

#define QARGS                                                                                                     \
    const int32_t *coeff_ptr, intptr_t n_coeffs, const int16_t *zbin_ptr, const int16_t *round_ptr,               \
        const int16_t *quant_ptr, const int16_t *quant_shift_ptr, int32_t *qcoeff_ptr, int32_t *dqcoeff_ptr,      \
        const int16_t *dequant_ptr, uint16_t *eob_ptr, const int16_t *scan, const int16_t *iscan
#define QPASS coeff_ptr, n_coeffs, zbin_ptr, round_ptr, quant_ptr, quant_shift_ptr, qcoeff_ptr, dqcoeff_ptr, dequant_ptr, eob_ptr, scan

extern "C" void svt_b200_aom_quantize_b(QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_B_LBD, QPASS, qm_ptr, iqm_ptr, log_scale);
}
extern "C" void svt_b200_aom_highbd_quantize_b(QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_B_HBD, QPASS, qm_ptr, iqm_ptr, log_scale);
}
extern "C" void svt_b200_av1_quantize_b_qm(QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_B_LBD, QPASS, qm_ptr, iqm_ptr, log_scale);
}
extern "C" void svt_b200_av1_highbd_quantize_b_qm(QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int32_t log_scale) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_B_HBD, QPASS, qm_ptr, iqm_ptr, log_scale);
}
extern "C" void svt_b200_av1_quantize_fp(QARGS) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_FP_LBD, QPASS, nullptr, nullptr, 0);
}
extern "C" void svt_b200_av1_quantize_fp_32x32(QARGS) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_FP_LBD, QPASS, nullptr, nullptr, 1);
}
extern "C" void svt_b200_av1_quantize_fp_64x64(QARGS) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_FP_LBD, QPASS, nullptr, nullptr, 2);
}
extern "C" void svt_b200_av1_quantize_fp_qm(QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int16_t log_scale) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_FP_LBD, QPASS, qm_ptr, iqm_ptr, log_scale);
}
extern "C" void svt_b200_av1_highbd_quantize_fp(QARGS, int16_t log_scale) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_FP_HBD, QPASS, nullptr, nullptr, log_scale);
}
extern "C" void svt_b200_av1_highbd_quantize_fp_qm(QARGS, const uint8_t* qm_ptr, const uint8_t* iqm_ptr, int16_t log_scale) {
    (void)iscan;
    quant_t1(SVT_B200_QUANT_FP_HBD, QPASS, qm_ptr, iqm_ptr, log_scale);
}

extern "C" int svt_b200_quant_batch_dev(const int32_t* d_coeff, int32_t* d_qcoeff, int32_t* d_dqcoeff, const int16_t* d_scan,
                                        const int16_t* d_iscan, const uint8_t* d_qm, const SvtB200QuantItem* d_items, int n_items,
                                        uint16_t* d_eobs, void* stream) {
    require_ready();
    if (n_items < 0 || (!d_scan && !d_iscan)) return SVT_B200_ERR_BAD_ARG;
    launch_quant(d_coeff, d_qcoeff, d_dqcoeff, d_scan, d_iscan, d_qm, d_items, n_items, d_eobs, (cudaStream_t)stream);
    return SVT_B200_OK;
}
