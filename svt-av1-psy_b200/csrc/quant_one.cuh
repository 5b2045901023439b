// quant_one.cuh -- the per-coefficient quantise/dequantise arithmetic of K7, shared by quant.cu (batch
// and T1 quantizers) and txfm.cu (the fused transform / quantise / inverse-transform kernel).
// Reference: svt_aom_quantize_b_c_ii (Source/Lib/Codec/full_loop.c:29-79), svt_aom_highbd_quantize_b_c
// (:149-198), quantize_fp_helper_c (:282-342), highbd_quantize_fp_helper_c (:387-453).
//
// The arithmetic is quant_coef, specialised on the quantiser mode and on whether the item has a matrix; what is the same
// for every coefficient of an item (the DC / AC constants rounded by log_scale) is QuantK, computed once per item.  The
// fused kernel selects the specialisation once per item and runs a loop on it; quant_one selects it per coefficient.
#pragma once
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

constexpr int kQmBits = 5;

__device__ __forceinline__ int32_t round_pow2(int32_t v, int n) { return n == 0 ? v : ((v + (1 << (n - 1))) >> n); }

// an item's quantiser constants, [0] = DC, [1] = AC; zbin and round are already rounded by log_scale
struct QuantK {
    int32_t zbin[2], round[2], quant[2], quant_shift[2], dequant[2];
    int     ls;
};
__device__ __forceinline__ QuantK quant_consts(const SvtB200QuantItem& it) {
    QuantK k;
    k.ls = it.log_scale;
#pragma unroll
    for (int a = 0; a < 2; a++) {
        k.zbin[a]        = round_pow2(it.zbin[a], k.ls);
        k.round[a]       = round_pow2(it.round[a], k.ls);
        k.quant[a]       = it.quant[a];
        k.quant_shift[a] = it.quant_shift[a];
        k.dequant[a]     = it.dequant[a];
    }
    return k;
}
// the item has a quantisation matrix: either of its weight tables is given (a missing one weighs 1 << kQmBits)
__device__ __forceinline__ bool quant_has_qm(const SvtB200QuantItem& it) {
    return it.qm_off != SVT_B200_NO_QM || it.iqm_off != SVT_B200_NO_QM;
}

// One coefficient.  ac: 0 for the DC position, 1 otherwise; wt / iwt: the matrix weights at its position (read only when
// QM).  The constants are picked by ac with selects, so that a QuantK in registers is never indexed dynamically.
template <int MODE, bool QM>
__device__ __forceinline__ void quant_coef(const QuantK& k, int32_t coeff, int ac, int32_t wt_in, int32_t iwt_in, int32_t& q,
                                           int32_t& dq) {
    const int     ls          = k.ls;
    const int32_t zbin        = ac ? k.zbin[1] : k.zbin[0];
    const int32_t round       = ac ? k.round[1] : k.round[0];
    const int32_t quant       = ac ? k.quant[1] : k.quant[0];
    const int32_t quant_shift = ac ? k.quant_shift[1] : k.quant_shift[0];
    const int32_t dequant_ac  = ac ? k.dequant[1] : k.dequant[0];
    const int32_t sign        = coeff < 0 ? -1 : 0;
    const int32_t absc        = (coeff ^ sign) - sign;
    const int32_t wt          = QM ? wt_in : (1 << kQmBits);
    const int32_t iwt         = QM ? iwt_in : (1 << kQmBits);
    q = dq = 0;
    if constexpr (MODE == SVT_B200_QUANT_B_LBD) {
        if ((int32_t)((uint32_t)absc * (uint32_t)wt) >= (zbin << kQmBits)) {
            int32_t t = absc + round;
            t         = t < -32768 ? -32768 : (t > 32767 ? 32767 : t);
            long long tmp = (long long)t * wt;
            const int32_t tmp32 = (int32_t)(((((tmp * quant) >> 16) + tmp) * quant_shift) >> (16 - ls + kQmBits));
            q = (tmp32 ^ sign) - sign;
            const int32_t dequant = (dequant_ac * iwt + (1 << (kQmBits - 1))) >> kQmBits;
            const int32_t adq     = (int32_t)((uint32_t)tmp32 * (uint32_t)dequant) >> ls;
            dq = (adq ^ sign) - sign;
        }
    } else if constexpr (MODE == SVT_B200_QUANT_B_HBD) {
        const int32_t cw = (int32_t)((uint32_t)coeff * (uint32_t)wt);
        if (cw >= zbin * (1 << kQmBits) || cw <= -zbin * (1 << kQmBits)) {
            const long long tmp1 = (long long)absc + round;
            const long long tmpw = tmp1 * wt;
            const long long tmp2 = ((tmpw * quant) >> 16) + tmpw;
            const int32_t   aq   = (int32_t)((tmp2 * quant_shift) >> (16 - ls + kQmBits));
            q = (aq ^ sign) - sign;
            const int32_t dequant = (dequant_ac * iwt + (1 << (kQmBits - 1))) >> kQmBits;
            const int32_t adq     = (int32_t)((uint32_t)aq * (uint32_t)dequant) >> ls;
            dq = (adq ^ sign) - sign;
        }
    } else if constexpr (MODE == SVT_B200_QUANT_FP_LBD) {
        if constexpr (!QM) {
            if (((long long)absc << (1 + ls)) >= (long long)dequant_ac) {
                long long a = (long long)absc + round;
                a           = a < -32768 ? -32768 : (a > 32767 ? 32767 : a);
                const int32_t tmp32 = (int32_t)((a * quant) >> (16 - ls));
                if (tmp32) {
                    q = (tmp32 ^ sign) - sign;
                    const int32_t adq = (int32_t)((uint32_t)tmp32 * (uint32_t)dequant_ac) >> ls;
                    dq = (adq ^ sign) - sign;
                }
            }
        } else {
            const int32_t dequant = (dequant_ac * iwt + (1 << (kQmBits - 1))) >> kQmBits;
            if ((long long)absc * wt >= (long long)(dequant_ac << (kQmBits - (1 + ls)))) {
                long long a = (long long)absc + round;
                a           = a < -32768 ? -32768 : (a > 32767 ? 32767 : a);
                const int32_t tmp32 = (int32_t)((a * wt * quant) >> (16 - ls + kQmBits));
                q = (tmp32 ^ sign) - sign;
                const int32_t adq = (int32_t)((uint32_t)tmp32 * (uint32_t)dequant) >> ls;
                dq = (adq ^ sign) - sign;
            }
        }
    } else {  // SVT_B200_QUANT_FP_HBD
        const int shift = 16 - ls;
        if constexpr (QM) {
            const int32_t dequant = (dequant_ac * iwt + (1 << (kQmBits - 1))) >> kQmBits;
            if ((long long)absc * wt >= (long long)(dequant_ac << (kQmBits - (1 + ls)))) {
                const long long tmp = (long long)absc + round;
                const int32_t   aq  = (int32_t)((tmp * quant * wt) >> (shift + kQmBits));
                q = (aq ^ sign) - sign;
                const int32_t adq = (int32_t)((uint32_t)aq * (uint32_t)dequant) >> ls;
                dq = (adq ^ sign) - sign;
            }
        } else {
            if ((int32_t)((uint32_t)absc << (1 + ls)) >= dequant_ac) {
                const long long tmp = (long long)absc + round;
                const int32_t   aq  = (int32_t)((tmp * quant) >> shift);
                q = (aq ^ sign) - sign;
                const int32_t adq = (int32_t)((uint32_t)aq * (uint32_t)dequant_ac) >> ls;
                dq = (adq ^ sign) - sign;
            }
        }
    }
}

// one coefficient of an item, the specialisation chosen here (the batch quantiser, quant.cu)
__device__ __forceinline__ void quant_one(const SvtB200QuantItem& it, int32_t coeff, int rc, const uint8_t* qm,
                                          const uint8_t* iqm, int32_t& q, int32_t& dq) {
    const QuantK  k   = quant_consts(it);
    const int     ac  = rc != 0;
    const int32_t wt  = qm ? (int32_t)qm[rc] : (1 << kQmBits);
    const int32_t iwt = iqm ? (int32_t)iqm[rc] : (1 << kQmBits);
    const bool    has = qm || iqm;
    switch (it.mode) {
    case SVT_B200_QUANT_B_LBD:
        if (has) quant_coef<SVT_B200_QUANT_B_LBD, true>(k, coeff, ac, wt, iwt, q, dq);
        else quant_coef<SVT_B200_QUANT_B_LBD, false>(k, coeff, ac, wt, iwt, q, dq);
        break;
    case SVT_B200_QUANT_B_HBD:
        if (has) quant_coef<SVT_B200_QUANT_B_HBD, true>(k, coeff, ac, wt, iwt, q, dq);
        else quant_coef<SVT_B200_QUANT_B_HBD, false>(k, coeff, ac, wt, iwt, q, dq);
        break;
    case SVT_B200_QUANT_FP_LBD:
        if (has) quant_coef<SVT_B200_QUANT_FP_LBD, true>(k, coeff, ac, wt, iwt, q, dq);
        else quant_coef<SVT_B200_QUANT_FP_LBD, false>(k, coeff, ac, wt, iwt, q, dq);
        break;
    default:
        if (has) quant_coef<SVT_B200_QUANT_FP_HBD, true>(k, coeff, ac, wt, iwt, q, dq);
        else quant_coef<SVT_B200_QUANT_FP_HBD, false>(k, coeff, ac, wt, iwt, q, dq);
        break;
    }
}

}  // namespace b200
