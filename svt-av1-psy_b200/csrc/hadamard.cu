// hadamard.cu -- K4 Hadamard transforms and SATD (sm_90a).
//
// Reference behaviour restated: svt_aom_hadamard_{4x4,8x8,16x16,32x32}_c
// (Source/Lib/C_DEFAULT/picture_operators_c.c:188-330: 1-D butterflies on int16 with wrap, >>1 inside
// the 4-point column, >>1 / >>2 when four sub-blocks are merged) and svt_aom_satd_c
// (Source/Lib/Codec/common_dsp_rtcd.c:70-77).
//
// Mapping: one CTA per block; every 8x8 sub-block is owned by 8 threads (one per column, then one
// per row of the intermediate), the 16x16 / 32x32 merges are element-parallel.  The fused T2 entry
// (hadamard + sum |coeff|) never writes the coefficients to HBM.
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

__device__ __forceinline__ void had_col8(const int16_t* s, int st, int16_t* o) {
    const int16_t b0 = (int16_t)(s[0 * st] + s[1 * st]), b1 = (int16_t)(s[0 * st] - s[1 * st]);
    const int16_t b2 = (int16_t)(s[2 * st] + s[3 * st]), b3 = (int16_t)(s[2 * st] - s[3 * st]);
    const int16_t b4 = (int16_t)(s[4 * st] + s[5 * st]), b5 = (int16_t)(s[4 * st] - s[5 * st]);
    const int16_t b6 = (int16_t)(s[6 * st] + s[7 * st]), b7 = (int16_t)(s[6 * st] - s[7 * st]);
    const int16_t c0 = (int16_t)(b0 + b2), c1 = (int16_t)(b1 + b3), c2 = (int16_t)(b0 - b2), c3 = (int16_t)(b1 - b3);
    const int16_t c4 = (int16_t)(b4 + b6), c5 = (int16_t)(b5 + b7), c6 = (int16_t)(b4 - b6), c7 = (int16_t)(b5 - b7);
    o[0] = (int16_t)(c0 + c4);
    o[7] = (int16_t)(c1 + c5);
    o[3] = (int16_t)(c2 + c6);
    o[4] = (int16_t)(c3 + c7);
    o[2] = (int16_t)(c0 - c4);
    o[6] = (int16_t)(c1 - c5);
    o[1] = (int16_t)(c2 - c6);
    o[5] = (int16_t)(c3 - c7);
}
__device__ __forceinline__ void had_col4(const int16_t* s, int st, int16_t* o) {
    const int16_t b0 = (int16_t)((s[0 * st] + s[1 * st]) >> 1), b1 = (int16_t)((s[0 * st] - s[1 * st]) >> 1);
    const int16_t b2 = (int16_t)((s[2 * st] + s[3 * st]) >> 1), b3 = (int16_t)((s[2 * st] - s[3 * st]) >> 1);
    o[0] = (int16_t)(b0 + b2);
    o[1] = (int16_t)(b1 + b3);
    o[2] = (int16_t)(b0 - b2);
    o[3] = (int16_t)(b1 - b3);
}

// n = 4, 8, 16, 32.  in: n x n int16 in shared memory (pitch n).  out: n*n int32 in the reference's
// coefficient order.  128 threads.
__device__ void hadamard_block(const int16_t* in, int n, int16_t* t1, int16_t* t2, int32_t* out) {
    const int tid = threadIdx.x;
    if (n == 4) {
        if (tid < 4) had_col4(in + tid, 4, t1 + 4 * tid);
        __syncthreads();
        if (tid < 4) had_col4(t1 + tid, 4, t2 + 4 * tid);
        __syncthreads();
        if (tid < 16) out[tid] = (int32_t)t2[tid];
        __syncthreads();
        return;
    }
    const int nb = (n / 8) * (n / 8);  // 8x8 sub-blocks, 8 threads each
    const int sb = tid >> 3, k = tid & 7;
    // sub-block order of the reference: 32x32 -> four 16x16 (raster), each -> four 8x8 (raster)
    int by = 0, bx = 0;
    if (n == 8) {
        by = bx = 0;
    } else if (n == 16) {
        by = sb >> 1;
        bx = sb & 1;
    } else {
        const int q = sb >> 2, s = sb & 3;
        by = (q >> 1) * 2 + (s >> 1);
        bx = (q & 1) * 2 + (s & 1);
    }
    if (sb < nb) had_col8(in + (by * 8) * n + bx * 8 + k, n, t1 + sb * 64 + 8 * k);
    __syncthreads();
    if (sb < nb) had_col8(t1 + sb * 64 + k, 8, t2 + sb * 64 + 8 * k);
    __syncthreads();
    for (int i = tid; i < n * n; i += blockDim.x) out[i] = (int32_t)t2[i];
    __syncthreads();
    if (n >= 16) {  // merge 4 x 8x8 -> 16x16, >>1
        const int n16 = (n / 16) * (n / 16);
        for (int i = tid; i < n16 * 64; i += blockDim.x) {
            int32_t* c = out + (i >> 6) * 256 + (i & 63);
            const int32_t a0 = c[0], a1 = c[64], a2 = c[128], a3 = c[192];
            const int32_t b0 = (a0 + a1) >> 1, b1 = (a0 - a1) >> 1, b2 = (a2 + a3) >> 1, b3 = (a2 - a3) >> 1;
            c[0] = b0 + b2;
            c[64] = b1 + b3;
            c[128] = b0 - b2;
            c[192] = b1 - b3;
        }
        __syncthreads();
    }
    if (n == 32) {  // merge 4 x 16x16 -> 32x32, >>2
        for (int i = tid; i < 256; i += blockDim.x) {
            int32_t* c = out + i;
            const int32_t a0 = c[0], a1 = c[256], a2 = c[512], a3 = c[768];
            const int32_t b0 = (a0 + a1) >> 2, b1 = (a0 - a1) >> 2, b2 = (a2 + a3) >> 2, b3 = (a2 - a3) >> 2;
            c[0] = b0 + b2;
            c[256] = b1 + b3;
            c[512] = b0 - b2;
            c[768] = b1 - b3;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(128)
hadamard_kernel(const int16_t* __restrict__ src_base, const SvtB200HadamardItem* __restrict__ items, int n_items,
                int32_t* __restrict__ coeff_base, int32_t* __restrict__ satd_out) {
    __shared__ int16_t s_in[1024], s_t1[1024], s_t2[1024];
    __shared__ int32_t s_out[1024];
    __shared__ int32_t s_sum;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const SvtB200HadamardItem item = items[it];
        const int n = item.size;
        if (n != 4 && n != 8 && n != 16 && n != 32) {  // not a Hadamard size: sentinel result, nothing else touched (block-uniform branch)
            if (threadIdx.x == 0 && satd_out) satd_out[it] = -1;
            continue;
        }
        if (threadIdx.x == 0) s_sum = 0;
        for (int i = threadIdx.x; i < n * n; i += blockDim.x)
            s_in[i] = src_base[item.src_off + (size_t)(i / n) * item.src_stride + (i % n)];
        __syncthreads();
        hadamard_block(s_in, n, s_t1, s_t2, s_out);
        int32_t acc = 0;
        for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
            const int32_t v = s_out[i];
            if (coeff_base) coeff_base[item.coeff_off + i] = v;
            acc += v < 0 ? -v : v;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if ((threadIdx.x & 31) == 0) atomicAdd(&s_sum, acc);
        __syncthreads();
        if (threadIdx.x == 0 && satd_out) satd_out[it] = s_sum;
        __syncthreads();
    }
}

__global__ void satd_kernel(const int32_t* __restrict__ coeff, int length, int32_t* out) {
    __shared__ int32_t tot;
    if (threadIdx.x == 0) tot = 0;
    __syncthreads();
    int32_t acc = 0;
    for (int i = threadIdx.x; i < length; i += blockDim.x) {
        const int32_t v = coeff[i];
        acc += v < 0 ? -v : v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&tot, acc);
    __syncthreads();
    if (threadIdx.x == 0) *out = tot;
}

static void hadamard_t1(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff, int n) {
    require_ready();
    LaneGuard l;
    size_t o_src = l->alloc((size_t)n * n * 2), o_it = l->alloc(sizeof(SvtB200HadamardItem));
    size_t in_end = l->used;
    size_t o_c = l->alloc((size_t)n * n * 4);
    for (int r = 0; r < n; r++) memcpy(l->h<int16_t>(o_src) + r * n, src_diff + (ptrdiff_t)r * src_stride, n * 2);
    SvtB200HadamardItem* it = l->h<SvtB200HadamardItem>(o_it);
    memset(it, 0, sizeof(*it));
    it->src_stride = n;
    it->size = n;
    l->h2d(0, in_end);
    hadamard_kernel<<<1, 128, 0, l->stream>>>(l->d<int16_t>(o_src), l->d<SvtB200HadamardItem>(o_it), 1, l->d<int32_t>(o_c), nullptr);
    B200_LAUNCH_CHECK();
    l->d2h(o_c, (size_t)n * n * 4);
    l->sync();
    memcpy(coeff, l->h<int32_t>(o_c), (size_t)n * n * 4);
}

// ---- hadamard_path (enc_mode_config.c:2147-2212): residual -> Hadamard -> SATD of every transform block of a prediction block ----
// one CTA per transform block; the last block also leaves its residual / coefficients behind, as the reference's loop does
struct HadPathArgs {
    const uint8_t* input; const uint8_t* pred; int in_stride, pred_stride, n /*tx size 4..32*/, blocks_per_row, n_blocks;
};
__global__ void __launch_bounds__(128)
hadamard_path_kernel(const __grid_constant__ HadPathArgs a, int32_t* __restrict__ satd_out, int16_t* __restrict__ last_res, int32_t* __restrict__ last_coeff) {
    __shared__ int16_t s_in[1024], s_t1[1024], s_t2[1024];
    __shared__ int32_t s_out[1024];
    __shared__ int32_t s_sum;
    const int blk = blockIdx.x, n = a.n, brow = blk / a.blocks_per_row, bcol = blk - brow * a.blocks_per_row;
    if (threadIdx.x == 0) s_sum = 0;
    const uint8_t* ip = a.input + (size_t)(brow * n) * a.in_stride + bcol * n;
    const uint8_t* pp = a.pred + (size_t)(brow * n) * a.pred_stride + bcol * n;
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int r = i / n, c = i - r * n;
        s_in[i] = (int16_t)((int)ip[(size_t)r * a.in_stride + c] - (int)pp[(size_t)r * a.pred_stride + c]);
    }
    __syncthreads();
    hadamard_block(s_in, n, s_t1, s_t2, s_out);
    int32_t acc = 0;
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int32_t v = s_out[i];
        acc += v < 0 ? -v : v;
        if (blk == a.n_blocks - 1) { last_coeff[i] = v; last_res[i] = s_in[i]; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s_sum, acc);
    __syncthreads();
    if (threadIdx.x == 0) satd_out[blk] = s_sum;
}

// svt_av1_fwht4x4_c (transforms.c:3099-3150): the reversible Walsh-Hadamard of lossless blocks
__global__ void fwht4x4_kernel(const int16_t* __restrict__ in /*4x4 packed*/, int32_t* __restrict__ out) {
    __shared__ long long t[16];
    const int i = threadIdx.x;
    if (i < 4) {
        long long a1 = in[0 * 4 + i], b1 = in[1 * 4 + i], c1 = in[2 * 4 + i], d1 = in[3 * 4 + i];
        a1 += b1; d1 = d1 - c1;
        const long long e1 = (a1 - d1) >> 1;
        b1 = e1 - b1; c1 = e1 - c1; a1 -= c1; d1 += b1;
        t[4 * i + 0] = a1; t[4 * i + 1] = c1; t[4 * i + 2] = d1; t[4 * i + 3] = b1;
    }
    __syncthreads();
    if (i < 4) {
        long long a1 = (int32_t)t[4 * 0 + i], b1 = (int32_t)t[4 * 1 + i], c1 = (int32_t)t[4 * 2 + i], d1 = (int32_t)t[4 * 3 + i];
        a1 += b1; d1 -= c1;
        const long long e1 = (a1 - d1) >> 1;
        b1 = e1 - b1; c1 = e1 - c1; a1 -= c1; d1 += b1;
        out[4 * 0 + i] = (int32_t)(a1 * 4); out[4 * 1 + i] = (int32_t)(c1 * 4); out[4 * 2 + i] = (int32_t)(d1 * 4); out[4 * 3 + i] = (int32_t)(b1 * 4);
    }
}

// svt_av1_compute_cul_level_c (full_loop.c:1449-1465): min(63, sum of |level| over the first eob scan positions), DC sign in bits 6-7
__global__ void cul_level_kernel(const int16_t* __restrict__ scan, const int32_t* __restrict__ q, int eob, int32_t* __restrict__ out) {
    __shared__ unsigned int s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
    unsigned int acc = 0;
    for (int c = threadIdx.x; c < eob; c += blockDim.x) {
        const int32_t v = q[scan[c]];
        const unsigned int l = (unsigned int)(v < 0 ? -(long long)v : v);
        acc += l > 63u ? 63u : l;  // a single level >= 63 already saturates the result: clamping keeps the sum from wrapping
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s, acc);
    __syncthreads();
    if (threadIdx.x == 0) {
        int32_t cul = (int32_t)(s < 63u ? s : 63u);
        const int32_t dc = q[0];
        if (dc < 0) cul |= 1 << 6;
        else if (dc > 0) cul += 2 << 6;
        *out = cul;
    }
}

}  // namespace b200

using namespace b200;

// T1: hadamard_path (aom_dsp_rtcd.h:582).  Buf2D = {uint8_t* buf; uint8_t* buf0; int width, height, stride} (definitions.h:243).
extern "C" uint32_t svt_b200_hadamard_path(SvtB200Buf2D residual, SvtB200Buf2D coeff, SvtB200Buf2D input, SvtB200Buf2D pred, uint8_t bsize) {
    static const uint8_t wide[22] = {4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 128, 128, 4, 16, 8, 32, 16, 64};           // block_size_wide
    static const uint8_t maxtx[22] = {4, 4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 64, 4, 4, 8, 8, 16, 16};                // max_txsize_lookup, in pixels
    require_ready();
    if (bsize >= 22) { fprintf(stderr, "[svt_b200] FATAL: hadamard_path: bad block size %d\n", bsize); abort(); }
    const int n = maxtx[bsize] > 32 ? 32 : maxtx[bsize];  // AOMMIN(TX_32X32, max_txsize_lookup[bsize])
    const int side = wide[bsize];                          // the reference walks block_size_wide in BOTH directions
    const int per_row = side / n, nblk = per_row * per_row;
    LaneGuard l;
    size_t o_in = l->alloc((size_t)side * side), o_pr = l->alloc((size_t)side * side);
    size_t in_end = l->used;
    size_t o_satd = l->alloc((size_t)nblk * 4), o_res = l->alloc((size_t)n * n * 2), o_co = l->alloc((size_t)n * n * 4);
    for (int r = 0; r < side; r++) {
        memcpy(l->h<uint8_t>(o_in) + (size_t)r * side, input.buf + (size_t)r * input.stride, side);
        memcpy(l->h<uint8_t>(o_pr) + (size_t)r * side, pred.buf + (size_t)r * pred.stride, side);
    }
    l->h2d(0, in_end);
    HadPathArgs a = {l->d<uint8_t>(o_in), l->d<uint8_t>(o_pr), side, side, n, per_row, nblk};
    hadamard_path_kernel<<<nblk, 128, 0, l->stream>>>(a, l->d<int32_t>(o_satd), l->d<int16_t>(o_res), l->d<int32_t>(o_co));
    B200_LAUNCH_CHECK();
    l->d2h(o_satd, (o_co + (size_t)n * n * 4) - o_satd);
    l->sync();
    uint32_t cost = 0;
    for (int i = 0; i < nblk; i++) cost += (uint32_t)l->h<int32_t>(o_satd)[i];
    // the loop of the reference leaves the LAST block's residual (at its stride) and coefficients in the caller's buffers
    int16_t* rb = reinterpret_cast<int16_t*>(residual.buf);
    for (int r = 0; r < n; r++) memcpy(rb + (size_t)r * residual.stride, l->h<int16_t>(o_res) + (size_t)r * n, (size_t)n * 2);
    memcpy(coeff.buf, l->h<int32_t>(o_co), (size_t)n * n * 4);
    return cost;
}

// T1: svt_av1_fwht4x4 (aom_dsp_rtcd.h:208)
extern "C" void svt_b200_av1_fwht4x4(int16_t* input, int32_t* output, uint32_t stride) {
    require_ready();
    LaneGuard l;
    size_t o_in = l->alloc(32);
    size_t in_end = l->used;
    size_t o_out = l->alloc(64);
    for (int r = 0; r < 4; r++) memcpy(l->h<int16_t>(o_in) + 4 * r, input + (size_t)r * stride, 8);
    l->h2d(0, in_end);
    fwht4x4_kernel<<<1, 32, 0, l->stream>>>(l->d<int16_t>(o_in), l->d<int32_t>(o_out));
    B200_LAUNCH_CHECK();
    l->d2h(o_out, 64);
    l->sync();
    memcpy(output, l->h<int32_t>(o_out), 64);
}

// T1: svt_av1_compute_cul_level (aom_dsp_rtcd.h:904)
extern "C" uint8_t svt_b200_av1_compute_cul_level(const int16_t* const scan, const int32_t* const quant_coeff, uint16_t* eob) {
    require_ready();
    const int n = *eob;
    int maxpos = 0;
    for (int c = 0; c < n; c++) maxpos = scan[c] > maxpos ? scan[c] : maxpos;
    LaneGuard l;
    size_t o_sc = l->alloc((size_t)(n > 0 ? n : 1) * 2), o_q = l->alloc((size_t)(maxpos + 1) * 4);
    size_t in_end = l->used;
    size_t o_out = l->alloc(16);
    if (n) memcpy(l->h<int16_t>(o_sc), scan, (size_t)n * 2);
    memcpy(l->h<int32_t>(o_q), quant_coeff, (size_t)(maxpos + 1) * 4);
    l->h2d(0, in_end);
    cul_level_kernel<<<1, 128, 0, l->stream>>>(l->d<int16_t>(o_sc), l->d<int32_t>(o_q), n, l->d<int32_t>(o_out));
    B200_LAUNCH_CHECK();
    l->d2h(o_out, 4);
    l->sync();
    return (uint8_t)*l->h<int32_t>(o_out);
}

extern "C" void svt_b200_aom_hadamard_4x4(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff) { hadamard_t1(src_diff, src_stride, coeff, 4); }
extern "C" void svt_b200_aom_hadamard_8x8(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff) { hadamard_t1(src_diff, src_stride, coeff, 8); }
extern "C" void svt_b200_aom_hadamard_16x16(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff) { hadamard_t1(src_diff, src_stride, coeff, 16); }
extern "C" void svt_b200_aom_hadamard_32x32(const int16_t* src_diff, ptrdiff_t src_stride, int32_t* coeff) { hadamard_t1(src_diff, src_stride, coeff, 32); }

extern "C" int svt_b200_aom_satd(const int32_t* coeff, int length) {
    require_ready();
    if (length <= 0) return 0;
    LaneGuard l;
    size_t o_c = l->alloc((size_t)length * 4);
    size_t in_end = l->used;
    size_t o_o = l->alloc(16);
    memcpy(l->h<int32_t>(o_c), coeff, (size_t)length * 4);
    l->h2d(0, in_end);
    satd_kernel<<<1, 256, 0, l->stream>>>(l->d<int32_t>(o_c), length, l->d<int32_t>(o_o));
    B200_LAUNCH_CHECK();
    l->d2h(o_o, 4);
    l->sync();
    return *l->h<int32_t>(o_o);
}

extern "C" int svt_b200_hadamard_satd_batch_dev(const int16_t* d_residual, const SvtB200HadamardItem* d_items, int n_items,
                                                int32_t* d_coeff_or_null, int32_t* d_satd, void* stream) {
    require_ready();
    if (n_items <= 0) return n_items == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    hadamard_kernel<<<grid_for(n_items, 8), 128, 0, (cudaStream_t)stream>>>(d_residual, d_items, n_items, d_coeff_or_null, d_satd);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}
