// wiener_unit.cuh -- the arithmetic of one separable Wiener unit (<= 64 x 64) out of a staged shared-memory tile:
// shared by wiener_convolve_kernel (wiener.cu: plain units) and lr_filter_kernel (restoration.cu: stripe-aware units).
// s_src: rows -3 .. h+3 of the input in the picture's own pixel type at pitch kWienerTilePitch; element 0 of a row is
// column -4 (never read), so that the columns -3 .. w+4 the filter reads start one element into a 4-byte word and a
// stager can move whole aligned words; s_tmp: (64 + 8) x 64 uint16 scratch.
// Follows svt_av1_wiener_convolve_add_src_c / svt_av1_highbd_wiener_convolve_add_src_c (convolve.c:100-147, 194-237).
#pragma once
#include <cstdint>

namespace b200 {

constexpr int kWienerTilePitch = 80;      // elements: 4 + 64 + 5 columns, rounded up to whole 16-byte groups
constexpr int kWienerTileRows = 64 + 8;

__device__ __forceinline__ int round_pow2_s(int v, int n) { return (v + ((1 << n) >> 1)) >> n; }

// c + sum of four (unsigned byte of a) x (signed byte of b)
__device__ __forceinline__ int dp4a_u8s8(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// tile elements c .. c+11 of a row (c a multiple of 4): four adjacent outputs read elements 1 .. 11 of them
__device__ __forceinline__ void wiener_load12(const uint8_t* p, int x[12]) {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(p);
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const uint32_t v = q[i];
        x[4 * i] = (int)(v & 0xff); x[4 * i + 1] = (int)((v >> 8) & 0xff); x[4 * i + 2] = (int)((v >> 16) & 0xff); x[4 * i + 3] = (int)(v >> 24);
    }
}
__device__ __forceinline__ void wiener_load12(const uint16_t* p, int x[12]) {
    const uint2* q = reinterpret_cast<const uint2*>(p);
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const uint2 v = q[i];
        x[4 * i] = (int)(v.x & 0xffff); x[4 * i + 1] = (int)(v.x >> 16); x[4 * i + 2] = (int)(v.y & 0xffff); x[4 * i + 3] = (int)(v.y >> 16);
    }
}

// item i of a pass over rows of `w4` four-pixel groups -> (row, first column); 64- and 32-wide units need no division
__device__ __forceinline__ void wiener_item(int i, int w4, int& r, int& c) {
    if (w4 == 16) { r = i >> 4; c = (i & 15) << 2; }
    else if (w4 == 8) { r = i >> 3; c = (i & 7) << 2; }
    else { r = i / w4; c = (i - r * w4) << 2; }
}

template <typename PIX>
__device__ __forceinline__ void wiener_unit_compute(const PIX* s_src, uint16_t* s_tmp, PIX* dst, int dst_stride, int w, int h,
                                                    const int16_t* hfilter, const int16_t* vfilter, int bd, int round0, int round1,
                                                    int lbd_rows) {
    constexpr int P = kWienerTilePitch;
    const int sh = h + 7;
    const int limit = (1 << (bd + 1 + 7 - round0)) - 1;
    // horizontal: intermediate rows -3..h+3; the low-bit-depth reference computes h+6 rows and
    // zero-fills the last one (convolve.c:113-121)
    const int hrows = lbd_rows ? h + 6 : h + 7;
    const int pmax = (1 << bd) - 1;
    if ((w & 3) == 0) {
        // four adjacent outputs per thread in the horizontal pass, four columns of two rows in the vertical one
        int hf[8], vf[8];
        bool byte_taps = sizeof(PIX) == 1;  // every legal AV1 tap fits a signed byte; the ABI takes any int16
#pragma unroll
        for (int k = 0; k < 8; k++) {
            hf[k] = hfilter[k];
            vf[k] = vfilter[k];
            byte_taps = byte_taps && hf[k] >= -128 && hf[k] <= 127;
        }
        const int w4 = w >> 2;
        const int hoff = 1 << (bd + 6);
        if constexpr (sizeof(PIX) == 1) {
            if (byte_taps) {
                // bytes x signed-byte taps: the 8 taps of an output are two dp4a on words cut from the three loaded ones
                const uint32_t t_lo = (uint32_t)(hf[0] & 0xff) | ((uint32_t)(hf[1] & 0xff) << 8) | ((uint32_t)(hf[2] & 0xff) << 16) | ((uint32_t)(hf[3] & 0xff) << 24);
                const uint32_t t_hi = (uint32_t)(hf[4] & 0xff) | ((uint32_t)(hf[5] & 0xff) << 8) | ((uint32_t)(hf[6] & 0xff) << 16) | ((uint32_t)(hf[7] & 0xff) << 24);
                for (int i = threadIdx.x; i < sh * w4; i += blockDim.x) {
                    int r, c;
                    wiener_item(i, w4, r, c);
                    uint2 out = make_uint2(0u, 0u);
                    if (r < hrows) {
                        const uint32_t* q = reinterpret_cast<const uint32_t*>(s_src + r * P + c);
                        const uint32_t  a = q[0], b = q[1], d = q[2];
                        int v[4];
#pragma unroll
                        for (int o = 0; o < 4; o++) {
                            // output o reads elements o+1 .. o+8; its centre (add-src) pixel, element o+4, is the top byte of the low word
                            const uint32_t lo = o == 3 ? b : __funnelshift_r(a, b, 8 * (o + 1));
                            const uint32_t hi = o == 3 ? d : __funnelshift_r(b, d, 8 * (o + 1));
                            const int sum = dp4a_u8s8(hi, t_hi, dp4a_u8s8(lo, t_lo, (int)((lo >> 24) << 7) + hoff));
                            const int t = round_pow2_s(sum, round0);
                            v[o] = t < 0 ? 0 : (t > limit ? limit : t);
                        }
                        out = make_uint2((uint32_t)v[0] | ((uint32_t)v[1] << 16), (uint32_t)v[2] | ((uint32_t)v[3] << 16));
                    }
                    *reinterpret_cast<uint2*>(s_tmp + r * 64 + c) = out;
                }
            }
        }
        if (!byte_taps) {
            for (int i = threadIdx.x; i < sh * w4; i += blockDim.x) {
                int r, c;
                wiener_item(i, w4, r, c);
                uint2 out = make_uint2(0u, 0u);
                if (r < hrows) {
                    int x[12], v[4];
                    wiener_load12(s_src + r * P + c, x);
#pragma unroll
                    for (int o = 0; o < 4; o++) {
                        int sum = (x[o + 4] << 7) + hoff;
#pragma unroll
                        for (int k = 0; k < 8; k++) sum += x[o + 1 + k] * hf[k];
                        const int t = round_pow2_s(sum, round0);
                        v[o] = t < 0 ? 0 : (t > limit ? limit : t);
                    }
                    out = make_uint2((uint32_t)v[0] | ((uint32_t)v[1] << 16), (uint32_t)v[2] | ((uint32_t)v[3] << 16));
                }
                *reinterpret_cast<uint2*>(s_tmp + r * 64 + c) = out;
            }
        }
        __syncthreads();
        // one store per four pixels where the destination rows are aligned to it
        const bool wide = (((uintptr_t)dst | ((size_t)dst_stride * sizeof(PIX))) & (4 * sizeof(PIX) - 1)) == 0;
        const int  voff = 1 << (bd + round1 - 1);
        vf[3] += 128;  // the add-src term: the centre row once more, scaled by 1 << FILTER_BITS
        for (int i = threadIdx.x; i < ((h + 1) >> 1) * w4; i += blockDim.x) {
            int r, c;
            wiener_item(i, w4, r, c);
            r *= 2;
            int sum[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
#pragma unroll
            for (int k = 0; k < 9; k++) {  // rows r .. r+8 of the intermediate feed output rows r and r+1 (r+8 <= h+6 when row r+1 exists)
                const uint2 t = *reinterpret_cast<const uint2*>(s_tmp + (r + k) * 64 + c);
                const int   e[4] = {(int)(t.x & 0xffff), (int)(t.x >> 16), (int)(t.y & 0xffff), (int)(t.y >> 16)};
#pragma unroll
                for (int o = 0; o < 4; o++) {
                    if (k < 8) sum[0][o] += e[o] * vf[k];
                    if (k > 0) sum[1][o] += e[o] * vf[k - 1];
                }
            }
#pragma unroll
            for (int j = 0; j < 2; j++) {
                if (r + j >= h) break;
                int v[4];
#pragma unroll
                for (int o = 0; o < 4; o++) {
                    v[o] = round_pow2_s(sum[j][o] - voff, round1);
                    v[o] = v[o] < 0 ? 0 : (v[o] > pmax ? pmax : v[o]);
                }
                PIX* d = dst + (ptrdiff_t)(r + j) * dst_stride + c;
                if (!wide) {
#pragma unroll
                    for (int o = 0; o < 4; o++) d[o] = (PIX)v[o];
                } else if constexpr (sizeof(PIX) == 1) {
                    *reinterpret_cast<uint32_t*>(d) = (uint32_t)v[0] | ((uint32_t)v[1] << 8) | ((uint32_t)v[2] << 16) | ((uint32_t)v[3] << 24);
                } else {
                    *reinterpret_cast<uint2*>(d) = make_uint2((uint32_t)v[0] | ((uint32_t)v[1] << 16), (uint32_t)v[2] | ((uint32_t)v[3] << 16));
                }
            }
        }
        __syncthreads();
        return;
    }
    for (int i = threadIdx.x; i < sh * w; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        int v = 0;
        if (r < hrows) {
            int sum = ((int)s_src[r * P + c + 4] << 7) + (1 << (bd + 6));
#pragma unroll
            for (int k = 0; k < 8; k++) sum += (int)s_src[r * P + c + 1 + k] * (int)hfilter[k];
            v = round_pow2_s(sum, round0);
            v = v < 0 ? 0 : (v > limit ? limit : v);
        }
        s_tmp[r * 64 + c] = (uint16_t)v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < h * w; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        int sum = ((int)s_tmp[(r + 3) * 64 + c] << 7) - (1 << (bd + round1 - 1));
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (r + k < sh) sum += (int)s_tmp[(r + k) * 64 + c] * (int)vfilter[k];
        int v = round_pow2_s(sum, round1);
        v = v < 0 ? 0 : (v > pmax ? pmax : v);
        dst[(ptrdiff_t)r * dst_stride + c] = (PIX)v;
    }
    __syncthreads();
}

}  // namespace b200
