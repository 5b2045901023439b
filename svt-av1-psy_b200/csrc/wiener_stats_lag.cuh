// wiener_stats_lag.cuh -- K11 Wiener statistics by LAG sums (sm_90a), included by wiener.cu.
//
// Reference: svt_av1_compute_stats_c / _highbd_c (Source/Lib/Codec/restoration_pick.c:659-745).  With y_p(i,j) =
// dgd(i + lr_p, j + kc_p) - avg the window sample p of pixel (i,j) (p = (kc + half) * win + (lr + half)) and x = src - avg,
//     M[p] = sum_unit x y_p          H[p][q] = sum_unit y_p y_q .
// Brute force costs win^2 (win^2 + 1) / 2 + win^2 = 1274 multiply-accumulates per pixel (7x7).  But y_p y_q only depends on
// the LAG (dy, dx) = (lr_q - lr_p, kc_q - kc_p): H[p][q] is the sum of the lag's product image P(u,v) = Y(u,v) Y(u+dy, v+dx)
// over the unit rectangle shifted by (lr_p, kc_p).  All win^2 shifted rectangles of a lag share the CORE
// [vs+half, ve-half) x [hs+half, he-half) and differ in a frame of 2*half rows / columns around it.  So, exactly, in integers:
//     H[p][q] = CC(lag) + sum of the edge-row sums RS(lag, u) that the shifted rectangle contains
//                       + sum of the edge-column sums CS(lag, v) ...   + the <= (2 half)^2 corner products,
// with RAW pixels (no mean removed: products are non-negative, 8-bit pictures take four multiply-accumulates per DP4A) and
// the mean folded back in at the end:  sum (y-a)(z-a) = sum yz - a (sum y + sum z) + N a^2  (a = the integer average).
// That is (2 win - 1) win - (win - 1) = 85 lags + 49 cross lags for M per pixel instead of 1274, identical results, same code for
// 8 / 10 / 12 bit.  Measured on the previous target GPU (1080p, ncu): the 8-bit form cost more instructions than the
// tensor-core Gram matrix of that time (57 M vs 31 M warp instructions per picture -- the partner extraction dominates), so
// 8-bit pictures use the tensor cores (stats_imma_kernel, wiener.cu); for 10 / 12 bit, where no exact tensor-core form
// exists, it replaces the 49-MAC-per-pixel integer kernel and halves the call.
//
//   stats_lag_bulk_kernel   CC of every lag, sum x Y(shift) for M, plain pixel sums: one CTA per (8-row band, unit); warp g owns
//                           the lags with dy = g and the M shifts with lr = g - half; partner words come from a 5 / 7 word
//                           window per row with compile-time funnel shifts.
//   stats_lag_edges_kernel  RS / CS: the 4 half edge rows and columns of every lag.
//   stats_lag_finalize      assembles H (both triangles) and M, applies the mean correction and the bit-depth divider.
#pragma once

namespace b200 {

constexpr int kLagSlots = 92;                 // dy * 13 + (dx + 6) for the 7x7 geometry, slot 91 = "ones" (plain pixel sums)
constexpr int kLagOnes = 91;
constexpr int kLagAccStride = 144;            // per item: [0,92) CC, [92,141) sum x Y(shift p), [141] sum x
constexpr int kLagEdge = 12;                  // edge rows (columns) per lag: 2 groups of 2 * half <= 6
constexpr int kLagItemWords = kLagAccStride + 2 * kLagSlots * kLagEdge;  // + RS + CS  (uint64 each)
constexpr int kLagBandRows = 8;

template <typename PIX> struct LagPix;
template <> struct LagPix<uint8_t> {
    static constexpr int G = 4, OFFP = 8;     // pixels per 32-bit word; pixels between the tile row origin and the first core column
    static constexpr uint32_t ONES = 0x01010101u;
    static __device__ __forceinline__ uint32_t mac(uint32_t a, uint32_t b, uint32_t acc) { return __dp4a(a, b, acc); }
};
template <> struct LagPix<uint16_t> {
    static constexpr int G = 2, OFFP = 6;
    static constexpr uint32_t ONES = 0x00010001u;
    static __device__ __forceinline__ uint32_t mac(uint32_t a, uint32_t b, uint32_t acc) {
        return acc + (a & 0xffffu) * (b & 0xffffu) + (a >> 16) * (b >> 16);
    }
};

// edge rows of a unit: slot i < 2 half -> vs - half + i; slot 2 half + i -> max(ve - half, vs + half) + i (invalid when >= ve + half)
__host__ __device__ __forceinline__ int lag_edge_line(int lo, int hi, int half, int i) {
    if (i < 2 * half) return lo - half + i;
    const int b0 = (hi - half) > (lo + half) ? (hi - half) : (lo + half);
    const int l = b0 + (i - 2 * half);
    return l < hi + half ? l : 0x7fffffff;
}

constexpr int kLagSegW = 512;  // pixels per column segment of a work unit (any unit width is handled: segments are additive)

// grid = (CTAs per unit, units); a CTA walks the (row band, column segment) work units of its restoration unit
template <typename PIX, int WIN>
__global__ void __launch_bounds__(256)
stats_lag_bulk_kernel(const PIX* __restrict__ dgd_base, const PIX* __restrict__ src_base, const SvtB200StatsItem* __restrict__ items,
                      unsigned long long* __restrict__ acc_base) {
    using P = LagPix<PIX>;
    constexpr int HALF = WIN >> 1, S = (int)sizeof(PIX), G = P::G, OFFB = P::OFFP * S;
    constexpr int NW = (OFFB + (WIN - 1) * S + 3) / 4 + 1;  // words of the partner window of one core word (5 for 8-bit, 7 for 16-bit at 7x7)
    constexpr int PITCH = (OFFB + (kLagSegW + 2 * (WIN - 1)) * S + 3) / 4 + NW + 1;  // words per Y tile row
    constexpr int XPITCH = (kLagSegW * S + 3) / 4 + 1;
    constexpr int TROWS = kLagBandRows + 3 * HALF;
    const SvtB200StatsItem s = items[blockIdx.y];
    if (s.wiener_win != WIN) return;
    const int hs = s.h_start, he = s.h_end, vs = s.v_start, ve = s.v_end, w = he - hs, h = ve - vs;
    const int cu0 = vs + HALF, cu1 = ve - HALF, cv0 = hs + HALF, cv1 = he - HALF;
    extern __shared__ __align__(16) uint32_t lag_sm[];
    uint32_t* Yt = lag_sm;                  // rows [b0 - HALF, b1 + 2 HALF), row byte 0 = pixel column cv0 + c0 - OFFP; outside the halo'd unit: 0
    uint32_t* Xt = lag_sm + TROWS * PITCH;  // rows [b0, b1) of the source, word 0 = column hs + c0
    const PIX* dgd = dgd_base + s.dgd_off;
    const PIX* src = src_base + s.src_off;
    const int g = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __shared__ unsigned long long s_tot[kLagAccStride];  // the CTA's share of CC / sum x Y / sum x, flushed to global at the end
    for (int i = threadIdx.x; i < kLagAccStride; i += blockDim.x) s_tot[i] = 0;
    unsigned long long* acc = acc_base + (size_t)blockIdx.y * kLagItemWords;
    // warp-wide sum of a 32-bit partial (a work unit's partial cannot overflow: 8 rows x 512 columns / 32 lanes of <= 2 x 4095^2)
    auto wsum = [&](uint32_t v) {
        unsigned long long t = v;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        return t;
    };
    const int nbands = (h + kLagBandRows - 1) / kLagBandRows, nsegs = (w + kLagSegW - 1) / kLagSegW;
    for (int wu = blockIdx.x; wu < nbands * nsegs; wu += gridDim.x) {
        const int band = wu / nsegs, seg = wu - band * nsegs;
        const int b0 = vs + band * kLagBandRows, b1 = min(b0 + kLagBandRows, ve), c0 = seg * kLagSegW;
        const int cw = max(min(cv1 - (cv0 + c0), kLagSegW), 0);  // core columns of this segment
        const int xw = min(w - c0, kLagSegW);                      // unit columns of this segment
        __syncthreads();
        {
            PIX* yb = reinterpret_cast<PIX*>(Yt);
            constexpr int PPR = PITCH * 4 / S;  // pixels per tile row
            const int trows = (b1 - b0) + 3 * HALF;
            // only the columns this segment can touch (a 128-wide chroma unit does not pay for a 512-wide tile)
            int spx = P::OFFP + xw + 2 * WIN + 2 * G;
            spx = spx < PPR ? (spx + G - 1) / G * G : PPR;
            for (int tr = g; tr < trows; tr += 8) {  // a warp per tile row: no index division, coalesced runs
                const int u = b0 - HALF + tr;
                const bool rin = u >= vs - HALF && u < ve + HALF;
                const PIX* grow = dgd + (ptrdiff_t)u * s.dgd_stride + (cv0 + c0 - P::OFFP);
                PIX* trow_p = yb + tr * PPR;
                const int vlo = hs - HALF - (cv0 + c0 - P::OFFP), vhi = he + HALF - (cv0 + c0 - P::OFFP);  // valid tile columns
                for (int tc = lane; tc < spx; tc += 32) trow_p[tc] = (rin && tc >= vlo && tc < vhi) ? grow[tc] : (PIX)0;
            }
            PIX* xb = reinterpret_cast<PIX*>(Xt);
            constexpr int XPR = XPITCH * 4 / S;
            const int xsp = min(XPR, (xw + G - 1) / G * G + G);
            for (int tr = g; tr < b1 - b0; tr += 8) {
                const PIX* grow = src + (ptrdiff_t)(b0 + tr) * s.src_stride + hs + c0;
                for (int tc = lane; tc < xsp; tc += 32) xb[tr * XPR + tc] = tc < xw ? grow[tc] : (PIX)0;
            }
        }
        __syncthreads();
        uint32_t accH[2 * WIN - 1], accM[WIN], accY = 0, accX = 0;
#pragma unroll
        for (int k = 0; k < 2 * WIN - 1; k++) accH[k] = 0;
#pragma unroll
        for (int k = 0; k < WIN; k++) accM[k] = 0;
        const int ncw = (cw + G - 1) / G, nxw = (xw + G - 1) / G;  // words of a core row / of a unit row of this segment
        if (g < WIN) {
            // ---- H lags with dy = g: A = core-column word of row u, partner words from row u + g.  Core rows add up in accH (-> CC);
            // the unit's edge rows [vs - HALF, vs + HALF) and [ve - HALF, ve + HALF) are done the same way but each keeps its own sums
            // (-> RS).  Band b covers unit rows [b0, b1); the HALF rows above the unit ride with band 0, the HALF below with the last.
            const int dy = g;
            const int a0 = band == 0 ? vs - HALF : b0, a1 = (b1 == ve) ? ve + HALF : b1;
            for (int u = a0; u < a1; u++) {
                if (u + dy >= ve + HALF) break;  // partner row outside the halo: no shifted rectangle uses it
                const bool core_row = u >= cu0 && u < cu1;
                // rows [b0 - HALF, b0) of later bands were handled as rows of the previous band
                const int trow = u - (b0 - HALF);
                if (trow < 0 || trow + dy >= (b1 - b0) + 3 * HALF) continue;
                uint32_t accR[2 * WIN - 1];
#pragma unroll
                for (int k = 0; k < 2 * WIN - 1; k++) accR[k] = 0;
                const uint32_t* arow = Yt + trow * PITCH + OFFB / 4;
                const uint32_t* brow = Yt + (trow + dy) * PITCH;
                for (int wc = lane; wc < ncw; wc += 32) {
                    uint32_t a = arow[wc];
                    const int rem = cw - wc * G;  // pixels of this word inside the core columns
                    if (rem < G) a &= (1u << (rem * 8 * S)) - 1u;
                    uint32_t win_w[NW];
#pragma unroll
                    for (int k = 0; k < NW; k++) win_w[k] = brow[wc + k];
#pragma unroll
                    for (int k = 0; k < 2 * WIN - 1; k++) {
                        const int dx = k - (WIN - 1);
                        const int rel = OFFB + dx * S;  // byte offset of the partner inside the window (compile-time after unrolling)
                        const uint32_t b = (rel & 3) ? __funnelshift_r(win_w[rel >> 2], win_w[(rel >> 2) + 1], (rel & 3) * 8) : win_w[rel >> 2];
                        if (dy > 0 || dx >= 0) accR[k] = P::mac(a, b, accR[k]);
                    }
                }
                if (core_row) {
#pragma unroll
                    for (int k = 0; k < 2 * WIN - 1; k++) accH[k] += accR[k];
                } else {  // edge row: slot index of u in the unit's edge-row list
                    int ei = -1;
                    for (int i = 0; i < 4 * HALF; i++)
                        if (lag_edge_line(vs, ve, HALF, i) == u) ei = i;
#pragma unroll
                    for (int k = 0; k < 2 * WIN - 1; k++) {
                        if (!(dy > 0 || k >= WIN - 1)) continue;
                        const unsigned long long t = wsum(accR[k]);
                        if (lane == 0 && t && ei >= 0) atomicAdd(&acc[kLagAccStride + (dy * 13 + (k - (WIN - 1)) + 6) * kLagEdge + ei], t);
                    }
                }
            }
            // ---- M shifts with lr = g - HALF: A = source word of unit row u, partners = Y(u + lr, column + kc) -------------------
            const int lr = g - HALF;
            for (int u = b0; u < b1; u++) {
                const uint32_t* arow = Xt + (u - b0) * XPITCH;
                const uint32_t* brow = Yt + (u + lr - (b0 - HALF)) * PITCH;
                for (int wc = lane; wc < nxw; wc += 32) {
                    const uint32_t a = arow[wc];  // columns >= xw were staged as 0
                    uint32_t win_w[NW];
#pragma unroll
                    for (int k = 0; k < NW; k++) win_w[k] = brow[wc + k];
#pragma unroll
                    for (int k = 0; k < WIN; k++) {
                        const int kc = k - HALF;
                        const int rel = (P::OFFP - HALF + kc) * S;
                        const uint32_t b = (rel & 3) ? __funnelshift_r(win_w[rel >> 2], win_w[(rel >> 2) + 1], (rel & 3) * 8) : win_w[rel >> 2];
                        accM[k] = P::mac(a, b, accM[k]);
                    }
                }
            }
        } else if (g == WIN) {
            // ---- plain sums: Y over the core rows ("ones" lag; edge rows -> its RS), x over the unit rows --------------------------------
            const int a0 = band == 0 ? vs - HALF : b0, a1 = (b1 == ve) ? ve + HALF : b1;
            for (int u = a0; u < a1; u++) {
                const int trow = u - (b0 - HALF);
                if (trow < 0 || trow >= (b1 - b0) + 3 * HALF) continue;
                const bool core_row = u >= cu0 && u < cu1;
                uint32_t accR = 0;
                const uint32_t* arow = Yt + trow * PITCH + OFFB / 4;
                for (int wc = lane; wc < ncw; wc += 32) {
                    uint32_t a = arow[wc];
                    const int rem = cw - wc * G;
                    if (rem < G) a &= (1u << (rem * 8 * S)) - 1u;
                    accR = P::mac(a, P::ONES, accR);
                }
                if (core_row) accY += accR;
                else {
                    int ei = -1;
                    for (int i = 0; i < 4 * HALF; i++)
                        if (lag_edge_line(vs, ve, HALF, i) == u) ei = i;
                    const unsigned long long t = wsum(accR);
                    if (lane == 0 && t && ei >= 0) atomicAdd(&acc[kLagAccStride + kLagOnes * kLagEdge + ei], t);
                }
            }
            for (int u = b0; u < b1; u++) {
                const uint32_t* arow = Xt + (u - b0) * XPITCH;
                for (int wc = lane; wc < nxw; wc += 32) accX = P::mac(arow[wc], P::ONES, accX);
            }
        }
        // the work unit's partial sums: warp-reduce, then into the CTA's 64-bit totals
        if (g < WIN) {
#pragma unroll
            for (int k = 0; k < 2 * WIN - 1; k++) {
                if (!(g > 0 || k >= WIN - 1)) continue;
                const unsigned long long t = wsum(accH[k]);
                if (lane == 0 && t) atomicAdd(&s_tot[g * 13 + (k - (WIN - 1)) + 6], t);
            }
#pragma unroll
            for (int k = 0; k < WIN; k++) {
                const unsigned long long t = wsum(accM[k]);
                if (lane == 0 && t) atomicAdd(&s_tot[kLagSlots + k * WIN + g], t);  // p = (kc + half) * win + (lr + half)
            }
        } else if (g == WIN) {
            const unsigned long long ty = wsum(accY), tx = wsum(accX);
            if (lane == 0) { atomicAdd(&s_tot[kLagOnes], ty); atomicAdd(&s_tot[kLagSlots + 49], tx); }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kLagAccStride; i += blockDim.x)
        if (s_tot[i]) atomicAdd(&acc[i], s_tot[i]);
}

template <typename PIX, int WIN>
constexpr size_t lag_bulk_smem() {
    using P = LagPix<PIX>;
    constexpr int S = (int)sizeof(PIX), OFFB = P::OFFP * S, NW = (OFFB + (WIN - 1) * S + 3) / 4 + 1;
    constexpr int PITCH = (OFFB + (kLagSegW + 2 * (WIN - 1)) * S + 3) / 4 + NW + 1, XPITCH = (kLagSegW * S + 3) / 4 + 1;
    return (size_t)((kLagBandRows + 3 * (WIN >> 1)) * PITCH + kLagBandRows * XPITCH) * 4;
}

// CS(lag, edge column v) = sum over the core rows of P(u, v): one warp per (edge column, dy), lanes over the rows, all dx of the
// dy at once (the 2 win - 1 partners of a row are neighbours).  RS is produced by the bulk kernel.  grid = (12 edge columns, units), 8 warps
template <typename PIX>
__global__ void __launch_bounds__(256)
stats_lag_edges_kernel(const PIX* __restrict__ dgd_base, const SvtB200StatsItem* __restrict__ items, unsigned long long* __restrict__ acc_base) {
    const SvtB200StatsItem s = items[blockIdx.y];
    const int win = s.wiener_win, half = win >> 1;
    const int hs = s.h_start, he = s.h_end, vs = s.v_start, ve = s.v_end;
    const int cu0 = vs + half, cu1 = ve - half;
    const PIX* dgd = dgd_base + s.dgd_off;
    unsigned long long* CS = acc_base + (size_t)blockIdx.y * kLagItemWords + kLagAccStride + kLagSlots * kLagEdge;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if ((int)blockIdx.x >= 4 * half) return;  // grid.x = 12 edge columns of the 7x7 geometry
    for (int job = blockIdx.x * (win + 1) + warp; job < (blockIdx.x + 1) * (win + 1); job += 8) {
        const int i = job / (win + 1), dy = job - i * (win + 1);  // dy == win: the "ones" lag
        const int v = lag_edge_line(hs, he, half, i);
        if (v == 0x7fffffff) continue;
        if (dy == win) {
            unsigned long long t = 0;
            for (int u = cu0 + lane; u < cu1; u += 32) t += dgd[(ptrdiff_t)u * s.dgd_stride + v];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            if (lane == 0) CS[kLagOnes * kLagEdge + i] = t;
            continue;
        }
        unsigned long long t[13];
#pragma unroll
        for (int k = 0; k < 13; k++) t[k] = 0;
        for (int u = cu0 + lane; u < cu1; u += 32) {
            const unsigned long long a = dgd[(ptrdiff_t)u * s.dgd_stride + v];
            const PIX* prow = dgd + (ptrdiff_t)(u + dy) * s.dgd_stride + v;
#pragma unroll
            for (int k = 0; k < 13; k++) {
                const int dx = k - 6;
                if (dx > -win && dx < win && v + dx >= hs - half && v + dx < he + half) t[k] += a * (unsigned long long)prow[dx];
            }
        }
#pragma unroll
        for (int k = 0; k < 13; k++) {
            unsigned long long x = t[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            const int dx = k - 6;
            if (lane == 0 && dx > -win && dx < win && (dy > 0 || dx >= 0)) CS[(dy * 13 + k) * kLagEdge + i] = x;
        }
    }
}

// sum of a lag's product image over the unit rectangle shifted by (ar, ac): core + contained edge rows / columns + corners
template <typename PIX>
__device__ long long lag_rect_sum(const PIX* dgd, const SvtB200StatsItem& s, const unsigned long long* acc, int slot, bool ones, int dy, int dx,
                                  int ar, int ac) {
    const int half = s.wiener_win >> 1, hs = s.h_start, he = s.h_end, vs = s.v_start, ve = s.v_end;
    const unsigned long long* RS = acc + kLagAccStride + slot * kLagEdge;
    const unsigned long long* CS = acc + kLagAccStride + kLagSlots * kLagEdge + slot * kLagEdge;
    long long tot = (long long)acc[slot];
    for (int i = 0; i < 4 * half; i++) {
        const int u = lag_edge_line(vs, ve, half, i);
        if (u != 0x7fffffff && u >= vs + ar && u < ve + ar) tot += (long long)RS[i];
        const int v = lag_edge_line(hs, he, half, i);
        if (v != 0x7fffffff && v >= hs + ac && v < he + ac) tot += (long long)CS[i];
    }
    for (int i = 0; i < 4 * half; i++) {
        const int u = lag_edge_line(vs, ve, half, i);
        if (u == 0x7fffffff || u < vs + ar || u >= ve + ar) continue;
        for (int j = 0; j < 4 * half; j++) {
            const int v = lag_edge_line(hs, he, half, j);
            if (v == 0x7fffffff || v < hs + ac || v >= he + ac) continue;
            const long long a = dgd[(ptrdiff_t)u * s.dgd_stride + v];
            tot += ones ? a : a * (long long)dgd[(ptrdiff_t)(u + dy) * s.dgd_stride + v + dx];
        }
    }
    return tot;
}

// grid = (ceil((win2 (win2 + 1) / 2 + win2) / 128), items)
template <typename PIX>
__global__ void __launch_bounds__(128)
stats_lag_finalize_kernel(const PIX* __restrict__ dgd_base, const SvtB200StatsItem* __restrict__ items, const unsigned long long* __restrict__ acc_base,
                          const unsigned long long* __restrict__ tot, int divider, long long* __restrict__ M_out, long long* __restrict__ H_out) {
    const int it = blockIdx.y;
    const SvtB200StatsItem s = items[it];
    const int win = s.wiener_win, half = win >> 1, win2 = win * win;
    const int npairs = win2 * (win2 + 1) / 2;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long* acc = acc_base + (size_t)it * kLagItemWords;
    const PIX* dgd = dgd_base + s.dgd_off;
    __shared__ long long s_sy[49];  // plain pixel sums of the win^2 shifted rectangles (every H and M entry needs two / one of them)
    if (threadIdx.x < win2) s_sy[threadIdx.x] = lag_rect_sum<PIX>(dgd, s, acc, kLagOnes, true, 0, 0, threadIdx.x % win - half, threadIdx.x / win - half);
    __syncthreads();
    if (e >= npairs + win2) return;
    const long long N = (long long)(s.h_end - s.h_start) * (s.v_end - s.v_start);
    const long long avg = (long long)(tot[it] / (unsigned long long)N);  // find_average
    if (e >= npairs) {  // M[p] = sum x y_p - a sum x - a sum Y_p + N a^2
        const int p = e - npairs, kc = p / win - half, lr = p % win - half;
        const long long sy = s_sy[p];
        (void)kc; (void)lr;
        const long long m = (long long)acc[kLagSlots + p] - avg * (long long)acc[kLagSlots + 49] - avg * sy + N * avg * avg;
        M_out[(size_t)it * 49 + p] = m / divider;
        return;
    }
    // e -> (p, q), p <= q, rows of the upper triangle in order
    int p = 0, rem = e;
    while (rem >= win2 - p) { rem -= win2 - p; p++; }
    const int q = p + rem;
    const int kp = p / win - half, lp = p % win - half, kq = q / win - half, lq = q % win - half;
    int dy = lq - lp, dx = kq - kp, ar = lp, ac = kp;
    if (dy < 0 || (dy == 0 && dx < 0)) { dy = -dy; dx = -dx; ar = lq; ac = kq; }
    const long long syy = lag_rect_sum<PIX>(dgd, s, acc, dy * 13 + dx + 6, false, dy, dx, ar, ac);
    const long long sp = s_sy[p], sq = s_sy[q];
    const long long hv = (syy - avg * (sp + sq) + N * avg * avg) / divider;
    H_out[(size_t)it * 2401 + p * win2 + q] = hv;
    H_out[(size_t)it * 2401 + q * win2 + p] = hv;
}

}  // namespace b200
