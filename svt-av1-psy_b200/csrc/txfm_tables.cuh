// txfm_tables.cuh -- constant tables + the uniform 1-D butterfly evaluator of the 2-D transform kernel
// (txfm.cu), in its forward, inverse and fused-chain modes.
//
// AV1's 1-D DCT/ADST are multi-stage butterfly networks with a rounding shift after every rotation
// (reference: half_btf, Source/Lib/Codec/inv_transforms.h:264), so a GEMM cannot reproduce them
// bit-exactly (SURVEY.md F11).  We run the network itself: txfm_graphs.inc holds the networks as
// DATA (one packed node per (stage, element), extracted from the reference by a tool) and
// tools/gen_txfm_code.py turns that data into straight-line device functions (txfm_gen.inc) in which
// one thread holds one whole vector in registers -- stage permutations cost nothing and every
// butterfly is a handful of integer instructions.  A team of max(W,H) threads owns a block: thread v
// transforms column v, the block is handed over transposed through shared memory (odd pitch, so
// both directions are bank-conflict free), then thread r transforms row r.  In the 32- and 64-point classes a 32- or
// 64-point DCT vector is split across two lanes instead (txfm_pass_split).
#pragma once
#include <cstdint>
#include "common.cuh"

namespace b200 {

enum {  // TxfmType, Source/Lib/Codec/inv_transforms.h:91-108
    TT_DCT4, TT_DCT8, TT_DCT16, TT_DCT32, TT_DCT64, TT_ADST4, TT_ADST8, TT_ADST16, TT_ADST32,
    TT_IDTX4, TT_IDTX8, TT_IDTX16, TT_IDTX32, TT_IDTX64, TT_TYPES
};

struct TxCfg {  // per (tx_size, tx_type); dumped from the reference by tools/dump_txfm_cfg.py
    int8_t valid;
    int8_t f_ud, f_lr, f_s0, f_s1, f_s2, f_cbc, f_cbr, f_tc, f_tr;
    int8_t i_ud, i_lr, i_s0, i_s1, i_cbc, i_cbr, i_tc, i_tr;
};

// NOTE: this header is included by exactly one translation unit (txfm.cu): the symbols below are
// defined here so that no relocatable device code is needed.
__constant__ TxCfg     c_txcfg[19][16];

// cospi / sinpi of cosine bits 10..16 (dumped from the reference into txfm_cfg.inc) as compile-time tables: the networks
// take their cosine bit as a template parameter, so every weight they use folds to an instruction immediate
#define TXC(...)
#define TXSIN(...)
#define TXCOS(bit, ...) {__VA_ARGS__},
constexpr int32_t kTxCos[7][64] = {
#include "txfm_cfg.inc"
};
#undef TXCOS
#undef TXSIN
#define TXCOS(...)
#define TXSIN(bit, ...) {__VA_ARGS__},
constexpr int32_t kTxSin[7][5] = {
#include "txfm_cfg.inc"
};
#undef TXC
#undef TXCOS
#undef TXSIN
constexpr bool tx_trig_rows_in_order() {  // row k is cosine bit 10 + k: cospi[0] = 2^bit, sinpi[0] = 0
    for (int k = 0; k < 7; k++)
        if (kTxCos[k][0] != (1 << (10 + k)) || kTxCos[k][63] == 0 || kTxSin[k][0] != 0 || kTxSin[k][4] == 0) return false;
    return true;
}
static_assert(tx_trig_rows_in_order(), "txfm_cfg.inc: TXCOS / TXSIN rows of bits 10..16, in order");

// the cosine table of one cosine bit as a value: cosv[k] is a constant expression
template <int BIT> struct TxCosv {
    static_assert(BIT >= 10 && BIT <= 16, "cosine bits 10..16");
    __host__ __device__ constexpr int32_t operator[](int k) const { return kTxCos[BIT - 10][k]; }
};

// log2(dimension) - 2 of the 19 sizes, 3 bits each: a runtime-indexed constexpr array would be placed in local memory
constexpr unsigned long long kTxLgW = 0x1132846d2244688ull;  // W: 4 8 16 32 64 4 8 8 16 16 32 32 64 4 16 8 32 16 64
constexpr unsigned long long kTxLgH = 0x0a161389940c688ull;  // H: 4 8 16 32 64 8 4 16 8 32 16 64 32 16 4 32 8 64 16
__host__ __device__ constexpr int tx_w(int s) { return 4 << ((kTxLgW >> (3 * s)) & 7); }
__host__ __device__ constexpr int tx_h(int s) { return 4 << ((kTxLgH >> (3 * s)) & 7); }
constexpr bool tx_dims_packed_right() {
    constexpr int W[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
    constexpr int H[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};
    for (int s = 0; s < 19; s++)
        if (tx_w(s) != W[s] || tx_h(s) != H[s]) return false;
    return true;
}
static_assert(tx_dims_packed_right(), "kTxLgW / kTxLgH");
const TxCfg& host_txcfg(int size, int type);

constexpr int kNewSqrt2    = 5793;  // 2^12 * sqrt(2)
constexpr int kNewInvSqrt2 = 2896;  // 2^12 / sqrt(2)

__device__ __forceinline__ int32_t round_shift64(long long v, int bit) { return (int32_t)((v + (1ll << (bit - 1))) >> bit); }
// svt_av1_round_shift_array_c semantics (inv_transforms.c:2421): bit>0 rounding right shift, bit<0 multiply
__device__ __forceinline__ int32_t round_shift_arr(int32_t v, int bit) {
    if (bit == 0) return v;
    if (bit > 0) return round_shift64((long long)v, bit);
    return (int32_t)((uint32_t)v * (1u << (-bit)));
}
__device__ __forceinline__ int32_t clamp_bits(int32_t v, int bit) {
    if (bit <= 0) return v;
    const int32_t hi = (int32_t)((1ll << (bit - 1)) - 1), lo = (int32_t)(-(1ll << (bit - 1)));
    return v < lo ? lo : (v > hi ? hi : v);
}

// Team barrier.  Teams of < 32 threads share a warp with other teams that may be running a different
// block shape, so they synchronise on their own lane mask; a 64-thread team is a whole CTA.
template <int TEAM, bool SOLO = false>  // SOLO: the team is alone in its CTA and the whole CTA helps moving its data
__device__ __forceinline__ void team_sync() {
    if constexpr (TEAM >= 64 || SOLO)
        __syncthreads();
    else if constexpr (TEAM == 32)
        __syncwarp();
    else
        __syncwarp(((1u << TEAM) - 1u) << ((threadIdx.x & 31) / TEAM * TEAM));
}

// half_btf (inv_transforms.h:264): the two products wrap at 32 bits, their sum is taken in 64
__device__ __forceinline__ int32_t txg_hbtf(int32_t w0, int32_t in0, int32_t w1, int32_t in1, int bit) {
    const int32_t p0 = (int32_t)((uint32_t)w0 * (uint32_t)in0), p1 = (int32_t)((uint32_t)w1 * (uint32_t)in1);
    return (int32_t)(((long long)p0 + (long long)p1 + (1ll << (bit - 1))) >> bit);
}

// ... with one operand known to be zero
__device__ __forceinline__ int32_t txg_hbtf1(int32_t w0, int32_t in0, int bit) {
    const int32_t p0 = (int32_t)((uint32_t)w0 * (uint32_t)in0);
    return (int32_t)(((long long)p0 + (1ll << (bit - 1))) >> bit);
}

#include "txfm_gen.inc"

// Closed form of svt_av1_fadst4_new (transforms.c:1415-1502) / svt_av1_iadst4_new
// (inv_transforms.c:722-806): every intermediate is a 32-bit wrapping linear combination, so the
// four outputs are evaluated directly (mod 2^32) and rounded once.
template <bool INV, int COS_BIT>
__device__ __forceinline__ void txfm_adst4(int32_t (&x)[4]) {
    constexpr uint32_t s1 = kTxSin[COS_BIT - 10][1], s2 = kTxSin[COS_BIT - 10][2], s3 = kTxSin[COS_BIT - 10][3], s4 = kTxSin[COS_BIT - 10][4];
    const uint32_t x0 = x[0], x1 = x[1], x2 = x[2], x3 = x[3];
    uint32_t o0, o1, o2, o3;
    if (!INV) {
        o0 = s1 * x0 + s2 * x1 + s3 * x2 + s4 * x3;
        o1 = s3 * (x0 + x1 - x3);
        o2 = s4 * x0 - s1 * x1 - s3 * x2 + s2 * x3;
        o3 = (s4 * x0 - s1 * x1 + s2 * x3) - (s1 * x0 + s2 * x1 + s4 * x3) + s3 * x2;
    } else {
        const uint32_t a = s1 * x0 + s4 * x2 + s2 * x3;
        const uint32_t b = s2 * x0 - s1 * x2 - s4 * x3;
        const uint32_t c = s3 * x1;
        o0 = a + c;
        o1 = b + c;
        o2 = s3 * (x0 - x2 + x3);
        o3 = a + b - c;
    }
    x[0] = round_shift64((long long)(int32_t)o0, COS_BIT);
    x[1] = round_shift64((long long)(int32_t)o1, COS_BIT);
    x[2] = round_shift64((long long)(int32_t)o2, COS_BIT);
    x[3] = round_shift64((long long)(int32_t)o3, COS_BIT);
}

// identity kernels (transforms.c:2205-2236, inv_transforms.c:2331-2362)
template <int N>
__device__ __forceinline__ int32_t txfm_identity_one(int32_t xv) {
    if constexpr (N == 4) return round_shift64((long long)xv * kNewSqrt2, 12);
    else if constexpr (N == 8) return (int32_t)((uint32_t)xv * 2u);
    else if constexpr (N == 16) return round_shift64((long long)xv * 2 * kNewSqrt2, 12);
    else if constexpr (N == 32) return (int32_t)((uint32_t)xv * 4u);
    else return round_shift64((long long)xv * 4 * kNewSqrt2, 12);
}
template <int N>
__device__ __forceinline__ void txfm_identity(int32_t (&x)[N]) {
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = txfm_identity_one<N>(x[i]);
}

// one N-point vector in registers through the 1-D kernel `type` (a TT_* of that length)
// PACKED: the 64-point kernels work on the packed coefficient layout -- the forward one needs only its 32
// low outputs (x[32..63] are left undefined), the inverse one gets zeros in x[32..63].  COS_BIT: the pass's cosine bit.
template <int N, bool INV, bool PACKED, int COS_BIT>
__device__ __forceinline__ void txfm_vec(int type, int32_t (&x)[N], int clampb) {
    constexpr TxCosv<COS_BIT> cosv{};
    if constexpr (N == 4) {
        if (type == TT_DCT4) { if constexpr (INV) txg_IDCT4(x, cosv, clampb); else txg_FDCT4(x, cosv, clampb); }
        else if (type == TT_ADST4) txfm_adst4<INV, COS_BIT>(x);
        else txfm_identity<4>(x);
    } else if constexpr (N == 8) {
        if (type == TT_DCT8) { if constexpr (INV) txg_IDCT8(x, cosv, clampb); else txg_FDCT8(x, cosv, clampb); }
        else if (type == TT_ADST8) { if constexpr (INV) txg_IADST8(x, cosv, clampb); else txg_FADST8(x, cosv, clampb); }
        else txfm_identity<8>(x);
    } else if constexpr (N == 16) {
        if (type == TT_DCT16) { if constexpr (INV) txg_IDCT16(x, cosv, clampb); else txg_FDCT16(x, cosv, clampb); }
        else if (type == TT_ADST16) { if constexpr (INV) txg_IADST16(x, cosv, clampb); else txg_FADST16(x, cosv, clampb); }
        else txfm_identity<16>(x);
    } else if constexpr (N == 32) {
        if (type == TT_DCT32) { if constexpr (INV) txg_IDCT32(x, cosv, clampb); else txg_FDCT32(x, cosv, clampb); }
        else txfm_identity<32>(x);
    } else {
        if (type == TT_DCT64) {
            if constexpr (INV && PACKED) txg_IDCT64_in32(x, cosv, clampb);
            else if constexpr (INV) txg_IDCT64(x, cosv, clampb);
            else if constexpr (PACKED) txg_FDCT64_lo32(x, cosv, clampb);
            else txg_FDCT64(x, cosv, clampb);
        }
        else txfm_identity<64>(x);
    }
}

// One 1-D pass over the V vectors of N points of a block held element-major in shared memory
// (x[i*P + v]), in place: thread v of the team loads vector v, transforms it in registers, stores it.
template <int N, int TEAM, bool INV, bool PACKED, int COS_BIT>
__device__ __forceinline__ void txfm_pass_n(int type, int32_t* x, int V, int P, int clampb, int tid) {
    for (int v = tid; v < V; v += TEAM) {
        int32_t r[N];
#pragma unroll
        for (int i = 0; i < N; i++) r[i] = x[i * P + v];
        txfm_vec<N, INV, PACKED, COS_BIT>(type, r, clampb);
#pragma unroll
        for (int i = 0; i < N; i++) x[i * P + v] = r[i];
    }
}
// a team of TEAM = max(W,H) threads only ever sees vector lengths TEAM/4 .. TEAM
template <int TEAM, bool INV, bool PACKED, int COS_BIT>
__device__ __forceinline__ void txfm_pass_1d(int type, int32_t* x, int N, int V, int P, int clampb, int tid) {
    if constexpr (TEAM <= 16) { if (N == 4) return txfm_pass_n<4, TEAM, INV, PACKED, COS_BIT>(type, x, V, P, clampb, tid); }
    if constexpr (TEAM >= 8 && TEAM <= 32) { if (N == 8) return txfm_pass_n<8, TEAM, INV, PACKED, COS_BIT>(type, x, V, P, clampb, tid); }
    if constexpr (TEAM >= 16) { if (N == 16) return txfm_pass_n<16, TEAM, INV, PACKED, COS_BIT>(type, x, V, P, clampb, tid); }
    if constexpr (TEAM >= 32) { if (N == 32) return txfm_pass_n<32, TEAM, INV, PACKED, COS_BIT>(type, x, V, P, clampb, tid); }
    if constexpr (TEAM >= 64) { if (N == 64) return txfm_pass_n<64, TEAM, INV, PACKED, COS_BIT>(type, x, V, P, clampb, tid); }
}

// One 1-D pass of N = 32 or 64 points with every vector split across two lanes, for a block that has its CTA of
// THREADS threads to itself: thread (g, v) = (tid / HALF, tid % HALF), HALF = THREADS / 2 >= V, runs lane group g
// of vector v.  HALF >= 32, so g is warp-uniform and the two groups' different code never diverges within a warp.
// DCT: the generated split (txfm_gen.inc, TxgSplit_*): forward, each group loads the vector and computes its own
// outputs; inverse, each group computes its half of the values before the combining last stage, the halves meet
// in shared memory, and each group runs the last stage for its outputs.  Identity: each group takes half the
// elements.  Every thread of the CTA must call it (it holds the CTA's barriers).
template <class S, int G, int N, int COS_BIT>
__device__ __forceinline__ void split_mid(int32_t (&r)[N], int32_t* x, int P, int v, TxCosv<COS_BIT> cosv, int clampb) {
    S::template mid<G>(r, cosv, clampb);
    if constexpr (S::kTail) {
        constexpr unsigned long long MID = G ? S::kMid1 : S::kMid0;
#pragma unroll
        for (int i = 0; i < N; i++)
            if ((MID >> i) & 1) x[i * P + v] = r[i];
    }
}
template <class S, int G, int N, int COS_BIT>
__device__ __forceinline__ void split_tail(int32_t (&r)[N], int32_t* x, int P, int v, TxCosv<COS_BIT> cosv, int clampb) {
    constexpr unsigned long long MID = G ? S::kMid1 : S::kMid0;
#pragma unroll
    for (int i = 0; i < N; i++)
        if (!((MID >> i) & 1)) r[i] = x[i * P + v];  // the other group's values
    S::template tail<G>(r, cosv, clampb);
}
template <class S, int G, int N>
__device__ __forceinline__ void split_store(const int32_t (&r)[N], int32_t* x, int P, int v) {
    constexpr unsigned long long OUT = G ? S::kOut1 : S::kOut0;
#pragma unroll
    for (int i = 0; i < N; i++)
        if ((OUT >> i) & 1) x[i * P + v] = r[i];
}
template <class S, int N, int COS_BIT>
__device__ __forceinline__ void txfm_pass_split_dct(int32_t* x, int V, int P, int clampb, int g, int v) {
    constexpr TxCosv<COS_BIT> cosv{};
    const bool on = v < V;
    int32_t r[N];
    if (on) {
#pragma unroll
        for (int i = 0; i < N; i++) r[i] = x[i * P + v];  // loads outside the group's network are dead
    }
    __syncthreads();  // both groups have read the vector before either writes over it
    if (on) {
        if (g == 0) split_mid<S, 0>(r, x, P, v, cosv, clampb);
        else split_mid<S, 1>(r, x, P, v, cosv, clampb);
    }
    if constexpr (S::kTail) {
        __syncthreads();  // both halves are in shared memory
        if (on) {
            if (g == 0) split_tail<S, 0>(r, x, P, v, cosv, clampb);
            else split_tail<S, 1>(r, x, P, v, cosv, clampb);
        }
        __syncthreads();  // both groups have read the other's half before the outputs go over it
    }
    if (on) {
        if (g == 0) split_store<S, 0>(r, x, P, v);
        else split_store<S, 1>(r, x, P, v);
    }
}
template <int N, int THREADS, bool INV, int COS_BIT>
__device__ __forceinline__ void txfm_pass_split(int type, int32_t* x, int V, int P, int clampb, int tid) {
    static_assert(N == 32 || N == 64, "two-lane splits exist for 32 and 64 points");
    constexpr int HALF = THREADS / 2;
    static_assert(HALF >= 32 && HALF % 32 == 0, "lane groups are whole warps");
    const int g = tid / HALF, v = tid % HALF;
    if (type == (N == 32 ? TT_DCT32 : TT_DCT64)) {
        if constexpr (N == 32 && INV) txfm_pass_split_dct<TxgSplit_IDCT32, 32, COS_BIT>(x, V, P, clampb, g, v);
        else if constexpr (N == 32) txfm_pass_split_dct<TxgSplit_FDCT32, 32, COS_BIT>(x, V, P, clampb, g, v);
        else if constexpr (INV) txfm_pass_split_dct<TxgSplit_IDCT64_in32, 64, COS_BIT>(x, V, P, clampb, g, v);
        else txfm_pass_split_dct<TxgSplit_FDCT64_lo32, 64, COS_BIT>(x, V, P, clampb, g, v);
    } else if (v < V) {
        // identity, element-wise.  64 points are packed: the forward's elements 32..63 are not kept, the inverse's
        // are zero and stay zero
        constexpr int PER = (N == 64 ? 32 : N) / 2;
#pragma unroll
        for (int k = 0; k < PER; k++) {
            const int i = g * PER + k;
            x[i * P + v] = txfm_identity_one<N>(x[i * P + v]);
        }
    }
}

}  // namespace b200
