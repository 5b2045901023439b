// txfm.cu -- K5 forward 2-D transforms, K6 inverse 2-D transforms + reconstruction, and the fused chain of both
// with the quantiser between them (sm_90a).
//
// Reference behaviour restated: av1_tranform_two_d_core_c (Source/Lib/Codec/transforms.c:2259-2324)
// and inv_txfm2d_add_c (Source/Lib/Codec/inv_transforms.c:2459-2534), for all 19 transform sizes and
// 16 transform types, 8/10/12-bit.  The 2-D configuration table (flips, per-pass kernel, cos_bit,
// shifts) is dumped from the reference (txfm_cfg.inc); the 1-D networks are txfm_graphs.inc.  The cosine bits and
// stage shifts depend on the size alone and are compile-time constants of each size body (kTxSizeCfg); the flips and
// the 1-D kernel types depend on the transform type and are read per item.
//
// H100 mapping: one kernel, txfm_kernel, whose modes are the forward batch, the inverse batch and the fused chain.
// A transform block belongs to a team sized by its team class, log2(max(W,H)) - 2.  In the 4-, 8- and 16-point
// classes a team is max(W,H) threads and several teams share a CTA: one thread per column in the column pass and one
// per row in the row pass, each running the generated straight-line network on its vector in registers
// (txfm_tables.cuh).  In the 32- and 64-point classes a block has a CTA of 2 * max(W,H) threads to itself, and its
// 32- and 64-point vectors run split across two lanes.  The block sits in shared memory in element-major order with
// an odd pitch, so the passes and the transposing hand-over are bank-conflict free; pixel, residual and coefficient
// rows move between global memory and the planes in 4- to 16-byte words where the item's origin and stride allow it.
#include <type_traits>
#include <utility>
#include "txfm_tables.cuh"
#include "quant_one.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

// The constants of a 2-D transform that depend on its size alone: the forward's column and row cosine bits and its three
// stage shifts, the inverse's two stage shifts (all as TxCfg holds them); the inverse's cosine bit is kInvCosBit at every
// size.  They are compile-time constants of each size body, so the networks' weights and every rounding shift become
// instruction immediates.  txfm_tables_init checks them against the table dumped from the reference for every valid
// (size, type).
struct TxSizeCfg {
    int8_t f_cbc, f_cbr, f_s0, f_s1, f_s2, i_s0, i_s1;
};
constexpr int       kInvCosBit = 12;
constexpr TxSizeCfg kTxSizeCfg[19] = {
    {13, 13, 2, 0, 0, 0, -4},    // 0: 4x4
    {13, 13, 2, -1, 0, -1, -4},  // 1: 8x8
    {13, 12, 2, -2, 0, -2, -4},  // 2: 16x16
    {12, 12, 2, -4, 0, -2, -4},  // 3: 32x32
    {13, 10, 0, -2, -2, -2, -4}, // 4: 64x64
    {13, 13, 2, -1, 0, 0, -4},   // 5: 4x8
    {13, 13, 2, -1, 0, 0, -4},   // 6: 8x4
    {13, 13, 2, -2, 0, -1, -4},  // 7: 8x16
    {13, 13, 2, -2, 0, -1, -4},  // 8: 16x8
    {12, 13, 2, -4, 0, -1, -4},  // 9: 16x32
    {13, 13, 2, -4, 0, -1, -4},  // 10: 32x16
    {13, 11, 0, -2, -2, -1, -4}, // 11: 32x64
    {12, 11, 2, -4, -2, -1, -4}, // 12: 64x32
    {13, 12, 2, -1, 0, -1, -4},  // 13: 4x16
    {13, 13, 2, -1, 0, -1, -4},  // 14: 16x4
    {12, 12, 2, -2, 0, -2, -4},  // 15: 8x32
    {13, 12, 2, -2, 0, -2, -4},  // 16: 32x8
    {13, 12, 0, -2, 0, -2, -4},  // 17: 16x64
    {13, 12, 2, -4, 0, -2, -4},  // 18: 64x16
};

static TxCfg h_txcfg[19][16];
const TxCfg& host_txcfg(int size, int type) { return h_txcfg[size][type]; }

void txfm_tables_init() {
    memset(h_txcfg, 0, sizeof(h_txcfg));
#define TXC(sz, ty, v, fud, flr, fs0, fs1, fs2, fcbc, fcbr, ftc, ftr, iud, ilr, is0, is1, icbc, icbr, itc, itr) \
    h_txcfg[sz][ty] = TxCfg{v, fud, flr, fs0, fs1, fs2, fcbc, fcbr, ftc, ftr, iud, ilr, is0, is1, icbc, icbr, itc, itr};
#define TXCOS(...)
#define TXSIN(...)
#include "txfm_cfg.inc"
#undef TXC
#undef TXCOS
#undef TXSIN
    for (int sz = 0; sz < 19; sz++)
        for (int ty = 0; ty < 16; ty++) {
            const TxCfg& c = h_txcfg[sz][ty];
            const TxSizeCfg& k = kTxSizeCfg[sz];
            if (c.valid && (c.f_cbc != k.f_cbc || c.f_cbr != k.f_cbr || c.f_s0 != k.f_s0 || c.f_s1 != k.f_s1 || c.f_s2 != k.f_s2 ||
                            c.i_s0 != k.i_s0 || c.i_s1 != k.i_s1 || c.i_cbc != kInvCosBit || c.i_cbr != kInvCosBit)) {
                fprintf(stderr, "[svt_b200] FATAL %s:%d: the compile-time transform constants of tx_size %d differ from the "
                                "reference's table at tx_type %d\n", __FILE__, __LINE__, sz, ty);
                abort();
            }
        }
    B200_CUDA_CHECK(cudaMemcpyToSymbol(c_txcfg, h_txcfg, sizeof(h_txcfg)));
}

// ints between the shared-memory areas (two planes) of consecutive teams.  Teams that share a warp must not
// land on the same banks: a team of T lanes covers T banks with its odd pitch, so the stride is made
// congruent to T modulo 32.
__host__ __device__ constexpr int team_stride(int team) {
    return team == 4 ? 68 : (team == 8 ? 152 : (team == 16 ? 560 : 2 * team * (team + 1)));
}

// ------------------------------------------------------------------------------------------------
// One block body for the three batch calls, as the modes of txfm_kernel:
//   Forward (svt_b200_fwd_txfm_batch_dev): residual -> coefficients;
//   Inverse (svt_b200_inv_txfm_batch_dev): dequantised coefficients + prediction -> reconstruction;
//   Chain   (the fused calls): the per-block chain of the final encode pass (coding_loop.c:405-658), forward transform
//           -> quantise -> inverse transform + reconstruction without leaving shared memory: the coefficients and the
//           dequantised levels never travel through HBM between the steps.
// The fused calls are bit-identical to the separate ones because each step is the same code in every mode.
// The body is a template on the transform size (txfm_block<..., SZ>): every element loop has a constant trip count and
// constant index arithmetic.  A class launch holds the bodies of its sizes and picks one per item (dispatch_size).
// ------------------------------------------------------------------------------------------------
struct Forward { using Item = SvtB200FwdTxfmItem; };
struct Inverse { using Item = SvtB200InvTxfmItem; };
struct Chain { using Item = SvtB200TrioItem; };

// the forward and the inverse part of an item: a Chain item has both, a Forward or an Inverse item is its own only part
template <class I> __device__ __forceinline__ const I& fwd_part(const I& i) { return i; }
template <class I> __device__ __forceinline__ const I& inv_part(const I& i) { return i; }
__device__ __forceinline__ const SvtB200FwdTxfmItem& fwd_part(const SvtB200TrioItem& i) { return i.fwd; }
__device__ __forceinline__ const SvtB200InvTxfmItem& inv_part(const SvtB200TrioItem& i) { return i.inv; }
// the part that holds a block's tx_size and tx_type: a Chain item's forward part, otherwise the item itself
template <class I> __device__ __forceinline__ const auto& shape_part(const I& i) { return fwd_part(i); }

// the forward's last steps on one coefficient: final shift, then the scaling of 2:1 rectangles
template <int RECT, int F_S2>
__device__ __forceinline__ int32_t fwd_out(int32_t v) {
    v = round_shift_arr(v, -F_S2);
    if constexpr (RECT == 1 || RECT == -1) v = round_shift64((long long)v * kNewSqrt2, 12);
    return v;
}
// the inverse's first steps on one dequantised coefficient: the scaling of 2:1 rectangles, then the row clamp
template <int RECT>
__device__ __forceinline__ int32_t inv_in(int32_t v, int row_clamp) {
    if constexpr (RECT == 1 || RECT == -1) v = round_shift64((long long)v * kNewInvSqrt2, 12);
    return clamp_bits(v, row_clamp);
}

// A 1-D pass.  In the 32- and 64-point classes (one block per CTA of 2 * TEAM threads) 32- and 64-point vectors run split
// across two lanes, shorter ones one per thread.  FULL64: 64-point vectors run whole on one thread, so that all 64 outputs
// exist (the forward batch's unpacked items); otherwise the 64-point networks are the packed ones.  COS_BIT: the pass's
// cosine bit.
template <int TEAM, int THREADS, bool INV, bool FULL64, int N, int V, int P, int COS_BIT>
__device__ __forceinline__ void txfm_pass(int type, int32_t* x, int clampb, int tid) {
    if constexpr (TEAM >= 32 && N == 32) {
        static_assert(THREADS == 2 * TEAM, "a lane pair per vector");
        return txfm_pass_split<32, THREADS, INV, COS_BIT>(type, x, V, P, clampb, tid);
    } else if constexpr (TEAM >= 64 && N == 64 && !FULL64) {
        return txfm_pass_split<64, THREADS, INV, COS_BIT>(type, x, V, P, clampb, tid);
    } else {
        txfm_pass_1d<TEAM, INV, !FULL64, COS_BIT>(type, x, N, V, P, clampb, tid);
    }
}

// ---- element loops -------------------------------------------------------------------------------------------------
// The words of V elements of a region of R rows of W elements, spread over the MOVERS threads of a team: f(r, c) for
// every word this thread moves (c: the word's first column).  Trip count and index split are constants.
template <int W, int R, int V, int MOVERS, class F>
__device__ __forceinline__ void for_words(int tid, F&& f) {
    static_assert(W % V == 0, "whole words per row");
    constexpr int PER_ROW = W / V, N = PER_ROW * R;
#pragma unroll 2
    for (int k = 0; k < (N + MOVERS - 1) / MOVERS; k++) {
        const int w = tid + k * MOVERS;
        if (N % MOVERS == 0 || w < N) f(w / PER_ROW, (w % PER_ROW) * V);
    }
}

// V consecutive elements of global memory: one 4-, 8- or 16-byte word when VEC (the caller has checked the alignment:
// row_words), V element moves otherwise
template <int V, typename T> union Word {
    using U = std::conditional_t<V * sizeof(T) == 4, uint32_t, std::conditional_t<V * sizeof(T) == 8, uint2, uint4>>;
    static_assert(V * sizeof(T) == 4 || V * sizeof(T) == 8 || V * sizeof(T) == 16, "a word is 4, 8 or 16 bytes");
    U u;
    T e[V];
};
template <bool VEC, int V, typename T>
__device__ __forceinline__ void ld_word(const T* p, T (&v)[V]) {
    if constexpr (VEC) {
        Word<V, T> w;
        w.u = *reinterpret_cast<const typename Word<V, T>::U*>(p);
#pragma unroll
        for (int j = 0; j < V; j++) v[j] = w.e[j];
    } else {
#pragma unroll
        for (int j = 0; j < V; j++) v[j] = p[j];
    }
}
template <bool VEC, int V, typename T>
__device__ __forceinline__ void st_word(T* p, const T (&v)[V]) {
    if constexpr (VEC) {
        Word<V, T> w;
#pragma unroll
        for (int j = 0; j < V; j++) w.e[j] = v[j];
        *reinterpret_cast<typename Word<V, T>::U*>(p) = w.u;
    } else {
#pragma unroll
        for (int j = 0; j < V; j++) p[j] = v[j];
    }
}
// the rows of a block starting at p with the given stride (in elements) can move in words of V elements.  A per-item,
// hence team-uniform, predicate: the block's origin and its stride are whole words.
template <int V, typename T>
__device__ __forceinline__ bool row_words(const T* p, size_t stride) {
    constexpr int BYTES = V * (int)sizeof(T);
    return ((uintptr_t)p % BYTES) == 0 && (stride * sizeof(T)) % BYTES == 0;
}
// runs f(std::true_type) or f(std::false_type): the word or the element form of a loop
template <class F> __device__ __forceinline__ void with_words(bool vec, F&& f) {
    if (vec) f(std::true_type{});
    else f(std::false_type{});
}
// the word widths: pixels and residual samples up to 16 bytes and at most a row; coefficients, levels, scan positions
// and matrix weights 4 at a time (int4, 4 x int16, u32)
template <int W, typename T> constexpr int kRowWord = W < 16 / (int)sizeof(T) ? W : 16 / (int)sizeof(T);
constexpr int kCoefWord = 4;

// the device buffers of a batch call, in txfm_kernel's order; each mode uses its own
template <typename PIX>
struct TxfmPtrs {
    const int16_t* src_base;    // residual (Forward; Chain without source)
    const PIX*     srcpix_base; // Chain, non-null: residual = source - prediction, formed here
    const PIX*     pred_base;
    PIX*           recon_base;
    int32_t*       coef_base;   // Forward: the coefficients; Chain: the quantised levels
    int32_t*       dq_base;     // Chain: the dequantised levels, may be null
    const int16_t* iscan_base;
    const uint8_t* qm_base;
    uint16_t*      eobs;
    const int32_t* dq_in;       // Inverse: the dequantised coefficients
};

// One block of size SZ.  A and B: the team's two shared-memory planes.
template <class M, int TEAM, int THREADS, typename PIX, int SZ>
__device__ __forceinline__ void txfm_block(const TxfmPtrs<PIX>& g, const typename M::Item& item, int it, int32_t* A, int32_t* B,
                                           int tid, int& s_eob) {
    constexpr bool FWD = !std::is_same_v<M, Inverse>, INV = !std::is_same_v<M, Forward>, CHAIN = FWD && INV;
    constexpr bool SOLO = TEAM >= 32;
    constexpr int  MOVERS = SOLO ? THREADS : TEAM;
    constexpr int  W = tx_w(SZ), H = tx_h(SZ);
    static_assert((W > H ? W : H) == TEAM, "a size runs in the team class of its longer side");
    constexpr int  RECT = W == H ? 0 : (W > H ? (W == 2 * H ? 1 : (W == 4 * H ? 2 : 3)) : (H == 2 * W ? -1 : (H == 4 * W ? -2 : -3)));  // get_rect_tx_log_ratio
    constexpr int  Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;  // 64-point dimensions are packed (inv_transforms.c:2567-2686)
    constexpr int  PW = W + 1, PH = H + 1;  // odd pitches: a plane holds the block as [r * PW + c] or as [c * PH + r]
    constexpr int  VP = kRowWord<W, PIX>, VR = kRowWord<W, int16_t>, VC = kCoefWord;
    // the size's cosine bits and stage shifts are constants; the flips and the 1-D kernel types come with the type
    constexpr int  F_CBC = kTxSizeCfg[SZ].f_cbc, F_CBR = kTxSizeCfg[SZ].f_cbr;
    constexpr int  F_S0 = kTxSizeCfg[SZ].f_s0, F_S1 = kTxSizeCfg[SZ].f_s1, F_S2 = kTxSizeCfg[SZ].f_s2;
    constexpr int  I_S0 = kTxSizeCfg[SZ].i_s0, I_S1 = kTxSizeCfg[SZ].i_s1;
    const auto&    fi  = fwd_part(item);
    const TxCfg    cfg = c_txcfg[SZ][shape_part(item).tx_type];
    // 1-byte pixels are 8-bit ones: there the bit depth, and every clamp and range derived from it, is a constant too
    int            bd  = 0;
    if constexpr (INV) bd = std::is_same_v<PIX, uint8_t> ? 8 : inv_part(item).bd;
    if constexpr (FWD) {  // ---- forward transform (transforms.c:2286-2318) ----
        const size_t sstride = fi.src_stride;
        // load, optional up/down flip, pre-shift
        bool from_source = false;
        if constexpr (CHAIN) from_source = g.srcpix_base != nullptr;
        if constexpr (CHAIN) if (from_source) {  // svt_aom_residual_kernel fused in: the source picture shares the residual plane's geometry
            const PIX*   sp = g.srcpix_base + fi.src_off;
            const PIX*   pp = g.pred_base + item.inv.pred_off;
            const size_t pstride = item.inv.pred_stride;
            with_words(row_words<VP>(sp, sstride) && row_words<VP>(pp, pstride), [&](auto vec) {
                for_words<W, H, VP, MOVERS>(tid, [&](int r, int c) {
                    const int rr = cfg.f_ud ? (H - 1 - r) : r;
                    PIX s[VP], p[VP];
                    ld_word<decltype(vec)::value>(sp + rr * sstride + c, s);
                    ld_word<decltype(vec)::value>(pp + rr * pstride + c, p);
#pragma unroll
                    for (int j = 0; j < VP; j++) A[r * PW + c + j] = round_shift_arr((int32_t)s[j] - (int32_t)p[j], -F_S0);
                });
            });
        }
        if (!from_source) {
            const int16_t* src = g.src_base + fi.src_off;
            with_words(row_words<VR>(src, sstride), [&](auto vec) {
                for_words<W, H, VR, MOVERS>(tid, [&](int r, int c) {
                    const int rr = cfg.f_ud ? (H - 1 - r) : r;
                    int16_t   s[VR];
                    ld_word<decltype(vec)::value>(src + rr * sstride + c, s);
#pragma unroll
                    for (int j = 0; j < VR; j++) A[r * PW + c + j] = round_shift_arr((int32_t)s[j], -F_S0);
                });
            });
        }
        team_sync<TEAM, SOLO>();
        // columns: vector v = column v (Chain: rows >= Hp of the result are not needed)
        txfm_pass<TEAM, THREADS, false, !INV, H, W, PW, F_CBC>(cfg.f_tc, A, 0, tid);
        team_sync<TEAM, SOLO>();
        // round-shift, optional left/right flip, hand over transposed (element = column); Chain: only the Hp rows that
        // survive the packing
        constexpr int Hk = INV ? Hp : H;
        for_words<W, Hk, 1, MOVERS>(tid, [&](int r, int c) {
            const int cc = cfg.f_lr ? (W - 1 - c) : c;
            B[cc * PH + r] = round_shift_arr(A[r * PW + c], -F_S1);
        });
        team_sync<TEAM, SOLO>();
        txfm_pass<TEAM, THREADS, false, !INV, W, Hk, PH, F_CBR>(cfg.f_tr, B, 0, tid);  // rows: vector v = row v
        team_sync<TEAM, SOLO>();
    }
    if constexpr (!INV) {  // ---- Forward: the coefficients out ----
        int32_t*  dst = g.coef_base + fi.dst_off;
        const int part_shift = (fi.reserved >> 1) & 3;  // 0 full, 1 = N2, 2 = N4
        const int keep_h = max(H >> part_shift, 1), keep_w = max(W >> part_shift, 1);
        // WO x HO coefficients in rows of WO: packed output keeps the top-left min(W,32) x min(H,32) (svt_handle_transform64x64
        // repack, transforms.c:2374), otherwise all of them
        auto out = [&](auto vec, auto wo, auto ho) {
            constexpr int WO = decltype(wo)::value, HO = decltype(ho)::value;
            for_words<WO, HO, VC, MOVERS>(tid, [&](int r, int c) {
                int32_t v[VC];
#pragma unroll
                for (int j = 0; j < VC; j++) {
                    v[j] = fwd_out<RECT, F_S2>(B[(c + j) * PH + r]);
                    // N2 / N4 (av1_tranform_two_d_core_N2_c / _N4_c, transforms.c:5202, 6769): the top-left half / quarter
                    // of every dimension, identical to the full transform's values there, zero everywhere else
                    if (part_shift && (r >= keep_h || c + j >= keep_w)) v[j] = 0;
                }
                st_word<decltype(vec)::value>(dst + r * WO + c, v);
            });
        };
        with_words(row_words<VC>(dst, 0), [&](auto vec) {
            if ((fi.reserved & 1) && (W != Wp || H != Hp)) out(vec, std::integral_constant<int, Wp>{}, std::integral_constant<int, Hp>{});
            else out(vec, std::integral_constant<int, W>{}, std::integral_constant<int, H>{});
        });
        team_sync<TEAM, SOLO>();
    } else {
        // the inverse's input plane, rows first: A[c * PH + r], element = column, vector = row; zero outside the packed
        // Wp x Hp, which the passes keep zero
        const auto& ii = inv_part(item);
        const int   row_clamp = bd + 8;
        int eob = 0;
        if constexpr (CHAIN) {  // ---- quantise the (packed) coefficients; the dequantised levels are the input ----
            const SvtB200QuantItem& qi = item.quant;
            const QuantK   k   = quant_consts(qi);
            const uint8_t* qm  = qi.qm_off == SVT_B200_NO_QM ? nullptr : g.qm_base + qi.qm_off;
            const uint8_t* iqm = qi.iqm_off == SVT_B200_NO_QM ? nullptr : g.qm_base + qi.iqm_off;
            const int16_t* iscan = g.iscan_base + qi.scan_off;
            int32_t*       qc = g.coef_base + qi.q_off;
            int32_t*       dqc = g.dq_base ? g.dq_base + qi.dq_off : nullptr;
            if (SOLO && threadIdx.x == 0) s_eob = 0;
            const bool vec = row_words<VC>(qc, 0) && (!dqc || row_words<VC>(dqc, 0)) && row_words<VC>(iscan, 0) &&
                             (!qm || row_words<VC>(qm, 0)) && (!iqm || row_words<VC>(iqm, 0));
            // the packed coefficients are one run of Wp * Hp; a word is VC of them in one row
            auto quant = [&](auto vec_c, auto mode_c, auto qm_c) {
                constexpr bool VEC = decltype(vec_c)::value, QM = decltype(qm_c)::value;
                constexpr int  MODE = decltype(mode_c)::value;
                for_words<Wp, Hp, VC, MOVERS>(tid, [&](int r, int c) {
                    const int rc = r * Wp + c;
                    int16_t   pos[VC];
                    uint8_t   wt[VC], iwt[VC];
                    int32_t   q[VC], dq[VC];
                    ld_word<VEC>(iscan + rc, pos);
                    if constexpr (QM) {
                        if (qm) ld_word<VEC>(qm + rc, wt);
                        else {
#pragma unroll
                            for (int j = 0; j < VC; j++) wt[j] = 1 << kQmBits;
                        }
                        if (iqm) ld_word<VEC>(iqm + rc, iwt);
                        else {
#pragma unroll
                            for (int j = 0; j < VC; j++) iwt[j] = 1 << kQmBits;
                        }
                    }
#pragma unroll
                    for (int j = 0; j < VC; j++) {
                        const int32_t v = fwd_out<RECT, F_S2>(B[(c + j) * PH + r]);
                        quant_coef<MODE, QM>(k, v, rc + j != 0, QM ? wt[j] : 0, QM ? iwt[j] : 0, q[j], dq[j]);
                        if (q[j]) eob = max(eob, (int)pos[j] + 1);
                        A[(c + j) * PH + r] = inv_in<RECT>(dq[j], row_clamp);
                    }
                    st_word<VEC>(qc + rc, q);
                    if (dqc) st_word<VEC>(dqc + rc, dq);
                });
            };
            // the quantiser's mode and matrix once per item, then a loop specialised on them
            with_words(vec, [&](auto vec_c) {
                auto by_qm = [&](auto mode_c) {
                    if (quant_has_qm(qi)) quant(vec_c, mode_c, std::true_type{});
                    else quant(vec_c, mode_c, std::false_type{});
                };
                switch (qi.mode) {
                case SVT_B200_QUANT_B_LBD: by_qm(std::integral_constant<int, SVT_B200_QUANT_B_LBD>{}); break;
                case SVT_B200_QUANT_B_HBD: by_qm(std::integral_constant<int, SVT_B200_QUANT_B_HBD>{}); break;
                case SVT_B200_QUANT_FP_LBD: by_qm(std::integral_constant<int, SVT_B200_QUANT_FP_LBD>{}); break;
                default: by_qm(std::integral_constant<int, SVT_B200_QUANT_FP_HBD>{}); break;
                }
            });
        } else {  // ---- Inverse: the packed dequantised coefficients are the input ----
            const int32_t* in = g.dq_in + ii.coef_off;
            with_words(row_words<VC>(in, 0), [&](auto vec) {
                for_words<Wp, Hp, VC, MOVERS>(tid, [&](int r, int c) {
                    int32_t v[VC];
                    ld_word<decltype(vec)::value>(in + r * Wp + c, v);
#pragma unroll
                    for (int j = 0; j < VC; j++) A[(c + j) * PH + r] = inv_in<RECT>(v[j], row_clamp);
                });
            });
        }
        // zero outside the packed Wp x Hp
        if constexpr (W > Wp) for_words<W - Wp, H, 1, MOVERS>(tid, [&](int r, int c) { A[(Wp + c) * PH + r] = 0; });
        if constexpr (H > Hp) for_words<Wp, H - Hp, 1, MOVERS>(tid, [&](int r, int c) { A[c * PH + Hp + r] = 0; });
        if constexpr (CHAIN) {
            if constexpr (SOLO) {
                __syncthreads();
                if (eob) atomicMax(&s_eob, eob);
                __syncthreads();
                eob = s_eob;
                if (threadIdx.x == 0) g.eobs[it] = (uint16_t)eob;
            } else {
                const unsigned mask = TEAM == 32 ? 0xffffffffu : (((1u << TEAM) - 1u) << ((threadIdx.x & 31) / TEAM * TEAM));
#pragma unroll
                for (int o = TEAM / 2; o > 0; o >>= 1) eob = max(eob, __shfl_xor_sync(mask, eob, o));
                if (tid == 0) g.eobs[it] = (uint16_t)eob;
                team_sync<TEAM, SOLO>();
            }
        } else {
            team_sync<TEAM, SOLO>();
        }
        const PIX*   pr = g.pred_base + ii.pred_off;
        PIX*         pw = g.recon_base + ii.recon_off;
        const size_t pstride = ii.pred_stride, rstride = ii.recon_stride;
        const bool   vec = row_words<VP>(pr, pstride) && row_words<VP>(pw, rstride);
        if (CHAIN && eob == 0) {
            // every level is zero: the inverse of an all-zero plane is zero, the reconstruction is the prediction
            // (the encode pass takes the same shortcut, coding_loop.c: eob == 0 -> prediction copied); team-uniform branch
            if (pr != pw) {
                with_words(vec, [&](auto vec_c) {
                    for_words<W, H, VP, MOVERS>(tid, [&](int r, int c) {
                        PIX p[VP];
                        ld_word<decltype(vec_c)::value>(pr + r * pstride + c, p);
                        st_word<decltype(vec_c)::value>(pw + r * rstride + c, p);
                    });
                });
            }
            team_sync<TEAM, SOLO>();
        } else {  // ---- inverse transform + reconstruction (inv_transforms.c:2459-2534) ----
            const int col_clamp = (bd + 6) > 16 ? (bd + 6) : 16;
            const int opt_row = bd == 8 ? 16 : (bd == 10 ? 18 : 20);  // svt_av1_gen_inv_stage_range
            const int opt_col = bd == 12 ? 18 : 16;
            txfm_pass<TEAM, THREADS, true, false, W, Hp, PH, kInvCosBit>(cfg.i_tr, A, opt_row, tid);  // rows >= Hp are zero and stay zero
            team_sync<TEAM, SOLO>();
            for_words<W, H, 1, MOVERS>(tid, [&](int r, int c) {
                const int cs = cfg.i_lr ? (W - 1 - c) : c;
                B[r * PW + c] = clamp_bits(round_shift_arr(A[cs * PH + r], -I_S0), col_clamp);
            });
            team_sync<TEAM, SOLO>();
            txfm_pass<TEAM, THREADS, true, false, H, W, PW, kInvCosBit>(cfg.i_tc, B, opt_col, tid);
            team_sync<TEAM, SOLO>();
            const long long int_max = (1ll << (7 + bd)) - 1 + (914ll << (bd - 7));  // check_range, inv_transforms.c:2401
            const int       pix_max = (1 << bd) - 1;
            with_words(vec, [&](auto vec_c) {
                for_words<W, H, VP, MOVERS>(tid, [&](int r, int c) {
                    const int rs = cfg.i_ud ? (H - 1 - r) : r;
                    PIX       p[VP];
                    ld_word<decltype(vec_c)::value>(pr + r * pstride + c, p);
#pragma unroll
                    for (int j = 0; j < VP; j++) {
                        long long t = (long long)round_shift_arr(B[rs * PW + c + j], -I_S1);
                        t           = t < -int_max - 1 ? -int_max - 1 : (t > int_max ? int_max : t);
                        int v       = (int)p[j] + (int)t;
                        p[j]        = (PIX)(v < 0 ? 0 : (v > pix_max ? pix_max : v));
                    }
                    st_word<decltype(vec_c)::value>(pw + r * rstride + c, p);
                });
            });
            team_sync<TEAM, SOLO>();
        }
    }
}

// the transform sizes of a team class (max(W,H) = TEAM), in tx_size numbers
template <int TEAM> struct ClassSizes;
template <> struct ClassSizes<4> { using type = std::integer_sequence<int, 0>; };
template <> struct ClassSizes<8> { using type = std::integer_sequence<int, 1, 5, 6>; };
template <> struct ClassSizes<16> { using type = std::integer_sequence<int, 2, 7, 8, 13, 14>; };
template <> struct ClassSizes<32> { using type = std::integer_sequence<int, 3, 9, 10, 15, 16>; };
template <> struct ClassSizes<64> { using type = std::integer_sequence<int, 4, 11, 12, 17, 18>; };

// the item's size body, chosen once per item (team-uniform: a team runs one item)
template <class M, int TEAM, int THREADS, typename PIX, int... SZ>
__device__ __forceinline__ void dispatch_size(std::integer_sequence<int, SZ...>, int sz, const TxfmPtrs<PIX>& g,
                                              const typename M::Item& item, int it, int32_t* A, int32_t* B, int tid, int& s_eob) {
    (void)((sz == SZ && (txfm_block<M, TEAM, THREADS, PIX, SZ>(g, item, it, A, B, tid, s_eob), true)) || ...);
}

// CTAs per SM that the register allocation of a class must leave room for: what the class's kernels held before their
// bodies were specialised by size (168 / 96 / 64 / 64 / 64 registers).  The calls of a step run concurrently on several
// streams, so a CTA that takes more of an SM's register file keeps other kernels' CTAs off that SM; left free, ptxas
// gives the specialised bodies up to 208 registers and the step is slower even where the class's own kernel is faster.
// Tighter bounds spill heavily (the 64-point class at 4 CTAs per SM: over 1 KB of spill stores).
template <int TEAM> constexpr int class_min_ctas() { return TEAM == 64 ? 3 : (TEAM == 32 ? 10 : (TEAM == 16 ? 8 : 4)); }

template <class M, int TEAM, int THREADS, typename PIX>
__global__ void __launch_bounds__(THREADS, class_min_ctas<TEAM>())
txfm_kernel(const TxfmPtrs<PIX> g, const typename M::Item* __restrict__ items, int n_items) {
    extern __shared__ __align__(16) int32_t tsm[];
    // big blocks are few: one block per CTA (SOLO) of 2 * TEAM threads; all of them move its data, and lane pairs run
    // its 32- and 64-point vectors (txfm_pass)
    constexpr bool SOLO = TEAM >= 32;
    constexpr int  TEAMS = SOLO ? 1 : THREADS / TEAM, PLANE = TEAM * (TEAM + 1);
    const int      team  = SOLO ? 0 : threadIdx.x / TEAM, tid = SOLO ? threadIdx.x : threadIdx.x % TEAM;
    int32_t*       A     = tsm + (size_t)team * team_stride(TEAM);
    int32_t*       B     = A + PLANE;
    __shared__ int s_eob;

    // a Forward or Inverse item is small and is copied into registers; a Chain item is read once by its team, in 8-byte
    // words, into shared memory, and its fields are read from there where they are used
    using Item = typename M::Item;
    constexpr bool STAGE = std::is_same_v<M, Chain>;
    static_assert(sizeof(Item) % 8 == 0 && alignof(Item) == 8, "an item is whole 8-byte words");
    __shared__ __align__(16) Item s_item[STAGE ? TEAMS : 1];
    for (int it = blockIdx.x * TEAMS + team; it < n_items; it += gridDim.x * TEAMS) {
        if constexpr (STAGE) {
            constexpr int MOVERS = SOLO ? THREADS : TEAM, WORDS = (int)(sizeof(Item) / 8);
            for (int w = tid; w < WORDS; w += MOVERS)
                reinterpret_cast<uint2*>(&s_item[team])[w] = reinterpret_cast<const uint2*>(items + it)[w];
            team_sync<TEAM, SOLO>();
            const Item& item = s_item[team];  // every body ends on a team barrier: the next item's copy waits for its readers
            dispatch_size<M, TEAM, THREADS, PIX>(typename ClassSizes<TEAM>::type{}, shape_part(item).tx_size, g, item, it, A, B, tid, s_eob);
        } else {
            const Item item = items[it];
            dispatch_size<M, TEAM, THREADS, PIX>(typename ClassSizes<TEAM>::type{}, shape_part(item).tx_size, g, item, it, A, B, tid, s_eob);
        }
    }
}

// team class of a transform size: log2(max(W,H)) - 2
static inline int tx_class(int sz) {
    const int m = tx_w(sz) > tx_h(sz) ? tx_w(sz) : tx_h(sz);
    return m == 4 ? 0 : (m == 8 ? 1 : (m == 16 ? 2 : (m == 32 ? 3 : 4)));
}

// CTA size per team class: small enough that a picture's worth of blocks of that class spreads over all SMs.  A 32- or
// 64-point block has its CTA of 2 * TEAM threads to itself (a lane pair per vector in the passes).
template <int TEAM> constexpr int class_threads() { return TEAM >= 32 ? 2 * TEAM : (TEAM == 16 ? 128 : 256); }

// the device buffers of a batch call as the entry points fill them, untyped; launch makes them a TxfmPtrs<PIX>
struct TxfmBufs {
    const int16_t* residual = nullptr;
    const void*    source   = nullptr;
    const void*    pred     = nullptr;
    void*          recon    = nullptr;
    int32_t*       coef     = nullptr;
    int32_t*       dq       = nullptr;
    const int16_t* iscan    = nullptr;
    const uint8_t* qm       = nullptr;
    const int32_t* dq_in    = nullptr;
};

template <class M, int TEAM, typename PIX>
static void launch(const TxfmBufs& b, const typename M::Item* items, int n, uint16_t* eobs, cudaStream_t st) {
    if (n <= 0) return;
    constexpr int    THREADS = class_threads<TEAM>(), TEAMS = TEAM >= 32 ? 1 : THREADS / TEAM;
    constexpr size_t smem = (size_t)TEAMS * team_stride(TEAM) * 4;
    static_assert(smem <= 48 * 1024, "the default dynamic shared-memory limit: no attribute to set");
    constexpr int per_sm = (int)((200 * 1024) / (smem + 1024)) < 2048 / THREADS ? (int)((200 * 1024) / (smem + 1024)) : 2048 / THREADS;
    const TxfmPtrs<PIX> g{b.residual, (const PIX*)b.source, (const PIX*)b.pred, (PIX*)b.recon, b.coef, b.dq, b.iscan, b.qm, eobs, b.dq_in};
    txfm_kernel<M, TEAM, THREADS, PIX><<<grid_for((n + TEAMS - 1) / TEAMS, per_sm), THREADS, smem, st>>>(g, items, n);
    B200_LAUNCH_CHECK();
}
// the n items of team class cls
template <class M, typename PIX>
static void launch_class(int cls, const TxfmBufs& b, const typename M::Item* items, int n, uint16_t* eobs, cudaStream_t st) {
    switch (cls) {
    case 0: launch<M, 4, PIX>(b, items, n, eobs, st); break;
    case 1: launch<M, 8, PIX>(b, items, n, eobs, st); break;
    case 2: launch<M, 16, PIX>(b, items, n, eobs, st); break;
    case 3: launch<M, 32, PIX>(b, items, n, eobs, st); break;
    default: launch<M, 64, PIX>(b, items, n, eobs, st); break;
    }
}
// A batch ordered by class.  The five class launches are independent: the three big-block classes (few, long-running CTAs)
// go to side streams forked from the caller's stream and joined back into it, so the many small blocks fill the SMs the
// big ones leave idle.
template <class M, typename PIX>
static void launch_batch(const TxfmBufs& b, const typename M::Item* items, const int* n_per_class, uint16_t* eobs, cudaStream_t user) {
    int first[SVT_B200_TXFM_CLASSES + 1] = {0};
    for (int c = 0; c < SVT_B200_TXFM_CLASSES; c++) first[c + 1] = first[c] + n_per_class[c];
    ForkJoin& fj = fork_streams(user);
    for (int c = SVT_B200_TXFM_CLASSES - 1; c >= 0; c--)
        launch_class<M, PIX>(c, b, items + first[c], n_per_class[c], eobs ? eobs + first[c] : nullptr, c >= 2 ? fj.side[c - 2] : user);
    join_streams(fj, user);
}
static bool class_counts_ok(const int* n_per_class) {
    if (!n_per_class) return false;
    for (int c = 0; c < SVT_B200_TXFM_CLASSES; c++)
        if (n_per_class[c] < 0) return false;
    return true;
}

}  // namespace b200

using namespace b200;

extern "C" int svt_b200_txfm_valid(int tx_size, int tx_type) {
    if (tx_size < 0 || tx_size >= 19 || tx_type < 0 || tx_type >= 16) return 0;
    require_ready();
    return host_txcfg(tx_size, tx_type).valid;
}

extern "C" int svt_b200_txfm_team_class(int tx_size) { return (tx_size < 0 || tx_size >= 19) ? -1 : tx_class(tx_size); }

extern "C" int svt_b200_fwd_txfm_batch_dev(const int16_t* d_residual, int32_t* d_coeff, const SvtB200FwdTxfmItem* d_items,
                                           const int n_per_class[SVT_B200_TXFM_CLASSES], void* stream) {
    require_ready();
    if (!class_counts_ok(n_per_class)) return SVT_B200_ERR_BAD_ARG;
    TxfmBufs b;
    b.residual = d_residual;
    b.coef     = d_coeff;
    launch_batch<Forward, uint8_t>(b, d_items, n_per_class, nullptr, (cudaStream_t)stream);  // (the forward has no pixels)
    return SVT_B200_OK;
}

extern "C" int svt_b200_inv_txfm_batch_dev(const int32_t* d_coeff, const void* d_pred, void* d_recon,
                                           const SvtB200InvTxfmItem* d_items, const int n_per_class[SVT_B200_TXFM_CLASSES],
                                           int pixel_bytes, void* stream) {
    require_ready();
    if (!class_counts_ok(n_per_class) || (pixel_bytes != 1 && pixel_bytes != 2)) return SVT_B200_ERR_BAD_ARG;
    TxfmBufs b;
    b.pred  = d_pred;
    b.recon = d_recon;
    b.dq_in = d_coeff;
    if (pixel_bytes == 1) launch_batch<Inverse, uint8_t>(b, d_items, n_per_class, nullptr, (cudaStream_t)stream);
    else launch_batch<Inverse, uint16_t>(b, d_items, n_per_class, nullptr, (cudaStream_t)stream);
    return SVT_B200_OK;
}

static int trio_entry(const int16_t* d_residual, const void* d_source, const void* d_pred, void* d_recon, int32_t* d_qcoeff,
                      int32_t* d_dqcoeff, const int16_t* d_iscan, const uint8_t* d_qm, const SvtB200TrioItem* d_items,
                      const int n_per_class[SVT_B200_TXFM_CLASSES], uint16_t* d_eobs, int pixel_bytes, void* stream) {
    require_ready();
    if (!class_counts_ok(n_per_class) || !d_iscan || !d_qcoeff || !d_eobs || (pixel_bytes != 1 && pixel_bytes != 2)) return SVT_B200_ERR_BAD_ARG;
    if (!d_residual == !d_source) return SVT_B200_ERR_BAD_ARG;  // exactly one of the two inputs
    const TxfmBufs b{d_residual, d_source, d_pred, d_recon, d_qcoeff, d_dqcoeff, d_iscan, d_qm};
    if (pixel_bytes == 1) launch_batch<Chain, uint8_t>(b, d_items, n_per_class, d_eobs, (cudaStream_t)stream);
    else launch_batch<Chain, uint16_t>(b, d_items, n_per_class, d_eobs, (cudaStream_t)stream);
    return SVT_B200_OK;
}
extern "C" int svt_b200_txfm_trio_batch_dev(const int16_t* d_residual, const void* d_pred, void* d_recon, int32_t* d_qcoeff,
                                            int32_t* d_dqcoeff, const int16_t* d_iscan, const uint8_t* d_qm,
                                            const SvtB200TrioItem* d_items, const int n_per_class[SVT_B200_TXFM_CLASSES],
                                            uint16_t* d_eobs, int pixel_bytes, void* stream) {
    return trio_entry(d_residual, nullptr, d_pred, d_recon, d_qcoeff, d_dqcoeff, d_iscan, d_qm, d_items, n_per_class, d_eobs, pixel_bytes, stream);
}
extern "C" int svt_b200_residual_txfm_trio_batch_dev(const void* d_source, const void* d_pred, void* d_recon, int32_t* d_qcoeff,
                                                     int32_t* d_dqcoeff, const int16_t* d_iscan, const uint8_t* d_qm,
                                                     const SvtB200TrioItem* d_items, const int n_per_class[SVT_B200_TXFM_CLASSES],
                                                     uint16_t* d_eobs, int pixel_bytes, void* stream) {
    return trio_entry(nullptr, d_source, d_pred, d_recon, d_qcoeff, d_dqcoeff, d_iscan, d_qm, d_items, n_per_class, d_eobs, pixel_bytes, stream);
}

// ---- svt_aom_residual_kernel (pic_operators.c:218; rtcd svt_residual_kernel8bit / 16bit, common_dsp_rtcd.h) on planes -----
template <typename PIX>
__global__ void residual_planes_kernel(const PIX* __restrict__ src, const PIX* __restrict__ pred, int16_t* __restrict__ res,
                                       const __grid_constant__ SvtB200ResidualPlanes pl) {
    const SvtB200ResidualPlane& e = pl.p[blockIdx.y];
    const long long n = (long long)e.w * e.h;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(idx / e.w), x = (int)(idx - (long long)y * e.w);
        res[e.res_off + (size_t)y * e.res_stride + x] =
            (int16_t)((int)src[e.src_off + (size_t)y * e.src_stride + x] - (int)pred[e.pred_off + (size_t)y * e.pred_stride + x]);
    }
}
extern "C" int svt_b200_residual_planes_dev(const void* d_source, const void* d_pred, int16_t* d_residual, const SvtB200ResidualPlanes* planes,
                                            int n_planes, int pixel_bytes, void* stream) {
    require_ready();
    if (!planes || n_planes <= 0 || n_planes > 3 || (pixel_bytes != 1 && pixel_bytes != 2)) return SVT_B200_ERR_BAD_ARG;
    long long mx = 0;
    for (int i = 0; i < n_planes; i++) mx = mx > (long long)planes->p[i].w * planes->p[i].h ? mx : (long long)planes->p[i].w * planes->p[i].h;
    const dim3 grid(grid_for((mx + 255) / 256, 8), n_planes);
    if (pixel_bytes == 1)
        residual_planes_kernel<uint8_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t*)d_source, (const uint8_t*)d_pred, d_residual, *planes);
    else
        residual_planes_kernel<uint16_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)d_source, (const uint16_t*)d_pred, d_residual, *planes);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

// ---- eob-bounded scan-order packing of the quantised levels (what the entropy coder consumes: the first eob levels of
// each block in scan order, coding_loop.c / entropy_coding.c) -- the device->host transfer of a picture's coefficients then
// carries sum(eob) levels instead of every coefficient position --------------------------------------------------------------
// pass 1: per-chunk sums of the eobs (256 blocks per CTA; a picture has a few hundred chunks)
constexpr int kPackChunk = 256;
__global__ void __launch_bounds__(256) eob_chunk_sum_kernel(const uint16_t* __restrict__ eobs, int n, uint32_t* __restrict__ sums,
                                                            uint32_t* __restrict__ offs) {
    __shared__ uint32_t s_tot;
    if (threadIdx.x == 0) s_tot = 0;
    if (threadIdx.x == 0 && blockIdx.x == 0) offs[n + 1] = 0;  // the count of levels that did not fit (pass 2 adds to it)
    __syncthreads();
    const int base = blockIdx.x * kPackChunk;
    uint32_t acc = 0;
    for (int i = threadIdx.x; i < kPackChunk; i += blockDim.x) acc += base + i < n ? eobs[base + i] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&s_tot, acc);
    __syncthreads();
    if (threadIdx.x == 0) sums[blockIdx.x] = s_tot;
}
// pass 2, one CTA per chunk of 256 blocks: exclusive offsets of the chunk (warp + shared-memory scan) on top of the levels of all
// chunks before it
__global__ void __launch_bounds__(kPackChunk) eob_offsets_kernel(const uint16_t* __restrict__ eobs, const uint32_t* __restrict__ sums,
                                                                 uint32_t* __restrict__ offs, int n) {
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, base = blockIdx.x * kPackChunk, i = base + threadIdx.x;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    {
        uint32_t b = 0;
        for (int c = threadIdx.x; c < (int)blockIdx.x; c += blockDim.x) b += sums[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
        if (lane == 0 && b) atomicAdd(&s_base, b);
    }
    __syncthreads();
    if (threadIdx.x == 0 && blockIdx.x == gridDim.x - 1) offs[n] = s_base + sums[blockIdx.x];
    const uint32_t v = i < n ? eobs[i] : 0;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < (kPackChunk >> 5) ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    if (i < n) offs[i] = x - v + (warp ? s_warp[warp - 1] : 0) + s_base;
}
// pass 3, one warp per block, as many warps in flight as the GPU holds: the block's coefficients are read in RASTER order
// (coalesced, four independent loads per lane in flight) and each level with scan position < eob goes to its place -- the scatter
// stays inside the block's eob-long output run
template <typename LVL>
__global__ void __launch_bounds__(256) pack_levels_kernel(const int32_t* __restrict__ q_base, const int16_t* __restrict__ iscan_base,
                                                           const SvtB200TrioItem* __restrict__ items, const uint16_t* __restrict__ eobs,
                                                           uint32_t* __restrict__ offs, int n, LVL* __restrict__ out, uint32_t cap) {
    const int lane = threadIdx.x & 31;
    for (int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < n; b += gridDim.x * (blockDim.x >> 5)) {
        const int eob = eobs[b];
        if (!eob) continue;
        const SvtB200QuantItem& qi = items[b].quant;
        const int32_t* q = q_base + qi.q_off;
        const int16_t* isc = iscan_base + qi.scan_off;
        const uint32_t o = offs[b];
        const int nc = qi.n_coeffs;
        for (int rc0 = 0; rc0 < nc; rc0 += 128) {
            int k[4];
            int32_t lv[4];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int rc = rc0 + 32 * j + lane;
                k[j] = rc < nc ? (int)isc[rc] : 0x7fff;
                lv[j] = rc < nc ? q[rc] : 0;
            }
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (k[j] >= eob || o + k[j] >= cap) continue;
                if (sizeof(LVL) == 2 && (lv[j] < -32768 || lv[j] > 32767)) atomicAdd(&offs[n + 1], 1u);  // cannot happen for 8-bit pictures; counted, never silent
                out[o + k[j]] = (LVL)lv[j];
            }
        }
    }
}
extern "C" int svt_b200_pack_levels_dev(const int32_t* d_qcoeff, const int16_t* d_iscan, const SvtB200TrioItem* d_items, const uint16_t* d_eobs,
                                        int n_items, uint32_t* d_offsets, void* d_levels, int level_bytes, uint32_t capacity, void* stream) {
    require_ready();
    if (n_items <= 0 || !d_offsets || !d_levels || !d_iscan || (level_bytes != 2 && level_bytes != 4)) return SVT_B200_ERR_BAD_ARG;
    const int chunks = (n_items + kPackChunk - 1) / kPackChunk;
    if (chunks > 4096) return SVT_B200_ERR_BAD_ARG;  // the chunk sums' scratch holds 4096
    static char key;  // the chunk sums, in this stream's scratch
    uint32_t* d_sums = (uint32_t*)stream_scratch(&key, (cudaStream_t)stream, 4096 * sizeof(uint32_t));
    eob_chunk_sum_kernel<<<chunks, 256, 0, (cudaStream_t)stream>>>(d_eobs, n_items, d_sums, d_offsets);
    B200_LAUNCH_CHECK();
    eob_offsets_kernel<<<chunks, kPackChunk, 0, (cudaStream_t)stream>>>(d_eobs, d_sums, d_offsets, n_items);
    B200_LAUNCH_CHECK();
    const int grid = grid_for((n_items + 7) / 8, 8);
    if (level_bytes == 2)
        pack_levels_kernel<int16_t><<<grid, 256, 0, (cudaStream_t)stream>>>(d_qcoeff, d_iscan, d_items, d_eobs, d_offsets, n_items, (int16_t*)d_levels,
                                                                           capacity);
    else
        pack_levels_kernel<int32_t><<<grid, 256, 0, (cudaStream_t)stream>>>(d_qcoeff, d_iscan, d_items, d_eobs, d_offsets, n_items, (int32_t*)d_levels,
                                                                           capacity);
    B200_LAUNCH_CHECK();
    return SVT_B200_OK;
}

// ---- T1: svt_av1_fwd_txfm2d_WxH (aom_dsp_rtcd.h:121-197; C: transforms.c:2388-2631) ----------------
extern "C" void svt_b200_fwd_txfm2d(int16_t* input, int32_t* output, uint32_t input_stride, int tx_type, int tx_size,
                                    uint8_t bit_depth) {
    svt_b200_fwd_txfm2d_partial(input, output, input_stride, tx_type, tx_size, bit_depth, 0);
}

extern "C" void svt_b200_fwd_txfm2d_partial(int16_t* input, int32_t* output, uint32_t input_stride, int tx_type, int tx_size,
                                            uint8_t bit_depth, int level) {
    (void)bit_depth;  // the forward arithmetic does not depend on it (stage ranges are assert-only)
    require_ready();
    if (level < 0 || level > 2) {
        fprintf(stderr, "[svt_b200] FATAL: partial-transform level %d\n", level);
        abort();
    }
    const int W = tx_w(tx_size), H = tx_h(tx_size);
    if (!host_txcfg(tx_size, tx_type).valid) {
        fprintf(stderr, "[svt_b200] FATAL: invalid (tx_size=%d, tx_type=%d)\n", tx_size, tx_type);
        abort();
    }
    RoundTrip rt;
    SvtB200FwdTxfmItem item{};
    item.src_stride = W;
    item.tx_size = (uint8_t)tx_size;
    item.tx_type = (uint8_t)tx_type;
    item.reserved = (uint16_t)(level << 1);
    auto src = rt.in_rows(input, input_stride, W, H);
    auto it = rt.in(&item, 1);
    auto dst = rt.out(output, (size_t)W * H);
    TxfmBufs b;
    b.residual = rt.dev(src);
    b.coef     = rt.dev(dst);
    launch_class<Forward, uint8_t>(tx_class(tx_size), b, rt.dev(it), 1, nullptr, rt.stream());
    rt.finish();
}

// ---- T1: svt_av1_inv_txfm2d_add_WxH (common_dsp_rtcd.h:106-142; C: inv_transforms.c:2545-2716) on 16-bit pixels, and
// svt_b200_inv_txfm_add_8bit on 8-bit ones ----
template <typename PIX>
static void inv_txfm_add_t1(const int32_t* input, const PIX* pred, int32_t stride_r, PIX* out, int32_t stride_w, int tx_type,
                            int tx_size, int bd) {
    require_ready();
    const int W = tx_w(tx_size), H = tx_h(tx_size);
    const int Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;
    if (!host_txcfg(tx_size, tx_type).valid) {
        fprintf(stderr, "[svt_b200] FATAL: invalid (tx_size=%d, tx_type=%d)\n", tx_size, tx_type);
        abort();
    }
    RoundTrip rt;
    SvtB200InvTxfmItem item{};
    item.pred_stride = item.recon_stride = W;
    item.tx_size = (uint8_t)tx_size;
    item.tx_type = (uint8_t)tx_type;
    item.bd = (uint8_t)bd;
    auto in = rt.in(input, (size_t)Wp * Hp);
    auto pr = rt.in_rows(pred, stride_r, W, H);
    auto it = rt.in(&item, 1);
    auto rec = rt.out_rows(out, stride_w, W, H);
    TxfmBufs b;
    b.pred  = rt.dev(pr);
    b.recon = rt.dev(rec);
    b.dq_in = rt.dev(in);
    launch_class<Inverse, PIX>(tx_class(tx_size), b, rt.dev(it), 1, nullptr, rt.stream());
    rt.finish();
}
extern "C" void svt_b200_inv_txfm2d_add(const int32_t* input, uint16_t* output_r, int32_t stride_r, uint16_t* output_w,
                                        int32_t stride_w, int tx_type, int tx_size, int32_t bd) {
    inv_txfm_add_t1(input, output_r, stride_r, output_w, stride_w, tx_type, tx_size, bd);
}
extern "C" void svt_b200_inv_txfm_add_8bit(const int32_t* dqcoeff, uint8_t* dst_r, int32_t stride_r, uint8_t* dst_w,
                                           int32_t stride_w, int tx_type, int tx_size) {
    inv_txfm_add_t1(dqcoeff, dst_r, stride_r, dst_w, stride_w, tx_type, tx_size, 8);
}

// T2 host variants: caller-owned host planes, one call per batch.
extern "C" int svt_b200_fwd_txfm_batch_host(const int16_t* residual, size_t residual_elems, int32_t* coeff, size_t coeff_elems,
                                            const SvtB200FwdTxfmItem* items, int n_items) {
    require_ready();
    if (n_items <= 0) return n_items == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    int cnt[SVT_B200_TXFM_CLASSES] = {0, 0, 0, 0, 0}, pos[SVT_B200_TXFM_CLASSES];
    for (int i = 0; i < n_items; i++) {
        if (items[i].tx_size >= 19 || !host_txcfg(items[i].tx_size, items[i].tx_type).valid) return SVT_B200_ERR_BAD_ARG;
        cnt[tx_class(items[i].tx_size)]++;
    }
    RoundTrip rt;
    auto src = rt.in(residual, residual_elems);
    auto it = rt.in<SvtB200FwdTxfmItem>(nullptr, n_items);
    auto dst = rt.out<int32_t>(nullptr, coeff_elems);
    SvtB200FwdTxfmItem* hi = rt.fill(it);  // the items grouped by transform class
    for (int c = 0, first = 0; c < SVT_B200_TXFM_CLASSES; first += cnt[c], c++) pos[c] = first;
    for (int i = 0; i < n_items; i++) hi[pos[tx_class(items[i].tx_size)]++] = items[i];
    TxfmBufs b;
    b.residual = rt.dev(src);
    b.coef     = rt.dev(dst);
    launch_batch<Forward, uint8_t>(b, rt.dev(it), cnt, nullptr, rt.stream());
    rt.finish();
    // only the regions the items cover were written; copy those back
    for (int i = 0; i < n_items; i++) {
        const int W = tx_w(items[i].tx_size), H = tx_h(items[i].tx_size);
        memcpy(coeff + items[i].dst_off, rt.host(dst) + items[i].dst_off, (size_t)W * H * 4);
    }
    return SVT_B200_OK;
}

// ---- T1: svt_handle_transform{16x64,32x64,64x16,64x32,64x64}{,_N2_N4} (aom_dsp_rtcd.h:216-240; C: transforms.c:2374-2543)
// Energy of the coefficients a 64-point transform drops (everything outside the top-left
// min(W,32) x min(H,32)), then, for 64-wide blocks, the in-place re-pack of the kept rows to stride 32
// (rows 1..Hp-1 move to offset 32*row; nothing else of the buffer is touched, exactly like the memcpy loop
// of the reference).  The N2_N4 variants only re-pack and return 0.
namespace b200 {
__global__ void __launch_bounds__(256)
handle_transform_kernel(int32_t* __restrict__ buf, int W, int H, int with_energy, unsigned long long* __restrict__ energy) {
    __shared__ int32_t            keep[32 * 32];
    __shared__ unsigned long long tot;
    const int Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;
    if (threadIdx.x == 0) tot = 0;
    __syncthreads();
    unsigned long long e = 0;
    for (int i = threadIdx.x; i < W * H; i += blockDim.x) {
        const int r = i / W, c = i - r * W;
        const int32_t v = buf[i];
        if (r < Hp && c < Wp) keep[r * 32 + c] = v;
        else if (with_energy) e += (unsigned long long)((long long)v * (long long)v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if ((threadIdx.x & 31) == 0 && e) atomicAdd(&tot, e);
    __syncthreads();
    if (W == 64)
        for (int i = threadIdx.x; i < (Hp - 1) * 32; i += blockDim.x) buf[32 + i] = keep[32 + i];  // rows 1..Hp-1
    if (threadIdx.x == 0) *energy = tot;
}
}  // namespace b200

static uint64_t handle_transform_t1(int32_t* output, int W, int H, int with_energy) {
    require_ready();
    RoundTrip rt;
    auto buf = rt.inout(output, (size_t)W * H);
    auto e = rt.out<unsigned long long>(nullptr, 2);
    handle_transform_kernel<<<1, 256, 0, rt.stream()>>>(rt.dev(buf), W, H, with_energy, rt.dev(e));
    B200_LAUNCH_CHECK();
    rt.finish();
    return (uint64_t)*rt.host(e);
}
#define B200_HANDLE(WxH, W, H)                                                                                    \
    extern "C" uint64_t svt_b200_handle_transform##WxH(int32_t* output) { return handle_transform_t1(output, W, H, 1); } \
    extern "C" uint64_t svt_b200_handle_transform##WxH##_N2_N4(int32_t* output) { return W == 64 ? handle_transform_t1(output, W, H, 0) : 0; }
B200_HANDLE(16x64, 16, 64) B200_HANDLE(32x64, 32, 64) B200_HANDLE(64x16, 64, 16) B200_HANDLE(64x32, 64, 32) B200_HANDLE(64x64, 64, 64)
#undef B200_HANDLE

// ---- named T1 wrappers: one symbol per reference function pointer --------------------------------
#define B200_FWD(WxH, SZ)                                                                                       \
    extern "C" void svt_b200_av1_fwd_txfm2d_##WxH(int16_t* input, int32_t* output, uint32_t input_stride,        \
                                                  uint8_t transform_type, uint8_t bit_depth) {                       \
        svt_b200_fwd_txfm2d(input, output, input_stride, transform_type, SZ, bit_depth);                         \
    }
B200_FWD(4x4, 0) B200_FWD(8x8, 1) B200_FWD(16x16, 2) B200_FWD(32x32, 3) B200_FWD(64x64, 4) B200_FWD(4x8, 5) B200_FWD(8x4, 6)
B200_FWD(8x16, 7) B200_FWD(16x8, 8) B200_FWD(16x32, 9) B200_FWD(32x16, 10) B200_FWD(32x64, 11) B200_FWD(64x32, 12)
B200_FWD(4x16, 13) B200_FWD(16x4, 14) B200_FWD(8x32, 15) B200_FWD(32x8, 16) B200_FWD(16x64, 17) B200_FWD(64x16, 18)
#define B200_FWD_PART(WxH, SZ)                                                                                  \
    extern "C" void svt_b200_av1_fwd_txfm2d_##WxH##_N2(int16_t* input, int32_t* output, uint32_t input_stride,   \
                                                       uint8_t transform_type, uint8_t bit_depth) {                  \
        svt_b200_fwd_txfm2d_partial(input, output, input_stride, transform_type, SZ, bit_depth, 1);              \
    }                                                                                                           \
    extern "C" void svt_b200_av1_fwd_txfm2d_##WxH##_N4(int16_t* input, int32_t* output, uint32_t input_stride,   \
                                                       uint8_t transform_type, uint8_t bit_depth) {                  \
        svt_b200_fwd_txfm2d_partial(input, output, input_stride, transform_type, SZ, bit_depth, 2);              \
    }
B200_FWD_PART(4x4, 0) B200_FWD_PART(8x8, 1) B200_FWD_PART(16x16, 2) B200_FWD_PART(32x32, 3) B200_FWD_PART(64x64, 4) B200_FWD_PART(4x8, 5)
B200_FWD_PART(8x4, 6) B200_FWD_PART(8x16, 7) B200_FWD_PART(16x8, 8) B200_FWD_PART(16x32, 9) B200_FWD_PART(32x16, 10) B200_FWD_PART(32x64, 11)
B200_FWD_PART(64x32, 12) B200_FWD_PART(4x16, 13) B200_FWD_PART(16x4, 14) B200_FWD_PART(8x32, 15) B200_FWD_PART(32x8, 16) B200_FWD_PART(16x64, 17)
B200_FWD_PART(64x16, 18)
#define B200_INV_A(WxH, SZ)                                                                                     \
    extern "C" void svt_b200_av1_inv_txfm2d_add_##WxH(const int32_t* input, uint16_t* output_r, int32_t stride_r, \
                                                      uint16_t* output_w, int32_t stride_w, uint8_t tx_type, int32_t bd) { \
        svt_b200_inv_txfm2d_add(input, output_r, stride_r, output_w, stride_w, tx_type, SZ, bd);                 \
    }
#define B200_INV_B(WxH, SZ)                                                                                     \
    extern "C" void svt_b200_av1_inv_txfm2d_add_##WxH(const int32_t* input, uint16_t* output_r, int32_t stride_r, \
                                                      uint16_t* output_w, int32_t stride_w, uint8_t tx_type,     \
                                                      uint8_t tx_size, int32_t bd) {                             \
        (void)tx_size;                                                                                           \
        svt_b200_inv_txfm2d_add(input, output_r, stride_r, output_w, stride_w, tx_type, SZ, bd);                 \
    }
#define B200_INV_C(WxH, SZ)                                                                                     \
    extern "C" void svt_b200_av1_inv_txfm2d_add_##WxH(const int32_t* input, uint16_t* output_r, int32_t stride_r, \
                                                      uint16_t* output_w, int32_t stride_w, uint8_t tx_type,     \
                                                      uint8_t tx_size, int32_t eob, int32_t bd) {                \
        (void)tx_size;                                                                                           \
        (void)eob;                                                                                               \
        svt_b200_inv_txfm2d_add(input, output_r, stride_r, output_w, stride_w, tx_type, SZ, bd);                 \
    }
B200_INV_A(4x4, 0) B200_INV_A(8x8, 1) B200_INV_A(16x16, 2) B200_INV_A(32x32, 3) B200_INV_A(64x64, 4)
B200_INV_B(4x8, 5) B200_INV_B(8x4, 6) B200_INV_B(4x16, 13) B200_INV_B(16x4, 14)
B200_INV_C(8x16, 7) B200_INV_C(16x8, 8) B200_INV_C(16x32, 9) B200_INV_C(32x16, 10) B200_INV_C(32x64, 11) B200_INV_C(64x32, 12)
B200_INV_C(8x32, 15) B200_INV_C(32x8, 16) B200_INV_C(16x64, 17) B200_INV_C(64x16, 18)
