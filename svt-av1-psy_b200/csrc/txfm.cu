// txfm.cu -- K5 forward 2-D transforms, K6 inverse 2-D transforms + reconstruction (sm_90a).
//
// Reference behaviour restated: av1_tranform_two_d_core_c (Source/Lib/Codec/transforms.c:2259-2324)
// and inv_txfm2d_add_c (Source/Lib/Codec/inv_transforms.c:2459-2534), for all 19 transform sizes and
// 16 transform types, 8/10/12-bit.  The 2-D configuration table (flips, per-pass kernel, cos_bit,
// shifts) is dumped from the reference (txfm_cfg.inc); the 1-D networks are txfm_graphs.inc.
//
// H100 mapping: a team of max(W,H) threads per transform block (4, 8, 16, 32 or 64: the block's
// "team class"), one thread per column in the column pass and one per row in the row pass, each
// running the generated straight-line network on its vector in registers (txfm_tables.cuh).  The
// block sits in shared memory in element-major order with an odd pitch, so the passes and the
// transposing hand-over are bank-conflict free; residual loads / coefficient stores are coalesced rows.
#include <map>
#include <mutex>
#include "txfm_tables.cuh"
#include "quant_one.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

static TxCfg h_txcfg[19][16];
const TxCfg& host_txcfg(int size, int type) { return h_txcfg[size][type]; }

void txfm_tables_init() {
    memset(h_txcfg, 0, sizeof(h_txcfg));
    static int32_t cosv[7][64], sinv[7][5];
#define TXC(sz, ty, v, fud, flr, fs0, fs1, fs2, fcbc, fcbr, ftc, ftr, iud, ilr, is0, is1, icbc, icbr, itc, itr) \
    h_txcfg[sz][ty] = TxCfg{v, fud, flr, fs0, fs1, fs2, fcbc, fcbr, ftc, ftr, iud, ilr, is0, is1, icbc, icbr, itc, itr};
#define TXCOS(bit, ...) { const int32_t t[64] = {__VA_ARGS__}; memcpy(cosv[bit - 10], t, sizeof(t)); }
#define TXSIN(bit, ...) { const int32_t t[5] = {__VA_ARGS__}; memcpy(sinv[bit - 10], t, sizeof(t)); }
#include "txfm_cfg.inc"
#undef TXC
#undef TXCOS
#undef TXSIN
    B200_CUDA_CHECK(cudaMemcpyToSymbol(c_txcfg, h_txcfg, sizeof(h_txcfg)));
    B200_CUDA_CHECK(cudaMemcpyToSymbol(c_cospi, cosv, sizeof(cosv)));
    B200_CUDA_CHECK(cudaMemcpyToSymbol(c_sinpi, sinv, sizeof(sinv)));
}

// ints between the shared-memory areas (two planes) of consecutive teams.  Teams that share a warp must not
// land on the same banks: a team of T lanes covers T banks with its odd pitch, so the stride is made
// congruent to T modulo 32.
__host__ __device__ constexpr int team_stride(int team) {
    return team == 4 ? 68 : (team == 8 ? 152 : (team == 16 ? 560 : 2 * team * (team + 1)));
}

__host__ __device__ inline int rect_log_ratio(int w, int h) {  // get_rect_tx_log_ratio
    if (w == h) return 0;
    if (w > h) return w == 2 * h ? 1 : (w == 4 * h ? 2 : 3);
    return h == 2 * w ? -1 : (h == 4 * w ? -2 : -3);
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <int TEAM, int THREADS>
__global__ void __launch_bounds__(THREADS)
fwd_txfm_kernel(const int16_t* __restrict__ src_base, int32_t* __restrict__ dst_base,
                const SvtB200FwdTxfmItem* __restrict__ items, int n_items) {
    extern __shared__ __align__(16) int32_t tsm[];
    // a 64-point block is alone in its CTA: all THREADS move data, the first 64 run the passes
    constexpr int TEAMS = TEAM >= 64 ? 1 : THREADS / TEAM, PLANE = TEAM * (TEAM + 1), MOVERS = TEAM >= 64 ? THREADS : TEAM;
    const int     team  = TEAM >= 64 ? 0 : threadIdx.x / TEAM, tid = TEAM >= 64 ? threadIdx.x : threadIdx.x % TEAM;
    int32_t*      A     = tsm + (size_t)team * team_stride(TEAM);
    int32_t*      B     = A + PLANE;

    for (int it = blockIdx.x * TEAMS + team; it < n_items; it += gridDim.x * TEAMS) {
        const SvtB200FwdTxfmItem item = items[it];
        const int   sz = item.tx_size, W = tx_w(sz), H = tx_h(sz);
        const int   lgW = 31 - __clz(W);
        const TxCfg cfg = c_txcfg[sz][item.tx_type];
        const int16_t* src = src_base + item.src_off;
        int32_t*       dst = dst_base + item.dst_off;
        const int P1 = W + 1, P2 = H + 1;
        const int part_shift = (item.reserved >> 1) & 3;  // 0 full, 1 = N2, 2 = N4
        // load, optional up/down flip, pre-shift (transforms.c:2286-2294)
        for (int idx = tid; idx < W * H; idx += MOVERS) {
            const int r = idx >> lgW, c = idx & (W - 1);
            const int rr = cfg.f_ud ? (H - 1 - r) : r;
            A[r * P1 + c] = round_shift_arr((int32_t)src[(size_t)rr * item.src_stride + c], -cfg.f_s0);
        }
        team_sync<TEAM>();
        txfm_pass_1d<TEAM, false>(cfg.f_tc, A, H, W, P1, cfg.f_cbc, 0, tid);  // columns: vector v = column v
        team_sync<TEAM>();
        // round-shift, optional left/right flip, hand over transposed (element = column)
        for (int idx = tid; idx < W * H; idx += MOVERS) {
            const int r = idx >> lgW, c = idx & (W - 1);
            const int cc = cfg.f_lr ? (W - 1 - c) : c;
            B[cc * P2 + r] = round_shift_arr(A[r * P1 + c], -cfg.f_s1);
        }
        team_sync<TEAM>();
        txfm_pass_1d<TEAM, false>(cfg.f_tr, B, W, H, P2, cfg.f_cbr, 0, tid);  // rows: vector v = row v
        team_sync<TEAM>();
        const int rect = rect_log_ratio(W, H);
        for (int idx = tid; idx < W * H; idx += MOVERS) {
            const int r = idx >> lgW, c = idx & (W - 1);
            int32_t   v = round_shift_arr(B[c * P2 + r], -cfg.f_s2);
            if (rect == 1 || rect == -1) v = round_shift64((long long)v * kNewSqrt2, 12);
            // N2 / N4 (av1_tranform_two_d_core_N2_c / _N4_c, transforms.c:5202, 6769): the top-left half / quarter
            // of every dimension, identical to the full transform's values there, zero everywhere else
            if (part_shift && (r >= max(H >> part_shift, 1) || c >= max(W >> part_shift, 1))) v = 0;
            if (item.reserved & 1) {  // packed output: keep the top-left min(W,32) x min(H,32) (svt_handle_transform64x64 repack, transforms.c:2374)
                const int Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;
                if (r < Hp && c < Wp) dst[r * Wp + c] = v;
            } else
                dst[idx] = v;
        }
        team_sync<TEAM>();
    }
}

// ------------------------------------------------------------------------------------------------
// inverse + reconstruction
// ------------------------------------------------------------------------------------------------
template <int TEAM, int THREADS, typename PIX>
__global__ void __launch_bounds__(THREADS)
inv_txfm_kernel(const int32_t* __restrict__ coef_base, const PIX* __restrict__ pred_base, PIX* __restrict__ recon_base,
                const SvtB200InvTxfmItem* __restrict__ items, int n_items) {
    extern __shared__ __align__(16) int32_t tsm[];
    // a 64-point block is alone in its CTA: all THREADS move data, the first 64 run the passes
    constexpr int TEAMS = TEAM >= 64 ? 1 : THREADS / TEAM, PLANE = TEAM * (TEAM + 1), MOVERS = TEAM >= 64 ? THREADS : TEAM;
    const int     team  = TEAM >= 64 ? 0 : threadIdx.x / TEAM, tid = TEAM >= 64 ? threadIdx.x : threadIdx.x % TEAM;
    int32_t*      A     = tsm + (size_t)team * team_stride(TEAM);
    int32_t*      B     = A + PLANE;

    for (int it = blockIdx.x * TEAMS + team; it < n_items; it += gridDim.x * TEAMS) {
        const SvtB200InvTxfmItem item = items[it];
        const int   sz = item.tx_size, W = tx_w(sz), H = tx_h(sz), bd = item.bd;
        const int   lgW = 31 - __clz(W);
        const TxCfg cfg = c_txcfg[sz][item.tx_type];
        const int32_t* in = coef_base + item.coef_off;
        const int Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;  // 64-point dims arrive packed (inv_transforms.c:2567-2686)
        const int P1 = H + 1, P2 = W + 1;
        const int rect = rect_log_ratio(W, H);
        const int row_clamp = bd + 8;
        const int col_clamp = (bd + 6) > 16 ? (bd + 6) : 16;
        const int opt_row = bd == 8 ? 16 : (bd == 10 ? 18 : 20);  // svt_av1_gen_inv_stage_range
        const int opt_col = bd == 12 ? 18 : 16;
        // rows first: element = column, vector = row
        for (int idx = tid; idx < W * H; idx += MOVERS) {
            const int r = idx >> lgW, c = idx & (W - 1);
            int32_t   v = (r < Hp && c < Wp) ? in[r * Wp + c] : 0;
            if (rect == 1 || rect == -1) v = round_shift64((long long)v * kNewInvSqrt2, 12);
            A[c * P1 + r] = clamp_bits(v, row_clamp);
        }
        team_sync<TEAM>();
        txfm_pass_1d<TEAM, true>(cfg.i_tr, A, W, H, P1, cfg.i_cbr, opt_row, tid);
        team_sync<TEAM>();
        for (int idx = tid; idx < W * H; idx += MOVERS) {
            const int r = idx >> lgW, c = idx & (W - 1);
            const int cs = cfg.i_lr ? (W - 1 - c) : c;
            B[r * P2 + c] = clamp_bits(round_shift_arr(A[cs * P1 + r], -cfg.i_s0), col_clamp);
        }
        team_sync<TEAM>();
        txfm_pass_1d<TEAM, true>(cfg.i_tc, B, H, W, P2, cfg.i_cbc, opt_col, tid);
        team_sync<TEAM>();
        const PIX* pr = pred_base + item.pred_off;
        PIX*       pw = recon_base + item.recon_off;
        const long long int_max = (1ll << (7 + bd)) - 1 + (914ll << (bd - 7));  // check_range, inv_transforms.c:2401
        const int       pix_max = (1 << bd) - 1;
        for (int idx = tid; idx < W * H; idx += MOVERS) {
            const int r = idx >> lgW, c = idx & (W - 1);
            const int rs = cfg.i_ud ? (H - 1 - r) : r;
            long long t  = (long long)round_shift_arr(B[rs * P2 + c], -cfg.i_s1);
            t            = t < -int_max - 1 ? -int_max - 1 : (t > int_max ? int_max : t);
            int p        = (int)pr[(size_t)r * item.pred_stride + c] + (int)t;
            p            = p < 0 ? 0 : (p > pix_max ? pix_max : p);
            pw[(size_t)r * item.recon_stride + c] = (PIX)p;
        }
        team_sync<TEAM>();
    }
}

// ------------------------------------------------------------------------------------------------
// fused: forward transform -> quantise -> inverse transform + reconstruction of one block
// (the per-block chain of the final encode pass, coding_loop.c:405-658) without leaving shared memory:
// the coefficients and the dequantised levels never travel through HBM between the three steps.
// ------------------------------------------------------------------------------------------------
template <int TEAM, int THREADS, typename PIX>
__global__ void __launch_bounds__(THREADS)
trio_txfm_kernel(const int16_t* __restrict__ src_base, const PIX* __restrict__ srcpix_base /*non-null: residual = source - prediction, formed here*/,
                 const PIX* __restrict__ pred_base, PIX* __restrict__ recon_base,
                 int32_t* __restrict__ q_base, int32_t* __restrict__ dq_base /*may be null*/, const int16_t* __restrict__ iscan_base,
                 const uint8_t* __restrict__ qm_base, const SvtB200TrioItem* __restrict__ items, int n_items,
                 uint16_t* __restrict__ eobs) {
    extern __shared__ __align__(16) int32_t tsm[];
    // big blocks are few: one block per CTA (SOLO), all THREADS move its data, the first TEAM run the passes --
    // the block's critical path is global-memory round trips, and 4x the movers means 4x fewer of them
    constexpr bool SOLO = TEAM >= 32;
    constexpr int  TEAMS = SOLO ? 1 : THREADS / TEAM, PLANE = TEAM * (TEAM + 1), MOVERS = SOLO ? THREADS : TEAM;
    const int      team  = SOLO ? 0 : threadIdx.x / TEAM, tid = SOLO ? threadIdx.x : threadIdx.x % TEAM;
    int32_t*      A     = tsm + (size_t)team * team_stride(TEAM);
    int32_t*      B     = A + PLANE;
    __shared__ int s_eob;

    for (int it = blockIdx.x * TEAMS + team; it < n_items; it += gridDim.x * TEAMS) {
        const SvtB200TrioItem& item = items[it];
        const int   sz = item.fwd.tx_size, W = tx_w(sz), H = tx_h(sz), bd = item.inv.bd;
        const int   lgW = 31 - __clz(W);
        const TxCfg cfg = c_txcfg[sz][item.fwd.tx_type];
        const int   rect = rect_log_ratio(W, H);
        const int   Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;
        {   // ---- forward (fwd_txfm_kernel) ----
            const int P1 = W + 1, P2 = H + 1, sstride = item.fwd.src_stride;
            if (srcpix_base) {  // svt_aom_residual_kernel fused in: the source picture shares the residual plane's geometry
                const PIX* sp = srcpix_base + item.fwd.src_off;
                const PIX* pp = pred_base + item.inv.pred_off;
                const int  pstride = item.inv.pred_stride;
#pragma unroll 4
                for (int idx = tid; idx < W * H; idx += MOVERS) {
                    const int r = idx >> lgW, c = idx & (W - 1);
                    const int rr = cfg.f_ud ? (H - 1 - r) : r;
                    const int32_t d = (int32_t)sp[(size_t)rr * sstride + c] - (int32_t)pp[(size_t)rr * pstride + c];
                    A[r * P1 + c] = round_shift_arr(d, -cfg.f_s0);
                }
            } else {
                const int16_t* src = src_base + item.fwd.src_off;
#pragma unroll 4
                for (int idx = tid; idx < W * H; idx += MOVERS) {
                    const int r = idx >> lgW, c = idx & (W - 1);
                    const int rr = cfg.f_ud ? (H - 1 - r) : r;
                    A[r * P1 + c] = round_shift_arr((int32_t)src[(size_t)rr * sstride + c], -cfg.f_s0);
                }
            }
            team_sync<TEAM, SOLO>();
            txfm_pass_1d<TEAM, false, true>(cfg.f_tc, A, H, W, P1, cfg.f_cbc, 0, tid);  // rows >= Hp of the result are not needed
            team_sync<TEAM, SOLO>();
#pragma unroll 4
            for (int idx = tid; idx < W * Hp; idx += MOVERS) {  // only the Hp rows that survive the packing
                const int r = idx >> lgW, c = idx & (W - 1);
                const int cc = cfg.f_lr ? (W - 1 - c) : c;
                B[cc * P2 + r] = round_shift_arr(A[r * P1 + c], -cfg.f_s1);
            }
            team_sync<TEAM, SOLO>();
            txfm_pass_1d<TEAM, false, true>(cfg.f_tr, B, W, Hp, P2, cfg.f_cbr, 0, tid);
            team_sync<TEAM, SOLO>();
        }
        int block_eob = 0;
        {   // ---- quantise the (packed) coefficients; the dequantised levels become the inverse's input plane ----
            const SvtB200QuantItem qi = item.quant;
            const uint8_t* qm  = qi.qm_off == SVT_B200_NO_QM ? nullptr : qm_base + qi.qm_off;
            const uint8_t* iqm = qi.iqm_off == SVT_B200_NO_QM ? nullptr : qm_base + qi.iqm_off;
            const int16_t* iscan = iscan_base + qi.scan_off;
            int32_t*       qc = q_base + qi.q_off;
            int32_t*       dqc = dq_base ? dq_base + qi.dq_off : nullptr;
            const int P2 = H + 1, P1i = H + 1;  // forward result: B[c*P2 + r]; inverse input: A[c*P1i + r]
            const int row_clamp = bd + 8;
            if (SOLO && threadIdx.x == 0) s_eob = 0;
            int eob = 0;
#pragma unroll 4
            for (int idx = tid; idx < W * H; idx += MOVERS) {
                const int r = idx >> lgW, c = idx & (W - 1);
                int32_t   dq = 0;
                if (r < Hp && c < Wp) {
                    int32_t v = round_shift_arr(B[c * P2 + r], -cfg.f_s2);
                    if (rect == 1 || rect == -1) v = round_shift64((long long)v * kNewSqrt2, 12);
                    const int rc = r * Wp + c;
                    int32_t   q;
                    quant_one(qi, v, rc, qm, iqm, q, dq);
                    qc[rc] = q;
                    if (dqc) dqc[rc] = dq;
                    if (q) eob = max(eob, (int)iscan[rc] + 1);
                    if (rect == 1 || rect == -1) dq = round_shift64((long long)dq * kNewInvSqrt2, 12);
                    dq = clamp_bits(dq, row_clamp);
                }
                A[c * P1i + r] = dq;  // rows first: element = column, vector = row
            }
            if constexpr (SOLO) {
                __syncthreads();
                if (eob) atomicMax(&s_eob, eob);
                __syncthreads();
                eob = s_eob;
                if (threadIdx.x == 0) eobs[it] = (uint16_t)eob;
            } else {
                const unsigned mask = TEAM == 32 ? 0xffffffffu : (((1u << TEAM) - 1u) << ((threadIdx.x & 31) / TEAM * TEAM));
#pragma unroll
                for (int o = TEAM / 2; o > 0; o >>= 1) eob = max(eob, __shfl_xor_sync(mask, eob, o));
                if (tid == 0) eobs[it] = (uint16_t)eob;
                team_sync<TEAM, SOLO>();
            }
            block_eob = eob;
        }
        if (block_eob == 0) {
            // every level is zero: the inverse of an all-zero plane is zero, the reconstruction is the prediction
            // (the encode pass takes the same shortcut, coding_loop.c: eob == 0 -> prediction copied); team-uniform branch
            const PIX* pr = pred_base + item.inv.pred_off;
            PIX*       pw = recon_base + item.inv.recon_off;
            if (pr != pw) {
#pragma unroll 4
                for (int idx = tid; idx < W * H; idx += MOVERS) {
                    const int r = idx >> lgW, c = idx & (W - 1);
                    pw[(size_t)r * item.inv.recon_stride + c] = pr[(size_t)r * item.inv.pred_stride + c];
                }
            }
            team_sync<TEAM, SOLO>();
        } else {   // ---- inverse + reconstruction (inv_txfm_kernel) ----
            const int P1 = H + 1, P2 = W + 1;
            const int col_clamp = (bd + 6) > 16 ? (bd + 6) : 16;
            const int opt_row = bd == 8 ? 16 : (bd == 10 ? 18 : 20);
            const int opt_col = bd == 12 ? 18 : 16;
            txfm_pass_1d<TEAM, true, true>(cfg.i_tr, A, W, Hp, P1, cfg.i_cbr, opt_row, tid);  // rows >= Hp are zero and stay zero
            team_sync<TEAM, SOLO>();
#pragma unroll 4
            for (int idx = tid; idx < W * H; idx += MOVERS) {
                const int r = idx >> lgW, c = idx & (W - 1);
                const int cs = cfg.i_lr ? (W - 1 - c) : c;
                B[r * P2 + c] = clamp_bits(round_shift_arr(A[cs * P1 + r], -cfg.i_s0), col_clamp);
            }
            team_sync<TEAM, SOLO>();
            txfm_pass_1d<TEAM, true, true>(cfg.i_tc, B, H, W, P2, cfg.i_cbc, opt_col, tid);
            team_sync<TEAM, SOLO>();
            const PIX* pr = pred_base + item.inv.pred_off;
            PIX*       pw = recon_base + item.inv.recon_off;
            const long long int_max = (1ll << (7 + bd)) - 1 + (914ll << (bd - 7));
            const int       pix_max = (1 << bd) - 1;
#pragma unroll 4
            for (int idx = tid; idx < W * H; idx += MOVERS) {
                const int r = idx >> lgW, c = idx & (W - 1);
                const int rs = cfg.i_ud ? (H - 1 - r) : r;
                long long t  = (long long)round_shift_arr(B[rs * P2 + c], -cfg.i_s1);
                t            = t < -int_max - 1 ? -int_max - 1 : (t > int_max ? int_max : t);
                int p        = (int)pr[(size_t)r * item.inv.pred_stride + c] + (int)t;
                p            = p < 0 ? 0 : (p > pix_max ? pix_max : p);
                pw[(size_t)r * item.inv.recon_stride + c] = (PIX)p;
            }
            team_sync<TEAM, SOLO>();
        }
    }
}

// team class of a transform size: log2(max(W,H)) - 2
static inline int tx_class(int sz) {
    const int m = tx_w(sz) > tx_h(sz) ? tx_w(sz) : tx_h(sz);
    return m == 4 ? 0 : (m == 8 ? 1 : (m == 16 ? 2 : (m == 32 ? 3 : 4)));
}

template <typename K>
static void set_smem_attr(K kernel, size_t smem) {
    if (smem > 48 * 1024) B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
}

// CTA size per team class: small enough that a picture's worth of blocks of that class spreads over all SMs
template <int TEAM> constexpr int class_threads() { return TEAM == 16 ? 128 : (TEAM == 32 ? 64 : 256); }

template <int TEAM>
static void launch_fwd_class(const int16_t* d_src, int32_t* d_dst, const SvtB200FwdTxfmItem* d_items, int n, cudaStream_t st) {
    constexpr int    THREADS = class_threads<TEAM>(), TEAMS = TEAM >= 64 ? 1 : THREADS / TEAM;
    constexpr size_t smem = (size_t)TEAMS * team_stride(TEAM) * 4;
    static int attr = -1;  // the initialisation (epoch) the attribute was applied in
    if (attr != epoch()) { set_smem_attr(fwd_txfm_kernel<TEAM, THREADS>, smem); attr = epoch(); }
    const int per_sm = (int)((200 * 1024) / (smem + 1024)) < 2048 / THREADS ? (int)((200 * 1024) / (smem + 1024)) : 2048 / THREADS;
    fwd_txfm_kernel<TEAM, THREADS><<<grid_for((n + TEAMS - 1) / TEAMS, per_sm), THREADS, smem, st>>>(d_src, d_dst, d_items, n);
    B200_LAUNCH_CHECK();
}
void launch_fwd_txfm(const int16_t* d_src, int32_t* d_dst, const SvtB200FwdTxfmItem* d_items, int n, int cls, cudaStream_t st) {
    if (n <= 0) return;
    switch (cls) {
    case 0: launch_fwd_class<4>(d_src, d_dst, d_items, n, st); break;
    case 1: launch_fwd_class<8>(d_src, d_dst, d_items, n, st); break;
    case 2: launch_fwd_class<16>(d_src, d_dst, d_items, n, st); break;
    case 3: launch_fwd_class<32>(d_src, d_dst, d_items, n, st); break;
    default: launch_fwd_class<64>(d_src, d_dst, d_items, n, st); break;
    }
}

template <int TEAM, typename PIX>
static void launch_inv_class(const int32_t* d_coef, const PIX* d_pred, PIX* d_recon, const SvtB200InvTxfmItem* d_items, int n,
                             cudaStream_t st) {
    constexpr int    THREADS = class_threads<TEAM>(), TEAMS = TEAM >= 64 ? 1 : THREADS / TEAM;
    constexpr size_t smem = (size_t)TEAMS * team_stride(TEAM) * 4;
    static int attr = -1;  // the initialisation (epoch) the attribute was applied in
    if (attr != epoch()) { set_smem_attr(inv_txfm_kernel<TEAM, THREADS, PIX>, smem); attr = epoch(); }
    const int per_sm = (int)((200 * 1024) / (smem + 1024)) < 2048 / THREADS ? (int)((200 * 1024) / (smem + 1024)) : 2048 / THREADS;
    inv_txfm_kernel<TEAM, THREADS, PIX><<<grid_for((n + TEAMS - 1) / TEAMS, per_sm), THREADS, smem, st>>>(d_coef, d_pred, d_recon, d_items, n);
    B200_LAUNCH_CHECK();
}
template <typename PIX>
void launch_inv_txfm(const int32_t* d_coef, const PIX* d_pred, PIX* d_recon, const SvtB200InvTxfmItem* d_items, int n, int cls,
                     cudaStream_t st) {
    if (n <= 0) return;
    switch (cls) {
    case 0: launch_inv_class<4, PIX>(d_coef, d_pred, d_recon, d_items, n, st); break;
    case 1: launch_inv_class<8, PIX>(d_coef, d_pred, d_recon, d_items, n, st); break;
    case 2: launch_inv_class<16, PIX>(d_coef, d_pred, d_recon, d_items, n, st); break;
    case 3: launch_inv_class<32, PIX>(d_coef, d_pred, d_recon, d_items, n, st); break;
    default: launch_inv_class<64, PIX>(d_coef, d_pred, d_recon, d_items, n, st); break;
    }
}

template <int TEAM, typename PIX>
static void launch_trio_class(const int16_t* d_src, const PIX* d_srcpix, const PIX* d_pred, PIX* d_recon, int32_t* d_q, int32_t* d_dq, const int16_t* d_iscan,
                              const uint8_t* d_qm, const SvtB200TrioItem* d_items, int n, uint16_t* d_eobs, cudaStream_t st) {
    if (n <= 0) return;
    constexpr int    THREADS = TEAM == 32 ? 128 : class_threads<TEAM>(), TEAMS = TEAM >= 32 ? 1 : THREADS / TEAM;
    constexpr size_t smem = (size_t)TEAMS * team_stride(TEAM) * 4;
    static int attr = -1;  // the initialisation (epoch) the attribute was applied in
    if (attr != epoch()) { set_smem_attr(trio_txfm_kernel<TEAM, THREADS, PIX>, smem); attr = epoch(); }
    const int per_sm = (int)((200 * 1024) / (smem + 1024)) < 2048 / THREADS ? (int)((200 * 1024) / (smem + 1024)) : 2048 / THREADS;
    trio_txfm_kernel<TEAM, THREADS, PIX><<<grid_for((n + TEAMS - 1) / TEAMS, per_sm), THREADS, smem, st>>>(d_src, d_srcpix, d_pred, d_recon, d_q, d_dq, d_iscan,
                                                                                                     d_qm, d_items, n, d_eobs);
    B200_LAUNCH_CHECK();
}
template <typename PIX>
static void launch_trio(const int16_t* d_src, const PIX* d_srcpix, const PIX* d_pred, PIX* d_recon, int32_t* d_q, int32_t* d_dq, const int16_t* d_iscan,
                        const uint8_t* d_qm, const SvtB200TrioItem* d_items, const int* n_per_class, uint16_t* d_eobs, cudaStream_t user) {
    int first[SVT_B200_TXFM_CLASSES + 1] = {0};
    for (int c = 0; c < SVT_B200_TXFM_CLASSES; c++) first[c + 1] = first[c] + n_per_class[c];
    ForkJoin& fj = fork_streams(user);
    for (int c = SVT_B200_TXFM_CLASSES - 1; c >= 0; c--) {
        cudaStream_t st = c >= 2 ? fj.side[c - 2] : user;
        const SvtB200TrioItem* it = d_items + first[c];
        uint16_t* eo = d_eobs + first[c];
        const int n = n_per_class[c];
        switch (c) {
        case 0: launch_trio_class<4, PIX>(d_src, d_srcpix, d_pred, d_recon, d_q, d_dq, d_iscan, d_qm, it, n, eo, st); break;
        case 1: launch_trio_class<8, PIX>(d_src, d_srcpix, d_pred, d_recon, d_q, d_dq, d_iscan, d_qm, it, n, eo, st); break;
        case 2: launch_trio_class<16, PIX>(d_src, d_srcpix, d_pred, d_recon, d_q, d_dq, d_iscan, d_qm, it, n, eo, st); break;
        case 3: launch_trio_class<32, PIX>(d_src, d_srcpix, d_pred, d_recon, d_q, d_dq, d_iscan, d_qm, it, n, eo, st); break;
        default: launch_trio_class<64, PIX>(d_src, d_srcpix, d_pred, d_recon, d_q, d_dq, d_iscan, d_qm, it, n, eo, st); break;
        }
    }
    join_streams(fj, user);
}

}  // namespace b200

using namespace b200;

extern "C" int svt_b200_txfm_valid(int tx_size, int tx_type) {
    if (tx_size < 0 || tx_size >= 19 || tx_type < 0 || tx_type >= 16) return 0;
    require_ready();
    return host_txcfg(tx_size, tx_type).valid;
}

extern "C" int svt_b200_txfm_team_class(int tx_size) { return (tx_size < 0 || tx_size >= 19) ? -1 : tx_class(tx_size); }

// The five class launches of a batch are independent: the three big-block classes (few, long-running
// CTAs) go to side streams forked from the caller's stream and joined back into it, so the many
// small blocks fill the SMs the big ones leave idle.
extern "C" int svt_b200_fwd_txfm_batch_dev(const int16_t* d_residual, int32_t* d_coeff, const SvtB200FwdTxfmItem* d_items,
                                           const int n_per_class[SVT_B200_TXFM_CLASSES], void* stream) {
    require_ready();
    if (!n_per_class) return SVT_B200_ERR_BAD_ARG;
    int first[SVT_B200_TXFM_CLASSES + 1] = {0};
    for (int c = 0; c < SVT_B200_TXFM_CLASSES; c++) {
        if (n_per_class[c] < 0) return SVT_B200_ERR_BAD_ARG;
        first[c + 1] = first[c] + n_per_class[c];
    }
    ForkJoin& fj = fork_streams((cudaStream_t)stream);
    for (int c = SVT_B200_TXFM_CLASSES - 1; c >= 0; c--)
        launch_fwd_txfm(d_residual, d_coeff, d_items + first[c], n_per_class[c], c, c >= 2 ? fj.side[c - 2] : (cudaStream_t)stream);
    join_streams(fj, (cudaStream_t)stream);
    return SVT_B200_OK;
}

extern "C" int svt_b200_inv_txfm_batch_dev(const int32_t* d_coeff, const void* d_pred, void* d_recon,
                                           const SvtB200InvTxfmItem* d_items, const int n_per_class[SVT_B200_TXFM_CLASSES],
                                           int pixel_bytes, void* stream) {
    require_ready();
    if (!n_per_class || (pixel_bytes != 1 && pixel_bytes != 2)) return SVT_B200_ERR_BAD_ARG;
    int first[SVT_B200_TXFM_CLASSES + 1] = {0};
    for (int c = 0; c < SVT_B200_TXFM_CLASSES; c++) {
        if (n_per_class[c] < 0) return SVT_B200_ERR_BAD_ARG;
        first[c + 1] = first[c] + n_per_class[c];
    }
    ForkJoin& fj = fork_streams((cudaStream_t)stream);
    for (int c = SVT_B200_TXFM_CLASSES - 1; c >= 0; c--) {
        cudaStream_t st = c >= 2 ? fj.side[c - 2] : (cudaStream_t)stream;
        if (pixel_bytes == 1) launch_inv_txfm<uint8_t>(d_coeff, (const uint8_t*)d_pred, (uint8_t*)d_recon, d_items + first[c], n_per_class[c], c, st);
        else launch_inv_txfm<uint16_t>(d_coeff, (const uint16_t*)d_pred, (uint16_t*)d_recon, d_items + first[c], n_per_class[c], c, st);
    }
    join_streams(fj, (cudaStream_t)stream);
    return SVT_B200_OK;
}

static int trio_entry(const int16_t* d_residual, const void* d_source, const void* d_pred, void* d_recon, int32_t* d_qcoeff,
                      int32_t* d_dqcoeff, const int16_t* d_iscan, const uint8_t* d_qm, const SvtB200TrioItem* d_items,
                      const int n_per_class[SVT_B200_TXFM_CLASSES], uint16_t* d_eobs, int pixel_bytes, void* stream) {
    require_ready();
    if (!n_per_class || !d_iscan || !d_qcoeff || !d_eobs || (pixel_bytes != 1 && pixel_bytes != 2)) return SVT_B200_ERR_BAD_ARG;
    if (!d_residual == !d_source) return SVT_B200_ERR_BAD_ARG;  // exactly one of the two inputs
    for (int c = 0; c < SVT_B200_TXFM_CLASSES; c++)
        if (n_per_class[c] < 0) return SVT_B200_ERR_BAD_ARG;
    if (pixel_bytes == 1)
        launch_trio<uint8_t>(d_residual, (const uint8_t*)d_source, (const uint8_t*)d_pred, (uint8_t*)d_recon, d_qcoeff, d_dqcoeff, d_iscan, d_qm,
                             d_items, n_per_class, d_eobs, (cudaStream_t)stream);
    else
        launch_trio<uint16_t>(d_residual, (const uint16_t*)d_source, (const uint16_t*)d_pred, (uint16_t*)d_recon, d_qcoeff, d_dqcoeff, d_iscan, d_qm,
                              d_items, n_per_class, d_eobs, (cudaStream_t)stream);
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
    if (chunks > 4096) return SVT_B200_ERR_BAD_ARG;  // the chunk sums live in the tail of the offsets buffer's lane scratch
    static std::mutex mu;
    static std::map<cudaStream_t, uint32_t*> sums_of;  // per-stream scratch: concurrent frames on different streams do not share it
    uint32_t* d_sums;
    {
        std::lock_guard<std::mutex> lk(mu);
        auto it = sums_of.find((cudaStream_t)stream);
        static ResetHook hook([] { sums_of.clear(); });
        if (it == sums_of.end()) {
            d_sums = (uint32_t*)scratch_alloc(4096 * sizeof(uint32_t));
            sums_of[(cudaStream_t)stream] = d_sums;
        } else
            d_sums = it->second;
    }
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
    LaneGuard l;
    size_t o_src = l->alloc((size_t)W * H * 2), o_it = l->alloc(sizeof(SvtB200FwdTxfmItem));
    size_t in_end = l->used;
    size_t o_dst = l->alloc((size_t)W * H * 4);
    for (int r = 0; r < H; r++) memcpy(l->h<int16_t>(o_src) + r * W, input + (size_t)r * input_stride, W * 2);
    SvtB200FwdTxfmItem* it = l->h<SvtB200FwdTxfmItem>(o_it);
    memset(it, 0, sizeof(*it));
    it->src_stride = W;
    it->tx_size = (uint8_t)tx_size;
    it->tx_type = (uint8_t)tx_type;
    it->reserved = (uint16_t)(level << 1);
    l->h2d(0, in_end);
    launch_fwd_txfm(l->d<int16_t>(o_src), l->d<int32_t>(o_dst), l->d<SvtB200FwdTxfmItem>(o_it), 1, tx_class(tx_size), l->stream);
    l->d2h(o_dst, (size_t)W * H * 4);
    l->sync();
    memcpy(output, l->h<int32_t>(o_dst), (size_t)W * H * 4);
}

// ---- T1: svt_av1_inv_txfm2d_add_WxH (common_dsp_rtcd.h:106-142; C: inv_transforms.c:2545-2716) ----
extern "C" void svt_b200_inv_txfm2d_add(const int32_t* input, uint16_t* output_r, int32_t stride_r, uint16_t* output_w,
                                        int32_t stride_w, int tx_type, int tx_size, int32_t bd) {
    require_ready();
    const int W = tx_w(tx_size), H = tx_h(tx_size);
    const int Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;
    if (!host_txcfg(tx_size, tx_type).valid) {
        fprintf(stderr, "[svt_b200] FATAL: invalid (tx_size=%d, tx_type=%d)\n", tx_size, tx_type);
        abort();
    }
    LaneGuard l;
    size_t o_in = l->alloc((size_t)Wp * Hp * 4), o_pred = l->alloc((size_t)W * H * 2), o_it = l->alloc(sizeof(SvtB200InvTxfmItem));
    size_t in_end = l->used;
    size_t o_out = l->alloc((size_t)W * H * 2);
    memcpy(l->h<int32_t>(o_in), input, (size_t)Wp * Hp * 4);
    for (int r = 0; r < H; r++) memcpy(l->h<uint16_t>(o_pred) + r * W, output_r + (size_t)r * stride_r, W * 2);
    SvtB200InvTxfmItem* it = l->h<SvtB200InvTxfmItem>(o_it);
    memset(it, 0, sizeof(*it));
    it->pred_stride = it->recon_stride = W;
    it->tx_size = (uint8_t)tx_size;
    it->tx_type = (uint8_t)tx_type;
    it->bd = (uint8_t)bd;
    l->h2d(0, in_end);
    launch_inv_txfm<uint16_t>(l->d<int32_t>(o_in), l->d<uint16_t>(o_pred), l->d<uint16_t>(o_out), l->d<SvtB200InvTxfmItem>(o_it), 1,
                              tx_class(tx_size), l->stream);
    l->d2h(o_out, (size_t)W * H * 2);
    l->sync();
    for (int r = 0; r < H; r++) memcpy(output_w + (size_t)r * stride_w, l->h<uint16_t>(o_out) + r * W, W * 2);
}

// T2 host variants: caller-owned host planes, one call per batch.
extern "C" int svt_b200_fwd_txfm_batch_host(const int16_t* residual, size_t residual_elems, int32_t* coeff, size_t coeff_elems,
                                            const SvtB200FwdTxfmItem* items, int n_items) {
    require_ready();
    if (n_items <= 0) return n_items == 0 ? SVT_B200_OK : SVT_B200_ERR_BAD_ARG;
    LaneGuard l;
    size_t o_src = l->alloc(residual_elems * 2), o_it = l->alloc(sizeof(SvtB200FwdTxfmItem) * n_items);
    size_t in_end = l->used;
    size_t o_dst = l->alloc(coeff_elems * 4);
    memcpy(l->h<int16_t>(o_src), residual, residual_elems * 2);
    SvtB200FwdTxfmItem* hi = l->h<SvtB200FwdTxfmItem>(o_it);
    int cnt[SVT_B200_TXFM_CLASSES] = {0, 0, 0, 0, 0}, pos[SVT_B200_TXFM_CLASSES];
    for (int i = 0; i < n_items; i++) {
        if (items[i].tx_size >= 19 || !host_txcfg(items[i].tx_size, items[i].tx_type).valid) return SVT_B200_ERR_BAD_ARG;
        cnt[tx_class(items[i].tx_size)]++;
    }
    for (int c = 0, first = 0; c < SVT_B200_TXFM_CLASSES; first += cnt[c], c++) pos[c] = first;
    for (int i = 0; i < n_items; i++) hi[pos[tx_class(items[i].tx_size)]++] = items[i];
    l->h2d(0, in_end);
    for (int c = 0, first = 0; c < SVT_B200_TXFM_CLASSES; first += cnt[c], c++)
        launch_fwd_txfm(l->d<int16_t>(o_src), l->d<int32_t>(o_dst), l->d<SvtB200FwdTxfmItem>(o_it) + first, cnt[c], c, l->stream);
    l->d2h(o_dst, coeff_elems * 4);
    l->sync();
    // only the regions the items cover were written; copy those back
    for (int i = 0; i < n_items; i++) {
        const int W = tx_w(items[i].tx_size), H = tx_h(items[i].tx_size);
        memcpy(coeff + items[i].dst_off, l->h<int32_t>(o_dst) + items[i].dst_off, (size_t)W * H * 4);
    }
    return SVT_B200_OK;
}

extern "C" void svt_b200_inv_txfm_add_8bit(const int32_t* dqcoeff, uint8_t* dst_r, int32_t stride_r, uint8_t* dst_w,
                                           int32_t stride_w, int tx_type, int tx_size) {
    require_ready();
    const int W = tx_w(tx_size), H = tx_h(tx_size);
    const int Wp = W > 32 ? 32 : W, Hp = H > 32 ? 32 : H;
    if (!host_txcfg(tx_size, tx_type).valid) {
        fprintf(stderr, "[svt_b200] FATAL: invalid (tx_size=%d, tx_type=%d)\n", tx_size, tx_type);
        abort();
    }
    LaneGuard l;
    size_t o_in = l->alloc((size_t)Wp * Hp * 4), o_pred = l->alloc((size_t)W * H), o_it = l->alloc(sizeof(SvtB200InvTxfmItem));
    size_t in_end = l->used;
    size_t o_out = l->alloc((size_t)W * H);
    memcpy(l->h<int32_t>(o_in), dqcoeff, (size_t)Wp * Hp * 4);
    for (int r = 0; r < H; r++) memcpy(l->h<uint8_t>(o_pred) + r * W, dst_r + (size_t)r * stride_r, W);
    SvtB200InvTxfmItem* it = l->h<SvtB200InvTxfmItem>(o_it);
    memset(it, 0, sizeof(*it));
    it->pred_stride = it->recon_stride = W;
    it->tx_size = (uint8_t)tx_size;
    it->tx_type = (uint8_t)tx_type;
    it->bd = 8;
    l->h2d(0, in_end);
    launch_inv_txfm<uint8_t>(l->d<int32_t>(o_in), l->d<uint8_t>(o_pred), l->d<uint8_t>(o_out), l->d<SvtB200InvTxfmItem>(o_it), 1,
                             tx_class(tx_size), l->stream);
    l->d2h(o_out, (size_t)W * H);
    l->sync();
    for (int r = 0; r < H; r++) memcpy(dst_w + (size_t)r * stride_w, l->h<uint8_t>(o_out) + r * W, W);
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
    LaneGuard l;
    const size_t n = (size_t)W * H;
    size_t o_buf = l->alloc(n * 4), o_e = l->alloc(16);
    memcpy(l->h<int32_t>(o_buf), output, n * 4);
    l->h2d(o_buf, n * 4);
    handle_transform_kernel<<<1, 256, 0, l->stream>>>(l->d<int32_t>(o_buf), W, H, with_energy, l->d<unsigned long long>(o_e));
    B200_LAUNCH_CHECK();
    l->d2h(o_buf, (o_e + 16) - o_buf);
    l->sync();
    memcpy(output, l->h<int32_t>(o_buf), n * 4);
    return (uint64_t)*l->h<unsigned long long>(o_e);
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
