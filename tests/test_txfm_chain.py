"""The transform chain of the encode pass, block by block against the reference's C kernels (ref_set_tier(0)),
bit for bit, at every tx size x valid type, 8 / 10 / 12 bit, every quantiser mode with and without matrices:

- the fused batch calls svt_b200_residual_txfm_trio_batch_dev / svt_b200_txfm_trio_batch_dev (with and without the
  dequantised output, in place, in the workload's order and with unlike neighbouring teams, and with enough blocks
  that every class's grid-stride loop runs at least twice);
- the separate calls svt_b200_residual_planes_dev + svt_b200_fwd_txfm_batch_dev + svt_b200_quant_batch_dev (raster
  and scan-order walks) + svt_b200_inv_txfm_batch_dev;
- the forward batch's packed / N2 / N4 bits, and svt_b200_pack_levels_dev (offsets, runs, capacity, int16 overflow
  count, argument limits).

The inputs come from chain_helpers; test_generator_reaches_the_edges checks on the CPU that they reach the
saturation, clamp and overflow paths they are built for."""
import ctypes as ct

import numpy as np
import pytest

import chain_helpers as ch
from helpers import rng
from oracle_libs import refc  # noqa: F401  (a fixture: overrides conftest.py's refc in this module)
from txfm_helpers import TX_H, TX_W, ref_fwd_partial

BAD_ARG = -4  # SVT_B200_ERR_BAD_ARG
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(refc):
    """the reference's C kernels with every host CPU on the batches"""
    refc.ref_set_tier(0)
    refc.ref_set_threads(0)
    return refc


@pytest.fixture(scope="module")
def matrix(ref):
    """bit depth -> (case, reference results) of the coverage matrix"""
    out = {}
    for bd in (8, 10, 12):
        case = ch.build_case(ch.matrix_blocks(bd), bd, rng(400 + bd))
        out[bd] = (case, ch.reference_chain(ref, case))
    return out


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _host(t, dtype):
    return t.cpu().numpy().view(dtype)


def _describe(case, i):
    b = case.blocks[i]
    return "block %d: %dx%d type %d mode %d qm %d step (%d, %d) %s" % (
        i, TX_W[b["sz"]], TX_H[b["sz"]], b["ty"], b["mode"], b["qm"], b["dc"], b["ac"], ch.KINDS[b["kind"]])


def _check_coeffs(case, got, want, what):
    if np.array_equal(got, want):
        return
    k = int(np.flatnonzero(got != want)[0])
    i = int(np.searchsorted(case.items["quant"]["q_off"].astype(np.int64), k, side="right")) - 1
    pytest.fail("%s differs at %d (got %d, want %d), %s" % (what, k, got[k], want[k], _describe(case, i)))


def _check_eobs(case, got, want):
    if not np.array_equal(got, want):
        i = int(np.flatnonzero(got != want)[0])
        pytest.fail("eob %d != %d, %s" % (got[i], want[i], _describe(case, i)))


def _check_recon(case, got, want, off_field="recon_off", stride=None):
    if np.array_equal(got, want):
        return
    stride = stride or case.recon_stride
    rr, cc = np.argwhere(got != want)[0]
    off = case.items["inv"][off_field].astype(np.int64)
    by, bx = off // stride, off % stride
    inside = (by <= rr) & (rr < by + np.array(TX_H)[case.blocks["sz"]]) & (bx <= cc) & (cc < bx + np.array(TX_W)[case.blocks["sz"]])
    where = _describe(case, int(np.flatnonzero(inside)[0])) if inside.any() else "outside every block"
    pytest.fail("recon differs at (%d, %d) in %d pixels (got %d, want %d), %s" % (rr, cc, int((got != want).sum()), got[rr, cc], want[rr, cc], where))


def _run_trio(b200, torch, case, entry, order=None, with_dq=True, in_place=False):
    """one fused call; returns q, dq, eobs (in block order) and the written plane"""
    order = np.arange(len(case.items)) if order is None else order
    items = case.items[order].copy()
    if in_place:
        items["inv"]["recon_off"], items["inv"]["recon_stride"] = items["inv"]["pred_off"], items["inv"]["pred_stride"]
    d_pred = _dev(torch, case.pred)
    d_recon = d_pred if in_place else _dev(torch, case.recon0)
    d_q = torch.full((case.n_coef,), ch.SENT32, dtype=torch.int32, device="cuda")
    d_dq = torch.full((case.n_coef,), ch.SENT32, dtype=torch.int32, device="cuda") if with_dq else None
    d_eobs = torch.full((len(items),), -1, dtype=torch.int16, device="cuda")
    d_iscan, d_qm, d_items = _dev(torch, case.iscan), _dev(torch, case.qm), _dev(torch, items)
    npc = (ct.c_int * 5)(*[int((case.cls[order] == k).sum()) for k in range(5)])
    s = torch.cuda.current_stream().cuda_stream
    if entry == "residual":
        d_in = _dev(torch, case.src)
        fn = b200.lib.svt_b200_residual_txfm_trio_batch_dev
    else:
        d_in = _dev(torch, case.residual)
        fn = b200.lib.svt_b200_txfm_trio_batch_dev
    rc = fn(d_in.data_ptr(), d_pred.data_ptr(), d_recon.data_ptr(), d_q.data_ptr(), d_dq.data_ptr() if with_dq else None, d_iscan.data_ptr(),
            d_qm.data_ptr(), d_items.data_ptr(), npc, d_eobs.data_ptr(), case.pixel_bytes, s)
    assert rc == 0
    torch.cuda.synchronize()
    eobs = np.empty(len(items), np.uint16)
    eobs[order] = _host(d_eobs, np.uint16)
    pix = case.pred.dtype
    plane = _host(d_recon, pix).reshape(case.pred.shape if in_place else case.recon0.shape)
    return {"q": _host(d_q, np.int32), "dq": _host(d_dq, np.int32) if with_dq else None, "eobs": eobs, "recon": plane}


def _check_trio(case, got, want):
    _check_eobs(case, got["eobs"], want["eobs"])
    _check_coeffs(case, got["q"], want["q"], "qcoeff")
    if got["dq"] is not None:
        _check_coeffs(case, got["dq"], want["dq"], "dqcoeff")
    _check_recon(case, got["recon"], want["recon"])


def _in_place_want(case, want):
    """what an in-place call leaves in the prediction plane: the prediction, with every block replaced by its reconstruction"""
    plane = case.pred.copy().reshape(-1)
    inv = case.items["inv"]
    ch.paste_blocks(plane, inv["pred_off"], case.pred_stride, want["recon"].reshape(-1), inv["recon_off"], case.recon_stride, case.blocks["sz"])
    return plane.reshape(case.pred.shape)


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_fused_chain_matches_reference(b200, matrix, bd):
    import torch
    case, want = matrix[bd]
    shuffled = ch.shuffled_order(case, rng(410 + bd))
    assert np.any(case.blocks["sz"][shuffled][1:] != case.blocks["sz"][shuffled][:-1])
    for entry in ("residual", "residual_plane"):
        for order in (None, shuffled):
            _check_trio(case, _run_trio(b200, torch, case, entry, order), want)
        got = _run_trio(b200, torch, case, entry, shuffled, with_dq=False)  # d_dqcoeff = NULL: the rest is unchanged
        _check_trio(case, got, want)
        got = _run_trio(b200, torch, case, entry, in_place=True)  # d_recon == d_pred
        _check_eobs(case, got["eobs"], want["eobs"])
        _check_coeffs(case, got["q"], want["q"], "qcoeff")
        _check_coeffs(case, got["dq"], want["dq"], "dqcoeff")
        _check_recon(case, got["recon"], _in_place_want(case, want), "pred_off", case.pred_stride)


def _three_calls(b200, torch, case, use_iscan):
    """svt_b200_residual_planes_dev -> svt_b200_fwd_txfm_batch_dev -> svt_b200_quant_batch_dev -> svt_b200_inv_txfm_batch_dev"""
    n = len(case.items)
    s = torch.cuda.current_stream().cuda_stream
    d_src, d_pred, d_recon = _dev(torch, case.src), _dev(torch, case.pred), _dev(torch, case.recon0)
    d_res = torch.full((case.residual.size,), 0x5a5a, dtype=torch.int16, device="cuda")
    planes = b200.ResidualPlanes()
    rows = case.src.shape[0]
    planes.p[0] = b200.ResidualPlane(0, 0, 0, case.src_stride, case.pred_stride, case.src_stride, case.src_stride, rows, 0)
    assert b200.lib.svt_b200_residual_planes_dev(d_src.data_ptr(), d_pred.data_ptr(), d_res.data_ptr(), ct.byref(planes), 1, case.pixel_bytes, s) == 0
    npc = (ct.c_int * 5)(*case.n_per_class)
    d_coeff = torch.full((case.n_coef,), ch.SENT32, dtype=torch.int32, device="cuda")
    d_fwd = _dev(torch, case.items["fwd"])
    assert b200.lib.svt_b200_fwd_txfm_batch_dev(d_res.data_ptr(), d_coeff.data_ptr(), d_fwd.data_ptr(), npc, s) == 0
    d_q = torch.full((case.n_coef,), ch.SENT32, dtype=torch.int32, device="cuda")
    d_dq = torch.full((case.n_coef,), ch.SENT32, dtype=torch.int32, device="cuda")
    d_eobs = torch.full((n,), -1, dtype=torch.int16, device="cuda")
    d_scan, d_iscan, d_qm, d_quant = _dev(torch, case.scan), _dev(torch, case.iscan), _dev(torch, case.qm), _dev(torch, case.items["quant"])
    assert b200.lib.svt_b200_quant_batch_dev(d_coeff.data_ptr(), d_q.data_ptr(), d_dq.data_ptr(), d_scan.data_ptr(), d_iscan.data_ptr() if use_iscan else None,
                                             d_qm.data_ptr(), d_quant.data_ptr(), n, d_eobs.data_ptr(), s) == 0
    d_inv = _dev(torch, case.items["inv"])
    assert b200.lib.svt_b200_inv_txfm_batch_dev(d_dq.data_ptr(), d_pred.data_ptr(), d_recon.data_ptr(), d_inv.data_ptr(), npc, case.pixel_bytes, s) == 0
    torch.cuda.synchronize()
    return {"residual": _host(d_res, np.int16).reshape(case.residual.shape), "coeff": _host(d_coeff, np.int32), "q": _host(d_q, np.int32),
            "dq": _host(d_dq, np.int32), "eobs": _host(d_eobs, np.uint16), "recon": _host(d_recon, case.pred.dtype).reshape(case.recon0.shape)}


def _check_three_calls(case, got, want):
    assert np.array_equal(got["residual"], case.residual)
    _check_coeffs(case, got["coeff"], want["coeff"], "forward coefficients")
    _check_trio(case, got, want)


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_three_call_chain_matches_reference(b200, matrix, bd):
    """the separate calls equal the reference (and so the fused call), quantiser walking raster order (d_iscan) or scan order"""
    import torch
    case, want = matrix[bd]
    for use_iscan in (True, False):
        _check_three_calls(case, _three_calls(b200, torch, case, use_iscan), want)


def trio_grid_capacity(team):
    """(CTAs per SM, teams per CTA) of one team class's launch, as launch (txfm.cu) derives them for all three modes of
    txfm_kernel (the fused call and the separate forward and inverse calls): THREADS = class_threads (256, 256, 128 for
    the 4- .. 16-point classes, 2 * TEAM = 64 and 128 for the 32- and 64-point classes); one team per CTA for the 32- and
    64-point classes, THREADS / TEAM otherwise; dynamic shared memory = teams * team_stride(TEAM) * 4 bytes; CTAs per SM
    = min(200 KB / (shared memory + 1 KB), 2048 / THREADS), and the grid is min(CTAs needed, sm_count * CTAs per SM)
    (grid_for).  A class with more blocks than sm_count * CTAs per SM * teams per CTA walks its grid-stride loop more
    than once."""
    threads = 2 * team if team >= 32 else {4: 256, 8: 256, 16: 128}[team]
    teams = 1 if team >= 32 else threads // team
    stride = {4: 68, 8: 152, 16: 560}.get(team, 2 * team * (team + 1))
    smem = teams * stride * 4
    return min(200 * 1024 // (smem + 1024), 2048 // threads), teams


@gpu
def test_grid_stride_loops_run_twice(b200, ref):
    """per class 2 x sm_count x CTAs per SM x teams per CTA blocks (+ a partial third pass): (8, 64), (8, 32), (10, 8),
    (21, 1), (5, 1) CTAs per SM x teams per CTA for the 4- .. 64-point classes, so every CTA of every class loops at least
    twice.  Fused and separate calls: they launch the same geometry."""
    import torch
    sms = int(b200.lib.svt_b200_sm_count())
    assert sms > 0
    counts = []
    for team in (4, 8, 16, 32, 64):
        per_sm, teams = trio_grid_capacity(team)
        counts.append(2 * sms * per_sm * teams + 37)
    assert [trio_grid_capacity(t) for t in (4, 8, 16, 32, 64)] == [(8, 64), (8, 32), (10, 8), (21, 1), (5, 1)]
    r = rng(420)
    case = ch.build_case(ch.random_blocks(8, counts, r), 8, r, width=2048)
    assert case.n_per_class == counts
    want = ch.reference_chain(ref, case)
    _check_trio(case, _run_trio(b200, torch, case, "residual"), want)
    _check_three_calls(case, _three_calls(b200, torch, case, True), want)


@gpu
@pytest.mark.parametrize("bd", [8, 12])
def test_fwd_batch_packed_n2_n4_bits(b200, ref, bd):
    """svt_b200_fwd_txfm_batch_dev with reserved = 0, packed, N2, N4, N2 | packed, N4 | packed, every size x valid type,
    against ref_fwd_txfm_batch_bd (full) and the reference's N2 / N4 kernels (ref_fwd_partial)"""
    import torch
    r = rng(430 + bd)
    blocks = []
    for sz in range(19):
        for ty in ch.valid_types(sz):
            blocks += [(sz, ty, 0, 0, 4, 4, ch.KINDS.index(k)) for k in ("uniform", "checker")]
    case = ch.build_case(np.array(blocks, ch.BLOCK_DTYPE), bd, r)
    res = case.residual.reshape(-1)
    fwd = np.ascontiguousarray(case.items["fwd"])
    W, H = np.array(TX_W)[fwd["tx_size"]], np.array(TX_H)[fwd["tx_size"]]
    s = torch.cuda.current_stream().cuda_stream
    d_res, npc = _dev(torch, case.residual), (ct.c_int * 5)(*case.n_per_class)
    for reserved in (0, 1, 2, 4, 3, 5):
        packed, level = reserved & 1, reserved >> 1
        n = np.where(packed, np.minimum(W, 32) * np.minimum(H, 32), W * H) + 2  # two sentinel words after each block
        items = fwd.copy()
        items["reserved"] = reserved
        items["dst_off"] = np.concatenate(([0], np.cumsum(n)[:-1]))
        want = np.full(int(n.sum()), ch.SENT32, np.int32)
        if level == 0:
            ref.ref_fwd_txfm_batch_bd(ch.ptr(case.residual), ch.ptr(want), ch.ptr(items), ct.c_int(len(items)), ct.c_int(bd))
        else:
            for it in items:
                sz, o = int(it["tx_size"]), int(it["dst_off"])
                c = ref_fwd_partial(ref, res[int(it["src_off"]):], int(it["src_stride"]), int(it["tx_type"]), sz, level, bd)
                c = c.reshape(TX_H[sz], TX_W[sz])[:min(TX_H[sz], 32), :min(TX_W[sz], 32)] if packed else c
                want[o:o + c.size] = c.reshape(-1)
        d_out = torch.full((want.size,), ch.SENT32, dtype=torch.int32, device="cuda")
        d_items = _dev(torch, items)
        assert b200.lib.svt_b200_fwd_txfm_batch_dev(d_res.data_ptr(), d_out.data_ptr(), d_items.data_ptr(), npc, s) == 0
        torch.cuda.synchronize()
        got = _host(d_out, np.int32)
        if not np.array_equal(got, want):
            k = int(np.flatnonzero(got != want)[0])
            i = int(np.searchsorted(items["dst_off"].astype(np.int64), k, side="right")) - 1
            pytest.fail("reserved %d: %s" % (reserved, _describe(case, i)))


# ---- svt_b200_pack_levels_dev ---------------------------------------------------------------------------------------
def _pack_case(r, n, lo, hi):
    """n blocks of random sizes / types with levels in [lo, hi] (a third of them near zero) and random eobs, a fifth 0"""
    tb = ch.av1_tables()
    sz = r.integers(0, 19, n)
    ty = np.array([r.choice(ch.valid_types(int(s))) for s in sz])
    ncoef = np.minimum(np.array(TX_W)[sz], 32) * np.minimum(np.array(TX_H)[sz], 32)
    items = np.zeros(n, ch.dsp.TRIO_ITEM_DTYPE)
    q_off = np.concatenate(([0], np.cumsum(ncoef)[:-1]))
    items["quant"]["q_off"], items["quant"]["n_coeffs"] = q_off, ncoef
    items["quant"]["scan_off"] = tb["scan_off"][sz, ty]
    q = r.integers(lo, hi + 1, int(ncoef.sum())).astype(np.int32)
    q[r.random(q.size) < 0.3] //= 4096
    eobs = r.integers(0, ncoef + 1).astype(np.uint16)
    eobs[r.random(n) < 0.2] = 0
    return items, q, eobs


def _pack_want(items, q, eobs):
    scan = ch.av1_tables()["scan"]
    qi = items["quant"]
    runs = [q[int(qi["q_off"][i]) + scan[int(qi["scan_off"][i]):int(qi["scan_off"][i]) + int(eobs[i])].astype(np.int64)]
            for i in range(len(items))]
    return np.concatenate(runs + [np.zeros(0, np.int32)]).astype(np.int32)


def _pack(b200, torch, items, q, eobs, level_bytes, capacity, alloc, n=None):
    n = len(items) if n is None else n
    lvl = np.int16 if level_bytes == 2 else np.int32
    d_q, d_isc, d_items, d_eobs = _dev(torch, q), _dev(torch, ch.av1_tables()["iscan"].astype(np.int16)), _dev(torch, items), _dev(torch, eobs)
    d_off = torch.full((len(items) + 2,), ch.SENT32, dtype=torch.int32, device="cuda")
    d_lv = torch.full((alloc,), 0x5a5a if level_bytes == 2 else ch.SENT32, dtype=torch.int16 if level_bytes == 2 else torch.int32, device="cuda")
    rc = b200.lib.svt_b200_pack_levels_dev(d_q.data_ptr(), d_isc.data_ptr(), d_items.data_ptr(), d_eobs.data_ptr(), n, d_off.data_ptr(),
                                           d_lv.data_ptr(), level_bytes, capacity, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, _host(d_off, np.uint32), _host(d_lv, lvl)


@gpu
@pytest.mark.parametrize("n", [1, 256, 257, 16 * 256 + 37])
def test_pack_levels_offsets_and_runs(b200, n):
    """offsets = exclusive prefix sum of the eobs (total at [n], 0 overflows at [n + 1]); block i's run = q[scan[:eob]];
    nothing written past the total; 4-byte levels beyond int16 and 2-byte levels that fit"""
    import torch
    r = rng(440 + n)
    for level_bytes, (lo, hi) in ((4, (-600000, 600000)), (2, (-32768, 32767))):
        items, q, eobs = _pack_case(r, n, lo, hi)
        want = _pack_want(items, q, eobs)
        total = want.size
        rc, offs, lv = _pack(b200, torch, items, q, eobs, level_bytes, total, total + 64)
        assert rc == 0
        excl = np.concatenate(([0], np.cumsum(eobs.astype(np.int64))[:-1]))
        assert np.array_equal(offs[:n], excl) and offs[n] == total and offs[n + 1] == 0
        assert np.array_equal(lv[:total], want), level_bytes
        assert np.all(lv[total:] == (0x5a5a if level_bytes == 2 else 0x5a5a5a5a))


@gpu
def test_pack_levels_capacity_and_int16_overflow(b200):
    """capacity below the total: offsets[n] is still the total and nothing lands at or past capacity; 2-byte levels of
    10 / 12-bit blocks: offsets[n + 1] counts the written levels outside int16 (both signs), the rest are exact"""
    import torch
    r = rng(450)
    n = 3 * 256 + 5
    for level_bytes, (lo, hi) in ((4, (-600000, 600000)), (2, (-32768, 32767)), (2, (-300000, 300000))):
        items, q, eobs = _pack_case(r, n, lo, hi)
        want = _pack_want(items, q, eobs)
        for capacity in (want.size, want.size // 2 + 3, 0):
            rc, offs, lv = _pack(b200, torch, items, q, eobs, level_bytes, capacity, want.size + 64)
            assert rc == 0 and offs[n] == want.size
            kept = want[:capacity]
            outside = (kept < -32768) | (kept > 32767)
            if level_bytes == 2:
                assert offs[n + 1] == int(outside.sum()), capacity
                assert np.array_equal(lv[:capacity], kept.astype(np.int16)), capacity
                assert np.all(lv[capacity:] == 0x5a5a), capacity
            else:
                assert offs[n + 1] == 0 and np.array_equal(lv[:capacity], kept) and np.all(lv[capacity:] == 0x5a5a5a5a)
        if hi > 32767:
            assert (want < -32768).any() and (want > 32767).any()


@gpu
def test_pack_levels_chunk_limit(b200):
    """4096 chunks of 256 blocks are accepted and packed; one block more is SVT_B200_ERR_BAD_ARG with nothing written
    (the buffers hold all the blocks, so a broken check could not read outside them)"""
    import torch
    n = 4096 * 256
    r = rng(460)
    items = np.zeros(n + 1, ch.dsp.TRIO_ITEM_DTYPE)  # every block: the same 4x4 DCT_DCT coefficients at offset 0
    items["quant"]["n_coeffs"] = 16
    q = r.integers(-50, 51, 16).astype(np.int32)
    eobs = r.integers(0, 17, n + 1).astype(np.uint16)
    rc, offs, lv = _pack(b200, torch, items, q, eobs, 4, 1 << 24, 1 << 24, n=n + 1)
    assert rc == BAD_ARG
    assert np.all(offs == ch.SENT32) and np.all(lv == 0x5a5a5a5a)
    rc, offs, lv = _pack(b200, torch, items, q, eobs, 4, 1 << 24, 1 << 24, n=n)
    assert rc == 0
    e = eobs[:n].astype(np.int64)
    excl = np.concatenate(([0], np.cumsum(e)[:-1]))
    assert np.array_equal(offs[:n], excl) and offs[n] == e.sum() and offs[n + 1] == 0
    k = np.arange(int(e.sum())) - np.repeat(excl, e)
    scan = ch.av1_tables()["scan"][:16].astype(np.int64)
    assert np.array_equal(lv[:int(e.sum())], q[scan[k]])


# ---- the generator reaches what it is built for (CPU) -----------------------------------------------------------------
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_generator_reaches_the_edges(refc, bd):
    """On the reference's own results for the coverage matrix: every (size, type, mode, QM on / off) has blocks with
    eob > 0 and every class blocks with eob = 0; the LBD quantisers' int16 saturation is hit (modes 0 and 2, past the
    dead zone); some dequantised value exceeds the inverse's bd + 8 row clamp; 10 / 12-bit levels leave int16."""
    refc.ref_set_tier(0)
    refc.ref_set_threads(0)
    case = ch.build_case(ch.matrix_blocks(bd), bd, rng(400 + bd))
    out = ch.reference_chain(refc, case)
    b, qi, eobs = case.blocks, case.items["quant"], out["eobs"]
    combos = {(int(x["sz"]), int(x["ty"]), int(x["mode"]), bool(x["qm"])) for x in b}
    live = {(int(x["sz"]), int(x["ty"]), int(x["mode"]), bool(x["qm"])) for x, e in zip(b, eobs) if e > 0}
    assert combos - live == set()
    assert len(combos) == sum(len(ch.valid_types(sz)) for sz in range(19)) * len(ch.MODES[bd]) * 2
    assert set(case.cls[eobs == 0].tolist()) == set(range(5))
    assert np.all(case.items["fwd"]["src_off"] > 0) and case.n_per_class == [int((case.cls == k).sum()) for k in range(5)]

    # per coefficient: its block, its position, the reference's forward output, level and dequantised value
    nc = qi["n_coeffs"].astype(np.int64)
    blk = np.repeat(np.arange(len(b)), nc)
    rc = np.arange(int(nc.sum())) - np.repeat(np.cumsum(nc) - nc, nc)
    idx = qi["q_off"].astype(np.int64)[blk] + rc
    coeff, q, dq = (out[k][idx].astype(np.int64) for k in ("coeff", "q", "dq"))
    ac = (rc != 0).astype(np.int64)
    ls = qi["log_scale"].astype(np.int64)[blk]
    rnd = qi["round"].astype(np.int64)[blk, ac]
    rnd = np.where(ls > 0, (rnd + (1 << np.maximum(ls - 1, 0))) >> ls, rnd)
    absc = np.abs(coeff)
    wt = np.where(b["qm"][blk] != ch.QM_NONE, case.qm[np.where(b["qm"][blk] != ch.QM_NONE, qi["qm_off"].astype(np.int64)[blk] + rc, 0)], 32)
    mode = qi["mode"][blk]
    zbin = qi["zbin"].astype(np.int64)[blk, ac]
    zbin = np.where(ls > 0, (zbin + (1 << np.maximum(ls - 1, 0))) >> ls, zbin)
    deq = qi["dequant"].astype(np.int64)[blk, ac]
    past_b = absc * wt >= zbin << 5  # quantize_b dead zone (full_loop.c svt_aom_quantize_b_c_ii)
    past_fp = np.where(b["qm"][blk] != ch.QM_NONE, absc * wt >= deq << (5 - (1 + ls)), absc << (1 + ls) >= deq)
    sat = absc + rnd > 32767
    if bd == 8:
        assert np.any(sat & past_b & (mode == ch.dsp.QUANT_B_LBD)), "quantize_b int16 saturation not reached"
        assert np.any(sat & past_fp & (mode == ch.dsp.QUANT_FP_LBD)), "quantize_fp int16 saturation not reached"
    W, H = np.array(TX_W)[b["sz"]][blk], np.array(TX_H)[b["sz"]][blk]
    rect2 = (W == 2 * H) | (H == 2 * W)
    dq_in = np.where(rect2, (dq * 2896 + 2048) >> 12, dq)  # the inverse's input after the 2:1 rescale (kNewInvSqrt2)
    assert np.any(dq_in > (1 << (bd + 7)) - 1) and np.any(dq_in < -(1 << (bd + 7))), "bd + 8 row clamp not reached"
    assert np.any(rect2 & (np.abs(dq_in) > (1 << (bd + 7))))
    if bd > 8:
        assert np.any(q > 32767) and np.any(q < -32768), "levels outside int16 not reached"
