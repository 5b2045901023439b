"""The transform chain's word moves: the fused and separate transform calls on planes and buffers whose rows can move
in 4-, 8- and 16-byte words, alone and side by side with blocks whose rows cannot, against the reference's C kernels.

txfm_kernel picks, per item, the word or the element form of each of its global moves from the item's own offsets and
strides (row_words in txfm.cu):
- source and prediction rows of the residual (min(W, 16 / pixel bytes) pixels a word);
- int16 residual rows (min(W, 8) samples);
- prediction loads and reconstruction stores (min(W, 16 / pixel bytes) pixels; also the eob == 0 copy);
- the quantiser's streams: levels and dequantised levels (int4), scan positions (4 x int16), matrix weights (u32);
- the forward batch's coefficient stores and the inverse batch's coefficient loads (int4).
`word_paths` restates that predicate, and the tests assert that every path takes the word form for every size and
pixel type and, in the mixed batches, the element form too.  The existing chain tests use odd strides, so they reach
only the element forms."""
import ctypes as ct

import numpy as np
import pytest

import chain_helpers as ch
from helpers import rng
from oracle_libs import refc  # noqa: F401  (a fixture: overrides conftest.py's refc in this module)
from quant_helpers import tables_for
from svt_av1_psy_b200.workload import av1_tables
from txfm_helpers import TX_H, TX_W

gpu = pytest.mark.gpu
PAD = 16


def layout_case(blocks, bd, r, misalign, width=1024):
    """ch.build_case's batch on planes with 16-element-aligned strides.  A block with misalign[i] (in block order) sits
    one column right of a 16-column boundary in the source / prediction / residual planes, three columns right in the
    reconstruction, and its coefficient run, and its random matrices, start on an odd element; the other blocks start on
    multiples of 16 everywhere."""
    c = ch.Case()
    n = len(blocks)
    c.bd, c.pixel_bytes = bd, 1 if bd == 8 else 2
    pix = np.uint8 if bd == 8 else np.uint16
    mx = (1 << bd) - 1
    W = np.array(TX_W)[blocks["sz"]].astype(np.int64)
    H = np.array(TX_H)[blocks["sz"]].astype(np.int64)
    x = np.zeros(n, np.int64)
    y = np.zeros(n, np.int64)
    cx = cy = shelf = 0
    for i in np.argsort(-H, kind="stable"):  # shelves of 16-column slots with a free slot between blocks
        slot = (W[i] + 16 + 15) // 16 * 16
        if cx + slot > width:
            cx, cy, shelf = 0, cy + shelf + 16, 0
        x[i], y[i] = cx + (1 if misalign[i] else 0), cy
        cx += slot
        shelf = max(shelf, H[i])
    rows = cy + shelf + 2 * PAD
    c.src_stride = c.pred_stride = width + 2 * PAD + 16
    c.recon_stride = width + 2 * PAD + 48
    c.src = r.integers(0, mx + 1, (rows, c.src_stride)).astype(pix)
    c.pred = r.integers(0, mx + 1, (rows, c.pred_stride)).astype(pix)
    for i in np.flatnonzero(blocks["kind"] != ch.KINDS.index("uniform")):
        ch._fill(c.src, c.pred, PAD + int(y[i]), PAD + int(x[i]), int(H[i]), int(W[i]), ch.KINDS[blocks["kind"][i]], mx, r)
    c.residual = (c.src.astype(np.int32) - c.pred).astype(np.int16)
    c.sentinel = 0xa5 if bd == 8 else 0xa5a5
    c.recon0 = np.full((rows, c.recon_stride), c.sentinel, pix)

    cls = np.array([ch.team_class(int(s)) for s in blocks["sz"]])
    order = np.lexsort((blocks["ty"], blocks["sz"], cls))
    b, x, y, W, H, mis = blocks[order], x[order], y[order], W[order], H[order], np.asarray(misalign)[order]
    c.blocks, c.cls, c.misalign = b, cls[order], mis
    c.n_per_class = [int((c.cls == k).sum()) for k in range(5)]
    ncoef = np.minimum(W, 32) * np.minimum(H, 32)
    coef = np.zeros(n, np.int64)
    pos = 0
    for i in range(n):  # runs on multiples of 16, a misaligned one 1 past; 16 untouched elements between runs
        coef[i] = pos + (1 if mis[i] else 0)
        pos = (coef[i] + ncoef[i] + 16 + 15) // 16 * 16
    c.n_coef = int(pos) + 16

    tb = av1_tables()
    nq = tb["qm"].shape[2]
    qm_parts = [tb["qm"].reshape(-1), tb["iqm"].reshape(-1)]
    iqm_base = tb["qm"].size
    qm_off = np.full(n, ch.dsp.NO_QM, np.int64)
    iqm_off = np.full(n, ch.dsp.NO_QM, np.int64)
    ref_m = b["qm"] == ch.QM_REF
    lvl, pt = r.integers(0, tb["qm"].shape[0], n), r.integers(0, 2, n)
    base = (lvl * 2 + pt) * nq + tb["qm_off"][b["sz"]]
    qm_off[ref_m], iqm_off[ref_m] = base[ref_m], iqm_base + base[ref_m]
    qpos = 2 * iqm_base
    for i in np.flatnonzero(b["qm"] == ch.QM_RAND):
        m = int(ncoef[i])
        lead = 1 if mis[i] else 0
        qm_parts.append(np.concatenate([np.full(lead, 77, np.uint8), r.integers(12, 256, 2 * m).astype(np.uint8)]))
        qm_off[i], iqm_off[i] = qpos + lead, qpos + lead + m
        qpos += lead + 2 * m
    c.qm = np.ascontiguousarray(np.concatenate(qm_parts), np.uint8)
    c.scan, c.iscan = np.ascontiguousarray(tb["scan"], np.int16), np.ascontiguousarray(tb["iscan"], np.int16)

    it = np.zeros(n, ch.dsp.TRIO_ITEM_DTYPE)
    f, q, v = it["fwd"], it["quant"], it["inv"]
    f["src_off"] = (PAD + y) * c.src_stride + PAD + x
    f["dst_off"] = coef
    f["src_stride"] = c.src_stride
    f["tx_size"], f["tx_type"] = b["sz"], b["ty"]
    f["reserved"] = 1
    q["coeff_off"] = q["q_off"] = q["dq_off"] = coef
    q["scan_off"] = tb["scan_off"][b["sz"], b["ty"]]
    q["qm_off"], q["iqm_off"] = qm_off, iqm_off
    q["n_coeffs"] = ncoef
    for (dc, ac) in set(zip(b["dc"].tolist(), b["ac"].tolist())):
        tq, tfp = tables_for(dc, ac)
        for is_fp, t in ((False, tq), (True, tfp)):
            m = (b["dc"] == dc) & (b["ac"] == ac) & (np.isin(b["mode"], (ch.dsp.QUANT_FP_LBD, ch.dsp.QUANT_FP_HBD)) == is_fp)
            for name in ("zbin", "round", "quant", "quant_shift", "dequant"):
                q[name][m] = t[name]
    q["mode"] = b["mode"]
    q["log_scale"] = [ch.log_scale(int(s)) for s in b["sz"]]
    v["coef_off"] = coef
    v["pred_off"] = (PAD + y) * c.pred_stride + PAD + x
    v["recon_off"] = (PAD + y) * c.recon_stride + PAD + x + np.where(mis, 2, 0)
    v["pred_stride"], v["recon_stride"] = c.pred_stride, c.recon_stride
    v["tx_size"], v["tx_type"], v["bd"] = b["sz"], b["ty"], bd
    c.items = it
    return c


def _words(off, stride, elem_bytes, v):
    """row_words<V>: the block's origin and its row stride are whole words of v elements (device buffers are allocated
    on 256-byte boundaries)"""
    wb = v * elem_bytes
    return ((np.asarray(off, np.int64) * elem_bytes) % wb == 0) & ((np.asarray(stride, np.int64) * elem_bytes) % wb == 0)


def word_paths(items, pixel_bytes, in_place=False):
    """per item, whether each word path of txfm_kernel takes its word form (the kernel's predicate, restated)"""
    f, q, v = items["fwd"], items["quant"], items["inv"]
    W = np.array(TX_W)[f["tx_size"]]
    vp = np.minimum(W, 16 // pixel_bytes)
    vr = np.minimum(W, 8)
    recon_off = v["pred_off"] if in_place else v["recon_off"]
    recon_stride = v["pred_stride"] if in_place else v["recon_stride"]
    has_qm = q["qm_off"] != ch.dsp.NO_QM
    has_iqm = q["iqm_off"] != ch.dsp.NO_QM
    pix_ok = lambda off, st: np.array([bool(_words(o, s, pixel_bytes, k)) for o, s, k in zip(off, st, vp)])  # noqa: E731
    return {
        "source": pix_ok(f["src_off"], f["src_stride"]) & pix_ok(v["pred_off"], v["pred_stride"]),
        "residual": np.array([bool(_words(o, s, 2, k)) for o, s, k in zip(f["src_off"], f["src_stride"], vr)]),
        "recon": pix_ok(v["pred_off"], v["pred_stride"]) & pix_ok(recon_off, recon_stride),
        "quant": (_words(q["q_off"], 0, 4, 4) & _words(q["dq_off"], 0, 4, 4) & _words(q["scan_off"], 0, 2, 4)
                  & (~has_qm | _words(np.where(has_qm, q["qm_off"], 0), 0, 1, 4))
                  & (~has_iqm | _words(np.where(has_iqm, q["iqm_off"], 0), 0, 1, 4))),
        "fwd_out": _words(f["dst_off"], 0, 4, 4),
        "inv_in": _words(v["coef_off"], 0, 4, 4),
    }


def _assert_reached(case, mixed):
    paths = word_paths(case.items, case.pixel_bytes)
    sizes = case.blocks["sz"]
    for name, on in paths.items():
        for sz in range(19):
            m = sizes == sz
            assert on[m].any(), "%s: the word form is not reached at size %d" % (name, sz)
            if mixed:
                assert (~on[m]).any(), "%s: the element form is not reached at size %d" % (name, sz)


@pytest.fixture(scope="module")
def ref(refc):
    refc.ref_set_tier(0)
    refc.ref_set_threads(0)
    return refc


@pytest.fixture(scope="module")
def cases(ref):
    """(bit depth, mixed) -> (case, reference results): the coverage matrix of ch.matrix_blocks, every block aligned, or
    every other block of each (size, type) misaligned"""
    out = {}
    for bd in (8, 10, 12):
        blocks = ch.matrix_blocks(bd)
        for mixed in (False, True):
            mis = (np.arange(len(blocks)) % 2 == 1) if mixed else np.zeros(len(blocks), bool)
            case = layout_case(blocks, bd, rng(470 + bd + 10 * mixed), mis)
            out[bd, mixed] = (case, ch.reference_chain(ref, case))
    return out


@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("mixed", [False, True])
def test_cases_reach_every_word_path(bd, mixed):
    """CPU: the layouts put every size of every pixel type on every word path (and, mixed, on every element path too)"""
    blocks = ch.matrix_blocks(bd)
    mis = (np.arange(len(blocks)) % 2 == 1) if mixed else np.zeros(len(blocks), bool)
    case = layout_case(blocks, bd, rng(470 + bd + 10 * mixed), mis)
    _assert_reached(case, mixed)
    paths = word_paths(case.items, case.pixel_bytes, in_place=True)
    for sz in range(19):
        assert paths["recon"][case.blocks["sz"] == sz].any()
    if not mixed:
        assert all(v.all() for v in paths.values())


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("mixed", [False, True])
def test_fused_chain_on_word_layouts(b200, cases, bd, mixed):
    """both fused forms, with and without the dequantised output, out of place and in place, workload and shuffled orders"""
    import torch
    from test_txfm_chain import _check_coeffs, _check_eobs, _check_recon, _check_trio, _in_place_want, _run_trio
    case, want = cases[bd, mixed]
    shuffled = ch.shuffled_order(case, rng(480 + bd))
    for entry in ("residual", "residual_plane"):
        _check_trio(case, _run_trio(b200, torch, case, entry), want)
        _check_trio(case, _run_trio(b200, torch, case, entry, shuffled, with_dq=False), want)
        got = _run_trio(b200, torch, case, entry, shuffled, in_place=True)
        _check_eobs(case, got["eobs"], want["eobs"])
        _check_coeffs(case, got["q"], want["q"], "qcoeff")
        _check_coeffs(case, got["dq"], want["dq"], "dqcoeff")
        _check_recon(case, got["recon"], _in_place_want(case, want), "pred_off", case.pred_stride)


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("mixed", [False, True])
def test_separate_calls_on_word_layouts(b200, cases, bd, mixed):
    """the residual, forward, quantise and inverse calls on the same layouts"""
    import torch
    from test_txfm_chain import _check_three_calls, _three_calls
    case, want = cases[bd, mixed]
    _check_three_calls(case, _three_calls(b200, torch, case, True), want)


def test_word_paths_predicate():
    """the restated predicate on hand-made items: origin and stride must both be whole words"""
    it = np.zeros(4, ch.dsp.TRIO_ITEM_DTYPE)
    it["fwd"]["tx_size"] = [0, 2, 4, 2]  # 4x4, 16x16, 64x64, 16x16
    it["fwd"]["src_off"] = [4, 16, 32, 17]
    it["fwd"]["src_stride"] = [1040, 1040, 1040, 1040]
    it["inv"]["pred_off"] = it["fwd"]["src_off"]
    it["inv"]["pred_stride"] = 1040
    it["inv"]["recon_off"] = [0, 8, 16, 16]
    it["inv"]["recon_stride"] = [1072, 1072, 1072, 1076]
    it["quant"]["qm_off"] = it["quant"]["iqm_off"] = ch.dsp.NO_QM
    p8 = word_paths(it, 1)
    assert p8["source"].tolist() == [True, True, True, False]
    assert p8["recon"].tolist() == [True, False, True, False]
    assert p8["residual"].tolist() == [True, True, True, False]
    p16 = word_paths(it, 2)
    assert p16["recon"].tolist() == [True, True, True, False]
