"""The transform constants that txfm.cu compiles into each size body, against the table dumped from the reference.

The forward column / row cosine bits and stage shifts and the inverse stage shifts depend on the transform size alone;
txfm.cu holds them as the constexpr table kTxSizeCfg (and the inverse cosine bit as kInvCosBit), and the generated
networks take their cosine bit as a template parameter.  On the CPU: the table read back from the source equals the
TXC rows of txfm_cfg.inc at every valid (size, type), and no generated network reads its weights at run time.  On the
GPU: every size x valid type through the fused chain at 8, 10 and 12 bit, full-scale residuals and the finest
quantiser steps (so the forward outputs and the inverse's clamps reach their extremes), bit for bit against the
reference's C kernels."""
import ctypes as ct
import os
import re

import numpy as np
import pytest

import chain_helpers as ch
from helpers import rng
from oracle_libs import refc  # noqa: F401  (a fixture: overrides conftest.py's refc in this module)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "svt-av1-psy_b200", "csrc")
FIELDS = ("f_cbc", "f_cbr", "f_s0", "f_s1", "f_s2", "i_s0", "i_s1")
TXC_FIELDS = ("size", "type", "valid", "f_ud", "f_lr", "f_s0", "f_s1", "f_s2", "f_cbc", "f_cbr", "f_tc", "f_tr",
              "i_ud", "i_lr", "i_s0", "i_s1", "i_cbc", "i_cbr", "i_tc", "i_tr")
EXTREME = ("flat_pos", "flat_neg", "checker", "impulse")
gpu = pytest.mark.gpu


def _src(name):
    return open(os.path.join(CSRC, name)).read()


def size_table():
    """kTxSizeCfg and kInvCosBit as txfm.cu defines them"""
    text = _src("txfm.cu")
    m = re.search(r"struct TxSizeCfg \{\s*int8_t ([^;]*);", text)
    assert m, "struct TxSizeCfg"
    assert tuple(f.strip() for f in m.group(1).split(",")) == FIELDS
    m = re.search(r"constexpr TxSizeCfg kTxSizeCfg\[19\] = \{(.*?)\n\};", text, re.S)
    assert m, "kTxSizeCfg"
    rows = [tuple(int(v) for v in r.split(",")) for r in re.findall(r"\{([-\d,\s]+)\}", m.group(1))]
    inv_bit = int(re.search(r"constexpr int\s+kInvCosBit = (\d+);", text).group(1))
    return rows, inv_bit


def dumped_rows():
    rows = []
    for m in re.finditer(r"^TXC\(([^)]*)\)", _src("txfm_cfg.inc"), re.M):
        rows.append(dict(zip(TXC_FIELDS, (int(v) for v in m.group(1).split(",")))))
    return rows


def test_size_constants_match_the_dumped_table():
    table, inv_bit = size_table()
    assert len(table) == 19 and all(len(r) == len(FIELDS) for r in table)
    rows = dumped_rows()
    assert len(rows) == 19 * 16
    checked = 0
    for row in rows:
        if not row["valid"]:
            continue
        want = dict(zip(FIELDS, table[row["size"]]))
        for f in FIELDS:
            assert row[f] == want[f], (row["size"], row["type"], f)
        assert row["i_cbc"] == inv_bit and row["i_cbr"] == inv_bit, (row["size"], row["type"])
        checked += 1
    assert checked == sum(len(ch.valid_types(sz)) for sz in range(19))


def test_networks_take_the_cosine_bit_at_compile_time():
    """every generated network and split function is a template on cos_bit whose weights come from TxCosv<cos_bit>"""
    text = _src("txfm_gen.inc")
    heads = re.findall(r"^(.*)\n__device__ __forceinline__ void txg_(\w+)\(int32_t \(&x\)\[\d+\]([^{]*)\{", text, re.M)
    assert len(heads) >= 14 + 2 + 12
    for tmpl, name, params in heads:
        assert tmpl == "template <int cos_bit>", name
        assert params.strip() == ", TxCosv<cos_bit> cosv, const int clampb)", name
    assert "c_cospi" not in text and "const int32_t*" not in text


def _run_fused(b200, torch, case):
    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()

    d_src, d_pred, d_recon = dev(case.src), dev(case.pred), dev(case.recon0)
    d_q = torch.full((case.n_coef,), ch.SENT32, dtype=torch.int32, device="cuda")
    d_dq = torch.full((case.n_coef,), ch.SENT32, dtype=torch.int32, device="cuda")
    d_eobs = torch.full((len(case.items),), -1, dtype=torch.int16, device="cuda")
    d_iscan, d_qm, d_items = dev(case.iscan), dev(case.qm), dev(case.items)
    npc = (ct.c_int * 5)(*case.n_per_class)
    s = torch.cuda.current_stream().cuda_stream
    rc = b200.lib.svt_b200_residual_txfm_trio_batch_dev(d_src.data_ptr(), d_pred.data_ptr(), d_recon.data_ptr(), d_q.data_ptr(),
                                                         d_dq.data_ptr(), d_iscan.data_ptr(), d_qm.data_ptr(), d_items.data_ptr(),
                                                         npc, d_eobs.data_ptr(), case.pixel_bytes, s)
    assert rc == 0
    torch.cuda.synchronize()
    return {"q": d_q.cpu().numpy(), "dq": d_dq.cpu().numpy(), "eobs": d_eobs.cpu().numpy().view(np.uint16),
            "recon": d_recon.cpu().numpy().view(case.pred.dtype).reshape(case.recon0.shape)}


@gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_every_size_and_type_with_extreme_residuals(b200, refc, bd):
    import torch
    refc.ref_set_tier(0)
    refc.ref_set_threads(0)
    blocks = []
    for sz in range(19):
        for ty in ch.valid_types(sz):
            for mode in ch.MODES[bd][:2]:
                for kind in EXTREME:
                    blocks.append((sz, ty, mode, ch.QM_NONE, 4, 4, ch.KINDS.index(kind)))
    case = ch.build_case(np.array(blocks, ch.BLOCK_DTYPE), bd, rng(470 + bd))
    want = ch.reference_chain(refc, case)
    got = _run_fused(b200, torch, case)
    assert np.any(want["eobs"] > 0)
    for k in ("eobs", "q", "dq", "recon"):
        if not np.array_equal(got[k], want[k]):
            bad = np.flatnonzero(got[k].reshape(-1) != want[k].reshape(-1))
            pytest.fail("bd %d: %s differs at %d places, first %d" % (bd, k, bad.size, int(bad[0])))
