"""CPU-only checks of the host side: the C structs of include/svt_b200.h against their ctypes twins in layout.py,
the batch-ordering rules of the transform calls, the synthetic workload's invariants, and the oracle pin of
the N2 / N4 partial transforms (the fact the CUDA kernels rely on)."""
import ctypes as ct
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from oracle_libs import refc  # noqa: F401  (a fixture: overrides conftest.py's refc in this module)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _c_layout(classes):
    """{(struct, None): sizeof, (struct, field): (offsetof, sizeof member)} of the header, for the fields of each class"""
    lines = []
    for n, cls in classes.items():
        lines.append('printf("%s - %%zu\\n", sizeof(SvtB200%s));' % (n, n))
        lines += ['printf("%s %s %%zu %%zu\\n", offsetof(SvtB200%s, %s), sizeof(((SvtB200%s*)0)->%s));' % (n, f, n, f, n, f)
                  for f, *_ in cls._fields_]
    src = '#include <stddef.h>\n#include <stdio.h>\n#include "svt_b200.h"\nint main(void){\n' + "\n".join(lines) + "\nreturn 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        open(c, "w").write(src)
        r = subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    got = {}
    for l in out.splitlines():
        n, f, *v = l.split()
        got[n, None if f == "-" else f] = int(v[0]) if f == "-" else tuple(map(int, v))
    return got


def test_struct_layouts_match_the_header():
    """Every `typedef struct SvtB200X` of the header has a twin layout.X and no class lacks one; every field of a twin has
    the header's offset and size, and the fields tile the struct without gaps (only tail padding may stay unnamed)."""
    import svt_av1_psy_b200
    from svt_av1_psy_b200 import layout
    txt = subprocess.run(["gcc", "-E", "-P", svt_av1_psy_b200.HEADER_PATH], capture_output=True, text=True, check=True).stdout
    header = sorted(n[len("SvtB200"):] for n in set(re.findall(r"\btypedef\s+struct\s+(SvtB200\w+)", txt)))
    classes = {n: c for n, c in vars(layout).items() if isinstance(c, type) and issubclass(c, ct.Structure)}
    assert sorted(classes) == header
    mine = {}
    for n, cls in classes.items():
        mine[n, None] = ct.sizeof(cls)
        end = 0
        for f, *_ in cls._fields_:
            d = getattr(cls, f)
            mine[n, f] = (d.offset, d.size)
            assert d.offset == end, "%s: %d unnamed bytes before %s" % (n, d.offset - end, f)
            end = d.offset + d.size
    assert mine == _c_layout(classes)


def test_team_class_rule_and_library_agree():
    from svt_av1_psy_b200 import dsp
    for sz in range(19):
        assert dsp.lib.svt_b200_txfm_team_class(sz) == dsp.txfm_team_class(sz)
        assert dsp.txfm_team_class(sz) == {4: 0, 8: 1, 16: 2, 32: 3, 64: 4}[max(dsp.TX_W[sz], dsp.TX_H[sz])]
    assert dsp.lib.svt_b200_txfm_team_class(19) == -1 and dsp.lib.svt_b200_txfm_team_class(-1) == -1


def test_workload_invariants():
    from svt_av1_psy_b200 import dsp
    from svt_av1_psy_b200.workload import FrameWorkload
    wl = FrameWorkload(384, 256)
    n = len(wl.fwd_items)
    assert n == len(wl.inv_items) == len(wl.quant_items) == len(wl.trio_items) == sum(wl.tx_class_counts)
    cls = np.array([dsp.txfm_team_class(int(s)) for s in wl.fwd_items["tx_size"]])
    assert np.all(np.diff(cls) >= 0), "items must be ordered by team class"
    # every sample of the three planes is covered exactly once by the transform blocks
    covered = sum(int(dsp.TX_W[s]) * int(dsp.TX_H[s]) for s in wl.fwd_items["tx_size"])
    assert covered == 384 * 256 * 3 // 2
    # the three views of the fused item are the separate items
    assert np.array_equal(wl.trio_items["fwd"], wl.fwd_items) and np.array_equal(wl.trio_items["quant"], wl.quant_items)
    assert np.array_equal(wl.trio_items["inv"], wl.inv_items)
    # scan / iscan tables are inverse permutations of each other, block by block
    for it in wl.quant_items[:: max(1, n // 50)]:
        o, m = int(it["scan_off"]), int(it["n_coeffs"])
        sc, isc = wl.scan_table[o:o + m], wl.iscan_table[o:o + m]
        assert np.array_equal(isc[sc], np.arange(m))
    # another seed changes the pictures, not the work lists
    w2 = wl.with_seed(99)
    assert w2.trio_items is wl.trio_items and not np.array_equal(w2.cur[0], wl.cur[0])
    assert set(wl.algorithmic_bytes()) >= {"me_search", "txfm_trio", "cdef_search", "wiener_stats"}


def test_reference_n2_n4_equal_the_masked_full_transform(oracle, refc):
    """What svt_b200_fwd_txfm2d_partial implements: the reference's N2 / N4 kernels give the full transform's
    top-left half / quarter (of each dimension) and zero elsewhere."""
    import txfm_helpers as th
    r = np.random.default_rng(5)
    for sz in range(19):
        w, h = th.TX_W[sz], th.TX_H[sz]
        for ty in (0, 3, 9, 12):
            if not th.valid(sz, ty):
                continue
            res, stride = th.residual_input(r, sz, 8, "random")
            full = th.ref_fwd(refc, res, stride, ty, sz).reshape(h, w)
            for level in (1, 2):
                want = full.copy()
                want[max(h >> level, 1):, :] = 0
                want[:, max(w >> level, 1):] = 0
                assert np.array_equal(th.ref_fwd_partial(refc, res, stride, ty, sz, level).reshape(h, w), want), (sz, ty, level)
