"""The two-lane splits of the 32- and 64-point DCTs (txfm_gen.inc, written by tools/gen_txfm_code.py) against the
whole networks of txfm_graphs.inc, without a GPU.

The generated split functions are read back from txfm_gen.inc and evaluated in numpy with the device arithmetic
(32-bit wrapping sums and products, half_btf's 64-bit sum and rounding shift, stage clamps); the whole network is
evaluated straight from the graph data.  Inputs are random int32 vectors with the +-2^31 extremes mixed in, so the
wrapping products of half_btf are exercised."""
import importlib.util
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "svt-av1-psy_b200", "csrc")

_spec = importlib.util.spec_from_file_location("gen_txfm_code", os.path.join(ROOT, "tools", "gen_txfm_code.py"))
gen = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(gen)

GRAPHS = {tag: (n, stages) for tag, n, stages in gen.parse(gen.SRC)}
GEN_TEXT = open(os.path.join(CSRC, "txfm_gen.inc")).read()


def _cospi():
    text = open(os.path.join(CSRC, "txfm_cfg.inc")).read()
    tab = {}
    for m in re.finditer(r"TXCOS\((\d+),([^)]*)\)", text):
        tab[int(m.group(1))] = [int(v) for v in m.group(2).split(",") if v.strip()]
    return tab


COSPI = _cospi()


def w32(v):
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def hbtf(w0, in0, w1, in1, bit):
    return w32((w32(w0 * in0) + w32(w1 * in1) + (1 << (bit - 1))) >> bit)


def hbtf1(w0, in0, bit):
    return w32((w32(w0 * in0) + (1 << (bit - 1))) >> bit)


def clamp_bits(v, bit):
    return v if bit <= 0 else np.clip(v, -(1 << (bit - 1)), (1 << (bit - 1)) - 1)


def whole(tag, x, cos_bit, clampb):
    """the network straight from the graph data (TXG_NODE semantics of txfm_graphs.inc)"""
    n, stages = GRAPHS[tag]
    cos = COSPI[cos_bit]
    cur = [x[i] for i in range(n)]
    for st in stages:
        new = []
        for btf, wa, a, wb, b, cl in st:
            if btf:
                assert not cl
                terms = [(w, cur[o]) for w, o in ((wa, a), (wb, b)) if w]
                ws = [(1 if w > 0 else -1) * cos[abs(w)] for w, _ in terms]
                v = hbtf(ws[0], terms[0][1], ws[1], terms[1][1], cos_bit) if len(terms) == 2 else hbtf1(ws[0], terms[0][1], cos_bit)
            else:
                v = w32(wa * cur[a] + wb * cur[b])
                if cl:
                    v = clamp_bits(v, clampb)
            new.append(v)
        cur = new
    return cur


def function_source(name, text=GEN_TEXT):
    m = re.search(r"__device__ __forceinline__ void txg_%s\(int32_t \(&x\)\[(\d+)\][^{]*\{\n(.*?)\n\}" % re.escape(name), text, re.S)
    assert m, name
    return int(m.group(1)), m.group(2)


def run_generated(name, x, cos_bit, clampb, text=GEN_TEXT):
    """evaluate the generated device function txg_<name> on the vectors x (list of int64 arrays), as the GPU does"""
    n, body = function_source(name, text)
    py = []
    for ln in body.splitlines():
        ln = ln.strip()
        if ln.startswith("(void)"):
            continue
        ln = ln.replace("const int32_t ", "").replace("(uint32_t)", "").replace("(int32_t)(", "w32(").rstrip(";")
        py.append(re.sub(r"\b0u\b", "0", ln))
    env = {"w32": w32, "txg_hbtf": hbtf, "txg_hbtf1": hbtf1, "clamp_bits": clamp_bits, "cosv": COSPI[cos_bit],
           "cos_bit": cos_bit, "clampb": clampb, "x": list(x)}
    exec("\n".join(py), env)  # noqa: S102 -- generated straight-line arithmetic of this repository
    return env["x"]


def struct_masks(name, text=GEN_TEXT):
    m = re.search(r"struct TxgSplit_%s \{(.*?)\n\};" % re.escape(name), text, re.S)
    assert m, name
    body = m.group(1)
    tail = "kTail = true" in body
    masks = {k: int(v, 16) for k, v in re.findall(r"(k(?:Mid|Out)[01]) = (0x[0-9a-f]+)ull", body)}
    return tail, masks


def run_split(name, x, cos_bit, clampb, text=GEN_TEXT):
    """what txfm_pass_split_dct does with one vector: both lane groups, their exchange through memory, the stores"""
    n = len(x)
    tail, m = struct_masks(name, text)
    bits = lambda mask: [i for i in range(n) if (mask >> i) & 1]  # noqa: E731
    if not tail:
        out = [None] * n
        for g in range(2):
            r = run_generated("%s_g%d" % (name, g), x, cos_bit, clampb, text)
            for i in bits(m["kOut%d" % g]):
                out[i] = r[i]
        return out
    cut = [None] * n
    for g in range(2):
        r = run_generated("%s_g%d" % (name, g), x, cos_bit, clampb, text)
        for i in bits(m["kMid%d" % g]):
            cut[i] = r[i]
    out = [None] * n
    for g in range(2):
        r = run_generated("%s_t%d" % (name, g), cut, cos_bit, clampb, text)
        for i in bits(m["kOut%d" % g]):
            out[i] = r[i]
    return out


def random_vectors(n, k, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(-(1 << 31), 1 << 31, size=(n, k), dtype=np.int64)
    small = rng.integers(-(1 << 17), 1 << 17, size=(n, k // 2), dtype=np.int64)  # realistic residual / coefficient ranges
    x[:, : k // 2] = small
    ext = np.array([-(1 << 31), (1 << 31) - 1, 0, -1, 1], dtype=np.int64)
    x[:, k // 2: k // 2 + 64] = rng.choice(ext, size=(n, 64))
    return [x[i] for i in range(n)]


def live_and_zero(name):
    for nm, tag, live_out, zero_in in gen.SPLITS:
        if nm == name:
            n = GRAPHS[tag][0]
            return tag, n, (list(range(n)) if live_out is None else list(live_out)), (zero_in or set())
    raise KeyError(name)


def check(name, cos_bit, clampb, seed=1, text=GEN_TEXT):
    tag, n, live, zero = live_and_zero(name)
    x = random_vectors(n, 512, seed)
    for i in zero:
        x[i] = np.zeros_like(x[i])
    ref = whole(tag, x, cos_bit, clampb)
    got = run_split(name, x, cos_bit, clampb, text)
    return all(got[i] is not None and np.array_equal(got[i], ref[i]) for i in live)


SPLIT_NAMES = [s[0] for s in gen.SPLITS]


def test_every_split_is_emitted():
    for name in SPLIT_NAMES:
        assert "struct TxgSplit_%s {" % name in GEN_TEXT


@pytest.mark.parametrize("name", SPLIT_NAMES)
def test_split_masks_partition_the_outputs(name):
    tag, n, live, _ = live_and_zero(name)
    tail, m = struct_masks(name)
    assert m["kOut0"] & m["kOut1"] == 0 and m["kOut0"] | m["kOut1"] == sum(1 << i for i in live)
    assert m["kOut0"] and m["kOut1"]
    if tail:
        assert m["kMid0"] & m["kMid1"] == 0 and m["kMid0"] | m["kMid1"] == (1 << n) - 1


@pytest.mark.parametrize("name", SPLIT_NAMES)
@pytest.mark.parametrize("cos_bit", [12, 13])
def test_split_matches_whole_network(name, cos_bit):
    clampb = 16 if name.startswith("I") else 0
    assert check(name, cos_bit, clampb)
    if name.startswith("I"):
        assert check(name, cos_bit, 18, seed=2) and check(name, cos_bit, 20, seed=3)


def test_a_wrong_pair_index_is_caught():
    """the comparison is sharp: one operand of one butterfly in one split function pointed at its neighbour fails it"""
    for name in SPLIT_NAMES:
        assert check(name, 12, 16 if name.startswith("I") else 0)
    _, body = function_source("FDCT64_lo32_g1")
    m = re.search(r"txg_hbtf\(([-\w]+), s(\d+)_(\d+),", body)
    assert m
    s, i = int(m.group(2)), int(m.group(3))
    bad_line = m.group(0).replace("s%d_%d," % (s, i), "s%d_%d," % (s, i ^ 1))
    mutated = GEN_TEXT.replace(body, body.replace(m.group(0), bad_line, 1))
    assert mutated != GEN_TEXT
    assert not check("FDCT64_lo32", 12, 0, text=mutated)
