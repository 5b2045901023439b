"""The self-guided restoration filter (SGR) against the reference's own C functions at 8, 10 and 12 bit, at every
parameter set, at the unit shapes and content where an integer kernel goes wrong, and in the shapes the encoder's
restoration search calls it with:

  * the T1 filter and apply (svt_av1_selfguided_restoration_c, svt_apply_selfguided_restoration_c): widths and heights
    from 1 up to what the reference's stack buffers hold, odd source strides, outputs written into the middle of wider
    buffers, all 16 parameter sets on random, flat, all-0, all-max, 0/max checkerboard, near-flat and gradient content,
    and xqd at the four corners of its legal box;
  * the projection calls (svt_av1_{lowbd,highbd}_pixel_proj_error_c, svt_get_proj_subspace_c) on whole restoration
    units up to 383 x 383 with padded strides, and the SGR half of search_selfguided_restoration (restoration_pick.c)
    run once on the reference functions and once on the H100 ones;
  * the same T1 calls from 8 host threads at once;
  * svt_b200_sgr_units_dev: mixed batches up to 128 x 128, more units than CTAs, two streams at once, its argument checks;
  * the striped filter with self-guided units at 8, 10 and 12 bit (oracle/ref_driver.c ref_lr_filter_plane).

Units larger than the reference filter takes are checked against the reference run on sub-tiles whose bands start an
even number of rows apart (rest_helpers.ref_sgr_tiled); the two CPU tests at the top show that this oracle equals the
whole call and that it would notice a band started on an odd row.  Every output buffer is filled with a sentinel first
and compared whole, so strides, gaps and the output of a radius-0 filter must keep it."""
import ctypes as ct
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import rest_helpers as rh
from helpers import rng
from oracle_libs import refc  # noqa: F401  (a fixture: overrides conftest.py's refc in this module)
from test_restoration_frame import PAD, _plane
from test_restoration_paths import _reference, _run

SENT = -0x2A2A2A2B  # int32 filter-output sentinel
BAD_ARG = -4        # SVT_B200_ERR_BAD_ARG
H100_SMS = 132      # svt_b200_sgr_units_dev launches at most 2 CTAs per SM
XQD_LO, XQD_HI = (-96, -32), (31, 95)  # SGRPROJ_PRJ_MIN0 / MIN1, SGRPROJ_PRJ_MAX0 / MAX1
XQD_CORNERS = [(a, b) for a in (XQD_LO[0], XQD_HI[0]) for b in (XQD_LO[1], XQD_HI[1])]
KINDS = ("random", "flat", "zeros", "max", "checker", "nearflat", "gradient")
# name -> (bit depth, pixel type): 8-bit content also runs through the 16-bit pipeline (highbd = 1)
MODES = {"b8": (8, np.uint8), "b8_in_u16": (8, np.uint16), "b10": (10, np.uint16), "b12": (12, np.uint16)}


def _content(r, kind, rows, cols, bd):
    mx = (1 << bd) - 1
    yy, xx = np.mgrid[0:rows, 0:cols]
    if kind == "random":
        a = r.integers(0, mx + 1, (rows, cols))
    elif kind == "flat":
        a = np.full((rows, cols), int(r.integers(0, mx + 1)))
    elif kind == "zeros":
        a = np.zeros((rows, cols), np.int64)
    elif kind == "max":
        a = np.full((rows, cols), mx)
    elif kind == "checker":  # the largest local variance: p * s and z at their largest
        a = ((yy + xx) & 1) * mx
    elif kind == "nearflat":  # at 10 / 12 bit the rounded moments give a * n < b * b, which the guard saturates to p = 0
        a = int(r.integers(mx // 4, 3 * mx // 4)) + r.integers(0, 2, (rows, cols))
    elif kind == "gradient":
        a = np.minimum((xx * 5 + yy * 3) << (bd - 8), mx)
    else:
        raise ValueError(kind)
    return a


def _sgr_smem(w, h):
    """the dynamic shared memory of sgr_filter_kernel for a w x h launch (sgr.cu sgr_smem)"""
    return (((w + 6) * (h + 6) * 2 + 15) & ~15) + 2 * (w + 2) * (h + 2) * 4


def _tile(r, kind, w, h, bd, dt, pad_x):
    """a w x h block with at least a 3-pixel border of the same content, in a plane of odd pitch: (plane, offset, stride)"""
    stride = (w + 8 + pad_x) | 1
    plane = _content(r, kind, h + 8, stride, bd).astype(dt).reshape(-1)
    return plane, 4 * stride + 4, stride


def _fbuf(w, h, fstride, lead):
    return np.full(lead + (h + 1) * fstride, SENT, np.int32)


def _outside(buf, foff, fstride, w, h):
    """the elements of buf that lie outside the w x h window at foff"""
    m = np.ones(buf.size, bool)
    for i in range(h):
        m[foff + i * fstride:foff + i * fstride + w] = False
    return buf[m]


# ---- the case lists (the CPU test below checks what they reach) --------------------------------------------------------
T1_WIDTHS = (1, 2, 3, 4, 5, 7, 8, 31, 32, 33, 63, 64, 75, 96, 128, 200)
T1_HEIGHTS = (1, 2, 3, 4, 7, 8, 33, 63, 64)
T1_SHAPES = [(w, h) for w in T1_WIDTHS for h in T1_HEIGHTS if rh.ref_sgr_fits(w, h)]


def t1_cases():
    """(w, h, params_idx, kind): every shape meets every parameter set; the content kind rotates with both, so each shape
    sees every kind and each set every kind"""
    for s, (w, h) in enumerate(T1_SHAPES):
        for idx in range(16):
            yield w, h, idx, KINDS[(idx + s) % len(KINDS)]


APPLY_SHAPES = [(1, 1), (2, 3), (7, 4), (33, 33), (64, 64), (63, 7), (75, 75), (200, 30)]


def apply_cases():
    """(kind, xqd): the corners of the xqd box on the extremes of content and on random content (a checkerboard is so
    variable that the filter returns it unchanged; random pixels make the projection clamp at both ends), random xqd on
    the rest"""
    r = rng(3101)
    out = [(kind, c) for kind in ("zeros", "max", "checker", "random") for c in XQD_CORNERS]
    out += [(kind, (int(r.integers(-96, 32)), int(r.integers(-32, 96)))) for kind in ("random", "gradient", "nearflat")]
    return out


PROJ_UNITS = [(1, 1), (7, 3), (64, 64), (129, 65), (256, 256), (383, 200), (200, 383), (383, 383)]
PROJ_SETS = (0, 7, 10, 13, 14, 15)  # both radii, r0 = 0, r1 = 0
PROJ_KINDS = ("noisy", "max", "checker", "flat", "flat_filter", "extreme")


def proj_xqds():
    r = rng(3102)
    return XQD_CORNERS + [(int(r.integers(-96, 32)), int(r.integers(-32, 96))) for _ in range(2)]


def sgr_batch(seed, n, max_wh, special=()):
    """units of one svt_b200_sgr_units_dev call as tuples (x, y, w, h, params_idx, flt_stride): the special sizes, then
    random sizes up to max_wh, parameter sets in turn, output pitches 1 .. 7 wider than the unit"""
    r = rng(seed)
    sizes = list(special) + [(int(r.integers(1, max_wh + 1)), int(r.integers(1, max_wh + 1))) for _ in range(n - len(special))]
    out, x, y, shelf, plane_w = [], 3, 3, 0, 1200
    for k, (w, h) in enumerate(sizes):
        if x + w + 3 > plane_w:
            x, y, shelf = 3, y + shelf + 7, 0
        out.append((x, y, w, h, (k * 7 + seed) % 16, w + 1 + k % 7))
        x += w + 7 + k % 3
        shelf = max(shelf, h)
    return out, plane_w, y + shelf + 3


BATCH_SPECIAL = [(1, 1), (128, 128), (127, 3), (3, 127), (65, 65), (2, 1), (1, 2), (33, 97), (128, 1), (1, 128), (75, 76), (64, 64),
                 (127, 127), (5, 8)]
BATCHES = {"mixed": (3201, 300, 128, BATCH_SPECIAL), "small": (3202, 40, 32, [(1, 1), (32, 32), (31, 1)])}


def striped_choice(k, plane, mix):
    """(restoration_type, sgr_ep, xqd corner or 4 = random) of unit k of a plane: the self-guided units take the 16 sets
    in turn and the xqd corners against them; `mix` puts Wiener and RESTORE_NONE units in between"""
    t = (2, 1, 2, 0, 2, 2)[k % 6] if mix else 2
    j = k - (k // 6) * 2 - (1 if k % 6 > 1 else 0) - (1 if k % 6 > 3 else 0) if mix else k  # index among the SGR units
    return t, (j + 3 * plane) % 16, (j // 5 + j) % 5


def striped_units(b200, n, plane, seed, mix):
    r = rng(seed)
    u = np.zeros(n, dtype=b200.LR_UNIT_DTYPE)
    for k in range(n):
        t, ep, c = striped_choice(k, plane, mix)
        u["restoration_type"][k] = t
        t0, t1, t2 = int(r.integers(-5, 11)), int(r.integers(-23, 9)), int(r.integers(-17, 47))
        taps = np.array([0 if plane else t0, t1, t2, -2 * ((0 if plane else t0) + t1 + t2), t2, t1, 0 if plane else t0, 0], np.int16)
        u["hfilter"][k] = taps
        u["vfilter"][k] = taps
        u["sgr_ep"][k] = ep
        u["sgr_xqd"][k] = XQD_CORNERS[c] if c < 4 else (int(r.integers(-96, 32)), int(r.integers(-32, 96)))
    return u


# (luma width, luma height, bit depth, luma unit size, frame_restoration_type, mixed unit types)
STRIPED_CASES = [(520, 301, 12, 64, 2, False), (520, 185, 12, 64, 3, True), (1000, 377, 12, 128, 0, True), (1100, 1040, 12, 256, 2, False),
                 (520, 301, 10, 64, 2, False), (1000, 377, 10, 128, 3, True), (1100, 1040, 10, 256, 0, False), (520, 185, 8, 64, 2, False)]


def _units_per_dim(size, us):
    return max(1, (size + us // 2) // us)


# ---- CPU: the oracle for large units, and what the cases reach --------------------------------------------------------
@pytest.mark.parametrize("bd", (8, 10, 12))
def test_tiled_reference_equals_whole_call(refc, bd):
    """the reference on sub-tiles whose bands start an even number of rows apart == one call on the unit; bands that
    start on an odd row change the r = 2 output (and only it), so the tiled oracle can tell the two apart"""
    r = rng(3000 + bd)
    dt = np.uint8 if bd == 8 else np.uint16
    odd_seen = 0
    for (w, h) in [(64, 64), (75, 75), (33, 63), (200, 30), (96, 33), (41, 50)]:
        plane, off, stride = _tile(r, "random", w, h, bd, dt, 5)
        fs = w + 3
        for idx in range(16):
            prm = rh.SGR_PARAMS[idx]
            whole = [_fbuf(w, h, fs, 2) for _ in range(2)]
            rh.ref_sgr_into(refc, plane, off, w, h, stride, idx, bd, whole[0], whole[1], 2, fs)
            tiled = [_fbuf(w, h, fs, 2) for _ in range(2)]
            rh.ref_sgr_tiled(refc, plane, off, w, h, stride, idx, bd, tiled[0], tiled[1], 2, fs, tw=13, rows=range(0, h, 16))
            assert np.array_equal(whole[0], tiled[0]) and np.array_equal(whole[1], tiled[1]), (w, h, idx)
            if h >= 8:
                odd = [_fbuf(w, h, fs, 2) for _ in range(2)]
                rh.ref_sgr_tiled(refc, plane, off, w, h, stride, idx, bd, odd[0], odd[1], 2, fs, tw=13, rows=[0, 7] + list(range(23, h, 16)))
                assert np.array_equal(whole[1], odd[1]), (w, h, idx)  # the r = 1 pass has no row parity
                if prm[0] > 0:
                    assert not np.array_equal(whole[0], odd[0]), (w, h, idx)
                    odd_seen += 1
    assert odd_seen > 0


@pytest.mark.parametrize("bd", (8, 10, 12))
def test_p_times_s_cannot_wrap(bd):
    """CPU: the filter's p * s (restoration.c:735) stays below 2^32 for every window of pixels in [0, (1 << bd) - 1], so
    the uint32 product never wraps and a 64-bit one would give the same z.  n * sum(x^2) - sum(x)^2 is convex in each
    pixel, so it is largest with k pixels at the maximum and the rest at 0, where it is k (n - k) max^2; rounding a and b
    to 8-bit scale adds at most n / 2 + sum / 2^(bd - 8).  A 0/max checkerboard puts n // 2 or n // 2 + 1 maxima in every
    window, which is where k (n - k) peaks, so the checkerboard cases run the largest p * s there is."""
    mx, d = (1 << bd) - 1, bd - 8
    worst = 0
    for prm in rh.SGR_PARAMS:
        for r, s in zip(prm[:2], prm[2:]):
            if r == 0:
                continue
            n = (2 * r + 1) ** 2
            k = max(range(n + 1), key=lambda k: k * (n - k))
            assert k in (n // 2, n // 2 + 1)
            bound = k * (n - k) * mx * mx / 4 ** d + n / 2 + n * mx / 2 ** d
            worst = max(worst, bound * s)
    assert worst < 2 ** 32, worst
    chk = _content(None, "checker", 6, 6, bd)
    assert all((chk[y:y + 3, x:x + 3] == mx).sum() in (4, 5) for y in range(4) for x in range(4))
    assert all((chk[y:y + 5, x:x + 5] == mx).sum() in (12, 13) for y in range(2) for x in range(2))


def test_cases_reach_every_boundary():
    """CPU: from the case lists alone, the GPU tests below reach every boundary they are meant to"""
    t1 = list(t1_cases())
    for (w, h) in T1_SHAPES:
        assert {c[2] for c in t1 if c[:2] == (w, h)} == set(range(16)), (w, h)       # every shape meets every set
        assert {c[3] for c in t1 if c[:2] == (w, h)} == set(KINDS), (w, h)          # ... and every content kind
    for idx in range(16):
        assert {c[3] for c in t1 if c[2] == idx} == set(KINDS), idx                 # every set meets every kind
    hs, ws = {h for _, h in T1_SHAPES}, {w for w, _ in T1_SHAPES}
    assert 1 in ws and 1 in hs and any(h % 2 for h in hs) and any(h % 2 == 0 for h in hs)
    assert {1, 2, 3, 4, 5, 7, 8, 31, 32, 33, 63, 64} <= ws and {1, 2, 3, 4, 7, 8, 33, 63, 64} <= hs
    assert all(rh.ref_sgr_fits(w, h) for w, h in T1_SHAPES + APPLY_SHAPES)
    assert any(_sgr_smem(w, h) > 48 * 1024 for w, h in T1_SHAPES)                    # the T1 launch above 48 KB
    assert any(_sgr_smem(w, h) <= 48 * 1024 for w, h in T1_SHAPES)
    assert max(w for w, _ in T1_SHAPES) == 200 and (75, 64) in T1_SHAPES
    # apply: every corner of the xqd box on the contents that clamp at both ends
    ac = apply_cases()
    for kind in ("zeros", "max", "checker", "random"):
        assert {x for k, x in ac if k == kind} >= set(XQD_CORNERS), kind
    assert set(XQD_CORNERS) <= set(proj_xqds())
    # projection: units up to the largest a search sees, every radius combination, the determinant's zero branch
    assert {(64, 64), (256, 256), (383, 200), (200, 383), (383, 383), (1, 1)} <= set(PROJ_UNITS)
    assert any(rh.SGR_PARAMS[i][0] and rh.SGR_PARAMS[i][1] for i in PROJ_SETS)
    assert any(not rh.SGR_PARAMS[i][0] for i in PROJ_SETS) and any(not rh.SGR_PARAMS[i][1] for i in PROJ_SETS)
    assert "flat" in PROJ_KINDS and "flat_filter" in PROJ_KINDS and "extreme" in PROJ_KINDS
    # the unit batches
    units, _, _ = sgr_batch(*BATCHES["mixed"])
    assert len(units) > 2 * H100_SMS                                                  # more units than CTAs
    assert {u[4] for u in units} == set(range(16))
    assert (1, 1) in {u[2:4] for u in units} and (128, 128) in {u[2:4] for u in units}
    assert any(u[3] % 2 for u in units) and any(u[3] % 2 == 0 for u in units)
    assert all(u[5] > u[2] for u in units) and max(max(u[2:4]) for u in units) == 128
    assert _sgr_smem(128, 128) > 48 * 1024 and _sgr_smem(32, 32) <= 48 * 1024
    small, _, _ = sgr_batch(*BATCHES["small"])
    assert max(max(u[2:4]) for u in small) == 32
    # striped: 12-bit self-guided units, all three unit sizes, every set on every plane, both frame types with SGR
    assert any(c[2] == 12 for c in STRIPED_CASES) and {c[3] for c in STRIPED_CASES if c[2] == 12} == {64, 128, 256}
    assert {c[4] for c in STRIPED_CASES} == {0, 2, 3} and {c[2] for c in STRIPED_CASES} == {8, 10, 12}
    for (W, H, bd, us, frt, mix) in STRIPED_CASES:
        for p in range(3):
            ss = 1 if p else 0
            w, h, usp = (W + ss) >> ss, (H + ss) >> ss, us >> ss
            n = _units_per_dim(w, usp) * _units_per_dim(h, usp)
            ch = [striped_choice(k, p, mix) for k in range(n)]
            assert {c[1] for c in ch if c[0] == 2} == set(range(16)), (W, H, us, p)
            assert {c[2] for c in ch if c[0] == 2} == set(range(5)), (W, H, us, p)
            assert not mix or {c[0] for c in ch} == {0, 1, 2}
            assert w % min(usp, 64), (W, p)                                           # a width that is not a multiple of the run
    assert any(((H + 8) % 64) % 2 for (W, H, *_rest) in STRIPED_CASES)                  # an odd last stripe
    assert any((H - 56) % 64 == 1 for (W, H, *_rest) in STRIPED_CASES)                 # a stripe ending 1 row above the border


# ---- T1 filter and apply ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_t1_filter_matches_reference(b200, refc, mode):
    """svt_b200_av1_selfguided_restoration == svt_av1_selfguided_restoration_c, every shape x set, outputs written at an
    offset into wider sentinel-filled buffers"""
    bd, dt = MODES[mode]
    r = rng(3300 + bd + (dt == np.uint16))
    hbd = int(dt == np.uint16)
    for k, (w, h, idx, kind) in enumerate(t1_cases()):
        plane, off, stride = _tile(r, kind, w, h, bd, dt, k % 4)
        fs = w + 1 + k % 6
        lead = fs + 3
        want = [_fbuf(w, h, fs, lead) for _ in range(2)]
        rh.ref_sgr_into(refc, plane, off, w, h, stride, idx, bd, want[0], want[1], lead, fs)
        got = [_fbuf(w, h, fs, lead) for _ in range(2)]
        b200.lib.svt_b200_av1_selfguided_restoration(rh.P(plane, off), w, h, stride, rh.P(got[0], lead), rh.P(got[1], lead), fs, idx, bd, hbd)
        for i in range(2):
            assert np.array_equal(got[i], want[i]), (mode, w, h, idx, kind, "flt%d" % i, np.argwhere(got[i] != want[i])[:4])
            if rh.SGR_PARAMS[idx][i] == 0:
                assert (got[i] == SENT).all()
            assert (_outside(got[i], lead, fs, w, h) == SENT).all()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_t1_apply_matches_reference(b200, refc, mode):
    """svt_b200_apply_selfguided_restoration == svt_apply_selfguided_restoration_c; the cases make the projection clamp
    at 0 and at (1 << bd) - 1"""
    bd, dt = MODES[mode]
    r = rng(3400 + bd + (dt == np.uint16))
    hbd = int(dt == np.uint16)
    mx = (1 << bd) - 1
    app = refc.svt_apply_selfguided_restoration_c; app.restype = None
    tmp = np.zeros(2 * 406 * 398 + 64, np.int32)  # 2 x RESTORATION_UNITPELS_MAX
    clamped = set()
    for s, (w, h) in enumerate(APPLY_SHAPES):
        for kind, xqd in apply_cases():
            plane, off, stride = _tile(r, kind, w, h, bd, dt, s)
            xqd_a = np.array(xqd, np.int32)
            for idx in range(16):
                ds = w + 3 + s
                want = np.full((h + 2) * ds, 0x5A, dt)
                got = want.copy()
                app(rh.bptr(plane, off), w, h, stride, idx, rh.P(xqd_a), rh.bptr(want, ds + 1), ds, rh.P(tmp), bd, hbd)
                b200.lib.svt_b200_apply_selfguided_restoration(rh.P(plane, off), w, h, stride, idx, rh.P(xqd_a), rh.P(got, ds + 1), ds, None, bd, hbd)
                assert np.array_equal(got, want), (mode, w, h, kind, xqd, idx, np.argwhere(got != want)[:4])
                # which clamp the reference applied: the projection before the clamp, from the reference filter outputs
                f = [np.zeros(w * h, np.int32) for _ in range(2)]
                rh.ref_sgr_into(refc, plane, off, w, h, stride, idx, bd, f[0], f[1], 0, w)
                u = plane[off + (np.arange(h)[:, None] * stride + np.arange(w)[None, :])].astype(np.int64).reshape(-1) << 4
                xq = rh.decode_xq(xqd, rh.SGR_PARAMS[idx])
                v = u << 7
                for i in range(2):
                    if rh.SGR_PARAMS[idx][i]:
                        v = v + xq[i] * (f[i].astype(np.int64) - u)
                wv = (v + 1024) >> 11
                clamped |= {"low"} if (wv < 0).any() else set()
                clamped |= {"high"} if (wv > mx).any() else set()
    assert clamped == {"low", "high"}, clamped


# ---- T1 projection calls on whole units -------------------------------------------------------------------------------
def _proj_unit(refc, r, kind, w, h, bd, dt, idx):
    """(src, dat, flt0, flt1) of a w x h restoration unit with padded strides: (array, offset, stride) each"""
    mx = (1 << bd) - 1
    ss, ds, f0s, f1s = w + 13, w + 8, w + 3, w + 11
    dat = _content(r, {"noisy": "gradient", "flat_filter": "flat", "extreme": "max"}.get(kind, kind), h + 8, ds, bd).astype(dt).reshape(-1)
    doff = 4 * ds + 4
    if kind == "noisy":
        dat = np.clip(dat.astype(np.int64) + r.integers(-(mx >> 4) - 1, (mx >> 4) + 2, dat.size), 0, mx).astype(dt)
    src = _content(r, "checker" if kind in ("max", "extreme") else ("flat" if kind.startswith("flat") else "gradient"), h + 1, ss, bd)
    if kind in ("max", "extreme"):
        src = mx - src  # the source against the saturated picture: s = (src << 4) - u at its largest
    src = src.astype(dt).reshape(-1)
    f0 = np.full(h * f0s + 5, SENT, np.int32); f1 = np.full(h * f1s + 9, SENT, np.int32)
    if kind == "extreme":  # filter outputs at both ends of the range the projection documents: |flt| < 2^15
        lim = (1 << 15) - 1
        f0[:] = r.choice([-lim, lim, 0], f0.size); f1[:] = r.choice([-lim, lim, 1], f1.size)
    elif kind == "flat_filter":  # both filters return the picture: H = 0, xq stays {0, 0}
        for i in range(h):
            f0[i * f0s:i * f0s + w] = dat[doff + i * ds:doff + i * ds + w].astype(np.int32) << 4
            f1[i * f1s:i * f1s + w] = dat[doff + i * ds:doff + i * ds + w].astype(np.int32) << 4
    else:
        t0 = np.full(h * f0s + 5, SENT, np.int32); t1 = np.full(h * f1s + 9, SENT, np.int32)
        g0, g1 = np.full(h * f1s + 9, SENT, np.int32), np.full(h * f1s + 9, SENT, np.int32)  # the pass not wanted at each pitch
        # the two outputs have different pitches: run the tiled reference once per pitch
        rh.ref_sgr_tiled(refc, dat, doff, w, h, ds, idx, bd, t0, g1, 0, f0s)
        rh.ref_sgr_tiled(refc, dat, doff, w, h, ds, idx, bd, g0, t1, 0, f1s)
        f0, f1 = t0, t1
    return (src, 0, ss), (dat, doff, ds), (f0, f0s), (f1, f1s)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_projection_on_whole_units(b200, refc, mode):
    """svt_b200_get_proj_subspace and svt_b200_av1_{lowbd,highbd}_pixel_proj_error == the reference on whole units up to
    383 x 383, padded strides, flt0_stride != flt1_stride"""
    bd, dt = MODES[mode]
    r = rng(3500 + bd + (dt == np.uint16))
    hbd = int(dt == np.uint16)
    gps = refc.svt_get_proj_subspace_c; gps.restype = None
    ppe = refc.svt_av1_highbd_pixel_proj_error_c if hbd else refc.svt_av1_lowbd_pixel_proj_error_c; ppe.restype = ct.c_int64
    dev_ppe = b200.lib.svt_b200_av1_highbd_pixel_proj_error if hbd else b200.lib.svt_b200_av1_lowbd_pixel_proj_error
    zero_det = 0
    for ui, (w, h) in enumerate(PROJ_UNITS):
        for ki, kind in enumerate(PROJ_KINDS):
            if kind in ("max", "checker", "extreme") and w * h > 64 * 64 and bd < 12 and (ui + ki) % 2:
                continue  # the largest moments are 12-bit; lower depths take every other unit of these kinds
            idx = PROJ_SETS[(ui + ki) % len(PROJ_SETS)]
            (src, so, ss), (dat, do, ds), (f0, f0s), (f1, f1s) = _proj_unit(refc, r, kind, w, h, bd, dt, idx)
            for idx2 in {idx, PROJ_SETS[(ui + ki + 3) % len(PROJ_SETS)]} if kind in ("extreme", "flat_filter") else {idx}:
                prm = np.array(rh.SGR_PARAMS[idx2], np.int32)
                xq_w = np.full(2, 77, np.int32); xq_g = np.full(2, 77, np.int32)
                gps(rh.bptr(src, so), w, h, ss, rh.bptr(dat, do), ds, hbd, rh.P(f0), f0s, rh.P(f1), f1s, rh.P(xq_w), rh.P(prm))
                b200.lib.svt_b200_get_proj_subspace(rh.P(src, so), w, h, ss, rh.P(dat, do), ds, hbd, rh.P(f0), f0s, rh.P(f1), f1s, rh.P(xq_g),
                                                    rh.P(prm))
                assert np.array_equal(xq_g, xq_w), (mode, w, h, kind, idx2, xq_g, xq_w)
                if kind == "flat_filter" or (kind == "flat" and prm[0] and prm[1]):
                    assert list(xq_w) == [0, 0], (w, h, kind, idx2)  # det < 1e-8: the default
                    zero_det += 1
                for xqd in proj_xqds() + [(int(xq_w[0]), int(xq_w[1]))]:
                    xq = np.array(rh.decode_xq(xqd, prm), np.int32)
                    ew = ppe(rh.bptr(src, so), w, h, ss, rh.bptr(dat, do), ds, rh.P(f0), f0s, rh.P(f1), f1s, rh.P(xq), rh.P(prm))
                    eg = dev_ppe(rh.P(src, so), w, h, ss, rh.P(dat, do), ds, rh.P(f0), f0s, rh.P(f1), f1s, rh.P(xq), rh.P(prm))
                    assert eg == ew, (mode, w, h, kind, idx2, xqd, eg, ew)
    assert zero_det > 0


class _RefSgr:
    """the SGR calls of search_selfguided_restoration, on the reference's C functions"""

    def __init__(self, refc, hbd):
        self.refc, self.hbd = refc, hbd
        self.gps = refc.svt_get_proj_subspace_c; self.gps.restype = None
        self.ppe = refc.svt_av1_highbd_pixel_proj_error_c if hbd else refc.svt_av1_lowbd_pixel_proj_error_c
        self.ppe.restype = ct.c_int64

    def filter(self, dat, off, w, h, stride, f0, f1, foff, fs, ep, bd):
        rh.ref_sgr_into(self.refc, dat, off, w, h, stride, ep, bd, f0, f1, foff, fs)

    def subspace(self, src, so, ss, dat, do, ds, w, h, f0, f1, fs, xq, prm):
        self.gps(rh.bptr(src, so), w, h, ss, rh.bptr(dat, do), ds, self.hbd, rh.P(f0), fs, rh.P(f1), fs, rh.P(xq), rh.P(prm))

    def error(self, src, so, ss, dat, do, ds, w, h, f0, f1, fs, xq, prm):
        return self.ppe(rh.bptr(src, so), w, h, ss, rh.bptr(dat, do), ds, rh.P(f0), fs, rh.P(f1), fs, rh.P(xq), rh.P(prm))


class _DevSgr(_RefSgr):
    """the same calls on the H100 T1 entry points"""

    def __init__(self, b200, hbd):
        self.lib, self.hbd = b200.lib, hbd
        self.ppe = self.lib.svt_b200_av1_highbd_pixel_proj_error if hbd else self.lib.svt_b200_av1_lowbd_pixel_proj_error

    def filter(self, dat, off, w, h, stride, f0, f1, foff, fs, ep, bd):
        self.lib.svt_b200_av1_selfguided_restoration(rh.P(dat, off), w, h, stride, rh.P(f0, foff), rh.P(f1, foff), fs, ep, bd, self.hbd)

    def subspace(self, src, so, ss, dat, do, ds, w, h, f0, f1, fs, xq, prm):
        self.lib.svt_b200_get_proj_subspace(rh.P(src, so), w, h, ss, rh.P(dat, do), ds, self.hbd, rh.P(f0), fs, rh.P(f1), fs, rh.P(xq), rh.P(prm))

    def error(self, src, so, ss, dat, do, ds, w, h, f0, f1, fs, xq, prm):
        return self.ppe(rh.P(src, so), w, h, ss, rh.P(dat, do), ds, rh.P(f0), fs, rh.P(f1), fs, rh.P(xq), rh.P(prm))


def _search(api, src, so, ss, dat, do, ds, w, h, bd, pu):
    """the SGR part of search_selfguided_restoration (restoration_pick.c:542-640) with no reference-frame eps (step < 16:
    every ep, refined): apply_sgr tiling into a unit-wide buffer, get_proj_subspace, encode_xq, then
    finer_search_pixel_proj_error from step 2.  Returns (ep, xqd, err) of every ep, the chosen one last."""
    fs = ((w + 7) & ~7) + 8
    f0 = np.full(h * fs + 8, SENT, np.int32); f1 = np.full(h * fs + 8, SENT, np.int32)
    trace, best = [], None
    lo, hi = XQD_LO, XQD_HI
    for ep in range(16):
        for i in range(0, h, pu):
            for j in range(0, w, pu):
                api.filter(dat, do + i * ds + j, min(pu, w - j), min(pu, h - i), ds, f0, f1, i * fs + j, fs, ep, bd)
        prm = np.array(rh.SGR_PARAMS[ep], np.int32)
        exq = np.zeros(2, np.int32)
        api.subspace(src, so, ss, dat, do, ds, w, h, f0, f1, fs, exq, prm)
        clamp = lambda v, a, b: max(a, min(b, v))  # noqa: E731
        if prm[0] == 0:
            xqd = [0, clamp(128 - int(exq[1]), lo[1], hi[1])]
        elif prm[1] == 0:
            xqd = [clamp(int(exq[0]), lo[0], hi[0])]
            xqd.append(clamp(128 - xqd[0], lo[1], hi[1]))
        else:
            xqd = [clamp(int(exq[0]), lo[0], hi[0])]
            xqd.append(clamp(128 - xqd[0] - int(exq[1]), lo[1], hi[1]))

        def err_of(q):
            return int(api.error(src, so, ss, dat, do, ds, w, h, f0, f1, fs, np.array(rh.decode_xq(q, prm), np.int32), prm))
        err = err_of(xqd)
        step = 2
        s = step
        while s >= 1:
            for p in range(2):
                if (prm[0] == 0 and p == 0) or (prm[1] == 0 and p == 1):
                    continue
                skip = False
                while xqd[p] - s >= lo[p]:
                    xqd[p] -= s
                    e2 = err_of(xqd)
                    if e2 > err:
                        xqd[p] += s
                        break
                    err, skip = e2, True
                    if s != step:
                        break
                if skip:
                    break
                while xqd[p] + s <= hi[p]:
                    xqd[p] += s
                    e2 = err_of(xqd)
                    if e2 > err:
                        xqd[p] -= s
                        break
                    err = e2
                    if s != step:
                        break
            s >>= 1
        trace.append((ep, tuple(xqd), err))
        if best is None or err < best[2]:
            best = (ep, tuple(xqd), err)
    return trace + [best]


# (w, h, noise): the noise is the picture's maximum over this; the noisiest unit drives xqd to the corners of its box,
# the cleanest keeps it inside
SEARCH_UNITS = [(64, 64, 40), (100, 71, 150), (160, 97, 400), (37, 90, 400)]


@pytest.mark.gpu
@pytest.mark.parametrize("pu", (32, 64))
@pytest.mark.parametrize("mode", list(MODES))
def test_search_call_sequence_matches_reference(b200, refc, mode, pu):
    """the SGR search of several units, once on the reference functions and once on the H100 ones: the same
    (ep, xqd, err) for every ep, and the same choice"""
    bd, dt = MODES[mode]
    r = rng(3600 + bd + pu + (dt == np.uint16))
    hbd = int(dt == np.uint16)
    mx = (1 << bd) - 1
    for (w, h, noise) in SEARCH_UNITS:
        ss, ds = w + 21, w + 10
        yy, xx = np.mgrid[0:h + 8, 0:ds]
        clean = np.clip((np.sin(xx / 7.0) + np.cos(yy / 5.0) + 2.0) / 4.0 * mx, 0, mx)
        dat = np.clip(np.round(clean + r.normal(0, mx / noise, clean.shape)), 0, mx).astype(dt).reshape(-1)
        src = np.zeros((h, ss), dt)
        src[:, :w] = np.round(clean[4:4 + h, 4:4 + w]).astype(dt)
        src = src.reshape(-1)
        want = _search(_RefSgr(refc, hbd), src, 0, ss, dat, 4 * ds + 4, ds, w, h, bd, pu)
        got = _search(_DevSgr(b200, hbd), src, 0, ss, dat, 4 * ds + 4, ds, w, h, bd, pu)
        assert got == want, (mode, pu, w, h, [(a, b) for a, b in zip(got, want) if a != b][:3])


# ---- concurrency ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_t1_calls_from_eight_threads(b200, refc):
    """the T1 filter, subspace and projection error from 8 host threads at once (ctypes releases the GIL), launches
    below and above 48 KB of shared memory mixed; units beyond the reference's buffer against the tiled oracle"""
    r = rng(3700)
    jobs = []
    sizes = [(64, 64), (72, 72), (80, 80), (100, 90), (128, 128), (33, 17), (200, 30), (75, 75)]
    for k in range(48):
        w, h = sizes[k % len(sizes)]
        bd, dt = list(MODES.values())[k % 4]
        idx = (k * 5) % 16
        plane, off, stride = _tile(r, ("random", "checker", "gradient")[k % 3], w, h, bd, dt, k % 3)
        fs = w + 2
        want = [_fbuf(w, h, fs, 1) for _ in range(2)]
        rh.ref_sgr_tiled(refc, plane, off, w, h, stride, idx, bd, want[0], want[1], 1, fs)
        src = r.integers(0, 1 << bd, h * w).astype(dt)
        prm = np.array(rh.SGR_PARAMS[idx], np.int32)
        xq = np.array(rh.decode_xq(XQD_CORNERS[k % 4], prm), np.int32)
        f0 = np.where(want[0] == SENT, 0, want[0]).astype(np.int32); f1 = np.where(want[1] == SENT, 0, want[1]).astype(np.int32)
        xq_w = np.zeros(2, np.int32)
        refc.svt_get_proj_subspace_c.restype = None
        refc.svt_get_proj_subspace_c(rh.bptr(src), w, h, w, rh.bptr(plane, off), stride, int(dt == np.uint16), rh.P(f0, 1), fs, rh.P(f1, 1), fs,
                                     rh.P(xq_w), rh.P(prm))
        ppe = refc.svt_av1_highbd_pixel_proj_error_c if dt == np.uint16 else refc.svt_av1_lowbd_pixel_proj_error_c
        ppe.restype = ct.c_int64
        e_w = ppe(rh.bptr(src), w, h, w, rh.bptr(plane, off), stride, rh.P(f0, 1), fs, rh.P(f1, 1), fs, rh.P(xq), rh.P(prm))
        jobs.append((w, h, bd, dt, idx, plane, off, stride, fs, want, src, prm, xq, f0, f1, xq_w, e_w))

    def run(job):
        w, h, bd, dt, idx, plane, off, stride, fs, want, src, prm, xq, f0, f1, xq_w, e_w = job
        hbd = int(dt == np.uint16)
        lib = b200.lib
        for _ in range(3):
            got = [_fbuf(w, h, fs, 1) for _ in range(2)]
            lib.svt_b200_av1_selfguided_restoration(rh.P(plane, off), w, h, stride, rh.P(got[0], 1), rh.P(got[1], 1), fs, idx, bd, hbd)
            xq_g = np.zeros(2, np.int32)
            lib.svt_b200_get_proj_subspace(rh.P(src), w, h, w, rh.P(plane, off), stride, hbd, rh.P(f0, 1), fs, rh.P(f1, 1), fs, rh.P(xq_g), rh.P(prm))
            fn = lib.svt_b200_av1_highbd_pixel_proj_error if hbd else lib.svt_b200_av1_lowbd_pixel_proj_error
            e_g = fn(rh.P(src), w, h, w, rh.P(plane, off), stride, rh.P(f0, 1), fs, rh.P(f1, 1), fs, rh.P(xq), rh.P(prm))
            if not (np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(xq_g, xq_w) and e_g == e_w):
                return (w, h, bd, idx)
        return None

    with ThreadPoolExecutor(8) as ex:
        bad = [x for x in ex.map(run, jobs) if x is not None]
    assert not bad, bad


# ---- svt_b200_sgr_units_dev -------------------------------------------------------------------------------------------
def _batch_arrays(b200, refc, r, name, bd):
    seed, n, max_wh, special = BATCHES[name]
    lst, pw, ph = sgr_batch(seed, n, max_wh, special)
    dt = np.uint8 if bd == 8 else np.uint16
    kinds = ("random", "checker", "nearflat", "gradient", "max")
    plane = np.concatenate([_content(r, kinds[i], ph // 5 + 1, pw, bd) for i in range(5)])[:ph].astype(dt).reshape(-1)
    units = np.zeros(len(lst), dtype=b200.SGR_UNIT_DTYPE)
    o0, o1 = 5, 3
    sizes1 = [h * fs + 11 for (_, _, w, h, _, fs) in lst]
    offs1 = np.cumsum([3] + sizes1[::-1])[:-1][::-1]  # flt1 in the reverse order of flt0, other gaps
    for k, (x, y, w, h, idx, fs) in enumerate(lst):
        units[k] = (y * pw + x, o0, int(offs1[k]), pw, fs, w, h, idx, 0)
        o0 += h * fs + 7
    n0, n1 = o0 + 5, int(offs1[0]) + sizes1[0] + 3
    want0, want1 = np.full(n0, SENT, np.int32), np.full(n1, SENT, np.int32)
    # the reference writes both outputs at one pitch and offset: the two passes separately, into each expected buffer
    scratch0, scratch1 = np.full(n1 + n0, SENT, np.int32), np.full(n0 + n1, SENT, np.int32)
    for (x, y, w, h, idx, fs), u in zip(lst, units):
        prm = rh.SGR_PARAMS[idx]
        rh.ref_sgr_tiled(refc, plane, y * pw + x, w, h, pw, idx, bd, want0, scratch1, int(u["flt0_off"]), fs)
        rh.ref_sgr_tiled(refc, plane, y * pw + x, w, h, pw, idx, bd, scratch0, want1, int(u["flt1_off"]), fs)
        assert prm[0] or (want0[int(u["flt0_off"])] == SENT)
    return plane, units, want0, want1, max_wh



def _launch_batch(b200, torch, plane, units, n0, n1, bd, max_wh, stream):
    d_plane = torch.from_numpy(plane.view(np.uint8)).to("cuda")
    d_units = torch.from_numpy(units.view(np.uint8)).to("cuda")
    d_f0 = torch.full((n0,), SENT, dtype=torch.int32, device="cuda")
    d_f1 = torch.full((n1,), SENT, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    rc = b200.lib.svt_b200_sgr_units_dev(d_plane.data_ptr(), d_units.data_ptr(), len(units), d_f0.data_ptr(), d_f1.data_ptr(), bd, max_wh, max_wh,
                                         stream.cuda_stream)
    return rc, (d_plane, d_units, d_f0, d_f1)


@pytest.mark.gpu
@pytest.mark.parametrize("bd", (8, 10, 12))
def test_sgr_units_dev_mixed_batch(b200, refc, bd):
    """one batch of every unit size up to 128 x 128, more units than CTAs, all 16 sets, flt0_off != flt1_off and
    flt_stride > w, against the tiled reference; whole sentinel-filled output buffers compared"""
    import torch
    r = rng(3800 + bd)
    plane, units, want0, want1, max_wh = _batch_arrays(b200, refc, r, "mixed", bd)
    st = torch.cuda.Stream()
    rc, keep = _launch_batch(b200, torch, plane, units, want0.size, want1.size, bd, max_wh, st)
    assert rc == 0
    st.synchronize()
    got0, got1 = keep[2].cpu().numpy(), keep[3].cpu().numpy()
    assert np.array_equal(got0, want0), ("flt0", np.argwhere(got0 != want0)[:4])
    assert np.array_equal(got1, want1), ("flt1", np.argwhere(got1 != want1)[:4])


@pytest.mark.gpu
@pytest.mark.parametrize("bd", (8, 10, 12))
def test_sgr_units_dev_two_streams_at_once(b200, refc, bd):
    """a 128-wide batch and a 32-wide batch launched from two host threads on two streams, three times each"""
    import torch
    r = rng(3900 + bd)
    batches = [_batch_arrays(b200, refc, r, name, bd) for name in ("mixed", "small")]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    barrier = threading.Barrier(2)

    def go(i):
        plane, units, want0, want1, max_wh = batches[i]
        out = []
        for _ in range(3):
            barrier.wait()
            with torch.cuda.stream(streams[i]):
                rc, keep = _launch_batch(b200, torch, plane, units, want0.size, want1.size, bd, max_wh, streams[i])
            streams[i].synchronize()
            out.append((rc, np.array_equal(keep[2].cpu().numpy(), want0), np.array_equal(keep[3].cpu().numpy(), want1)))
        return out

    with ThreadPoolExecutor(2) as ex:
        res = list(ex.map(go, range(2)))
    assert res == [[(0, True, True)] * 3] * 2, res


@pytest.mark.gpu
def test_sgr_units_dev_rejects_bad_arguments(b200):
    """depths other than 8, 10 and 12 and max_w / max_h outside 1 .. 128 return SVT_B200_ERR_BAD_ARG and launch nothing"""
    import torch
    d_plane = torch.zeros(64 * 64, dtype=torch.int16, device="cuda")
    units = np.zeros(1, dtype=b200.SGR_UNIT_DTYPE)
    units[0] = (3 * 64 + 3, 0, 0, 64, 8, 8, 8, 0, 0)
    d_units = torch.from_numpy(units.view(np.uint8)).cuda()
    d_f = torch.full((64,), SENT, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    l0 = b200.launch_count()
    for bd, mw, mh in [(9, 8, 8), (11, 8, 8), (0, 8, 8), (7, 8, 8), (16, 8, 8), (10, 0, 8), (10, 8, 0), (8, -1, 8), (12, 129, 8), (12, 8, 129)]:
        assert b200.lib.svt_b200_sgr_units_dev(d_plane.data_ptr(), d_units.data_ptr(), 1, d_f.data_ptr(), d_f.data_ptr(), bd, mw, mh, s) == BAD_ARG, \
            (bd, mw, mh)
    assert b200.lib.svt_b200_sgr_units_dev(d_plane.data_ptr(), d_units.data_ptr(), -1, d_f.data_ptr(), d_f.data_ptr(), 10, 8, 8, s) == BAD_ARG
    torch.cuda.synchronize()
    assert b200.launch_count() == l0 and (d_f.cpu().numpy() == SENT).all()
    assert b200.lib.svt_b200_sgr_units_dev(d_plane.data_ptr(), d_units.data_ptr(), 1, d_f.data_ptr(), d_f.data_ptr(), 10, 8, 8, s) == 0
    torch.cuda.synchronize()
    assert b200.launch_count() > l0


# ---- the striped filter with self-guided units ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("skew", (0, 1), ids=("aligned", "skewed"))
@pytest.mark.parametrize("case", STRIPED_CASES, ids=lambda c: "%dx%d_b%d_ru%d_frt%d_%s" % (c[:5] + ("mixed" if c[5] else "sgr",)))
def test_lr_frame_sgr_units_match_reference(b200, refc, case, skew):
    """svt_b200_lr_save_boundary_lines_dev, svt_b200_lr_filter_frame_dev (normal and optimized_lr stripes) and
    svt_b200_lr_unit_sse_dev on planes of self-guided (or mixed) units == ref_lr_filter_plane"""
    W, H, bd, us, frt, mix = case
    r = rng(4000 + W + H + bd + us)
    fills = ("random", "max", "zeros", "checker")

    def plane(p, w, h, which):
        buf = _plane(r, w, h, bd, (p + which) % 2 == 0)
        kind = fills[(p + 2 * which + skew) % 4]
        if kind != "random":
            buf[PAD:PAD + h, PAD:PAD + w] = _content(r, kind, h, w, bd)
        return buf
    _run(b200, W, H, bd, us, skew, lambda p, n: striped_units(b200, n, p, 4100 + p, mix), plane, _reference(refc, W, H, bd), frt=frt, sse=True)


@pytest.mark.gpu
@pytest.mark.parametrize("bd", (10, 12))
@pytest.mark.parametrize("fill", ("max", "zeros", "checker"))
def test_lr_frame_sgr_extreme_content(b200, refc, bd, fill):
    """every plane all-max, all-0 or 0/max checkerboard, before and after CDEF: with the xqd corners the projection
    clamps at both ends"""
    W, H, us = 520, 185, 64
    r = rng(4200 + bd)

    def plane(p, w, h, which):
        buf = _plane(r, w, h, bd, False)
        buf[PAD:PAD + h, PAD:PAD + w] = _content(r, fill, h, w, bd)
        return buf
    _run(b200, W, H, bd, us, 0, lambda p, n: striped_units(b200, n, p, 4300 + p, False), plane, _reference(refc, W, H, bd), frt=2, sse=True)
