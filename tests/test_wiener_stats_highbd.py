"""GPU parity of the 10- and 12-bit Wiener statistics batch call (svt_b200_compute_stats_batch_dev), which sums products
by lag (wiener_stats_lag.cuh), item by item against the reference's svt_av1_compute_stats_highbd_c on the C tier.

The lag decomposition splits a region into 8-row bands and 512-column segments, into the 2 * half edge rows / columns
on each side of a core rectangle (the two groups merge and the core is empty when a side is shorter than 2 * half + 1)
and corner products, and it spreads an item's work units over 1 to 64 CTAs depending on the batch size.  The cases
reach each of these on purpose: a mixed batch of 7x7, 5x5 and 3x3 items over planes with random padding, odd strides
and odd offsets, with random, all-0, all-max, 0/max checkerboard, halves and near-max content; a sweep of region sizes
on both sides of every boundary; batches of 1 item, of tens and of more than 8 items per SM; all-max regions whose
full 8 x 512 work units put the uint32 per-lane partials at their bound; a 1920x1080 region; the T1 entry point on
strided planes; and two streams at once, and a captured graph replayed after its stream's scratch has grown.
test_cases_reach_every_boundary checks from the item lists alone (no GPU) that the cases do reach all of this."""
from functools import lru_cache

import numpy as np
import pytest

import rest_helpers as rh
from helpers import rng
from oracle.support import layout
from oracle_libs import refc  # noqa: F401  (a fixture: overrides conftest.py's refc in this module)

gpu = pytest.mark.gpu

BAND_ROWS, SEG_COLS = 8, 512  # kLagBandRows, kLagSegW: the rows and columns of one work unit of the lag kernels
H100_SMS = 132
SENTINEL = -0x5A5A5A5A5A5A5A5B  # d_M / d_H entries beyond an item's win^2 / win^4 must keep it
BAD_ARG = -4  # SVT_B200_ERR_BAD_ARG


def _content(r, kind, w, h, mx):
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "random":
        return r.integers(0, mx + 1, (h, w)), r.integers(0, mx + 1, (h, w))
    if kind == "zero":
        return np.zeros((h, w), np.int64), np.zeros((h, w), np.int64)
    if kind == "max":
        return np.full((h, w), mx), np.full((h, w), mx)
    if kind == "checker":
        c = ((xx + yy) % 2) * mx
        return c, mx - c
    if kind == "halves":
        return (xx >= w // 2) * mx, (yy >= h // 2) * mx
    if kind == "bright":  # near the largest raw products, not constant
        return r.integers(mx - mx // 16, mx + 1, (h, w)), r.integers(0, mx + 1, (h, w))
    raise ValueError(kind)


class Batch:
    """dgd planes with padding on every side (pad_fill "random": any legal value, "same": the content's own value, so
    that an all-max plane stays all-max through its halo) and unpadded src planes, each plane with its own strides,
    packed into one uint16 dgd and one uint16 src buffer; items = (plane, window, h_start, h_end, v_start, v_end)"""

    def __init__(self, bd):
        self.bd, self.mx = bd, (1 << bd) - 1
        self.dgd, self.src, self.planes, self.regions = [], [], [], []
        self.dgd_len = self.src_len = 0

    def plane(self, r, kind, w, h, dgd_extra, src_extra, pad_fill="random"):
        left, right, top, bottom = (int(v) for v in r.integers(3, 9, 4))  # >= 3: the 7x7 halo of a region on the plane edge
        ds, ss = left + w + right + dgd_extra, w + src_extra
        pd, ps = _content(r, kind, w, h, self.mx)
        if pad_fill == "same":
            d = np.full((top + h + bottom, ds), pd.flat[0])
        else:
            d = r.integers(0, self.mx + 1, (top + h + bottom, ds))
        s = r.integers(0, self.mx + 1, (h, ss))
        d[top:top + h, left:left + w] = pd
        s[:, :w] = ps
        self.planes.append(dict(dgd_off=self.dgd_len + top * ds + left, src_off=self.src_len, ds=ds, ss=ss, w=w, h=h, kind=kind,
                                pad_fill=pad_fill))
        self.dgd.append(d.astype(np.uint16).reshape(-1))
        self.src.append(s.astype(np.uint16).reshape(-1))
        self.dgd_len += d.size
        self.src_len += s.size
        return len(self.planes) - 1

    def region(self, p, win, hs, he, vs, ve):
        q = self.planes[p]
        assert win in (3, 5, 7) and 0 <= hs < he <= q["w"] and 0 <= vs < ve <= q["h"], (p, win, hs, he, vs, ve)
        self.regions.append((p, win, hs, he, vs, ve))

    def place(self, p, win, w, h, where):
        """a w x h region of plane p on a corner, an edge or inside it"""
        q = self.planes[p]
        W, H = q["w"], q["h"]
        x = {"tl": 0, "bl": 0, "tr": W - w, "br": W - w, "t": (W - w) // 3, "b": (W - w) // 2, "l": 0, "r": W - w, "in": (W - w) // 2}[where]
        y = {"tl": 0, "tr": 0, "bl": H - h, "br": H - h, "t": 0, "b": H - h, "l": (H - h) // 2, "r": (H - h) // 3, "in": (H - h) // 3}[where]
        self.region(p, win, x, x + w, y, y + h)

    def finish(self):
        self.dgd_buf, self.src_buf = np.concatenate(self.dgd), np.concatenate(self.src)
        assert int(self.dgd_buf.max()) <= self.mx and int(self.src_buf.max()) <= self.mx  # the partial bounds assume legal pixels
        self.items = np.zeros(len(self.regions), dtype=layout.STATS_ITEM_DTYPE)
        for i, (p, win, hs, he, vs, ve) in enumerate(self.regions):
            q = self.planes[p]
            self.items[i] = (q["dgd_off"], q["src_off"], q["ds"], q["ss"], hs, he, vs, ve, win, 0)
        return self


def _mixed(bd):
    """(a): every content kind, all three windows in one batch, regions on every plane edge and inside"""
    r = rng(2100 + bd)
    b = Batch(bd)
    rnd = b.plane(r, "random", 300, 200, 5, 7)
    zero = b.plane(r, "zero", 96, 80, 16, 0)
    mx = b.plane(r, "max", 100, 70, 1, 3)
    mxs = b.plane(r, "max", 90, 41, 2, 1, pad_fill="same")
    chk = b.plane(r, "checker", 131, 90, 3, 17)
    hv = b.plane(r, "halves", 200, 121, 0, 2)
    brt = b.plane(r, "bright", 257, 150, 9, 5)
    for reg in [(rnd, 7, 10, 11, 20, 21), (rnd, 5, 0, 1, 0, 1), (rnd, 3, 299, 300, 199, 200), (rnd, 7, 5, 6, 3, 200),
                (rnd, 5, 0, 300, 17, 18), (rnd, 3, 40, 41, 0, 77), (rnd, 7, 3, 40, 5, 28), (rnd, 5, 101, 166, 7, 40),
                (rnd, 3, 13, 142, 60, 157), (rnd, 7, 0, 300, 0, 200), (rnd, 5, 233, 300, 111, 200), (rnd, 7, 0, 65, 167, 200),
                (zero, 7, 0, 96, 0, 80), (zero, 3, 7, 70, 9, 42),
                (mx, 7, 0, 100, 0, 70), (mx, 5, 31, 99, 1, 69), (mx, 3, 0, 1, 0, 70),
                (mxs, 7, 0, 90, 0, 41), (mxs, 5, 0, 90, 0, 41), (mxs, 3, 0, 90, 0, 41),
                (chk, 7, 0, 131, 0, 90), (chk, 5, 1, 128, 3, 89), (chk, 3, 64, 131, 32, 90),
                (hv, 7, 0, 200, 0, 121), (hv, 5, 50, 151, 30, 91), (hv, 3, 99, 101, 0, 121),
                (brt, 7, 0, 257, 0, 150), (brt, 5, 17, 257, 9, 150), (brt, 3, 0, 129, 0, 64)]:
        b.region(*reg)
    return b.finish()


def _sizes(half):
    """(b): region sizes on both sides of every boundary of the lag decomposition for one window"""
    small_w = sorted({1, 2, 2 * half - 1, 2 * half, 2 * half + 1, 2 * half + 2, 13} - {0})
    small_h = sorted({1, 2, 2 * half - 1, 2 * half, 2 * half + 1, 7, 8, 9, 15, 16, 17, 8 + 2 * half} - {0})
    pairs = [(w, h) for w in small_w for h in small_h]
    # wide regions: one, two and three segments, one with a last segment without core columns; paired with heights
    # that give an empty vertical core, one short band, full bands and a short last band
    pairs += [(511, 9), (512, 16), (513, 2 * half + 1), (512 + 2 * half, 8 + 2 * half), (512 + 2 * half + 1, 2),
              (1024 + 2 * half, 17), (1030, 7), (1031, 2 * half), (1029, 1), (383, 391)]
    return pairs


def _geometry(bd):
    r = rng(2200 + bd)
    b = Batch(bd)
    p = b.plane(r, "random", 1040, 400, 7, 11)
    spots = ("tl", "tr", "bl", "br", "t", "b", "l", "r", "in")
    k = 0
    for win in (7, 5, 3):
        for w, h in _sizes(win // 2):
            b.place(p, win, w, h, spots[k % len(spots)])
            k += 1
    return b.finish()


def _worst(bd):
    """(d): all-max, 0/max checkerboard and halves regions with full 8 x 512 work units, and a 1920x1080 region"""
    r = rng(2300 + bd)
    b = Batch(bd)
    mx = b.plane(r, "max", 1040, 70, 3, 1, pad_fill="same")
    chk = b.plane(r, "checker", 1036, 66, 0, 5)
    hv = b.plane(r, "halves", 1030, 64, 1, 0)
    big = b.plane(r, "random", 1920, 1080, 13, 0)
    b.region(mx, 7, 3, 1033, 2, 66)
    b.region(mx, 5, 0, 1040, 0, 70)
    b.region(chk, 7, 3, 1033, 1, 65)
    b.region(hv, 7, 0, 1030, 0, 64)
    b.region(big, 7, 0, 1920, 0, 1080)
    return b.finish()


def _single(bd):
    """(c) n = 1: every CTA but a few of the 64 of the item is idle"""
    r = rng(2400 + bd)
    b = Batch(bd)
    p = b.plane(r, "random", 90, 61, 1, 0)
    b.region(p, 5, 2, 89, 0, 61)
    return b.finish()


def _many(bd, n=None):
    """(c) n > 8 items per SM: one CTA per item, which walks every work unit of its item"""
    n = n or 8 * H100_SMS + 136
    r = rng(2500 + bd)
    b = Batch(bd)
    p = b.plane(r, "random", 240, 180, 3, 2)
    q = b.plane(r, "bright", 77, 50, 0, 1)
    for i in range(n):
        win = (7, 5, 3)[i % 3]
        pl = q if i % 5 == 4 else p
        W, H = b.planes[pl]["w"], b.planes[pl]["h"]
        w, h = int(r.integers(1, 41)), int(r.integers(1, 34))
        x, y = int(r.integers(0, W - w + 1)), int(r.integers(0, H - h + 1))
        if i % 7 == 0:
            x = 0 if i % 2 else W - w
        if i % 11 == 0:
            y = 0 if i % 2 else H - h
        b.region(pl, win, x, x + w, y, y + h)
    return b.finish()


@lru_cache(maxsize=None)
def batch(name, bd):
    return {"mixed": _mixed, "geometry": _geometry, "worst": _worst, "single": _single, "many": _many}[name](bd)


BATCHES = ("mixed", "geometry", "worst", "single", "many")


# ---- what the cases reach: from the item lists alone ---------------------------------------------------------------------
def _work_units(win, w, h):
    """the lag kernels' decomposition of a w x h region: per segment its core columns, per band its core rows"""
    half = win // 2
    nsegs, nbands = -(-w // SEG_COLS), -(-h // BAND_ROWS)
    core_cols = [max(min(w - 2 * half - s * SEG_COLS, SEG_COLS), 0) for s in range(nsegs)]
    core_rows = [max(0, min((b + 1) * BAND_ROWS, h, h - half) - max(b * BAND_ROWS, half)) for b in range(nbands)]
    return core_cols, core_rows


@pytest.mark.parametrize("bd", [10, 12])
def test_cases_reach_every_boundary(bd):
    """CPU: the batches put every window on every boundary of the lag decomposition, every batch size on its CTA spread"""
    seen = {}
    for name in BATCHES:
        b = batch(name, bd)
        edges = set()
        for p, win, hs, he, vs, ve in b.regions:
            q = b.planes[p]
            w, h, half = he - hs, ve - vs, win // 2
            cols, rows = _work_units(win, w, h)
            s = seen.setdefault(win, set())
            s.add("segments=%d" % min(len(cols), 3))
            if len(cols) > 1 and cols[-1] == 0:
                s.add("last segment without core")
            if w <= 2 * half:
                s.add("no core columns")
            if h <= 2 * half:
                s.add("no core rows")
            if len(rows) > 1 and h % BAND_ROWS:
                s.add("short last band")
            if w % 2:
                s.add("odd width")
            if hs and vs:
                s.add("inner origin")
            if w == 383 and h == 391:
                s.add("largest unit")
            if q["kind"] == "max" and q["pad_fill"] == "same" and win == 7 and SEG_COLS in cols and BAND_ROWS in rows:
                s.add("full all-max work unit")
            edges |= {e for e, hit in (("left", hs == 0), ("right", he == q["w"]), ("top", vs == 0), ("bottom", ve == q["h"])) if hit}
            if q["kind"] == "random" and w * h >= 1920 * 1080:
                s.add("1920x1080")
        if name in ("mixed", "geometry", "many"):
            assert edges == {"left", "right", "top", "bottom"}, (name, edges)
    want = {"segments=1", "segments=2", "segments=3", "last segment without core", "no core columns", "no core rows", "short last band",
            "odd width", "inner origin", "largest unit"}
    for win in (7, 5, 3):
        assert want <= seen[win], (win, want - seen[win])
    assert "full all-max work unit" in seen[7] and "1920x1080" in seen[7]
    for name in ("mixed", "geometry", "many"):
        assert set(batch(name, bd).items["wiener_win"]) == {3, 5, 7}, name
    mixed = batch("mixed", bd)
    assert set(mixed.items["dgd_off"] % 2) == {0, 1} and set(mixed.items["src_off"] % 2) == {0, 1}
    assert len(set(mixed.items["dgd_stride"])) == len(mixed.planes) and any(mixed.items["dgd_stride"] % 2) and any(mixed.items["src_stride"] % 2)
    n = {name: len(batch(name, bd).items) for name in BATCHES}
    cpi = {k: min(max(8 * H100_SMS // v, 1), 64) for k, v in n.items()}  # CTAs per item on an H100
    assert cpi["single"] == 64 and 2 <= cpi["mixed"] <= 63 and 2 <= cpi["geometry"] <= 63 and n["many"] > 8 * H100_SMS
    assert any(len(_work_units(int(it["wiener_win"]), int(it["h_end"] - it["h_start"]), int(it["v_end"] - it["v_start"]))[1]) > 1
               for it in batch("many", bd).items)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref(refc):
    refc.ref_set_tier(0)
    refc.ref_set_threads(0)
    refc.ref_compute_stats_batch_bd.restype = None
    return refc


@pytest.fixture(scope="module")
def expect(ref):
    """(batch name, bd) -> the reference's M [n][49] and H [n][2401] (entries beyond win^2 / win^4: 0)"""
    cache = {}

    def get(b):
        if b not in cache:
            n = len(b.items)
            M, H = np.zeros((n, 49), np.int64), np.zeros((n, 2401), np.int64)
            ref.ref_compute_stats_batch_bd(rh.P(b.dgd_buf), rh.P(b.src_buf), rh.P(b.items), n, rh.P(M), rh.P(H), b.bd)
            cache[b] = (M, H)
        return cache[b]
    return get


class _OnDevice:
    """a batch's buffers and sentinel-filled outputs on the device"""

    def __init__(self, torch, b):
        self.b = b
        self.dgd = torch.from_numpy(b.dgd_buf.view(np.int16)).cuda()
        self.src = torch.from_numpy(b.src_buf.view(np.int16)).cuda()
        self.items = torch.from_numpy(b.items.view(np.uint8).copy()).cuda()
        self.M = torch.full((len(b.items), 49), SENTINEL, dtype=torch.int64, device="cuda")
        self.H = torch.full((len(b.items), 2401), SENTINEL, dtype=torch.int64, device="cuda")

    def launch(self, b200, stream_handle):
        return b200.lib.svt_b200_compute_stats_batch_dev(self.dgd.data_ptr(), self.src.data_ptr(), self.items.data_ptr(), len(self.b.items),
                                                         self.b.bd, self.M.data_ptr(), self.H.data_ptr(), stream_handle)

    def result(self):
        return self.M.cpu().numpy(), self.H.cpu().numpy()


def _check(b, got, want, what, rest=SENTINEL):
    (M, H), (wM, wH) = got, want
    for i, (p, win, hs, he, vs, ve) in enumerate(b.regions):
        w2 = win * win
        tag = (what, b.bd, i, win, hs, he, vs, ve, b.planes[p]["kind"])
        assert np.array_equal(M[i, :w2], wM[i, :w2]), tag + ("M", np.argwhere(M[i, :w2] != wM[i, :w2])[:4])
        assert np.array_equal(H[i, :w2 * w2], wH[i, :w2 * w2]), tag + ("H", np.argwhere(H[i, :w2 * w2] != wH[i, :w2 * w2])[:4])
        assert (M[i, w2:] == rest).all() and (H[i, w2 * w2:] == rest).all(), tag + ("entries beyond the window written",)


@gpu
@pytest.mark.parametrize("name", ["mixed", "geometry", "worst", "single", "many"])
@pytest.mark.parametrize("bd", [10, 12])
def test_compute_stats_batch_highbd(b200, expect, name, bd):
    """(a) - (d): each batch in one call on the default stream, against the reference item by item"""
    import torch
    b = batch(name, bd)
    if name == "many" and len(b.items) <= 8 * torch.cuda.get_device_properties(0).multi_processor_count:
        b = _many(bd, 8 * torch.cuda.get_device_properties(0).multi_processor_count + 136)
    d = _OnDevice(torch, b)
    assert d.launch(b200, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    want = expect(b)
    _check(b, d.result(), want, name)
    if name == "worst":  # all-max through the halo: every sample equals the average
        for i, (p, win, *_) in enumerate(b.regions):
            if b.planes[p]["pad_fill"] == "same":
                assert not want[0][i].any() and not want[1][i].any(), i


@gpu
@pytest.mark.parametrize("bd", [10, 12])
def test_compute_stats_t1_on_strided_planes(b200, ref, bd):
    """(e) the T1 entry point on regions up to 383 x 320 inside wider planes, dgd and src with their own odd strides"""
    r = rng(2600 + bd)
    mx = (1 << bd) - 1
    W, Hh, ds, ss = 420, 360, 451, 433
    for kind in ("random", "checker"):
        dgd = r.integers(0, mx + 1, (Hh, ds))
        src = r.integers(0, mx + 1, (Hh, ss))
        if kind == "checker":
            yy, xx = np.mgrid[0:Hh, 0:W]
            dgd[:, :W] = ((xx + yy) % 2) * mx
            src[:, :W] = mx - dgd[:, :W]
        dgd, src = dgd.astype(np.uint16).reshape(-1), src.astype(np.uint16).reshape(-1)
        for win, hs, he, vs, ve in [(7, 3, 386, 3, 323), (5, 30, 413, 37, 357), (3, 1, 384, 1, 321), (7, 200, 417, 5, 200), (5, 2, 3, 2, 300)]:
            want_M, want_H = rh.ref_stats(ref, win, dgd, src, hs, he, vs, ve, ds, ss, bd)
            M, H = np.full(49, SENTINEL, np.int64), np.full(2401, SENTINEL, np.int64)
            b200.lib.svt_b200_av1_compute_stats_highbd(win, rh.P(dgd), rh.P(src), hs, he, vs, ve, ds, ss, rh.P(M), rh.P(H), bd)
            assert np.array_equal(M[:win * win], want_M), (bd, kind, win, hs, he, vs, ve)
            assert np.array_equal(H[:win ** 4], want_H), (bd, kind, win, hs, he, vs, ve)


@gpu
def test_compute_stats_two_streams_at_once(b200, expect):
    """(f) two different batches on two streams, launched back to back: each equals its result when run alone"""
    import torch
    runs = [(_OnDevice(torch, batch("mixed", 10)), torch.cuda.Stream()), (_OnDevice(torch, batch("geometry", 12)), torch.cuda.Stream())]
    alone = []
    for d, st in runs:  # one at a time; this also sizes each stream's scratch before the concurrent launches
        assert d.launch(b200, st.cuda_stream) == 0
        torch.cuda.synchronize()
        alone.append(d.result())
        _check(d.b, alone[-1], expect(d.b), "alone")
    for rep in range(2):
        for d, _ in runs:
            d.M.fill_(SENTINEL)
            d.H.fill_(SENTINEL)
        torch.cuda.synchronize()
        for d, st in runs:
            assert d.launch(b200, st.cuda_stream) == 0
        torch.cuda.synchronize()
        for (d, _), a in zip(runs, alone):
            M, H = d.result()
            assert np.array_equal(M, a[0]) and np.array_equal(H, a[1]), (rep, d.b.bd)


@gpu
def test_compute_stats_graph_replays_after_scratch_grows(b200, expect):
    """(f) a graph captured on a warmed-up stream still reads and writes the scratch it was captured with after a larger
    eager batch on the same stream has replaced that scratch"""
    import torch
    st = torch.cuda.Stream()
    a, big = _OnDevice(torch, batch("mixed", 10)), _OnDevice(torch, batch("many", 10))
    assert len(big.b.items) > 2 * len(a.b.items) + 400  # beyond what any stream has been grown to
    assert a.launch(b200, st.cuda_stream) == 0  # warm-up with the batch to be captured: no allocation inside the capture
    torch.cuda.synchronize()
    _check(a.b, a.result(), expect(a.b), "warm-up")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        assert a.launch(b200, st.cuda_stream) == 0
    a.M.zero_()
    a.H.zero_()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        assert big.launch(b200, st.cuda_stream) == 0
    torch.cuda.synchronize()
    _check(big.b, big.result(), expect(big.b), "larger eager batch")
    with torch.cuda.stream(st):
        g.replay()
    torch.cuda.synchronize()
    _check(a.b, a.result(), expect(a.b), "graph replay", rest=0)


@gpu
def test_compute_stats_rejects_other_bit_depths(b200):
    """only 8, 10 and 12 bit are accepted; any other depth returns SVT_B200_ERR_BAD_ARG before anything is launched"""
    import torch
    b = batch("single", 10)
    d = _OnDevice(torch, b)
    s = torch.cuda.current_stream().cuda_stream
    for bd in (0, 1, 7, 9, 11, 13, 16, -10):
        l0 = b200.launch_count()
        rc = b200.lib.svt_b200_compute_stats_batch_dev(d.dgd.data_ptr(), d.src.data_ptr(), d.items.data_ptr(), 1, bd, d.M.data_ptr(),
                                                       d.H.data_ptr(), s)
        assert rc == BAD_ARG and b200.launch_count() == l0, bd
    for bd in (8, 10, 12):
        assert b200.lib.svt_b200_compute_stats_batch_dev(None, None, None, 0, bd, None, None, s) == 0
    torch.cuda.synchronize()
    assert (d.M.cpu().numpy() == SENTINEL).all() and (d.H.cpu().numpy() == SENTINEL).all()
