"""GPU parity of the restoration stage where the other restoration tests do not go: the plain Wiener unit batch
(svt_b200_wiener_units_dev) at 8, 10 and 12 bit against the reference's svt_av1_wiener_convolve_add_src_c /
svt_av1_highbd_wiener_convolve_add_src_c (oracle/ref_driver.c ref_wiener_units_bd, C tier), unit sizes on both the
four-pixel and the scalar path, destinations aligned and not aligned to four pixels, legal, extreme and (8-bit) wider
than a byte taps, more units than the grid has CTAs; the striped filter, its boundary lines and the unit SSE at 12 bit,
the only depth with its own Wiener rounding (round0 = 5, round1 = 9); and two 10-bit frames in flight on two streams."""

import numpy as np
import pytest

import rest_helpers as rh
import test_restoration_frame as trf
from helpers import rng
from oracle.support import layout
from test_restoration_frame import PAD, _plane, _units
from test_restoration_paths import LEGAL_HI, LEGAL_LO, _reference, _run, _taps, _wiener_units

pytestmark = pytest.mark.gpu

BAD_ARG = -4  # SVT_B200_ERR_BAD_ARG
UNIT_W = (1, 2, 3, 4, 5, 8, 31, 32, 33, 60, 63, 64)  # multiples of 4 take the four-pixel path, the others the scalar one
UNIT_H = (1, 2, 3, 7, 8, 33, 63, 64)                  # odd: the last row pair of the vertical pass has one row
EXTREME_TAPS = [_taps(*LEGAL_LO), _taps(*LEGAL_HI), _taps(LEGAL_HI[0], LEGAL_LO[1], LEGAL_HI[2]), _taps(LEGAL_LO[0], LEGAL_HI[1], LEGAL_LO[2])]
WIDE_TAPS = [_taps(-40, -60, -50, centre=300), _taps(0, 0, 100, centre=-200)]  # beyond a signed byte: not the dp4a path


@pytest.fixture(scope="module")
def cref(refc):
    refc.ref_set_tier(0)
    refc.ref_wiener_units_bd.restype = None
    return refc


def _wiener_case(r, bd, n_min):
    """a source plane with random, all-max, all-0 and 0/max checkerboard areas; units of every (w, h) at random places in
    it, each with its own destination rectangle (origin and stride aligned to four pixels or not) inside one buffer"""
    mx = (1 << bd) - 1
    SW, SH = 700, 400
    src = r.integers(0, mx + 1, (SH, SW))
    src[:, 100:200] = mx
    src[:, 200:300] = 0
    yy, xx = np.mgrid[0:SH, 300:400]
    src[:, 300:400] = ((xx + yy) % 2) * mx
    sets = [EXTREME_TAPS] + ([WIDE_TAPS] if bd == 8 else [])
    shapes = [(w, h) for w in UNIT_W for h in UNIT_H]
    n = max(n_min, 6 * len(shapes))
    units = np.zeros(n, dtype=layout.WIENER_UNIT_DTYPE)
    dst_len = 0
    for k in range(n):
        w, h = shapes[k % len(shapes)]
        v = k // len(shapes)
        x, y = int(r.integers(3, SW - w - 4)), int(r.integers(3, SH - h - 3))
        align = (k + v) % 4  # 0: aligned origin and stride, 1: odd origin, 2: stride of 2 (mod 4), 3: both
        stride = w + (4 - w % 4) % 4 + 4 * int(r.integers(1, 4)) + (2 if align >= 2 else 0)
        off = (dst_len + 3) & ~3
        off += 1 if align in (1, 3) else 0
        dst_len = off + h * stride + 5
        pick = (k + v) % 3
        if pick == 0:
            hf, vf = rh.wiener_taps(r), rh.wiener_taps(r)
        else:
            ts = sets[(pick - 1) % len(sets)]
            hf, vf = ts[k % len(ts)], ts[(k // 2 + 1) % len(ts)]
        units[k] = (y * SW + x, off, SW, stride, w, h, 0, hf, vf)
    return src.astype(np.uint8 if bd == 8 else np.uint16), units, dst_len


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_wiener_units_match_reference(b200, cref, bd):
    """every unit of the batch, and nothing outside the units: the whole destination buffer is compared"""
    import torch
    r = rng(2700 + bd)
    n_min = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 17  # more units than CTAs: the grid loops
    src, units, dst_len = _wiener_case(r, bd, n_min)
    dt = src.dtype
    init = r.integers(0, 1 << bd, dst_len).astype(dt)
    want = init.copy()
    cref.ref_wiener_units_bd(rh.P(src), rh.P(want), rh.P(units), len(units), bd)
    T = lambda a: torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()  # noqa: E731
    d_src, d_dst, d_units = T(src.reshape(-1)), T(init.copy()), torch.from_numpy(units.view(np.uint8).copy()).cuda()
    assert d_dst.data_ptr() % 16 == 0
    rc = b200.lib.svt_b200_wiener_units_dev(d_src.data_ptr(), d_dst.data_ptr(), d_units.data_ptr(), len(units), bd,
                                            torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    got = d_dst.cpu().numpy().view(dt)
    if not np.array_equal(got, want):
        for k, u in enumerate(units):
            o, s, w, h = int(u["dst_off"]), int(u["dst_stride"]), int(u["w"]), int(u["h"])
            g = np.lib.stride_tricks.as_strided(got[o:], (h, w), (s * got.itemsize, got.itemsize))
            e = np.lib.stride_tricks.as_strided(want[o:], (h, w), (s * want.itemsize, want.itemsize))
            assert np.array_equal(g, e), (bd, k, w, h, o, s, list(u["hfilter"]), list(u["vfilter"]), np.argwhere(g != e)[:4])
        assert False, ("written outside the units", bd, np.argwhere(got != want)[:8])


def test_wiener_units_rejects_other_bit_depths(b200):
    """only 8, 10 and 12 bit are accepted; any other depth returns SVT_B200_ERR_BAD_ARG before anything is launched"""
    import torch
    units = np.zeros(1, dtype=layout.WIENER_UNIT_DTYPE)
    units[0] = (3 * 16 + 3, 0, 16, 8, 8, 4, 0, _taps(*LEGAL_HI), _taps(*LEGAL_LO))
    d_src = torch.zeros(16 * 16, dtype=torch.int16, device="cuda")
    d_dst = torch.full((64,), 77, dtype=torch.int16, device="cuda")
    d_units = torch.from_numpy(units.view(np.uint8).copy()).cuda()
    s = torch.cuda.current_stream().cuda_stream
    for bd in (0, 1, 7, 9, 11, 13, 16, -8):
        l0 = b200.launch_count()
        assert b200.lib.svt_b200_wiener_units_dev(d_src.data_ptr(), d_dst.data_ptr(), d_units.data_ptr(), 1, bd, s) == BAD_ARG, bd
        assert b200.launch_count() == l0, bd
    for bd in (8, 10, 12):
        assert b200.lib.svt_b200_wiener_units_dev(None, None, None, 0, bd, s) == 0
    torch.cuda.synchronize()
    assert (d_dst.cpu().numpy() == 77).all()


# ---- the striped filter at 12 bit ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("skew", (0, 1), ids=("aligned", "skewed"))
@pytest.mark.parametrize("us", (64, 256))
def test_lr_frame_12bit_word_and_pixel_moves_match_reference(b200, cref, us, skew):
    """Wiener, self-guided and none units over aligned and skewed planes: both boundary passes, both optimized_lr modes"""
    W, H, bd = 1000, 300, 12
    r = rng(2800 + us + skew)
    _run(b200, W, H, bd, us, skew, lambda p, n: _units(r, n, b200), lambda p, w, h, which: _plane(r, w, h, bd, (p + which) % 2 == 0),
         _reference(cref, W, H, bd))


@pytest.mark.parametrize("fill", ("zeros", "max", "checker"))
def test_lr_frame_12bit_extreme_legal_taps_match_reference(b200, cref, fill):
    """the extreme legal taps on all-0, all-4095 and 0/4095 checkerboard pictures: the 12-bit intermediate clamp"""
    W, H, bd, us = 328, 200, 12, 64
    r = rng(2900)
    chroma = [_taps(0, t[1], t[2]) for t in EXTREME_TAPS]  # 5-tap window

    def plane(p, w, h, which):
        buf = _plane(r, w, h, bd, False)
        yy, xx = np.mgrid[0:h, 0:w]
        buf[PAD:PAD + h, PAD:PAD + w] = {"zeros": 0, "max": 4095, "checker": ((xx + yy + which) % 2) * 4095}[fill]
        return buf
    _run(b200, W, H, bd, us, 0, lambda p, n: _wiener_units(n, b200, chroma if p else EXTREME_TAPS), plane, _reference(cref, W, H, bd))


@pytest.mark.parametrize("case", [(328, 200, 12, 64), (256, 121, 12, 128), (200, 57, 12, 64)], ids=lambda c: "%dx%d_b%d_ru%d" % c)
def test_lr_frame_12bit_matches_reference_with_unit_sse(b200, cref, case):
    """the filter, both boundary passes and svt_b200_lr_unit_sse_dev, as test_lr_frame_matches_reference checks them at
    8 and 10 bit"""
    trf.test_lr_frame_matches_reference(b200, cref, case)


# ---- two 10-bit frames in flight --------------------------------------------------------------------------------------------
def test_two_10bit_frames_in_flight_on_two_streams(b200):
    """two independent 10-bit frames on two streams, eager and as graph replays: the statistics' per-stream scratch (and
    every other per-stream buffer) keeps them apart, so the results equal the one-at-a-time results"""
    import torch
    from svt_av1_psy_b200.pipeline import FramePipeline
    from svt_av1_psy_b200.workload import FrameWorkload
    fps = [FramePipeline(FrameWorkload(384, 256, seed=1234 + 7 * k, bit_depth=10, preset=6), torch) for k in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    names = ("qcoeff", "eobs", "recon", "cdef_mse", "cdef_out", "M", "Hm", "final")
    me_names = ("total_me_candidate_index", "me_candidate_array", "me_mv_array", "distortion", "best_sad")
    want = []
    for fp, st in zip(fps, streams):  # one at a time (also warms up every lazily allocated scratch)
        with torch.cuda.stream(st):
            fp.load_inputs()
            fp.step()
        torch.cuda.synchronize()
        want.append([getattr(fp, n).clone() for n in names] + [fp.me[n].clone() for n in me_names])
    assert not torch.equal(want[0][5], want[1][5])  # the two frames' statistics differ: a swap would show
    graphs = []
    for fp, st in zip(fps, streams):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            fp.step()
        graphs.append(g)
    for rep in range(6):
        for fp in fps:
            for n in ("qcoeff", "eobs", "cdef_mse", "M", "Hm", "final"):
                getattr(fp, n).zero_()
            fp.me["me_mv_array"].zero_()
            fp.me["best_sad"].zero_()
        torch.cuda.synchronize()
        for g, st in zip(graphs, streams):
            with torch.cuda.stream(st):
                g.replay() if rep % 2 == 0 else None
        if rep % 2:  # eager launches, interleaved call by call
            for fp, st in zip(fps, streams):
                with torch.cuda.stream(st):
                    fp.step()
        torch.cuda.synchronize()
        for fp, w in zip(fps, want):
            for n, t in zip(names + me_names, w):
                assert torch.equal(getattr(fp, n) if n in names else fp.me[n], t), (rep, n)
