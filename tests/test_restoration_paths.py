"""GPU parity of the striped restoration drivers on the paths test_restoration_frame.py does not separate: planes whose
rows start on 16-byte boundaries with a stride larger than the width (tiles and boundary lines move as aligned words)
against the same picture through a view that starts one pixel later (everything moves pixel by pixel); widths that leave
a partial last column run, a chroma unit size of 32 (two 32-wide chunks of a 64-wide run would lie in different units);
Wiener taps at both ends of the legal range on all-0, all-maximum and random pictures (the packed signed-byte products and
both clamps); and taps beyond a signed byte, which the ABI accepts (the unpacked multiply path).  The oracle is the
reference's own filter (oracle/ref_driver.c ref_lr_filter_plane), except for the taps the reference's SIMD filter cannot
hold, which are checked against the add-src convolution written out in numpy."""
import ctypes as ct

import numpy as np
import pytest

from helpers import rng
from test_restoration_frame import PAD, _plane, _units

pytestmark = pytest.mark.gpu

LEGAL_LO, LEGAL_HI = (-5, -23, -17), (10, 8, 46)  # taps 0..2; the centre tap -2 * (t0 + t1 + t2) is then 90 and -128


def _taps(t0, t1, t2, centre=None):
    return np.array([t0, t1, t2, -2 * (t0 + t1 + t2) if centre is None else centre, t2, t1, t0, 0], np.int16)


def _wiener_units(n, b200, taps):
    u = np.zeros(n, dtype=b200.LR_UNIT_DTYPE)
    for k in range(n):
        u["restoration_type"][k] = 1
        u["hfilter"][k] = taps[k % len(taps)]
        u["vfilter"][k] = taps[(k + 1) % len(taps)]
    return u


def _device_view(torch, a, stride, skew):
    """a 2-D array on the device inside a flat buffer: rows `stride` elements apart, the first `skew` elements after a
    16-byte boundary"""
    h, w = a.shape
    flat = torch.zeros(h * stride + 16 + skew, dtype=torch.uint8 if a.dtype == np.uint8 else torch.int16, device="cuda")
    lead = (-flat.data_ptr() // flat.element_size()) % (16 // flat.element_size()) + skew
    v = flat[lead:lead + h * stride].view(h, stride)[:, :w]
    v.copy_(torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a))
    return flat, v


def _run(b200, W, H, bd, us, skew, make_units, make_plane, want_fn, frt=0, sse=False):
    """both boundary passes and the filter (normal and optimized_lr stripes) over three 4:2:0 planes; want_fn gives the
    expected boundary lines (or None) and the expected restored plane per mode.  frt is every plane's
    frame_restoration_type; with sse, the unit SSE of each restored plane against its CDEF input is checked as well"""
    import torch
    planes = (b200.LrPlane * 3)()
    keep, checks = [], []
    tdt = torch.uint8 if bd == 8 else torch.int16
    for p in range(3):
        ss = 1 if p else 0
        w, h, usp = (W + ss) >> ss, (H + ss) >> ss, us >> ss
        deb, cdf = make_plane(p, w, h, 0), make_plane(p, w, h, 1)
        nst = b200.lib.svt_b200_lr_num_stripes(h, ss)
        bstride = b200.lib.svt_b200_lr_boundary_stride(w)
        hu, vu = b200.lib.svt_b200_lr_units_per_dim(w, usp), b200.lib.svt_b200_lr_units_per_dim(h, usp)
        units = make_units(p, hu * vu)
        stride = ((w + 15) & ~15) + 16
        k_deb, d_deb = _device_view(torch, deb[PAD:PAD + h, PAD:PAD + w], stride, skew)
        k_cdf, d_cdf = _device_view(torch, cdf[PAD:PAD + h, PAD:PAD + w], stride, skew)
        k_dst, d_dst = _device_view(torch, np.zeros((h, w), deb.dtype), stride, skew)
        d_ab = torch.full((2 * nst * bstride,), 77, dtype=tdt, device="cuda")
        d_bl = torch.full((2 * nst * bstride,), 77, dtype=tdt, device="cuda")
        d_units = torch.from_numpy(units.view(np.uint8)).cuda()
        planes[p] = b200.LrPlane(d_deb.data_ptr(), d_cdf.data_ptr(), d_dst.data_ptr(), d_cdf.data_ptr(), d_ab.data_ptr(), d_bl.data_ptr(), stride,
                                 stride, stride, stride, bstride, w, h, ss, ss, usp, frt)
        assert d_cdf.data_ptr() % 16 == skew * d_cdf.element_size()
        d_sse = torch.full((hu * vu,), -1, dtype=torch.int64, device="cuda")
        keep.append((k_deb, k_cdf, k_dst, d_dst, d_ab, d_bl, d_units, d_sse, cdf[PAD:PAD + h, PAD:PAD + w].astype(np.int64), (w, h, usp, hu, vu)))
        checks.append(want_fn(p, deb, cdf, w, h, ss, usp, units, nst, bstride))
    s = torch.cuda.current_stream().cuda_stream
    assert b200.lib.svt_b200_lr_save_boundary_lines_dev(planes, 3, 0, bd, s) == 0
    assert b200.lib.svt_b200_lr_save_boundary_lines_dev(planes, 3, 1, bd, s) == 0
    torch.cuda.synchronize()
    for p in range(3):
        lines, want = checks[p]
        if lines is not None:
            assert np.array_equal(keep[p][4].cpu().numpy().view(lines[0].dtype), lines[0]), ("above lines", p)
            assert np.array_equal(keep[p][5].cpu().numpy().view(lines[1].dtype), lines[1]), ("below lines", p)
    unit_ptrs = (ct.c_void_p * 3)(*[k[6].data_ptr() for k in keep])
    sse_ptrs = (ct.c_void_p * 3)(*[k[7].data_ptr() for k in keep])
    for opt in (0, 1):
        for k in keep:
            k[3].zero_()
        assert b200.lib.svt_b200_lr_filter_frame_dev(planes, 3, unit_ptrs, opt, bd, s) == 0
        if sse:
            assert b200.lib.svt_b200_lr_unit_sse_dev(planes, 3, sse_ptrs, bd, s) == 0
        torch.cuda.synchronize()
        for p in range(3):
            want = checks[p][1][opt]
            got = keep[p][3].cpu().numpy().view(want.dtype)
            assert np.array_equal(got, want), ("restored plane", p, opt, np.argwhere(got != want)[:4])
            if sse:  # sse_restoration_unit over each unit's limits, rows shifted up by the 8-row (luma) stripe offset
                w, h, usp, hu, vu = keep[p][9]
                d2 = (want.astype(np.int64) - keep[p][8]) ** 2
                off = 8 >> (1 if p else 0)
                got_sse = keep[p][7].cpu().numpy()
                for ur in range(vu):
                    vs, ve = max(0, ur * usp - off), (h if ur == vu - 1 else (ur + 1) * usp - off)
                    for uc in range(hu):
                        hs, he = uc * usp, (w if uc == hu - 1 else (uc + 1) * usp)
                        assert int(got_sse[ur * hu + uc]) == int(d2[vs:ve, hs:he].sum()), ("unit sse", p, opt, ur, uc)


def _reference(refc, W, H, bd):
    refc.ref_lr_save_boundaries.restype = None
    refc.ref_lr_filter_plane.restype = None
    psz = 1 if bd == 8 else 2

    def want(p, deb, cdf, w, h, ss, usp, units, nst, bstride):
        pitch = deb.shape[1]
        ab = np.full(2 * nst * bstride, 77, deb.dtype)
        bl = np.full(2 * nst * bstride, 77, deb.dtype)
        org = (PAD * pitch + PAD) * psz
        V = lambda a, o=0: ct.c_void_p(a.ctypes.data + o)  # noqa: E731
        refc.ref_lr_save_boundaries(V(deb, org), pitch, w, h, bd, p, W, H, 0, V(ab), V(bl), bstride)
        refc.ref_lr_save_boundaries(V(cdf, org), pitch, w, h, bd, p, W, H, 1, V(ab), V(bl), bstride)
        out = {}
        for opt in (0, 1):
            data, res = cdf.copy(), np.zeros_like(cdf)
            refc.ref_lr_filter_plane(V(data, org), pitch, V(res, org), pitch, w, h, ss, ss, bd, usp, V(units), V(ab), V(bl), bstride, opt)
            out[opt] = res[PAD:PAD + h, PAD:PAD + w].copy()
        return (ab, bl), out
    return want


LAYOUT_CASES = [  # (luma width, luma height, bit depth, luma unit size)
    (1000, 300, 8, 64), (1000, 300, 8, 256), (1000, 300, 10, 64), (1000, 300, 10, 256)]


@pytest.mark.parametrize("skew", (0, 1), ids=("aligned", "skewed"))
@pytest.mark.parametrize("case", LAYOUT_CASES, ids=lambda c: "%dx%d_b%d_ru%d" % c)
def test_lr_frame_word_and_pixel_moves_match_reference(b200, refc, case, skew):
    W, H, bd, us = case
    r = rng(1400 + W + H + bd + us)
    _run(b200, W, H, bd, us, skew, lambda p, n: _units(r, n, b200), lambda p, w, h, which: _plane(r, w, h, bd, (p + which) % 2 == 0),
         _reference(refc, W, H, bd))


@pytest.mark.parametrize("fill", ("zeros", "max", "random"))
def test_lr_frame_extreme_legal_taps_match_reference(b200, refc, fill):
    W, H, bd, us = 328, 200, 8, 64
    r = rng(1500)
    taps = [_taps(*LEGAL_LO), _taps(*LEGAL_HI), _taps(LEGAL_HI[0], LEGAL_LO[1], LEGAL_HI[2])]
    chroma = [_taps(0, t[1], t[2]) for t in taps]  # 5-tap window

    def plane(p, w, h, which):
        buf = _plane(r, w, h, bd, False)
        if fill != "random":
            buf[PAD:PAD + h, PAD:PAD + w] = 0 if fill == "zeros" else 255
        return buf
    _run(b200, W, H, bd, us, 0, lambda p, n: _wiener_units(n, b200, chroma if p else taps), plane, _reference(refc, W, H, bd))


def _numpy_wiener(cdf, w, h, usp, hu, units):
    """add-src Wiener convolution of an edge-replicated 8-bit plane of one stripe (convolve.c:100-147), unit by unit"""
    x = np.pad(cdf.astype(np.int64), ((3, 3), (3, 4)), mode="edge")
    out = np.zeros((h, w), np.uint8)
    for k in range(len(units)):
        x0 = (k % hu) * usp
        x1 = w if k % hu == hu - 1 else x0 + usp
        hf, vf = units["hfilter"][k].astype(np.int64), units["vfilter"][k].astype(np.int64)
        seg = x[:, x0:x1 + 7]
        n = x1 - x0
        mid = (seg[:, 3:3 + n] << 7) + (1 << 14)
        for t in range(8):
            mid = mid + seg[:, t:t + n] * hf[t]
        mid = np.clip((mid + 4) >> 3, 0, (1 << 13) - 1)
        mid = np.vstack([mid, np.zeros((1, n), np.int64)])  # the 8-bit reference computes h + 6 intermediate rows and zero-fills the last
        acc = (mid[3:3 + h] << 7) - (1 << 18)
        for t in range(8):
            acc = acc + mid[t:t + h] * vf[t]
        out[:, x0:x1] = np.clip((acc + (1 << 10)) >> 11, 0, 255)
    return out


def test_lr_frame_taps_beyond_a_byte(b200):
    """one stripe per plane (no boundary substitution, one row of units), units alternating between legal taps, which
    check the numpy model against the device path the reference also checks, and taps outside [-128, 127]"""
    W, H, bd, us = 328, 56, 8, 64
    r = rng(1600)
    taps = [_taps(3, -7, 15), _taps(-40, -60, -50, centre=300), _taps(10, 8, 46), _taps(0, 0, 100, centre=-200)]

    def want(p, deb, cdf, w, h, ss, usp, units, nst, bstride):
        assert nst == 1
        hu = b200.lib.svt_b200_lr_units_per_dim(w, usp)
        res = _numpy_wiener(cdf[PAD:PAD + h, PAD:PAD + w], w, h, usp, hu, units)
        return None, {0: res, 1: res}
    _run(b200, W, H, bd, us, 0, lambda p, n: _wiener_units(n, b200, taps), lambda p, w, h, which: _plane(r, w, h, bd, which == 0), want)
