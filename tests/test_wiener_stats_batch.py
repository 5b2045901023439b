"""GPU parity of the 8-bit Wiener statistics batch call (svt_b200_compute_stats_batch_dev), item by item against the
reference's svt_av1_compute_stats_c.  One batch mixes 7x7, 5x5 and 3x3 windows; regions of 1x1, 1xN, Nx1, odd sizes
and the workload's 256x256 luma / 128x128 chroma units; regions on the picture edge whose halo reads the plane's
padding, on planes with different dgd and src strides; random, all-0, all-255, 0/255 checkerboard (src the inverse)
and half-black / half-white content; and one 1920x1080 item, large enough that every warp of the kernel passes the
33025-pixel bound of its int32 sums and folds them into the int64 totals."""
import ctypes as ct

import numpy as np
import pytest

import rest_helpers as rh
from helpers import rng
from oracle_libs import refc as ref  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu

PAD = 8  # the reference reads up to 3 pixels beyond the region: a region on the picture edge reads this padding


def _content(r, kind, w, h):
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "random":
        return r.integers(0, 256, (h, w)), r.integers(0, 256, (h, w))
    if kind == "zero":
        return np.zeros((h, w)), np.zeros((h, w))
    if kind == "max":
        return np.full((h, w), 255), np.full((h, w), 255)
    if kind == "checker":
        c = ((xx + yy) % 2) * 255
        return c, 255 - c
    if kind == "halves":
        return (xx >= w // 2) * 255, (yy >= h // 2) * 255
    if kind == "bright":  # near the largest raw products, not constant
        return r.integers(240, 256, (h, w)), r.integers(0, 256, (h, w))
    raise ValueError(kind)


class _Planes:
    """dgd planes with PAD pixels of random padding on every side, src planes unpadded; each with its own stride, all
    packed into one dgd and one src buffer"""

    def __init__(self):
        self.dgd, self.src, self.planes = [], [], []
        self.dgd_len = self.src_len = 0

    def add(self, r, kind, w, h, dgd_extra, src_extra):
        ds, ss = w + 2 * PAD + dgd_extra, w + src_extra
        d = r.integers(0, 256, (h + 2 * PAD, ds))
        s = r.integers(0, 256, (h, ss))
        pd, ps = _content(r, kind, w, h)
        d[PAD:PAD + h, PAD:PAD + w] = pd
        s[:, :w] = ps
        self.planes.append(dict(dgd_off=self.dgd_len + PAD * ds + PAD, src_off=self.src_len, ds=ds, ss=ss, w=w, h=h))
        self.dgd.append(d.astype(np.uint8).reshape(-1)); self.src.append(s.astype(np.uint8).reshape(-1))
        self.dgd_len += d.size; self.src_len += s.size
        return len(self.planes) - 1


def test_compute_stats_batch_8bit(b200, ref):
    import torch
    r = rng(97)
    pl = _Planes()
    rnd = pl.add(r, "random", 300, 200, 5, 7)
    zero = pl.add(r, "zero", 96, 80, 16, 0)
    mx = pl.add(r, "max", 100, 70, 1, 3)
    chk = pl.add(r, "checker", 130, 90, 3, 17)
    hv = pl.add(r, "halves", 200, 120, 0, 2)
    unit = pl.add(r, "random", 512, 320, 24, 0)
    big = pl.add(r, "bright", 1920, 1080, 32, 0)
    # (plane, window, h_start, h_end, v_start, v_end)
    regions = [(rnd, 7, 10, 11, 20, 21), (rnd, 5, 0, 1, 0, 1), (rnd, 3, 299, 300, 199, 200),
               (rnd, 7, 5, 6, 3, 200), (rnd, 5, 0, 300, 17, 18), (rnd, 3, 40, 41, 0, 77),
               (rnd, 7, 3, 40, 5, 28), (rnd, 5, 101, 166, 7, 40), (rnd, 3, 13, 142, 60, 157),
               (rnd, 7, 0, 300, 0, 200), (rnd, 5, 233, 300, 111, 200), (rnd, 7, 0, 65, 167, 200),
               (zero, 7, 0, 96, 0, 80), (zero, 3, 7, 70, 9, 42),
               (mx, 7, 0, 100, 0, 70), (mx, 5, 31, 99, 1, 69), (mx, 3, 0, 1, 0, 70),
               (chk, 7, 0, 130, 0, 90), (chk, 5, 1, 128, 3, 89), (chk, 3, 64, 130, 32, 90),
               (hv, 7, 0, 200, 0, 120), (hv, 5, 50, 151, 30, 91), (hv, 3, 99, 101, 0, 120),
               (unit, 7, 0, 256, 0, 256), (unit, 7, 256, 512, 0, 320), (unit, 5, 128, 256, 128, 256), (unit, 5, 384, 512, 192, 320),
               (big, 7, 0, 1920, 0, 1080)]
    items = np.zeros(len(regions), dtype=b200.STATS_ITEM_DTYPE)
    for i, (p, win, hs, he, vs, ve) in enumerate(regions):
        q = pl.planes[p]
        assert 0 <= hs < he <= q["w"] and 0 <= vs < ve <= q["h"]
        items[i] = (q["dgd_off"], q["src_off"], q["ds"], q["ss"], hs, he, vs, ve, win, 0)
    dgd, src = np.concatenate(pl.dgd), np.concatenate(pl.src)
    d_dgd, d_src = torch.from_numpy(dgd).cuda(), torch.from_numpy(src).cuda()
    d_items = torch.from_numpy(items.view(np.uint8).copy()).cuda()
    d_M = torch.full((len(items), 49), -7, dtype=torch.int64).cuda()
    d_H = torch.full((len(items), 2401), -7, dtype=torch.int64).cuda()
    rc = b200.lib.svt_b200_compute_stats_batch_dev(d_dgd.data_ptr(), d_src.data_ptr(), d_items.data_ptr(), len(items), 8, d_M.data_ptr(),
                                                   d_H.data_ptr(), None)
    assert rc == 0
    torch.cuda.synchronize()
    M, H = d_M.cpu().numpy(), d_H.cpu().numpy()
    for i, (p, win, hs, he, vs, ve) in enumerate(regions):
        q = pl.planes[p]
        want_M, want_H = rh.ref_stats(ref, win, dgd[q["dgd_off"]:], src[q["src_off"]:], hs, he, vs, ve, q["ds"], q["ss"], 8)
        assert np.array_equal(M[i, :win * win], want_M), (i, regions[i])
        assert np.array_equal(H[i, :win ** 4], want_H), (i, regions[i])
