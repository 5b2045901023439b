"""GPU parity of the whole-picture CDEF apply (svt_b200_cdef_apply_frame_dev) and, on the same frames, of the strength
search (svt_b200_cdef_search_frame_dev).  The expected values come from the reference functions: the apply replayed in
the order of svt_av1_cdef_frame (cdef_helpers.ref_cdef_apply), the search in the order of cdef_seg_search
(cdef_helpers.ref_cdef_search).

Each bit depth (8, 10, 12) runs dampings 3..6 over pictures from 8x8 to 456x264 with partial filter blocks on the right
and bottom, and applies every strength code 0..63 in luma and in chroma, including the pairs (0, 0), (0, x) and (x, 0)
and filter blocks left untouched (index -1).  Every picture runs in three plane layouts: aligned pitches, odd pitches
(8-bit planes also at an odd address) and planes one pixel past an aligned address.  Between them they take both the
paired and the per-pixel tile loads, and both the wide and the per-pixel stores.  Output planes sit between sentinel
guard bands that must stay untouched.  The apply runs with the directions the search found and with none (it then finds
them itself).  One more picture per bit depth has more (filter block, plane) pairs than either grid has CTAs, so every
CTA loops; it is checked against the C drivers of oracle/ref_driver.c to keep the run time down."""
import ctypes as ct

import numpy as np
import pytest

import cdef_helpers as ch
from helpers import rng

pytestmark = pytest.mark.gpu

SIZES = [(8, 8), (64, 8), (72, 72), (200, 136), (456, 264)]
DAMPINGS = (3, 4, 5, 6)
LAYOUTS = ("aligned", "odd", "offset")
GUARD, SENTINEL = 256, 0xA5  # sentinel bytes before and after every plane


def _geometry(layout, w, psz):
    """(pitch in pixels, byte offset of the first pixel past the guard band) of a plane w pixels wide"""
    if layout == "aligned":
        return (w + 63) // 64 * 64 + 64, 0
    if layout == "odd":  # odd pitch; 8-bit planes also start at an odd address
        return w + 13, 1 if psz == 1 else 0
    # 16-bit: one pixel past an aligned address; 8-bit: 4 bytes past it.  The pitch is not a multiple of 8.
    return (w + 7) // 8 * 8 + (4 if psz == 1 else 6), 4 if psz == 1 else 2


def _view(buf, start, h, pitch, bd):
    n = h * pitch * (1 if bd == 8 else 2)
    return buf[start:start + n].view(np.uint8 if bd == 8 else np.uint16).reshape(h, pitch)


def _host_planes(planes, bd, layout, fill):
    """host byte buffers holding the three planes as they are laid out on the device: [(buffer, first pixel, pitch)]"""
    out = []
    for p in planes:
        h, w = p.shape
        pitch, off = _geometry(layout, w, 1 if bd == 8 else 2)
        buf = fill(GUARD + off + h * pitch * (1 if bd == 8 else 2) + GUARD)
        _view(buf, GUARD + off, h, pitch, bd)[:, :w] = p
        out.append((buf, GUARD + off, pitch))
    return out


def _to_device(torch, hp):
    """device copies of _host_planes buffers: (tensors, first-pixel pointers, pitches)"""
    dev = [torch.from_numpy(b).cuda() for b, _, _ in hp]
    return dev, [d.data_ptr() + s for d, (_, s, _) in zip(dev, hp)], [pitch for _, _, pitch in hp]


def _expect_planes_equal(got, want, bd, what):
    psz = 1 if bd == 8 else 2
    for pli, (g, (w, start, pitch)) in enumerate(zip(got, want)):
        if not np.array_equal(g, w):
            k = int(np.flatnonzero(g != w)[0]) - start
            where = "guard band" if k < 0 or k >= len(w) - start - GUARD else "row %d, column %d" % (k // (pitch * psz), k % (pitch * psz) // psz)
            pytest.fail("%s: plane %d differs first at %s" % (what, pli, where))


def _tables(perm, di, si, nfb):
    """strength tables (16 entries) and per filter block indices of one picture.  The 456x264 pictures (si = 4) take a
    disjoint 16-code slice of the bit depth's permutation per damping and use every entry, so each code is applied in
    both planes; chroma reads the permutation 7 places on, which never pairs a 0 with a 0.  The smaller pictures take
    rotations of the same slices with a (0, 0) entry.  Some filter blocks are left untouched (-1)."""
    sl = [int(c) for c in perm[16 * di:16 * di + 16]]
    sy, su = sl, [int(perm[(16 * di + k + 7) % 64]) for k in range(16)]
    if si == len(SIZES) - 1:
        idx = np.arange(nfb) % 16
        idx[[21, 37]] = -1
    else:
        rot = 5 * si + di
        sy, su = sy[rot:] + sy[:rot], su[rot:] + su[:rot]
        sy[15] = su[15] = 0
        idx = (3 * np.arange(nfb) + si + di) % 16
        if nfb >= 4:
            idx[nfb - 2] = 15
            idx[2] = -1
    return sy, su, idx.astype(np.int8)


def _skip_map(skip, W, H):
    """on top of the random skips: the last filter block all skip, the first without a skip, and a single non-skip 8x8
    in the partial filter block at the right edge of the first row (every 8x8 of a one-block picture is non-skip)"""
    nhfb, nvfb = (W + 63) // 64, (H + 63) // 64
    if nhfb * nvfb == 1:
        skip[:] = 0
        return skip
    skip[(nvfb - 1) * 8:, (nhfb - 1) * 8:] = 1
    skip[:8, :8] = 0
    if W % 64:
        skip[:8, (nhfb - 1) * 8:] = 1
        skip[min(2, skip.shape[0] - 1), (nhfb - 1) * 8] = 0
    return skip


class Coverage:
    """what the fixture of one bit depth reaches, gathered from the reference's own results"""

    def __init__(self):
        self.dirs, self.y, self.uv, self.pair_load, self.wide = set(), set(), set(), set(), set()
        self.var0 = self.var_cap = self.edge_y = self.edge_uv = self.untouched = self.zero_pair = False
        self.pair_0x = self.pair_x0 = False

    def add(self, W, H, skip, sy, su, idx, filtered, dirs, vars_):
        nhfb = (W + 63) // 64
        for fb in range(len(idx)):
            fbr, fbc = divmod(fb, nhfb)
            lst = ch.fb_list(skip, fbr, fbc)
            if lst and idx[fb] < 0:
                self.untouched = True
            if lst and idx[fb] >= 0 and sy[idx[fb]] == 0 and su[idx[fb]] == 0:
                self.zero_pair = True
        for fb in filtered:
            fbr, fbc = divmod(fb, nhfb)
            cy, cuv = sy[idx[fb]], su[idx[fb]]
            self.y.add(cy)
            self.uv.add(cuv)
            self.pair_0x |= cy == 0 and cuv != 0
            self.pair_x0 |= cuv == 0 and cy != 0
            partial = W - 64 * fbc < 64 or H - 64 * fbr < 64
            self.edge_y |= partial and cy != 0
            self.edge_uv |= partial and cuv != 0
            for by, bx in ch.fb_list(skip, fbr, fbc):
                v = int(vars_[fb, by * 8 + bx])
                self.dirs.add(int(dirs[fb, by * 8 + bx]))
                self.var0 |= v == 0
                self.var_cap |= (v >> 6) >= 4096

    def add_layout(self, bd, rec_ptrs, rec_pitch, out_ptrs, out_pitch):
        """the kernels' own alignment tests: stage_cdef_tile's pair_load and cdef_apply_kernel's wide"""
        psz = 1 if bd == 8 else 2
        for pli in range(3):
            self.pair_load.add(((rec_ptrs[pli] | rec_pitch[pli] * psz) & (2 * psz - 1)) == 0)
            self.wide.add(((out_ptrs[pli] | out_pitch[pli] * psz) & ((8 >> (pli > 0)) * psz - 1)) == 0)

    def check(self):
        assert self.dirs == set(range(8)), sorted(self.dirs)
        assert self.var0 and self.var_cap
        assert self.y == set(range(64)), sorted(set(range(64)) - self.y)
        assert self.uv == set(range(64)), sorted(set(range(64)) - self.uv)
        assert self.zero_pair and self.pair_0x and self.pair_x0
        assert self.edge_y and self.edge_uv and self.untouched
        assert self.pair_load == {True, False} and self.wide == {True, False}


def _frame_desc(b200, rec_ptrs, rec_pitch, src_ptrs, src_pitch, W, H, bd, damping, subs):
    f = b200.CdefFrame()
    f.recon_y, f.recon_cb, f.recon_cr = rec_ptrs
    f.src_y, f.src_cb, f.src_cr = src_ptrs
    f.recon_stride_y, f.recon_stride_c, f.src_stride_y, f.src_stride_c = rec_pitch[0], rec_pitch[1], src_pitch[0], src_pitch[1]
    f.width, f.height, f.bit_depth, f.damping, f.subsampling_factor = W, H, bd, damping, subs
    return f


def _run(b200, refc, torch, r, cov, W, H, bd, damping, subs, rec, src, skip, sy, su, idx, large=False):
    """search + apply (with the search's directions, and without) of one picture in every layout against the reference"""
    tag = "%dx%d bd %d damping %d" % (W, H, bd, damping)
    nfb, n = len(idx), len(sy)
    want_mse, want_dir, want_var = (ch.c_cdef_search if large else ch.ref_cdef_search)(refc, rec, src, skip, W, H, bd, damping, subs, sy, su)
    dskip, didx = torch.from_numpy(skip).cuda(), torch.from_numpy(idx).cuda()
    dsy, dsu = torch.tensor(sy, dtype=torch.int32).cuda(), torch.tensor(su, dtype=torch.int32).cuda()
    noise = lambda k: r.integers(0, 256, k, dtype=np.uint8)  # noqa: E731  (input padding: its values must not matter)
    sentinel = lambda k: np.full(k, SENTINEL, np.uint8)  # noqa: E731
    for layout in LAYOUTS:
        what = "%s, %s layout" % (tag, layout)
        drec, rec_ptrs, rec_pitch = _to_device(torch, _host_planes(rec, bd, layout, noise))
        dsrc, src_ptrs, src_pitch = _to_device(torch, _host_planes(src, bd, layout, noise))
        fr = _frame_desc(b200, rec_ptrs, rec_pitch, src_ptrs, src_pitch, W, H, bd, damping, subs)
        dmse = torch.full((2, nfb, n), -1, dtype=torch.int64).cuda()  # the luma half must be written in full
        ddir = torch.zeros((nfb, 64), dtype=torch.uint8).cuda(); dvar = torch.zeros((nfb, 64), dtype=torch.int32).cuda()
        assert b200.lib.svt_b200_cdef_search_frame_dev(ct.byref(fr), dskip.data_ptr(), dsy.data_ptr(), dsu.data_ptr(), n, dmse.data_ptr(),
                                                       ddir.data_ptr(), dvar.data_ptr(), None) == 0
        torch.cuda.synchronize()
        assert np.array_equal(ddir.cpu().numpy(), want_dir), "search directions, " + what
        assert np.array_equal(dvar.cpu().numpy(), want_var), "search variances, " + what
        assert np.array_equal(dmse.cpu().numpy().astype(np.uint64), want_mse), "search distortions, " + what
        # the output starts as a copy of the input (the ABI), between guard bands
        init = _host_planes(rec, bd, layout, sentinel)
        want = [(b.copy(), s, p) for b, s, p in init]
        views = [_view(b, s, q.shape[0], p, bd) for (b, s, p), q in zip(want, rec)]
        if large:
            ch.c_cdef_apply(refc, rec, skip, W, H, bd, damping, idx, sy, su, views, [v.shape[1] for v in views])
        else:
            filtered, dirs, vars_ = ch.ref_cdef_apply(refc, rec, skip, W, H, bd, damping, idx, sy, su, views, [v.shape[1] for v in views])
            if layout == LAYOUTS[0]:
                cov.add(W, H, skip, sy, su, idx, filtered, dirs, vars_)
        for with_dirs in (True, False):
            dout, out_ptrs, out_pitch = _to_device(torch, init)
            assert out_pitch[1] == out_pitch[2]
            rc = b200.lib.svt_b200_cdef_apply_frame_dev(ct.byref(fr), dskip.data_ptr(), didx.data_ptr(), dsy.data_ptr(), dsu.data_ptr(),
                                                        ddir.data_ptr() if with_dirs else None, dvar.data_ptr() if with_dirs else None,
                                                        out_ptrs[0], out_ptrs[1], out_ptrs[2], out_pitch[0], out_pitch[1], None)
            assert rc == 0
            torch.cuda.synchronize()
            _expect_planes_equal([d.cpu().numpy() for d in dout], want, bd,
                                 "apply (%s), %s" % ("the search's directions" if with_dirs else "directions found by the apply", what))
        cov.add_layout(bd, rec_ptrs, rec_pitch, out_ptrs, out_pitch)


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_cdef_apply_frame_matches_reference(b200, refc, bd):
    import torch
    r = rng(200 + bd)
    perm = r.permutation(64)
    cov = Coverage()
    for di, damping in enumerate(DAMPINGS):
        for si, (W, H) in enumerate(SIZES):
            rec, src, skip = ch.make_mixed_frame(r, W, H, bd)
            skip = _skip_map(skip, W, H)
            nfb = ((W + 63) // 64) * ((H + 63) // 64)
            sy, su, idx = _tables(perm, di, si, nfb)
            _run(b200, refc, torch, r, cov, W, H, bd, damping, (1, 2, 4, 1)[di], rec, src, skip, sy, su, idx)
    cov.check()


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_cdef_frame_larger_than_the_grid(b200, refc, bd):
    """more (filter block, plane) pairs than the 16 CTAs per SM of the search and apply grids: every CTA loops"""
    import torch
    r = rng(210 + bd)
    sm = b200.lib.svt_b200_sm_count()
    H = 1544  # 25 filter block rows, the last one 8 rows high
    nhfb = 16 * sm // (3 * 25) + 1
    W = 64 * nhfb - 56  # the last filter block column 8 wide
    nfb = nhfb * 25
    assert 3 * nfb > 16 * sm
    rec, src, skip = ch.make_mixed_frame(r, W, H, bd)
    perm = [int(c) for c in r.permutation(64)]
    sy, su = perm[:16], perm[16:32]
    idx = r.integers(-1, 16, nfb).astype(np.int8)
    _run(b200, refc, torch, r, Coverage(), W, H, bd, {8: 4, 10: 6, 12: 3}[bd], 1, rec, src, skip, sy, su, idx, large=True)
