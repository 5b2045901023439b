"""GPU parity of the CDEF search and apply where one CTA takes both chroma planes of a filter block: it stages the Cb
and the Cr tile in one pass, evaluates both planes' segments in one loop and writes each chroma distortion once.

Cb and Cr share one pitch but not one alignment: one plane starts on a whole tile-load word (8 pixels) and the other
1-15 bytes past it, so one CTA stages one plane by words and the other pixel by pixel, and stores one plane's rows
whole and the other's pixel by pixel.  Every 8-bit origin offset 1-15 and every 16-bit one 2-14 is taken, in the luma
plane too.  The chroma strength lists of the search hold untested (-1) entries, or code 0 only; one filter block has no non-skip
8x8 and the distortion buffer starts as garbage, so its zero rows must be written by the search.  A last picture has
more filter blocks than the grids have CTAs, so CTAs go from chroma items to luma items and rebuild their constants
table.  The expected values come from the reference functions (cdef_helpers)."""
import ctypes as ct

import numpy as np
import pytest

import cdef_helpers as ch
from helpers import rng
from oracle_libs import refc  # noqa: F401  (a fixture: overrides conftest.py's refc in this module)

pytestmark = pytest.mark.gpu

GUARD = 256  # bytes before and after every plane
SY = [0, 4, 9, 17, 35, 63, 2, 41]
SU = {"untested": [0, -1, 5, 22, -1, 63, 3, 12], "zero": [0] * 8}


def _layout(bd, k):
    """byte offsets past an aligned address of the (Y, Cb, Cr) origins: Cb or Cr on a whole word, the other k bytes off"""
    return (k, 0, k) if (k // (1 if bd == 8 else 2)) % 2 else (k, k, 0)


def _host(planes, bd, offs, fill):
    """host byte buffers holding the planes at the given offsets, pitch a multiple of 16 pixels: [(buffer, start, pitch)]"""
    psz = 1 if bd == 8 else 2
    out = []
    for p, off in zip(planes, offs):
        h, w = p.shape
        pitch = (w + 8 + 15) // 16 * 16
        buf = fill(GUARD + off + h * pitch * psz + GUARD)
        _view(buf, GUARD + off, h, pitch, bd)[:, :w] = p
        out.append((buf, GUARD + off, pitch))
    return out


def _view(buf, start, h, pitch, bd):
    n = h * pitch * (1 if bd == 8 else 2)
    return buf[start:start + n].view(np.uint8 if bd == 8 else np.uint16).reshape(h, pitch)


def _device(torch, hp):
    dev = [torch.from_numpy(b).cuda() for b, _, _ in hp]
    return dev, [d.data_ptr() + s for d, (_, s, _) in zip(dev, hp)], [p for _, _, p in hp]


def _frame(b200, rp, rs, sp, ss, W, H, bd, damping, subs):
    f = b200.CdefFrame()
    f.recon_y, f.recon_cb, f.recon_cr = rp
    f.src_y, f.src_cb, f.src_cr = sp
    f.recon_stride_y, f.recon_stride_c, f.src_stride_y, f.src_stride_c = rs[0], rs[1], ss[0], ss[1]
    f.width, f.height, f.bit_depth, f.damping, f.subsampling_factor = W, H, bd, damping, subs
    return f


def _check(b200, refc, torch, r, W, H, bd, damping, subs, rec, src, skip, sy, su, idx, offs, large=False):
    nfb, n = len(idx), len(sy)
    search = ch.c_cdef_search if large else ch.ref_cdef_search
    want_mse, want_dir, want_var = search(refc, rec, src, skip, W, H, bd, damping, subs, sy, su)
    noise = lambda k: r.integers(0, 256, k, dtype=np.uint8)  # noqa: E731  (padding: its values must not matter)
    drec, rp, rs = _device(torch, _host(rec, bd, offs, noise))
    dsrc, sp, ss = _device(torch, _host(src, bd, offs, noise))
    word = 8 * (1 if bd == 8 else 2)
    assert rs[1] == rs[2] and rs[1] * (word // 8) % word == 0
    assert rp[1] % word == 0 or rp[2] % word == 0
    assert (rp[1] % word == 0) != (rp[2] % word == 0) or max(offs) % word == 0  # an 8-byte offset is still a word at 8 bit
    fr = _frame(b200, rp, rs, sp, ss, W, H, bd, damping, subs)
    dskip, didx = torch.from_numpy(skip).cuda(), torch.from_numpy(idx).cuda()
    dsy, dsu = torch.tensor(sy, dtype=torch.int32).cuda(), torch.tensor(su, dtype=torch.int32).cuda()
    dmse = torch.from_numpy(r.integers(-2**62, 2**62, (2, nfb, n), dtype=np.int64)).cuda()  # every entry must be written
    ddir = torch.zeros((nfb, 64), dtype=torch.uint8).cuda()
    dvar = torch.zeros((nfb, 64), dtype=torch.int32).cuda()
    assert b200.lib.svt_b200_cdef_search_frame_dev(ct.byref(fr), dskip.data_ptr(), dsy.data_ptr(), dsu.data_ptr(), n, dmse.data_ptr(),
                                                   ddir.data_ptr(), dvar.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(ddir.cpu().numpy(), want_dir)
    assert np.array_equal(dvar.cpu().numpy(), want_var)
    got = dmse.cpu().numpy().astype(np.uint64)
    assert np.array_equal(got[0], want_mse[0]), "luma distortions"
    assert np.array_equal(got[1], want_mse[1]), "chroma distortions"

    # the apply takes the strengths a search chose: no untested entries
    sy, su = [v if v >= 0 else 7 for v in sy], [v if v >= 0 else 7 for v in su]
    dsy, dsu = torch.tensor(sy, dtype=torch.int32).cuda(), torch.tensor(su, dtype=torch.int32).cuda()
    sentinel = lambda k: np.full(k, 0xA5, np.uint8)  # noqa: E731
    init = _host(rec, bd, offs, sentinel)
    want = [(b.copy(), s, p) for b, s, p in init]
    views = [_view(b, s, q.shape[0], p, bd) for (b, s, p), q in zip(want, rec)]
    (ch.c_cdef_apply if large else ch.ref_cdef_apply)(refc, rec, skip, W, H, bd, damping, idx, sy, su, views, [v.shape[1] for v in views])
    dout, op, osd = _device(torch, init)
    assert b200.lib.svt_b200_cdef_apply_frame_dev(ct.byref(fr), dskip.data_ptr(), didx.data_ptr(), dsy.data_ptr(), dsu.data_ptr(),
                                                  ddir.data_ptr(), dvar.data_ptr(), op[0], op[1], op[2], osd[0], osd[1], None) == 0
    torch.cuda.synchronize()
    for pli, (d, (w, _, _)) in enumerate(zip(dout, want)):
        assert np.array_equal(d.cpu().numpy(), w), "apply, plane %d" % pli


CASES = [(8, k) for k in range(1, 16)] + [(10, k) for k in range(2, 16, 2)]


@pytest.mark.parametrize("bd,k", CASES)
@pytest.mark.parametrize("uv", sorted(SU))
def test_cdef_chroma_pair_mixed_alignment(b200, refc, bd, k, uv):
    import torch
    r = rng(300 + 16 * bd + k)
    W, H = 200, 72  # partial filter blocks on the right and at the bottom
    rec, src, skip = ch.make_mixed_frame(r, W, H, bd)
    skip[0:8, 8:16] = 1  # a filter block without a non-skip 8x8
    skip[0:8, 0:8] = 0
    nfb = 4 * 2
    idx = (np.arange(nfb) % len(SY)).astype(np.int8)
    idx[5] = -1
    _check(b200, refc, torch, r, W, H, bd, 3 + k % 4, (1, 2, 4)[k % 3], rec, src, skip, SY, SU[uv], idx, _layout(bd, k))


@pytest.mark.parametrize("bd", [8, 10])
def test_cdef_chroma_pair_grid_loops(b200, refc, bd):
    """more filter blocks than the grids have CTAs: a CTA takes chroma items, then luma items"""
    import torch
    r = rng(330 + bd)
    sm = b200.lib.svt_b200_sm_count()
    nvfb = 9
    nhfb = 16 * sm // (2 * nvfb) + 1
    W, H = 64 * nhfb - 24, 64 * nvfb - 40
    nfb = nhfb * nvfb
    assert 2 * nfb > 16 * sm
    rec, src, skip = ch.make_mixed_frame(r, W, H, bd)
    skip[8:16, 16:24] = 1
    idx = r.integers(-1, len(SY), nfb).astype(np.int8)
    _check(b200, refc, torch, r, W, H, bd, 5, 1, rec, src, skip, SY, SU["untested"], idx, _layout(bd, 4 if bd == 8 else 6), large=True)
