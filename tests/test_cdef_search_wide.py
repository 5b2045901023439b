"""GPU parity of the whole-picture CDEF strength search at 12 bit and with more candidate strengths than a
search thread evaluates at once (8): the strength list is then taken in chunks, with primary codes that repeat
across a chunk boundary, code 0 and untested (-1) entries in later chunks, and up to the 64 the ABI allows.
The expected values come from the reference functions driven in the order of cdef_seg_search
(cdef_helpers.ref_cdef_search)."""
import ctypes as ct

import numpy as np
import pytest

import cdef_helpers as ch
from helpers import rng

pytestmark = pytest.mark.gpu


def _strengths(r, n):
    s = [int(v) for v in r.integers(0, 64, n)]
    s[0] = 0
    s[8] = (s[7] & ~3) | ((s[7] + 1) & 3)  # the first chunk's last primary code opens the second chunk
    for i in range(9, n, 7):  # code 0, a repeated primary code and an untested entry past the first chunk
        s[i] = 0
    for i in range(10, n, 7):
        s[i] = (s[i - 2] & ~3) | ((s[i - 2] + 1) & 3)
    for i in range(12, n, 11):
        s[i] = -1
    return s


@pytest.mark.parametrize("bd,subs,n", [(12, 1, 7), (12, 4, 7), (8, 4, 20), (10, 1, 64)])
def test_cdef_search_frame_t2_wide(b200, refc, bd, subs, n):
    import torch
    r = rng(90 + bd + subs + n)
    W, H = 208, 136
    rec, src, skip = ch.make_frame(r, W, H, bd)
    skip[0:8, 8:16] = 1  # one filter block without a single non-skip 8x8
    if n == 7:
        sy = [0, 4, 9, 17, 35, 63, 2]
        su = [0, 4, -1, 17, 20, 63, 3]
    else:
        sy, su = _strengths(r, n), _strengths(r, n)
    want = ch.ref_cdef_search(refc, rec, src, skip, W, H, bd, 5, subs, sy, su)
    dt = np.uint8 if bd == 8 else np.int16
    drec = [torch.from_numpy(p.astype(dt)).cuda() for p in rec]
    dsrc = [torch.from_numpy(p.astype(dt)).cuda() for p in src]
    dskip = torch.from_numpy(skip).cuda()
    dsy = torch.tensor(sy, dtype=torch.int32).cuda(); dsu = torch.tensor(su, dtype=torch.int32).cuda()
    nfb = ((W + 63) // 64) * ((H + 63) // 64)
    dmse = torch.full((2, nfb, n), -1, dtype=torch.int64).cuda()  # the luma half must be written in full
    ddir = torch.zeros((nfb, 64), dtype=torch.uint8).cuda(); dvar = torch.zeros((nfb, 64), dtype=torch.int32).cuda()
    fr = b200.cdef_frame_desc(drec, dsrc, W, H, bd, 5, subs)
    rc = b200.lib.svt_b200_cdef_search_frame_dev(ct.byref(fr), dskip.data_ptr(), dsy.data_ptr(), dsu.data_ptr(), n, dmse.data_ptr(),
                                                 ddir.data_ptr(), dvar.data_ptr(), None)
    assert rc == 0
    torch.cuda.synchronize()
    assert np.array_equal(ddir.cpu().numpy(), want[1])
    assert np.array_equal(dvar.cpu().numpy(), want[2])
    got = dmse.cpu().numpy().astype(np.uint64)
    assert np.array_equal(got, want[0])
