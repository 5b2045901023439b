"""The CDEF apply without directions (svt_b200_cdef_apply_frame_dev with d_dir = d_var = NULL) finds them itself in
scratch that belongs to the call's stream, like every other library scratch: the call only enqueues work, so two such
calls run on two streams at once and each can be captured in a CUDA graph.  Every result must equal, bit for bit, the
same apply given the directions and variances of the strength search."""
import ctypes as ct

import numpy as np
import pytest

import cdef_helpers as ch
from helpers import rng

pytestmark = pytest.mark.gpu


class _Picture:
    """one picture on the device: input planes, the search's directions, output planes and the output to expect"""

    def __init__(self, b200, torch, seed, W, H, bd, damping):
        r = rng(seed)
        rec, src, skip = ch.make_mixed_frame(r, W, H, bd)
        dt = np.uint8 if bd == 8 else np.uint16
        planes = lambda ps: [torch.from_numpy(p.astype(dt).reshape(-1).view(np.uint8)).cuda() for p in ps]  # noqa: E731
        nfb = ((W + 63) // 64) * ((H + 63) // 64)
        perm = [int(c) for c in r.permutation(64)]
        self.lib, self.W = b200.lib, W
        self.rec, self.src = planes(rec), planes(src)
        self.out = [p.clone() for p in self.rec]
        self.skip = torch.from_numpy(skip).cuda()
        self.idx = torch.from_numpy(r.integers(-1, 16, nfb).astype(np.int8)).cuda()
        self.sy = torch.tensor(perm[:16], dtype=torch.int32).cuda()
        self.su = torch.tensor(perm[16:32], dtype=torch.int32).cuda()
        f = self.frame = b200.CdefFrame()
        f.recon_y, f.recon_cb, f.recon_cr = (p.data_ptr() for p in self.rec)
        f.src_y, f.src_cb, f.src_cr = (p.data_ptr() for p in self.src)
        f.recon_stride_y = f.src_stride_y = W
        f.recon_stride_c = f.src_stride_c = W >> 1
        f.width, f.height, f.bit_depth, f.damping, f.subsampling_factor = W, H, bd, damping, 1
        mse = torch.empty((2, nfb, 16), dtype=torch.int64).cuda()
        self.dir = torch.zeros((nfb, 64), dtype=torch.uint8).cuda()
        self.var = torch.zeros((nfb, 64), dtype=torch.int32).cuda()
        assert self.lib.svt_b200_cdef_search_frame_dev(ct.byref(f), self.skip.data_ptr(), self.sy.data_ptr(), self.su.data_ptr(), 16,
                                                       mse.data_ptr(), self.dir.data_ptr(), self.var.data_ptr(), None) == 0
        assert self.apply(None, with_dirs=True) == 0
        torch.cuda.synchronize()
        self.want = self.result()
        assert any(not np.array_equal(w, p.cpu().numpy()) for w, p in zip(self.want, self.rec)), "the filter changed nothing"

    def apply(self, stream, with_dirs=False):
        return self.lib.svt_b200_cdef_apply_frame_dev(ct.byref(self.frame), self.skip.data_ptr(), self.idx.data_ptr(), self.sy.data_ptr(),
                                                      self.su.data_ptr(), self.dir.data_ptr() if with_dirs else None,
                                                      self.var.data_ptr() if with_dirs else None, self.out[0].data_ptr(),
                                                      self.out[1].data_ptr(), self.out[2].data_ptr(), self.W, self.W >> 1, stream)

    def reset(self):
        """outputs back to a copy of the input (the ABI: the apply writes only the filter blocks it filters)"""
        for o, p in zip(self.out, self.rec):
            o.copy_(p)

    def result(self):
        return [o.cpu().numpy() for o in self.out]

    def check(self, what):
        for pli, (got, want) in enumerate(zip(self.result(), self.want)):
            assert np.array_equal(got, want), "%s: %dx%d bd %d, plane %d" % (what, self.W, self.frame.height, self.frame.bit_depth, pli)


@pytest.fixture(scope="module")
def pictures(b200):
    """a small 10-bit and a large 8-bit picture: the large one needs more than twice the small one's scratch"""
    import torch
    return [_Picture(b200, torch, 400, 640, 360, 10, 4), _Picture(b200, torch, 401, 1920, 1080, 8, 5)]


def test_cdef_apply_without_directions_on_two_streams_at_once(pictures):
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rep in range(3):  # the first round also sizes each stream's scratch
        for p in pictures:
            p.reset()
        torch.cuda.synchronize()
        for p, st in zip(pictures, streams):
            assert p.apply(st.cuda_stream) == 0
        torch.cuda.synchronize()
        for p in pictures:
            p.check("two streams at once, round %d" % rep)


def test_cdef_apply_without_directions_in_graphs(pictures):
    """one graph captured per stream after a warm-up call; replayed on both streams at once, then again after the large
    picture, run eagerly on the small one's stream, has given that stream a larger scratch"""
    import torch
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    graphs = []
    for p, st in zip(pictures, streams):
        with torch.cuda.stream(st):
            assert p.apply(st.cuda_stream) == 0  # warm-up: no allocation inside the capture
        torch.cuda.synchronize()
        p.check("warm-up")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            assert p.apply(st.cuda_stream) == 0
        graphs.append(g)

    def replay(what):
        for p in pictures:
            p.reset()
        torch.cuda.synchronize()
        for g, st in zip(graphs, streams):
            with torch.cuda.stream(st):
                g.replay()
        torch.cuda.synchronize()
        for p in pictures:
            p.check(what)

    replay("graph replay")
    large = pictures[1]
    large.reset()
    torch.cuda.synchronize()
    assert large.apply(streams[0].cuda_stream) == 0
    torch.cuda.synchronize()
    large.check("eager on the other stream")
    replay("graph replay after the scratch grew")
