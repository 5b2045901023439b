"""TEST / BASELINE INFRASTRUCTURE: one frame of the synthetic hot-path workload bound to the reference's own
kernels (oracle/ref_driver.c inside oracle/_ref/libsvtav1_ref.so).

RefFrame owns the host buffers of one frame set and a RefFrameJob (the C struct ref_frame_step /
ref_frames_run take).  Nothing here imports the product package: the workload module is loaded
stand-alone (pure numpy), so a process that only times the CPU arm never maps libsvtav1_b200.so.
"""
import ctypes as ct
import importlib
import os
import sys

import numpy as np

from . import support as me_np

_PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "svt-av1-psy_b200")
vp = ct.c_void_p


def load_workload_module():
    """svt-av1-psy_b200/workload.py + layout.py as top-level modules (no package __init__, no .so)"""
    if "svt_av1_psy_b200.workload" in sys.modules:  # the product package is already imported (tests, H100 arm)
        return sys.modules["svt_av1_psy_b200.workload"]
    if _PKG not in sys.path:
        sys.path.append(_PKG)
    return importlib.import_module("workload")


class RefFrameJob(ct.Structure):
    _fields_ = [("width", ct.c_int32), ("height", ct.c_int32), ("bit_depth", ct.c_int32), ("n_refs", ct.c_int32),
                ("cur", vp), ("refs", vp), ("me_cfg", vp),
                ("me", me_np.RefMeB64Out),
                ("residual", vp), ("coeff", vp), ("q", vp), ("dq", vp), ("scan", vp), ("iscan", vp), ("qm", vp),
                ("fwd", vp), ("qi", vp), ("inv", vp), ("eobs", vp),
                ("n_tx", ct.c_int64), ("n_coeffs", ct.c_int64),
                ("pred", vp), ("recon", vp), ("cdef_out", vp), ("final", vp), ("src", vp),
                ("padded_elems", ct.c_int64),
                ("plane_off", ct.c_int64 * 3),
                ("plane_stride", ct.c_int32 * 3), ("plane_w", ct.c_int32 * 3), ("plane_h", ct.c_int32 * 3), ("pad", ct.c_int32),
                ("src_off", ct.c_int64 * 3), ("src_stride", ct.c_int32 * 3), ("reserved0", ct.c_int32),
                ("skip", vp), ("str_y", vp), ("str_uv", vp),
                ("n_str", ct.c_int32), ("damping", ct.c_int32), ("subsampling", ct.c_int32), ("reserved1", ct.c_int32),
                ("mse", vp), ("dir", vp), ("var", vp),
                ("fb_idx", vp), ("apply_y", vp), ("apply_uv", vp),
                ("stats", vp), ("M", vp), ("H", vp), ("units", vp), ("n_stats", ct.c_int32), ("n_units", ct.c_int32),
                ("lr_units", vp * 3), ("lr_above", vp * 3), ("lr_below", vp * 3), ("lr_unit_size", ct.c_int32 * 3), ("lr_bstride", ct.c_int32 * 3),
                ("lr_stripes", ct.c_int32 * 3), ("reserved2", ct.c_int32)]


def me_cfg_for(wl):
    """the RefMeB64Cfg of the workload's ME picture (workload.ME_PICTURE and friends)"""
    m = sys.modules[type(wl).__module__]
    mp = wl.me_picture
    return me_np.me_b64_cfg(preset=wl.preset, qp=mp["qp"], n_ref=mp["n_ref"], poc_dist=m.ME_DIST, temporal_layer_index=m.ME_TEMPORAL_LAYER,
                            hierarchical_levels=m.ME_HIERARCHICAL_LEVELS, is_ref=m.ME_IS_REF, max_l=mp["max_l"], only_l_bwd=mp["only_l_bwd"],
                            safe_limit_nref=mp["safe_limit_nref"], gm_enabled=mp["gm_enabled"])


def aligned_zeros(n, dtype, align=64):
    """numpy array whose data pointer is `align`-byte aligned (the AVX2 kernels use aligned stores)"""
    isz = np.dtype(dtype).itemsize
    raw = np.zeros(n * isz + align, np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + n * isz].view(dtype)


def bind(ref):
    ref.ref_frame_step.restype = None
    ref.ref_frame_step.argtypes = [ct.POINTER(RefFrameJob)]
    ref.ref_frames_run.restype = ct.c_double
    ref.ref_frames_run.argtypes = [ct.POINTER(RefFrameJob), ct.c_int, ct.c_int, ct.c_int]
    ref.ref_set_threads.restype = ct.c_int
    ref.ref_set_threads.argtypes = [ct.c_int]


class RefFrame:
    def __init__(self, wl, ref):
        self.wl, self.ref = wl, ref
        bind(ref)
        W, H = wl.width, wl.height
        pix = wl.pixel_dtype
        self.cur_pyr = me_np.build_pyramid_np(wl.me_luma(wl.cur), W, H, wl.me_shapes)
        self.ref_pyrs = [me_np.build_pyramid_np(wl.me_luma(r), W, H, wl.me_shapes) for r in wl.refs]
        self.cur_desc = me_np.ref_pic_desc(self.cur_pyr, wl.me_shapes)
        self.ref_descs = (me_np.RefMePicture * wl.n_refs)(*[me_np.ref_pic_desc(p, wl.me_shapes) for p in self.ref_pyrs])
        self.me_cfg = me_cfg_for(wl)
        nb = ((W + 63) // 64) * ((H + 63) // 64)
        mc, mr, n_pu = wl.me_controls["max_cand"], wl.me_controls["max_refs"], wl.me_n_pu
        # svt_aom_motion_estimation_b64's outputs: MeSbResults + the pcs distortion arrays + the per-reference state
        self.me = {"total_me_candidate_index": np.zeros((nb, n_pu), np.uint8), "me_candidate_array": np.zeros((nb, n_pu * mc), np.uint8),
                   "me_mv_array": np.zeros((nb, n_pu * mr), np.uint32), "distortion": np.zeros((nb, 6), np.uint32),
                   "flags": np.zeros((nb, 2), np.uint8), "do_ref": np.zeros((nb, 2, 4), np.uint8),
                   "hme_centre": np.zeros((nb, 2, 4, 2), np.int16), "zz_sad": np.zeros((nb, 2, 4), np.uint32)}
        self.cur_flat = np.concatenate([p.reshape(-1) for p in wl.cur])
        res = np.concatenate([p.reshape(-1) for p in wl.residual])
        self.residual = aligned_zeros(res.size, np.int16)
        self.residual[:] = res
        off, n_pad = wl.padded_offsets()
        self.pred = self._pad_planes(wl.pred)
        self.recon = aligned_zeros(n_pad, pix)
        self.cdef_out = aligned_zeros(n_pad, pix)
        self.final = aligned_zeros(n_pad, pix)
        self.coeff = aligned_zeros(wl.n_coeffs, np.int32)
        self.q = aligned_zeros(wl.n_coeffs, np.int32)
        self.dq = aligned_zeros(wl.n_coeffs, np.int32)
        self.eobs = np.zeros(len(wl.quant_items), np.uint16)
        self.fwd = np.ascontiguousarray(wl.fwd_items)
        self.inv = np.ascontiguousarray(wl.inv_items)
        self.qi = np.ascontiguousarray(wl.quant_items)
        self.mse = np.zeros((2, nb, len(wl.cdef_str_y)), np.uint64)
        self.dirs = np.zeros((nb, 64), np.uint8)
        self.vars = np.zeros((nb, 64), np.int32)
        self.stats = np.ascontiguousarray(wl.stats_items)
        self.lr_units = [np.ascontiguousarray(u) for u in wl.lr_units]
        self.lr_above = [np.zeros(2 * wl.lr_num_stripes(p) * wl.lr_boundary_stride(p), pix) for p in range(3)]
        self.lr_below = [np.zeros(2 * wl.lr_num_stripes(p) * wl.lr_boundary_stride(p), pix) for p in range(3)]
        self.M = np.zeros((len(wl.stats_items), 49), np.int64)
        self.Hm = np.zeros((len(wl.stats_items), 2401), np.int64)
        self.job = self._make_job()

    def _pad_planes(self, planes):
        wl = self.wl
        off, n = wl.padded_offsets()
        buf = aligned_zeros(n, wl.pixel_dtype)
        for p in range(3):
            th, st = wl.padded_shape(p)
            w, h = wl.plane_dims[p]
            buf[off[p]:off[p] + th * st].reshape(th, st)[:, :w + 2 * wl.PAD] = np.pad(planes[p], wl.PAD, mode="edge")
        return buf

    def _make_job(self):
        wl = self.wl
        j = RefFrameJob()
        P = lambda a: a.ctypes.data  # noqa: E731
        j.width, j.height, j.bit_depth, j.n_refs = wl.width, wl.height, wl.bit_depth, wl.n_refs
        j.cur, j.refs, j.me_cfg = ct.addressof(self.cur_desc), ct.addressof(self.ref_descs), ct.addressof(self.me_cfg)
        for k, a in self.me.items():
            setattr(j.me, k, P(a))
        j.me.best_sad = j.me.best_mv = None
        j.residual, j.coeff, j.q, j.dq = P(self.residual), P(self.coeff), P(self.q), P(self.dq)
        j.scan, j.iscan, j.qm = P(wl.scan_table), P(wl.iscan_table), P(wl.qm_table)
        j.fwd, j.qi, j.inv, j.eobs = P(self.fwd), P(self.qi), P(self.inv), P(self.eobs)
        j.n_tx, j.n_coeffs = len(self.fwd), wl.n_coeffs
        j.pred, j.recon, j.cdef_out, j.final, j.src = P(self.pred), P(self.recon), P(self.cdef_out), P(self.final), P(self.cur_flat)
        off, n_pad = wl.padded_offsets()
        soff, _ = wl.flat_offsets()
        j.padded_elems = n_pad
        for p in range(3):
            th, st = wl.padded_shape(p)
            j.plane_off[p], j.plane_stride[p] = off[p], st
            j.plane_w[p], j.plane_h[p] = wl.plane_dims[p]
            j.src_off[p], j.src_stride[p] = soff[p], wl.plane_dims[p][0]
        j.pad = wl.PAD
        j.skip, j.str_y, j.str_uv = P(wl.skip8x8), P(wl.cdef_str_y), P(wl.cdef_str_uv)
        j.n_str, j.damping, j.subsampling = len(wl.cdef_str_y), wl.cdef_damping, wl.cdef_subsampling
        j.mse, j.dir, j.var = P(self.mse), P(self.dirs), P(self.vars)
        j.fb_idx, j.apply_y, j.apply_uv = P(wl.cdef_fb_idx), P(wl.cdef_apply_y), P(wl.cdef_apply_uv)
        j.stats, j.M, j.H, j.units = P(self.stats), P(self.M), P(self.Hm), None
        j.n_stats, j.n_units = len(self.stats), 0
        for p in range(3):
            j.lr_units[p], j.lr_above[p], j.lr_below[p] = P(self.lr_units[p]), P(self.lr_above[p]), P(self.lr_below[p])
            j.lr_unit_size[p], j.lr_bstride[p], j.lr_stripes[p] = wl.lr_unit_size[p], wl.lr_boundary_stride(p), wl.lr_num_stripes(p)
        return j

    def step(self):
        """one frame through the reference's kernels, outputs into this frame's own buffers (parity checks)"""
        self.ref.ref_frame_step(ct.byref(self.job))


def run_frames(ref, frames, n_frames, n_threads):
    """n_frames whole frames in flight over a persistent, core-pinned pool of n_threads (<=0: every host CPU);
    frame i uses frames[i % len(frames)]'s inputs and the worker's private output buffers.  Returns seconds."""
    bind(ref)
    jobs = (RefFrameJob * len(frames))(*[f.job for f in frames])
    return float(ref.ref_frames_run(jobs, len(frames), int(n_frames), int(n_threads)))
