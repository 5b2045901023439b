"""TEST / BASELINE INFRASTRUCTURE: the structs oracle/ref_driver.c and oracle/ref_me_b64.c take beyond the product's
(include/svt_b200.h, described by svt-av1-psy_b200/layout.py) and the numpy input preparation (padded HME pyramid) shared by
tests/ and bench.py's reference arm."""
import ctypes as ct
import importlib
import os
import sys

import numpy as np

_PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "svt-av1-psy_b200")


def load_pkg_module(name):
    """svt-av1-psy_b200/<name>.py for the pure-numpy modules (layout, workload): the product package's own module when the
    package is already imported (tests, H100 arm), else the file as a top-level module (no package __init__, no .so)"""
    if "svt_av1_psy_b200." + name in sys.modules:
        return sys.modules["svt_av1_psy_b200." + name]
    if _PKG not in sys.path:
        sys.path.append(_PKG)
    return importlib.import_module(name)


layout = load_pkg_module("layout")
ME_CONTROL_FIELDS, MeControls, MePicture, CdefFrame = layout.ME_CONTROL_FIELDS, layout.MeControls, layout.MePicture, layout.CdefFrame


def pad_np(buf, pad, w, h):
    inner = buf[pad:pad + h, pad:pad + w].copy()
    buf[:, :] = np.pad(inner, ((pad, buf.shape[0] - pad - h), (pad, buf.shape[1] - pad - w)), mode="edge")
    return buf


def build_pyramid_np(full, width, height, shapes):
    """numpy restatement of svt_aom_downsample_2d_c + svt_aom_generate_padding
    (pic_analysis_process.c:130-160, 2138-2190).  tests/test_me_pyramid.py checks it against the device pyramid
    (test_build_hme_pyramid_dev), whose downsampling it checks against svt_aom_downsample_2d_c (test_downsample_2d_t1)."""
    planes = [None, None, None]
    th, stride, pad, w, h = shapes[2]
    buf = np.zeros((th, stride), np.uint8)
    buf[pad:pad + h, pad:pad + w] = full
    planes[2] = pad_np(buf, pad, w, h)
    src = full.astype(np.uint32)
    for lvl in (1, 0):
        th, stride, pad, w, h = shapes[lvl]
        d = ((src[0::2, 0::2] + src[0::2, 1::2] + src[1::2, 0::2] + src[1::2, 1::2] + 2) >> 2)[:h, :w]
        buf = np.zeros((th, stride), np.uint8)
        buf[pad:pad + h, pad:pad + w] = d
        planes[lvl] = pad_np(buf, pad, w, h)
        src = d.astype(np.uint32)
    return planes


def ref_pic_desc(planes, shapes):
    p = MePicture()
    for lvl, (th, stride, pad, w, h) in enumerate(shapes):
        p.plane[lvl] = planes[lvl].ctypes.data
        p.stride[lvl] = stride
        p.org_x[lvl] = p.org_y[lvl] = pad
        p.width[lvl] = w
        p.height[lvl] = h
    return p


# ---- oracle/ref_me_b64.c: the reference's own svt_aom_motion_estimation_b64 over a picture ------------------
class RefMeB64Cfg(ct.Structure):
    _fields_ = [(n, ct.c_int32) for n in ("enc_mode", "qp", "hierarchical_levels", "temporal_layer_index", "is_ref", "sc_class1")] + \
               [("n_ref", ct.c_int32 * 2), ("ref_poc_dist_sign", (ct.c_int32 * 4) * 2)] + \
               [(n, ct.c_int32) for n in ("enable_hme_flag", "enable_hme_level0_flag", "enable_hme_level1_flag", "enable_hme_level2_flag",
                                          "max_l0", "max_l1", "only_l_bwd", "safe_limit_nref", "safe_limit_zz_th", "similar_brightness_refs",
                                          "gm_enabled", "gm_use_distance_based_active_th", "frame_rate_q16")] + [("reserved", ct.c_int32 * 3)]


class RefMeB64Out(ct.Structure):
    _fields_ = [(n, ct.c_void_p) for n in ("total_me_candidate_index", "me_candidate_array", "me_mv_array", "distortion", "flags", "do_ref",
                                           "hme_centre", "zz_sad", "best_sad", "best_mv")]


def me_b64_cfg(preset=8, qp=30, n_ref=(2, 2), poc_dist=((-1, -3, 0, 0), (1, 3, 0, 0)), temporal_layer_index=3, hierarchical_levels=4,
               is_ref=0, max_l=(3, 2), only_l_bwd=1, safe_limit_nref=2, gm_enabled=0):
    """defaults: a non-base, non-reference B picture of the preset-8 CRF random-access configuration (MRP level 10,
    enc_handle.c:3559-3577: 2+2 references tried on non-base pictures, storage sized for 3+2; 5-layer hierarchy)"""
    c = RefMeB64Cfg()
    c.enc_mode, c.qp, c.hierarchical_levels, c.temporal_layer_index, c.is_ref, c.sc_class1 = preset, qp, hierarchical_levels, temporal_layer_index, is_ref, 0
    c.n_ref[0], c.n_ref[1] = n_ref
    for li in range(2):
        for r in range(4):
            c.ref_poc_dist_sign[li][r] = poc_dist[li][r]
    c.enable_hme_flag = c.enable_hme_level0_flag = c.enable_hme_level1_flag = c.enable_hme_level2_flag = 1
    c.max_l0, c.max_l1 = max_l
    c.only_l_bwd, c.safe_limit_nref, c.safe_limit_zz_th, c.similar_brightness_refs = only_l_bwd, safe_limit_nref, 0, 0
    c.gm_enabled, c.gm_use_distance_based_active_th, c.frame_rate_q16 = gm_enabled, 0, 30 << 16
    return c


def ref_me_b64_picture(ref, cur_pyr, ref_pyrs, shapes, cfg, run=True):
    """-> (controls dict, outputs dict of numpy arrays or None)"""
    W, H = shapes[2][3], shapes[2][4]
    nb = ((W + 63) // 64) * ((H + 63) // 64)
    ref.ref_me_b64_num_pus.restype = ct.c_int
    n_pu = ref.ref_me_b64_num_pus(cfg.enc_mode, W, H)
    cd = ref_pic_desc(cur_pyr, shapes)
    rd = (MePicture * len(ref_pyrs))(*[ref_pic_desc(p, shapes) for p in ref_pyrs])
    ctrl = MeControls()
    ref.ref_me_b64_picture.restype = ct.c_int
    ref.ref_me_b64_picture.argtypes = [ct.c_void_p] * 5
    if not run:
        ref.ref_me_b64_picture(ct.byref(cd), rd, ct.byref(cfg), ct.byref(ctrl), None)
        return ctrl, None
    ref.ref_me_b64_picture(ct.byref(cd), rd, ct.byref(cfg), ct.byref(ctrl), None)  # sizes first
    mc, mr = ctrl.max_cand, ctrl.max_refs
    arrs = {"total_me_candidate_index": np.zeros((nb, n_pu), np.uint8), "me_candidate_array": np.zeros((nb, n_pu * mc), np.uint8),
            "me_mv_array": np.zeros((nb, n_pu * mr), np.uint32), "distortion": np.zeros((nb, 6), np.uint32), "flags": np.zeros((nb, 2), np.uint8),
            "do_ref": np.zeros((nb, 2, 4), np.uint8), "hme_centre": np.zeros((nb, 2, 4, 2), np.int16), "zz_sad": np.zeros((nb, 2, 4), np.uint32),
            "best_sad": np.zeros((nb, 2, 4, 85), np.uint32), "best_mv": np.zeros((nb, 2, 4, 85), np.uint32)}
    out = RefMeB64Out()
    for n, _ in RefMeB64Out._fields_:
        setattr(out, n, arrs[n].ctypes.data)
    assert ref.ref_me_b64_picture(ct.byref(cd), rd, ct.byref(cfg), ct.byref(ctrl), ct.byref(out)) == 0
    return ctrl, arrs
