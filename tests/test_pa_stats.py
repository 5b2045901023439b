"""Picture-analysis statistics (svt_aom_gathering_picture_statistics, pic_analysis_process.c:1559): the four block-mean
dispatch pointers (aom_dsp_rtcd.h:858-862) against the reference's C functions, and the T2 call svt_b200_picture_statistics_dev
against oracle/ref_pa_stats.c -- the reference's own function on the same padded picture and 1/16 picture, with every output
pre-filled with a sentinel so that the entries it does not write are known.  The oracle derives the controls through the
integration glue (svt_b200_pa_controls_from_scs) and stores the device results back into a pcs through it
(svt_b200_pa_store_results)."""
import ctypes as ct

import numpy as np
import pytest

from helpers import rng
from oracle import support as sp
from oracle_libs import pa_stats, refc  # noqa: F401  (fixtures; refc overrides conftest.py's in this module)

layout = sp.layout

# sentinels (bit patterns) of the outputs: an entry that still holds one after a call was not written
S16, S32, S64 = 0xA5A5, 0xA5A5A5A5, 0xA5A5A5A5A5A5A5A5


class RefPaStatsCfg(ct.Structure):
    _fields_ = [(n, ct.c_int32) for n in ("calculate_variance", "block_mean_calc_prec", "enable_adaptive_quantization", "variance_octile",
                                          "calc_hist", "scene_change_detection", "regions_w", "regions_h")]


class RefPaStatsOut(ct.Structure):
    _fields_ = [(n, ct.c_void_p) for n in ("variance", "pic_avg_variance", "histogram", "average_intensity", "avg_luma")]


@pytest.fixture(scope="module")
def pa(pa_stats):
    pa_stats.ref_pa_stats.argtypes = [ct.c_void_p] * 4
    pa_stats.ref_pa_stats.restype = ct.c_int
    pa_stats.ref_pa_stats_store.argtypes = [ct.c_void_p, ct.c_void_p, ct.c_void_p, ct.c_uint16, ct.c_void_p, ct.c_void_p, ct.c_uint64, ct.c_void_p]
    pa_stats.ref_pa_stats_store.restype = ct.c_int
    return pa_stats


def cfg(var=1, sub=1, var8=1, hist=1, scd=0, regions=(4, 4)):
    """defaults: what the encoder runs with variance boost and the temporal filter on (enc_handle.c:4207-4254)"""
    c = RefPaStatsCfg()
    c.calculate_variance, c.block_mean_calc_prec, c.variance_octile, c.calc_hist, c.scene_change_detection = var, sub, 6 if var8 else 0, hist, scd
    c.enable_adaptive_quantization = 0
    c.regions_w, c.regions_h = regions
    return c


def picture(W, H, content, seed):
    r = rng(seed)
    if content == "flat":
        full = np.full((H, W), int(r.integers(0, 256)), np.uint8)
    elif content == "gradient":
        y, x = np.mgrid[0:H, 0:W]
        full = ((3 * x + 2 * y) // 5 % 256).astype(np.uint8)
    elif content == "extreme":
        full = np.where(r.random((H, W)) < 0.5, 0, 255).astype(np.uint8)
    else:
        full = r.integers(0, 256, (H, W), dtype=np.uint8)
    shapes = layout.me_plane_shapes(W, H)
    return sp.build_pyramid_np(full, W, H, shapes), shapes


def sentinel_outputs(n_b64, rw, rh):
    return {"variance": np.full((n_b64, 85), S16, np.uint16), "pic_avg_variance": np.full(1, S16, np.uint16),
            "histogram": np.full((rw, rh, 256), S32, np.uint32), "average_intensity": np.full((rw, rh), S64, np.uint64),
            "avg_luma": np.full(1, S64, np.uint64)}


def _out_struct(o):
    return RefPaStatsOut(*[o[n].ctypes.data for n, _ in RefPaStatsOut._fields_])


def ref_stats(pa, planes, shapes, c):
    """-> (glue controls, the reference's outputs)"""
    W, H = shapes[2][3], shapes[2][4]
    o = sentinel_outputs(((W + 63) // 64) * ((H + 63) // 64), c.regions_w, c.regions_h)
    ctl = layout.PaStatsControls()
    d = sp.ref_pic_desc(planes, shapes)
    assert pa.ref_pa_stats(ct.byref(d), ct.byref(c), ct.byref(ctl), ct.byref(_out_struct(o))) == 0
    return ctl, o


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle driver == a direct loop over the reference's T1 C functions
# ---------------------------------------------------------------------------------------------------------------------
def _tree(m8, q8):
    """the u64 '>> 2 of four' tree of compute_block_mean_compute_variance -> 85 variances (me_context.h:54 order)"""
    m8, q8 = m8.reshape(8, 8), q8.reshape(8, 8)
    quad = lambda a: (a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2]) >> np.uint64(2)  # noqa: E731
    m16, q16 = quad(m8), quad(q8)
    m32, q32 = quad(m16), quad(q16)
    m64, q64 = quad(m32), quad(q32)
    var = lambda q, m: ((q - m * m) >> np.uint64(16)).astype(np.uint16).reshape(-1)  # noqa: E731  (u64 wrap like the reference)
    return np.concatenate([var(q64, m64), var(q32, m32), var(q16, m16), var(q8, m8)])


def test_oracle_equals_a_loop_over_the_reference_t1_functions(pa, refc):
    W, H = 200, 136
    planes, shapes = picture(W, H, "random", 300)
    _, stride, pad, _, _ = shapes[2]
    full = planes[2].reshape(-1)
    P = lambda off: ct.c_void_p(full.ctypes.data + int(off))  # noqa: E731
    for f in (refc.svt_compute_mean_c, refc.svt_compute_mean_squared_values_c):
        f.restype = ct.c_uint64
        f.argtypes = [ct.c_void_p, ct.c_uint32, ct.c_uint32, ct.c_uint32]
    refc.svt_compute_interm_var_four8x8_c.argtypes = [ct.c_void_p, ct.c_uint16, ct.c_void_p, ct.c_void_p]
    refc.svt_compute_interm_var_four8x8_c.restype = None
    bw, bh = (W + 63) // 64, (H + 63) // 64
    for sub in (0, 1):
        _, got = ref_stats(pa, planes, shapes, cfg(sub=sub, hist=0))
        want = np.zeros((bw * bh, 85), np.uint16)
        for b in range(bw * bh):
            o = (pad + 64 * (b // bw)) * stride + pad + 64 * (b % bw)
            m8, q8 = np.zeros(64, np.uint64), np.zeros(64, np.uint64)
            for k in range(64):
                bo = o + 8 * (k // 8) * stride + 8 * (k % 8)
                if sub:
                    if k % 4 == 0:
                        refc.svt_compute_interm_var_four8x8_c(P(bo), stride, m8[k:].ctypes.data, q8[k:].ctypes.data)
                else:
                    m8[k] = refc.svt_compute_mean_c(P(bo), stride, 8, 8)
                    q8[k] = refc.svt_compute_mean_squared_values_c(P(bo), stride, 8, 8)
            want[b] = _tree(m8, q8)
        assert np.array_equal(got["variance"], want), sub
        assert int(got["pic_avg_variance"][0]) == int(want[:, 0].astype(np.uint64).sum()) // (bw * bh)
    # histograms: calculate_histogram (pic_analysis_process.c:166) per region, bins from 1, scaled by 16 * d^2
    refc.calculate_histogram.argtypes = [ct.c_void_p, ct.c_uint32, ct.c_uint32, ct.c_uint32, ct.c_uint8, ct.c_void_p, ct.c_void_p]
    refc.calculate_histogram.restype = None
    _, s16, p16, w16, h16 = shapes[0]
    six = planes[0].reshape(-1)
    for scd in (0, 1):
        d = 1 if scd else 4
        _, got = ref_stats(pa, planes, shapes, cfg(var=0, scd=scd))
        rw, rh = w16 // 4, h16 // 4
        total = 0
        for i in range(4):
            for j in range(4):
                ww, hh = rw + (w16 - 4 * rw if i == 3 else 0), rh + (h16 - 4 * rh if j == 3 else 0)
                hist, s = np.ones(256, np.uint32), ct.c_uint64(0)
                refc.calculate_histogram(ct.c_void_p(six.ctypes.data + (p16 + j * rh) * s16 + p16 + i * rw), ww, hh, s16, d, hist.ctypes.data,
                                         ct.byref(s))
                assert np.array_equal(got["histogram"][i, j], hist * np.uint32(16 * d * d)), (scd, i, j)
                ssum = s.value * d * d
                assert int(got["average_intensity"][i, j]) == ((ssum + (ww * hh >> 1)) // (ww * hh)) & 0xff
                total += ssum
        assert int(got["avg_luma"][0]) == total // (w16 * h16)
        assert int(got["pic_avg_variance"][0]) == 0  # calculate_variance off


# ---------------------------------------------------------------------------------------------------------------------
# GPU: T1 pointers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_t1_block_means_against_reference(b200, refc):
    r = rng(301)
    f_mean, f_sq = refc.svt_compute_mean_c, refc.svt_compute_mean_squared_values_c
    for f in (f_mean, f_sq):
        f.restype = ct.c_uint64
        f.argtypes = [ct.c_void_p, ct.c_uint32, ct.c_uint32, ct.c_uint32]
    refc.svt_compute_sub_mean_8x8_c.argtypes = [ct.c_void_p, ct.c_uint16]
    refc.svt_compute_sub_mean_8x8_c.restype = ct.c_uint64
    refc.svt_compute_interm_var_four8x8_c.argtypes = [ct.c_void_p, ct.c_uint16, ct.c_void_p, ct.c_void_p]
    refc.svt_compute_interm_var_four8x8_c.restype = None
    for trial in range(12):
        kind = ("random", "zero", "max")[trial % 3]
        stride = (40, 72, 8 + 32, 1000)[trial % 4]
        fill = lambda n: {"random": r.integers(0, 256, n, dtype=np.uint8), "zero": np.zeros(n, np.uint8),  # noqa: E731
                          "max": np.full(n, 255, np.uint8)}[kind]
        # every buffer ends exactly at the last pixel the call reads
        for w, h in ((8, 8), (16, 4), (5, 7)):
            buf = fill((h - 1) * stride + w)
            p = ct.c_void_p(buf.ctypes.data)
            assert b200.lib.svt_b200_compute_mean_8x8(p, stride, w, h) == f_mean(p, stride, w, h), (trial, w, h)
            assert b200.lib.svt_b200_compute_mean_square_values_8x8(p, stride, w, h) == f_sq(p, stride, w, h), (trial, w, h)
        buf = fill(6 * stride + 8)
        p = ct.c_void_p(buf.ctypes.data)
        assert b200.lib.svt_b200_compute_sub_mean_8x8(p, stride) == refc.svt_compute_sub_mean_8x8_c(p, stride), trial
        buf = fill(6 * stride + 32)
        p = ct.c_void_p(buf.ctypes.data)
        got = [np.full(4, S64, np.uint64) for _ in range(2)]
        want = [np.full(4, S64, np.uint64) for _ in range(2)]
        b200.lib.svt_b200_compute_interm_var_four8x8(p, stride, got[0].ctypes.data, got[1].ctypes.data)
        refc.svt_compute_interm_var_four8x8_c(p, stride, want[0].ctypes.data, want[1].ctypes.data)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), trial


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the whole-picture call against the reference's own function
# ---------------------------------------------------------------------------------------------------------------------
# the encoder's default; FULL precision with the 8x8 flag off and scene-change sampling; histograms only; variances only
CFGS = [dict(), dict(sub=0, var8=0, scd=1), dict(var=0, var8=0, scd=1), dict(sub=0, hist=0)]


def _device_planes(planes):
    import torch
    return [torch.from_numpy(p).cuda() for p in planes]


def _desc(dsp, dplanes, shapes):
    d = dsp.MePicture()
    for lvl, (th, stride, pad, w, h) in enumerate(shapes):
        d.plane[lvl] = dplanes[lvl].data_ptr()
        d.stride[lvl], d.org_x[lvl], d.org_y[lvl], d.width[lvl], d.height[lvl] = stride, pad, pad, w, h
    return d


def _check(b200, pa, planes, dplanes, shapes, c, label):
    import torch
    ctl, want = ref_stats(pa, planes, shapes, c)
    rc, out = b200.picture_statistics_dev(_desc(b200, dplanes, shapes), b200.PaStatsControls.from_buffer_copy(ctl), torch)
    assert rc == 0, label
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    got = {"variance": got["variance"].view(np.uint16), "pic_avg_variance": got["pic_avg_variance"].view(np.uint16),
           "histogram": got["histogram"].view(np.uint32), "average_intensity": got["average_intensity"],
           "avg_luma": got["avg_luma"].view(np.uint64)}
    if c.calculate_variance:
        assert np.array_equal(got["variance"][:, 0], want["variance"][:, 0]), label
        if c.variance_octile:
            assert np.array_equal(got["variance"], want["variance"]), label
        else:  # the reference leaves 1..84; the device writes 0 there
            assert np.all(want["variance"][:, 1:] == S16) and np.all(got["variance"][:, 1:] == 0), label
    else:
        assert np.all(want["variance"] == S16) and np.all(got["variance"] == S16), label
    if c.calc_hist:
        assert np.array_equal(got["histogram"], want["histogram"]), label
        assert np.array_equal(got["average_intensity"].astype(np.uint64), want["average_intensity"]), label
    else:
        assert np.all(want["histogram"] == S32) and np.all(got["histogram"] == S32), label
        assert np.all(want["average_intensity"] == S64) and np.all(got["average_intensity"] == 0xA5), label
    assert got["pic_avg_variance"][0] == want["pic_avg_variance"][0], label
    assert got["avg_luma"][0] == want["avg_luma"][0], label
    # the glue stores the device results into a pcs exactly as the reference's function left it
    back = sentinel_outputs(*want["variance"].shape[:1], c.regions_w, c.regions_h)
    assert pa.ref_pa_stats_store(ct.byref(sp.ref_pic_desc(planes, shapes)), ct.byref(c), got["variance"].ctypes.data,
                                 int(got["pic_avg_variance"][0]), got["histogram"].ctypes.data, got["average_intensity"].ctypes.data,
                                 int(got["avg_luma"][0]), ct.byref(_out_struct(back))) == 0
    for k in want:
        assert np.array_equal(back[k], want[k]), (label, k)


@pytest.mark.gpu
@pytest.mark.parametrize("content", ["flat", "random", "gradient", "extreme"])
@pytest.mark.parametrize("size", [(640, 360), (1920, 1080), (3840, 2160), (1000, 564), (48, 40)])
def test_picture_statistics_dev_against_reference(b200, pa, size, content):
    """every configuration of CFGS, bit for bit on every entry the reference writes; 1000x564: partial 64x64 blocks and regions
    with remainders; 48x40: the 1-region split the encoder uses below 64 pixels (enc_handle.c:4248)"""
    W, H = size
    planes, shapes = picture(W, H, content, 310 + W + H)
    dplanes = _device_planes(planes)
    regions = (4, 4) if W >= 64 else (1, 1)
    for k in CFGS:
        _check(b200, pa, planes, dplanes, shapes, cfg(regions=regions, **k), (size, content, k))


@pytest.mark.gpu
def test_picture_statistics_on_device_padded_pyramid(b200, pa):
    """the frame path's inputs: the full plane's padding replicated by svt_b200_extend_plane_dev and the 1/4 and 1/16 planes
    built by svt_b200_build_hme_pyramid_dev; region counts other than 4 x 4"""
    import torch
    W, H = 1000, 564
    shapes = layout.me_plane_shapes(W, H)
    full = rng(320).integers(0, 256, (H, W), dtype=np.uint8)
    dplanes = [torch.zeros((s[0], s[1]), dtype=torch.uint8, device="cuda") for s in shapes]
    pad = shapes[2][2]
    dplanes[2][pad:pad + H, pad:pad + W] = torch.from_numpy(full).cuda()
    assert b200.lib.svt_b200_extend_plane_dev(ct.c_void_p(dplanes[2].data_ptr()), shapes[2][1], W, H, pad, pad, None) == 0
    d = _desc(b200, dplanes, shapes)
    assert b200.lib.svt_b200_build_hme_pyramid_dev(ct.byref(d), None) == 0
    torch.cuda.synchronize()
    planes = [p.cpu().numpy() for p in dplanes]
    for regions in ((4, 4), (3, 2), (1, 4)):
        for k in CFGS[:2]:
            _check(b200, pa, planes, dplanes, shapes, cfg(regions=regions, **k), (regions, k))


@pytest.mark.gpu
def test_picture_statistics_rejects_bad_arguments(b200):
    import torch
    W, H = 320, 200
    planes, shapes = picture(W, H, "random", 330)
    dplanes = _device_planes(planes)
    good = b200.PaStatsControls(1, 1, 1, 1, 4, 4, 4, 0)
    assert b200.picture_statistics_dev(_desc(b200, dplanes, shapes), good, torch)[0] == 0

    def bad(ctl=None, **pic):
        d = _desc(b200, dplanes, shapes)
        for k, (lvl, v) in pic.items():
            getattr(d, k)[lvl] = v
        c = b200.PaStatsControls.from_buffer_copy(good)
        for k, v in (ctl or {}).items():
            setattr(c, k, v)
        l0 = b200.launch_count()
        rc, out = b200.picture_statistics_dev(d, c, torch)
        assert rc == -4 and b200.launch_count() == l0, (ctl, pic)

    bad(plane=(2, None))
    bad(plane=(0, None))
    bad({"regions_w": 0})
    bad({"regions_h": 0})
    bad({"regions_w": 5})
    bad({"decim_step": 2})
    bad({"block_mean_calc_prec": 2})
    bad(stride=(2, shapes[2][2] + W - 16), width=(2, W - 16))  # no room right of a partial 64x64 block
    bad(org_y=(2, 0), org_x=(2, 0), height=(2, 190))  # a partial bottom block without padding below
    bad(width=(0, 3))                               # 1/16 plane narrower than its regions
    bad(stride=(0, 10))
    # a disabled part's fields are not checked
    d = _desc(b200, dplanes, shapes)
    d.plane[0] = None
    c = b200.PaStatsControls.from_buffer_copy(good)
    c.calc_hist, c.regions_w = 0, 0
    assert b200.picture_statistics_dev(d, c, torch)[0] == 0
