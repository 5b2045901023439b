"""Host-side mirror of the reference's dispatched DSP functions, bound to libsvtav1_b200.so.

Function names and argument meaning follow the reference's function pointers
(Source/Lib/Codec/aom_dsp_rtcd.h / common_dsp_rtcd.h); buffers are numpy arrays where the C code
takes pointers.  Every call goes through the C ABI (include/svt_b200.h) -- nothing here computes.
"""
import ctypes as ct

import numpy as np

from . import lib, prototypes
from .layout import *  # noqa: F401,F403  (the header's structs and item dtypes, enum values, plane geometry: no library, shared with the CPU arm)

vp = ct.c_void_p


def _ptr(a, byte_off=0):
    """pointer to (a.data + byte_off); `a` must be a numpy array (kept alive by the caller)."""
    if a is None:
        return ct.cast(0, vp)
    return ct.cast(a.ctypes.data + int(byte_off), vp)


# every function of the C ABI gets the ctypes signature of its prototype in exports.txt
for _name, _ret, _params in prototypes():
    _f = getattr(lib, _name)
    _f.restype = ctype(_ret, returned=True)
    _f.argtypes = [ctype(_p) for _p in _params]

_initialised = False


def init(device=0):
    """Bind the library to a CUDA device (svt_b200_init).  Raises if no sm_90 device is usable."""
    global _initialised
    rc = lib.svt_b200_init(int(device))
    if rc != 0:
        raise RuntimeError("svt_b200_init(%d) failed with %d: an sm_90 (H100) device is required; "
                           "there is no CPU fallback" % (device, rc))
    _initialised = True
    return rc


def shutdown():
    global _initialised
    lib.svt_b200_shutdown()
    _initialised = False


def launch_count():
    return int(lib.svt_b200_launch_count())


# ------------------------------------------------------------------------------------------------
# K1 / K3
# ------------------------------------------------------------------------------------------------
def svt_sad_loop_kernel(src, src_off, src_stride, ref, ref_off, ref_stride, block_height, block_width,
                        src_stride_raw, skip_search_line, search_area_width, search_area_height,
                        x_init=0, y_init=0):
    """aom_dsp_rtcd.h:779.  `src`/`ref` are flat uint8 arrays, *_off the element offsets of the block /
    window origin.  Returns (best_sad, x_search_center, y_search_center)."""
    best = ct.c_uint64(0)
    xs = ct.c_int16(x_init)
    ys = ct.c_int16(y_init)
    lib.svt_b200_sad_loop_kernel(_ptr(src, src_off), src_stride, _ptr(ref, ref_off), ref_stride, block_height,
                                 block_width, ct.byref(best), ct.byref(xs), ct.byref(ys), src_stride_raw,
                                 skip_search_line, search_area_width, search_area_height)
    return int(best.value), int(xs.value), int(ys.value)


def svt_nxm_sad_kernel(src, src_off, src_stride, ref, ref_off, ref_stride, height, width):
    return int(lib.svt_b200_nxm_sad_kernel(_ptr(src, src_off), src_stride, _ptr(ref, ref_off), ref_stride,
                                           height, width))


def sad_search_batch_host(src_plane, ref_plane, items):
    """T2: items is a numpy structured array of SAD_ITEM_DTYPE; returns SAD_RESULT_DTYPE array."""
    items = np.ascontiguousarray(items, dtype=SAD_ITEM_DTYPE)
    res = np.zeros(len(items), dtype=SAD_RESULT_DTYPE)
    rc = lib.svt_b200_sad_search_batch_host(_ptr(src_plane), src_plane.nbytes, _ptr(ref_plane), ref_plane.nbytes,
                                            _ptr(items), len(items), _ptr(res))
    if rc != 0:
        raise RuntimeError("svt_b200_sad_search_batch_host rc=%d" % rc)
    return res


# ------------------------------------------------------------------------------------------------
# K5 / K6 transforms
# ------------------------------------------------------------------------------------------------
def txfm_valid(tx_size, tx_type):
    return bool(lib.svt_b200_txfm_valid(tx_size, tx_type))


def svt_av1_fwd_txfm2d(residual, stride, tx_type, tx_size, bit_depth=8, named=False):
    """svt_av1_fwd_txfm2d_WxH: int16 residual (flat, `stride`) -> int32[W*H]."""
    out = np.zeros(TX_W[tx_size] * TX_H[tx_size], np.int32)
    if named:
        getattr(lib, "svt_b200_av1_fwd_txfm2d_" + TX_NAME[tx_size])(_ptr(residual), _ptr(out), stride, tx_type, bit_depth)
    else:
        lib.svt_b200_fwd_txfm2d(_ptr(residual), _ptr(out), stride, tx_type, tx_size, bit_depth)
    return out


def svt_av1_fwd_txfm2d_partial(residual, stride, tx_type, tx_size, level, bit_depth=8, named=False):
    """svt_av1_fwd_txfm2d_WxH_N2 (level 1) / _N4 (level 2); the output buffer is pre-filled with a sentinel
    so that the test also sees that every element is written."""
    out = np.full(TX_W[tx_size] * TX_H[tx_size], 0x5a5a5a5a, np.int32)
    if named:
        getattr(lib, "svt_b200_av1_fwd_txfm2d_%s_N%d" % (TX_NAME[tx_size], 2 * level))(_ptr(residual), _ptr(out), stride, tx_type, bit_depth)
    else:
        lib.svt_b200_fwd_txfm2d_partial(_ptr(residual), _ptr(out), stride, tx_type, tx_size, bit_depth, level)
    return out


def svt_av1_inv_txfm2d_add(coeff, pred, stride_r, stride_w, tx_type, tx_size, bd):
    """svt_av1_inv_txfm2d_add_WxH on uint16 pixels; returns the written recon plane (H*stride_w)."""
    out = np.zeros(TX_H[tx_size] * stride_w, np.uint16)
    lib.svt_b200_inv_txfm2d_add(_ptr(coeff), _ptr(pred), stride_r, _ptr(out), stride_w, tx_type, tx_size, bd)
    return out


def svt_av1_inv_txfm2d_add_named(coeff, pred, stride_r, stride_w, tx_type, tx_size, bd):
    """the per-size named entry point (same argument list as the reference pointer of that size: after tx_type, the
    sizes take (bd), (tx_size, bd) or (tx_size, eob, bd))"""
    out = np.zeros(TX_H[tx_size] * stride_w, np.uint16)
    g = getattr(lib, "svt_b200_av1_inv_txfm2d_add_" + TX_NAME[tx_size])
    tail = {7: [bd], 8: [tx_size, bd], 9: [tx_size, TX_W[tx_size] * TX_H[tx_size], bd]}[len(g.argtypes)]
    g(_ptr(coeff), _ptr(pred), stride_r, _ptr(out), stride_w, tx_type, *tail)
    return out


def svt_av1_inv_txfm_add(coeff, pred8, stride_r, stride_w, tx_type, tx_size):
    out = np.zeros(TX_H[tx_size] * stride_w, np.uint8)
    lib.svt_b200_inv_txfm_add_8bit(_ptr(coeff), _ptr(pred8), stride_r, _ptr(out), stride_w, tx_type, tx_size)
    return out


def fwd_txfm_batch_host(residual, coeff, items):
    items = np.ascontiguousarray(items, dtype=FWD_ITEM_DTYPE)
    rc = lib.svt_b200_fwd_txfm_batch_host(_ptr(residual), residual.size, _ptr(coeff), coeff.size, _ptr(items), len(items))
    if rc != 0:
        raise RuntimeError("svt_b200_fwd_txfm_batch_host rc=%d" % rc)
    return coeff

# ------------------------------------------------------------------------------------------------
# K7 quantize / dequantize
# ------------------------------------------------------------------------------------------------
def quantize(name, coeff, tables, scan, qm=None, iqm=None, log_scale=None):
    """Call the T1 quantizer `name` (reference pointer name without the svt_ prefix, e.g.
    'aom_quantize_b', 'av1_quantize_fp_qm').  tables = dict(zbin, round, quant, quant_shift, dequant) of
    int16[2].  Returns (qcoeff, dqcoeff, eob)."""
    n = coeff.size
    q = np.full(n, 0x5a5a5a5a, np.int32)
    dq = np.full(n, 0x5a5a5a5a, np.int32)
    eob = ct.c_uint16(0xffff)
    args = [_ptr(coeff), n, _ptr(tables["zbin"]), _ptr(tables["round"]), _ptr(tables["quant"]),
            _ptr(tables["quant_shift"]), _ptr(q), _ptr(dq), _ptr(tables["dequant"]), ct.cast(ct.byref(eob), vp),
            _ptr(scan), _ptr(scan)]
    f = getattr(lib, "svt_b200_" + name)
    nextra = len(f.argtypes) - 12
    if nextra == 3:
        args += [_ptr(qm), _ptr(iqm), log_scale]
    elif nextra == 1:
        args += [log_scale]
    f(*args)
    return q, dq, int(eob.value)

# ------------------------------------------------------------------------------------------------
# K4 Hadamard / SATD, K2 SAD pyramid + full-pel search
# ------------------------------------------------------------------------------------------------
def svt_aom_hadamard(src_diff, stride, n):
    out = np.zeros(n * n, np.int32)
    getattr(lib, "svt_b200_aom_hadamard_%dx%d" % (n, n))(_ptr(src_diff), stride, _ptr(out))
    return out


def svt_aom_satd(coeff):
    return int(lib.svt_b200_aom_satd(_ptr(coeff), coeff.size))


def fullpel_search_batch_host(src_plane, ref_plane, items):
    items = np.ascontiguousarray(items, dtype=FULLPEL_ITEM_DTYPE)
    sad = np.zeros((len(items), 85), np.uint32)
    mv = np.zeros((len(items), 85), np.uint32)
    rc = lib.svt_b200_fullpel_search_batch_host(_ptr(src_plane), src_plane.nbytes, _ptr(ref_plane), ref_plane.nbytes,
                                                _ptr(items), len(items), _ptr(sad), _ptr(mv))
    if rc != 0:
        raise RuntimeError("svt_b200_fullpel_search_batch_host rc=%d" % rc)
    return sad, mv

# ------------------------------------------------------------------------------------------------
# K8 CDEF
# ------------------------------------------------------------------------------------------------
def cdef_frame_desc(rec, src, width, height, bit_depth, damping, subsampling):
    """rec/src: lists of three 2-D torch CUDA tensors (uint8 or int16/uint16 storage)."""
    f = CdefFrame()
    f.recon_y, f.recon_cb, f.recon_cr = (t.data_ptr() for t in rec)
    f.src_y, f.src_cb, f.src_cr = (t.data_ptr() for t in src)
    f.recon_stride_y, f.recon_stride_c = rec[0].stride(0), rec[1].stride(0)
    f.src_stride_y, f.src_stride_c = src[0].stride(0), src[1].stride(0)
    f.width, f.height, f.bit_depth, f.damping, f.subsampling_factor = width, height, bit_depth, damping, subsampling
    return f

# ------------------------------------------------------------------------------------------------
# K14 deblocking loop filter
# ------------------------------------------------------------------------------------------------
def svt_aom_lpf(direction, taps, buf, offset, pitch, blimit, limit, thresh, bd=None):
    """svt_aom_{,highbd_}lpf_<direction>_<taps> on a numpy buffer (uint8, or uint16 with bd) at element `offset`, in place"""
    hb = buf.dtype == np.uint16
    name = "svt_b200_aom_%slpf_%s_%d" % ("highbd_" if hb else "", direction, taps)
    th = [np.full(16, v, np.uint8) for v in (blimit, limit, thresh)]
    args = [_ptr(buf, byte_off=offset * buf.itemsize), pitch] + [_ptr(t) for t in th] + ([bd] if hb else [])
    getattr(lib, name)(*args)


def loop_filter_frame_dev(frame, d_mi, stream=0):
    """svt_b200_loop_filter_frame_dev: frame = DlfFrame with device plane pointers, d_mi = device records (data pointer)"""
    return lib.svt_b200_loop_filter_frame_dev(ct.byref(frame), vp(d_mi), vp(stream))


def dlf_level_sse_dev(frame, s, d_mi, d_sse, stream=0):
    """svt_b200_dlf_level_sse_dev: frame = DlfFrame, s = DlfLevelSse (device source planes and d_lvl), d_mi = device records,
    d_sse = device int64 [3 * s.n_levels] (data pointers)"""
    return lib.svt_b200_dlf_level_sse_dev(ct.byref(frame), ct.byref(s), vp(d_mi), vp(d_sse), vp(stream))

# ------------------------------------------------------------------------------------------------
# K13 + T2 open-loop ME for a whole picture
# ------------------------------------------------------------------------------------------------
def me_picture_desc(planes, width, height):
    """planes: three 2-D uint8 torch CUDA tensors (padded buffers) as laid out by me_plane_shapes()"""
    p = MePicture()
    for lvl, (th, stride, pad, w, h) in enumerate(me_plane_shapes(width, height)):
        p.plane[lvl] = planes[lvl].data_ptr()
        p.stride[lvl] = planes[lvl].stride(0)
        p.org_x[lvl] = pad
        p.org_y[lvl] = pad
        p.width[lvl] = w
        p.height[lvl] = h
    return p

# ------------------------------------------------------------------------------------------------
# K15 picture-analysis statistics
# ------------------------------------------------------------------------------------------------
def picture_statistics_dev(pic, ctl, torch, stream=0):
    """svt_b200_picture_statistics_dev on an ME picture (MePicture of device planes) with PaStatsControls `ctl`.  Returns
    (rc, dict of the torch CUDA result tensors: variance [n_b64, 85] int16, pic_avg_variance [1] int16, histogram
    [regions_w, regions_h, 256] int32, average_intensity [regions_w, regions_h] uint8, avg_luma [1] int64), all the bit
    patterns of the C types.  Every array is pre-filled with 0xa5 bytes, so unwritten entries stay recognisable."""
    n_b64 = ((pic.width[2] + 63) // 64) * ((pic.height[2] + 63) // 64)
    rw, rh = max(int(ctl.regions_w), 1), max(int(ctl.regions_h), 1)
    dev = torch.device("cuda")
    out = {"variance": torch.full((n_b64, 85), -0x5a5b, dtype=torch.int16, device=dev),
           "pic_avg_variance": torch.full((1,), -0x5a5b, dtype=torch.int16, device=dev),
           "histogram": torch.full((rw, rh, 256), -0x5a5a5a5b, dtype=torch.int32, device=dev),
           "average_intensity": torch.full((rw, rh), 0xa5, dtype=torch.uint8, device=dev),
           "avg_luma": torch.full((1,), -0x5a5a5a5a5a5a5a5b, dtype=torch.int64, device=dev)}
    res = PaStatsResults(*[out[n].data_ptr() for n, _ in PaStatsResults._fields_])
    rc = lib.svt_b200_picture_statistics_dev(ct.byref(pic), ct.byref(ctl), ct.byref(res), vp(stream))
    return rc, out
