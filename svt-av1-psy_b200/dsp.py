"""Host-side mirror of the reference's dispatched DSP functions, bound to libsvtav1_b200.so.

Function names and argument meaning follow the reference's function pointers
(Source/Lib/Codec/aom_dsp_rtcd.h / common_dsp_rtcd.h); buffers are numpy arrays where the C code
takes pointers.  Every call goes through the C ABI (include/svt_b200.h) -- nothing here computes.
"""
import ctypes as ct

import numpy as np

from . import lib
from .layout import *  # noqa: F401,F403  (the header's structs and item dtypes, enum values, plane geometry: no library, shared with the CPU arm)

c_u8p = ct.POINTER(ct.c_uint8)
c_u16p = ct.POINTER(ct.c_uint16)
c_i16p = ct.POINTER(ct.c_int16)
c_i32p = ct.POINTER(ct.c_int32)
c_u32p = ct.POINTER(ct.c_uint32)
c_i64p = ct.POINTER(ct.c_int64)
c_u64p = ct.POINTER(ct.c_uint64)
c_f64p = ct.POINTER(ct.c_double)
vp = ct.c_void_p


def _ptr(a, typ=vp, byte_off=0):
    """pointer to (a.data + byte_off); `a` must be a numpy array (kept alive by the caller)."""
    if a is None:
        return ct.cast(0, typ)
    return ct.cast(a.ctypes.data + int(byte_off), typ)


# ------------------------------------------------------------------------------------------------
# signatures
# ------------------------------------------------------------------------------------------------
lib.svt_b200_init.argtypes = [ct.c_int]
lib.svt_b200_init.restype = ct.c_int
lib.svt_b200_shutdown.restype = None
lib.svt_b200_sm_count.restype = ct.c_int
lib.svt_b200_launch_count.restype = ct.c_ulonglong
lib.svt_b200_version.restype = ct.c_char_p
lib.svt_b200_copy_async.argtypes = [vp, vp, ct.c_size_t, ct.c_int, vp]
lib.svt_b200_copy_async.restype = ct.c_int
lib.svt_b200_copy2d_async.argtypes = [vp, ct.c_size_t, vp, ct.c_size_t, ct.c_size_t, ct.c_size_t, ct.c_int, vp]
lib.svt_b200_copy2d_async.restype = ct.c_int

lib.svt_b200_sad_loop_kernel.argtypes = [vp, ct.c_uint32, vp, ct.c_uint32, ct.c_uint32, ct.c_uint32, c_u64p, c_i16p,
                                         c_i16p, ct.c_uint32, ct.c_uint8, ct.c_int16, ct.c_int16]
lib.svt_b200_sad_loop_kernel.restype = None
lib.svt_b200_nxm_sad_kernel.argtypes = [vp, ct.c_uint32, vp, ct.c_uint32, ct.c_uint32, ct.c_uint32]
lib.svt_b200_nxm_sad_kernel.restype = ct.c_uint32
lib.svt_b200_sad_search_batch_host.argtypes = [vp, ct.c_size_t, vp, ct.c_size_t, vp, ct.c_int, vp]
lib.svt_b200_sad_search_batch_host.restype = ct.c_int
lib.svt_b200_sad_search_batch_dev.argtypes = [vp, vp, vp, ct.c_int, vp, ct.c_int, ct.c_int, ct.c_int, ct.c_int,
                                              ct.c_int, vp]
lib.svt_b200_sad_search_batch_dev.restype = ct.c_int

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
    lib.svt_b200_sad_loop_kernel(_ptr(src, vp, src_off), src_stride, _ptr(ref, vp, ref_off), ref_stride, block_height,
                                 block_width, ct.byref(best), ct.byref(xs), ct.byref(ys), src_stride_raw,
                                 skip_search_line, search_area_width, search_area_height)
    return int(best.value), int(xs.value), int(ys.value)


def svt_nxm_sad_kernel(src, src_off, src_stride, ref, ref_off, ref_stride, height, width):
    return int(lib.svt_b200_nxm_sad_kernel(_ptr(src, vp, src_off), src_stride, _ptr(ref, vp, ref_off), ref_stride,
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




lib.svt_b200_fwd_txfm2d_partial.argtypes = [vp, vp, ct.c_uint32, ct.c_int, ct.c_int, ct.c_uint8, ct.c_int]
lib.svt_b200_fwd_txfm2d_partial.restype = None
lib.svt_b200_txfm_valid.argtypes = [ct.c_int, ct.c_int]
lib.svt_b200_txfm_valid.restype = ct.c_int
lib.svt_b200_fwd_txfm2d.argtypes = [vp, vp, ct.c_uint32, ct.c_int, ct.c_int, ct.c_uint8]
lib.svt_b200_fwd_txfm2d.restype = None
lib.svt_b200_inv_txfm2d_add.argtypes = [vp, vp, ct.c_int32, vp, ct.c_int32, ct.c_int, ct.c_int, ct.c_int32]
lib.svt_b200_inv_txfm2d_add.restype = None
lib.svt_b200_inv_txfm_add_8bit.argtypes = [vp, vp, ct.c_int32, vp, ct.c_int32, ct.c_int, ct.c_int]
lib.svt_b200_inv_txfm_add_8bit.restype = None
lib.svt_b200_fwd_txfm_batch_host.argtypes = [vp, ct.c_size_t, vp, ct.c_size_t, vp, ct.c_int]
lib.svt_b200_fwd_txfm_batch_host.restype = ct.c_int
lib.svt_b200_fwd_txfm_batch_dev.argtypes = [vp, vp, vp, ct.POINTER(ct.c_int), vp]
lib.svt_b200_fwd_txfm_batch_dev.restype = ct.c_int
lib.svt_b200_inv_txfm_batch_dev.argtypes = [vp, vp, vp, vp, ct.POINTER(ct.c_int), ct.c_int, vp]
lib.svt_b200_txfm_team_class.argtypes = [ct.c_int]
lib.svt_b200_txfm_team_class.restype = ct.c_int
lib.svt_b200_inv_txfm_batch_dev.restype = ct.c_int


def txfm_valid(tx_size, tx_type):
    return bool(lib.svt_b200_txfm_valid(tx_size, tx_type))


def svt_av1_fwd_txfm2d(residual, stride, tx_type, tx_size, bit_depth=8, named=False):
    """svt_av1_fwd_txfm2d_WxH: int16 residual (flat, `stride`) -> int32[W*H]."""
    out = np.zeros(TX_W[tx_size] * TX_H[tx_size], np.int32)
    if named:
        f = getattr(lib, "svt_b200_av1_fwd_txfm2d_" + TX_NAME[tx_size])
        f.argtypes = [vp, vp, ct.c_uint32, ct.c_uint8, ct.c_uint8]
        f.restype = None
        f(_ptr(residual), _ptr(out), stride, tx_type, bit_depth)
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
lib.svt_b200_txfm_trio_batch_dev.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, ct.POINTER(ct.c_int), vp, ct.c_int, vp]
lib.svt_b200_txfm_trio_batch_dev.restype = ct.c_int
_QA = [vp, ct.c_ssize_t, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
for _n, _extra in (("aom_quantize_b", [vp, vp, ct.c_int32]), ("aom_highbd_quantize_b", [vp, vp, ct.c_int32]),
                   ("av1_quantize_b_qm", [vp, vp, ct.c_int32]), ("av1_highbd_quantize_b_qm", [vp, vp, ct.c_int32]),
                   ("av1_quantize_fp", []), ("av1_quantize_fp_32x32", []), ("av1_quantize_fp_64x64", []),
                   ("av1_quantize_fp_qm", [vp, vp, ct.c_int16]), ("av1_highbd_quantize_fp", [ct.c_int16]),
                   ("av1_highbd_quantize_fp_qm", [vp, vp, ct.c_int16])):
    _f = getattr(lib, "svt_b200_" + _n)
    _f.argtypes = _QA + _extra
    _f.restype = None
lib.svt_b200_residual_txfm_trio_batch_dev.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, ct.POINTER(ct.c_int), vp, ct.c_int, vp]
lib.svt_b200_residual_txfm_trio_batch_dev.restype = ct.c_int
lib.svt_b200_residual_planes_dev.argtypes = [vp, vp, vp, ct.POINTER(ResidualPlanes), ct.c_int, ct.c_int, vp]
lib.svt_b200_residual_planes_dev.restype = ct.c_int
lib.svt_b200_pack_levels_dev.argtypes = [vp, vp, vp, vp, ct.c_int, vp, vp, ct.c_int, ct.c_uint32, vp]
lib.svt_b200_pack_levels_dev.restype = ct.c_int
lib.svt_b200_quant_batch_dev.argtypes = [vp, vp, vp, vp, vp, vp, vp, ct.c_int, vp, vp]
lib.svt_b200_quant_batch_dev.restype = ct.c_int


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
for _n in ("4x4", "8x8", "16x16", "32x32"):
    _f = getattr(lib, "svt_b200_aom_hadamard_" + _n)
    _f.argtypes = [vp, ct.c_ssize_t, vp]
    _f.restype = None
lib.svt_b200_aom_satd.argtypes = [vp, ct.c_int]
lib.svt_b200_aom_satd.restype = ct.c_int
lib.svt_b200_hadamard_path.argtypes = [Buf2D, Buf2D, Buf2D, Buf2D, ct.c_uint8]
lib.svt_b200_hadamard_path.restype = ct.c_uint32
lib.svt_b200_av1_fwht4x4.argtypes = [vp, vp, ct.c_uint32]
lib.svt_b200_av1_fwht4x4.restype = None
lib.svt_b200_av1_compute_cul_level.argtypes = [vp, vp, vp]
lib.svt_b200_av1_compute_cul_level.restype = ct.c_uint8
lib.svt_b200_hadamard_satd_batch_dev.argtypes = [vp, vp, ct.c_int, vp, vp, vp]
lib.svt_b200_hadamard_satd_batch_dev.restype = ct.c_int
lib.svt_b200_ext_all_sad_calculation_8x8_16x16.argtypes = [vp, ct.c_uint32, vp, ct.c_uint32, ct.c_uint32, vp, vp, vp, vp,
                                                           vp, vp, ct.c_uint8]
lib.svt_b200_ext_all_sad_calculation_8x8_16x16.restype = None
lib.svt_b200_ext_eight_sad_calculation_32x32_64x64.argtypes = [vp, vp, vp, vp, vp, ct.c_uint32, vp]
lib.svt_b200_ext_eight_sad_calculation_32x32_64x64.restype = None
lib.svt_b200_ext_sad_calculation_8x8_16x16.argtypes = [vp, ct.c_uint32, vp, ct.c_uint32, vp, vp, vp, vp, ct.c_uint32, vp,
                                                       vp, ct.c_uint8]
lib.svt_b200_ext_sad_calculation_8x8_16x16.restype = None
lib.svt_b200_ext_sad_calculation_32x32_64x64.argtypes = [vp, vp, vp, vp, vp, ct.c_uint32, vp]
lib.svt_b200_ext_sad_calculation_32x32_64x64.restype = None
lib.svt_b200_initialize_buffer_32bits.argtypes = [vp, ct.c_uint32, ct.c_uint32, ct.c_uint32]
lib.svt_b200_initialize_buffer_32bits.restype = None
lib.svt_b200_fullpel_search_batch_dev.argtypes = [vp, vp, vp, ct.c_int, vp, vp, vp]
lib.svt_b200_fullpel_search_batch_dev.restype = ct.c_int
lib.svt_b200_fullpel_search_batch_host.argtypes = [vp, ct.c_size_t, vp, ct.c_size_t, vp, ct.c_int, vp, vp]
lib.svt_b200_fullpel_search_batch_host.restype = ct.c_int


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
lib.svt_b200_aom_cdef_find_dir.argtypes = [vp, ct.c_int32, vp, ct.c_int32]
lib.svt_b200_aom_cdef_find_dir.restype = ct.c_uint8
lib.svt_b200_aom_cdef_find_dir_dual.argtypes = [vp, vp, ct.c_int, vp, vp, ct.c_int32, vp, vp]
lib.svt_b200_aom_cdef_find_dir_dual.restype = None
lib.svt_b200_cdef_filter_block.argtypes = [vp, vp, ct.c_int32, vp, ct.c_int32, ct.c_int32, ct.c_int32, ct.c_int32, ct.c_int32,
                                           ct.c_int32, ct.c_int32, ct.c_uint8]
lib.svt_b200_cdef_filter_block.restype = None
lib.svt_b200_aom_copy_rect8_8bit_to_16bit.argtypes = [vp, ct.c_int32, vp, ct.c_int32, ct.c_int32, ct.c_int32]
lib.svt_b200_aom_copy_rect8_8bit_to_16bit.restype = None
for _n in ("16bit", "8bit"):
    _f = getattr(lib, "svt_b200_compute_cdef_dist_" + _n)
    _f.argtypes = [vp, ct.c_int32, vp, vp, ct.c_int32, ct.c_uint8, ct.c_int32, ct.c_int32, ct.c_uint8]
    _f.restype = ct.c_uint64
lib.svt_b200_search_one_dual.argtypes = [vp, vp, ct.c_int, vp, ct.c_int, ct.c_int, ct.c_int]
lib.svt_b200_search_one_dual.restype = ct.c_uint64
lib.svt_b200_cdef_search_frame_dev.argtypes = [ct.POINTER(CdefFrame), vp, vp, vp, ct.c_int, vp, vp, vp, vp]
lib.svt_b200_cdef_search_frame_dev.restype = ct.c_int
lib.svt_b200_cdef_apply_frame_dev.argtypes = [ct.POINTER(CdefFrame), vp, vp, vp, vp, vp, vp, vp, vp, vp, ct.c_int, ct.c_int, vp]
lib.svt_b200_cdef_apply_frame_dev.restype = ct.c_int


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
LPF_TAPS = (4, 6, 8, 14)
for _d in ("horizontal", "vertical"):
    for _n in LPF_TAPS:
        _f = getattr(lib, "svt_b200_aom_lpf_%s_%d" % (_d, _n))
        _f.argtypes = [vp, ct.c_int32, vp, vp, vp]
        _f.restype = None
        _f = getattr(lib, "svt_b200_aom_highbd_lpf_%s_%d" % (_d, _n))
        _f.argtypes = [vp, ct.c_int32, vp, vp, vp, ct.c_int32]
        _f.restype = None
lib.svt_b200_loop_filter_frame_dev.argtypes = [ct.POINTER(DlfFrame), vp, vp]
lib.svt_b200_loop_filter_frame_dev.restype = ct.c_int
lib.svt_b200_dlf_level_sse_dev.argtypes = [ct.POINTER(DlfFrame), ct.POINTER(DlfLevelSse), vp, vp, vp]
lib.svt_b200_dlf_level_sse_dev.restype = ct.c_int


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
# K9 / K11 Wiener
# ------------------------------------------------------------------------------------------------
lib.svt_b200_av1_wiener_convolve_add_src.argtypes = [vp, ct.c_ssize_t, vp, ct.c_ssize_t, vp, vp, ct.c_int32, ct.c_int32,
                                                     ct.POINTER(ConvolveParams)]
lib.svt_b200_av1_wiener_convolve_add_src.restype = None
lib.svt_b200_av1_highbd_wiener_convolve_add_src.argtypes = [vp, ct.c_ssize_t, vp, ct.c_ssize_t, vp, vp, ct.c_int32, ct.c_int32,
                                                            ct.POINTER(ConvolveParams), ct.c_int32]
lib.svt_b200_av1_highbd_wiener_convolve_add_src.restype = None
lib.svt_b200_av1_compute_stats.argtypes = [ct.c_int32, vp, vp] + [ct.c_int32] * 6 + [vp, vp]
lib.svt_b200_av1_compute_stats.restype = None
lib.svt_b200_av1_compute_stats_highbd.argtypes = [ct.c_int32, vp, vp] + [ct.c_int32] * 6 + [vp, vp, ct.c_int32]
lib.svt_b200_av1_compute_stats_highbd.restype = None
lib.svt_b200_wiener_units_dev.argtypes = [vp, vp, vp, ct.c_int, ct.c_int, vp]
lib.svt_b200_wiener_units_dev.restype = ct.c_int
lib.svt_b200_compute_stats_batch_dev.argtypes = [vp, vp, vp, ct.c_int, ct.c_int, vp, vp, vp]
lib.svt_b200_compute_stats_batch_dev.restype = ct.c_int

# ------------------------------------------------------------------------------------------------
# K10 / K12 self-guided restoration
# ------------------------------------------------------------------------------------------------
lib.svt_b200_av1_selfguided_restoration.argtypes = [vp, ct.c_int32, ct.c_int32, ct.c_int32, vp, vp, ct.c_int32, ct.c_int32, ct.c_int32,
                                                    ct.c_int32]
lib.svt_b200_av1_selfguided_restoration.restype = None
lib.svt_b200_apply_selfguided_restoration.argtypes = [vp, ct.c_int32, ct.c_int32, ct.c_int32, ct.c_int32, vp, vp, ct.c_int32, vp,
                                                      ct.c_int32, ct.c_int32]
lib.svt_b200_apply_selfguided_restoration.restype = None
for _n in ("lowbd", "highbd"):
    _f = getattr(lib, "svt_b200_av1_%s_pixel_proj_error" % _n)
    _f.argtypes = [vp, ct.c_int32, ct.c_int32, ct.c_int32, vp, ct.c_int32, vp, ct.c_int32, vp, ct.c_int32, vp, vp]
    _f.restype = ct.c_int64
lib.svt_b200_get_proj_subspace.argtypes = [vp, ct.c_int, ct.c_int, ct.c_int, vp, ct.c_int, ct.c_int, vp, ct.c_int, vp, ct.c_int, vp, vp]
lib.svt_b200_get_proj_subspace.restype = None
lib.svt_b200_sgr_units_dev.argtypes = [vp, vp, ct.c_int, vp, vp, ct.c_int, ct.c_int, ct.c_int, vp]
lib.svt_b200_sgr_units_dev.restype = ct.c_int

# ------------------------------------------------------------------------------------------------
# a13 loop-restoration drivers
# ------------------------------------------------------------------------------------------------
lib.svt_b200_lr_num_stripes.argtypes = [ct.c_int, ct.c_int]
lib.svt_b200_lr_num_stripes.restype = ct.c_int
lib.svt_b200_lr_boundary_stride.argtypes = [ct.c_int]
lib.svt_b200_lr_boundary_stride.restype = ct.c_int
lib.svt_b200_lr_units_per_dim.argtypes = [ct.c_int, ct.c_int]
lib.svt_b200_lr_units_per_dim.restype = ct.c_int
lib.svt_b200_lr_save_boundary_lines_dev.argtypes = [ct.POINTER(LrPlane), ct.c_int, ct.c_int, ct.c_int, vp]
lib.svt_b200_lr_save_boundary_lines_dev.restype = ct.c_int
lib.svt_b200_lr_filter_frame_dev.argtypes = [ct.POINTER(LrPlane), ct.c_int, ct.POINTER(vp), ct.c_int, ct.c_int, vp]
lib.svt_b200_lr_filter_frame_dev.restype = ct.c_int
lib.svt_b200_lr_unit_sse_dev.argtypes = [ct.POINTER(LrPlane), ct.c_int, ct.POINTER(vp), ct.c_int, vp]
lib.svt_b200_lr_unit_sse_dev.restype = ct.c_int

# ------------------------------------------------------------------------------------------------
# K13 + T2 open-loop ME for a whole picture
# ------------------------------------------------------------------------------------------------
lib.svt_b200_downsample_2d.argtypes = [vp, ct.c_uint32, ct.c_uint32, ct.c_uint32, vp, ct.c_uint32, ct.c_uint32]
lib.svt_b200_downsample_2d.restype = None
lib.svt_b200_build_hme_pyramid_dev.argtypes = [ct.POINTER(MePicture), vp]
lib.svt_b200_build_hme_pyramid_dev.restype = ct.c_int
lib.svt_b200_me_b64_num_pus.argtypes = [ct.POINTER(MeControls)]
lib.svt_b200_me_b64_num_pus.restype = ct.c_int
lib.svt_b200_me_b64_picture_dev.argtypes = [ct.POINTER(MePicture), ct.POINTER(MePicture), ct.POINTER(MeControls), ct.POINTER(MeB64Results), vp]
lib.svt_b200_me_b64_picture_dev.restype = ct.c_int



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
for _n in ("svt_b200_compute_mean_8x8", "svt_b200_compute_mean_square_values_8x8"):
    getattr(lib, _n).argtypes = [vp, ct.c_uint32, ct.c_uint32, ct.c_uint32]
    getattr(lib, _n).restype = ct.c_uint64
lib.svt_b200_compute_sub_mean_8x8.argtypes = [vp, ct.c_uint16]
lib.svt_b200_compute_sub_mean_8x8.restype = ct.c_uint64
lib.svt_b200_compute_interm_var_four8x8.argtypes = [vp, ct.c_uint16, vp, vp]
lib.svt_b200_compute_interm_var_four8x8.restype = None
lib.svt_b200_picture_statistics_dev.argtypes = [ct.POINTER(MePicture), ct.POINTER(PaStatsControls), ct.POINTER(PaStatsResults), vp]
lib.svt_b200_picture_statistics_dev.restype = ct.c_int


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

lib.svt_b200_extend_plane_dev.argtypes = [vp, ct.c_int, ct.c_int, ct.c_int, ct.c_int, ct.c_int, vp]
lib.svt_b200_extend_plane_dev.restype = ct.c_int
lib.svt_b200_extend_planes_dev.argtypes = [ct.POINTER(PlaneExtent), ct.c_int, vp]
lib.svt_b200_extend_planes_dev.restype = ct.c_int


for _m, _n in SAD_SIZES:
    _f = getattr(lib, "svt_b200_aom_sad%dx%d" % (_m, _n))
    _f.argtypes = [vp, ct.c_int, vp, ct.c_int]
    _f.restype = ct.c_uint32
    _f = getattr(lib, "svt_b200_aom_sad%dx%dx4d" % (_m, _n))
    _f.argtypes = [vp, ct.c_int, ct.POINTER(ct.c_void_p), ct.c_int, vp]
    _f.restype = None


for _n in ("16x64", "32x64", "64x16", "64x32", "64x64"):
    for _sfx in ("", "_N2_N4"):
        _f = getattr(lib, "svt_b200_handle_transform" + _n + _sfx)
        _f.argtypes = [vp]
        _f.restype = ct.c_uint64

def unbound_symbols():
    """declared C-ABI symbols that have no ctypes signature yet (calling those would truncate pointers)"""
    from . import declared_symbols
    return [s for s in declared_symbols() if getattr(lib, s).argtypes is None and s not in
            ("svt_b200_shutdown", "svt_b200_sm_count", "svt_b200_launch_count", "svt_b200_version")]

for _i, _n in enumerate(TX_NAME):
    for _sfx in ("", "_N2", "_N4"):
        _f = getattr(lib, "svt_b200_av1_fwd_txfm2d_" + _n + _sfx)
        _f.argtypes = [vp, vp, ct.c_uint32, ct.c_uint8, ct.c_uint8]
        _f.restype = None
    _g = getattr(lib, "svt_b200_av1_inv_txfm2d_add_" + _n)
    _base = [vp, vp, ct.c_int32, vp, ct.c_int32, ct.c_uint8]
    if _i in (0, 1, 2, 3, 4):
        _g.argtypes = _base + [ct.c_int32]
    elif _i in (5, 6, 13, 14):
        _g.argtypes = _base + [ct.c_uint8, ct.c_int32]
    else:
        _g.argtypes = _base + [ct.c_uint8, ct.c_int32, ct.c_int32]
    _g.restype = None


def svt_av1_inv_txfm2d_add_named(coeff, pred, stride_r, stride_w, tx_type, tx_size, bd):
    """the per-size named entry point (same argument list as the reference pointer of that size)"""
    out = np.zeros(TX_H[tx_size] * stride_w, np.uint16)
    g = getattr(lib, "svt_b200_av1_inv_txfm2d_add_" + TX_NAME[tx_size])
    args = [_ptr(coeff), _ptr(pred), stride_r, _ptr(out), stride_w, tx_type]
    if tx_size in (0, 1, 2, 3, 4):
        args += [bd]
    elif tx_size in (5, 6, 13, 14):
        args += [tx_size, bd]
    else:
        args += [tx_size, TX_W[tx_size] * TX_H[tx_size], bd]
    g(*args)
    return out
