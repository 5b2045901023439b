"""ctypes callers for the restoration checkers (reference objects / port)."""
import ctypes as ct

import numpy as np


def P(a, off_elems=0):
    return ct.c_void_p(a.ctypes.data + off_elems * a.itemsize)


class RefConvolveParams(ct.Structure):  # ConvolveParams, definitions.h:572-585
    _fields_ = [("ref", ct.c_int32), ("do_average", ct.c_int32), ("dst", ct.c_void_p), ("dst_stride", ct.c_int32),
                ("round_0", ct.c_int32), ("round_1", ct.c_int32), ("plane", ct.c_int32), ("is_compound", ct.c_int32),
                ("use_jnt_comp_avg", ct.c_int32), ("fwd_offset", ct.c_int32), ("bck_offset", ct.c_int32),
                ("use_dist_wtd_comp_avg", ct.c_int32)]


def wiener_taps(r):
    """a legal symmetric 7-tap wiener kernel (+ zero 8th tap), 16-byte aligned inside a 256-B aligned block"""
    t0 = int(r.integers(-5, 11)); t1 = int(r.integers(-23, 9)); t2 = int(r.integers(-17, 47))
    k = np.zeros(8, np.int16)
    k[0] = k[6] = t0; k[1] = k[5] = t1; k[2] = k[4] = t2
    k[3] = -2 * (t0 + t1 + t2)
    return k


def aligned_filter(k):
    """the reference derives the kernel base by masking the low 8 address bits (convolve.c:48-56): hand it a
    256-byte aligned copy so that x0_q4 = 0."""
    buf = np.zeros(256 + 16, np.int16)
    off = ((-buf.ctypes.data) % 256) // 2
    buf[off:off + 8] = k
    return buf, off


def ref_wiener(refc, src, src_off, ss, w, h, fx, fy, bd):
    out = np.zeros(h * w, src.dtype)
    bx, ox = aligned_filter(fx); by, oy = aligned_filter(fy)
    cp = RefConvolveParams()
    cp.round_0 = 5 if bd == 12 else 3
    cp.round_1 = 14 - cp.round_0
    if src.dtype == np.uint8:
        f = refc.svt_av1_wiener_convolve_add_src_c; f.restype = None
        f(P(src, src_off), ct.c_ssize_t(ss), P(out), ct.c_ssize_t(w), P(bx, ox), P(by, oy), w, h, ct.byref(cp))
    else:
        f = refc.svt_av1_highbd_wiener_convolve_add_src_c; f.restype = None
        # CONVERT_TO_BYTEPTR(x) = (uint8_t*)(((uintptr_t)x) >> 1)
        f(ct.c_void_p((src.ctypes.data + 2 * src_off) >> 1), ct.c_ssize_t(ss), ct.c_void_p(out.ctypes.data >> 1), ct.c_ssize_t(w),
          P(bx, ox), P(by, oy), w, h, ct.byref(cp), bd)
    return out


def port_wiener(port, src16, src_off, ss, w, h, fx, fy, bd, lbd):
    out = np.zeros(h * w, np.uint16)
    port.port_wiener_convolve.restype = None
    r0 = 5 if bd == 12 else 3
    port.port_wiener_convolve(P(src16, src_off), ct.c_ssize_t(ss), P(out), ct.c_ssize_t(w), P(fx), P(fy), w, h, r0, 14 - r0, bd, lbd)
    return out


def ref_stats(refc, win, dgd, src, hs, he, vs, ve, dst, sst, bd):
    M = np.zeros(49, np.int64); H = np.zeros(2401, np.int64)
    if dgd.dtype == np.uint8:
        f = refc.svt_av1_compute_stats_c; f.restype = None
        f(win, P(dgd), P(src), hs, he, vs, ve, dst, sst, P(M), P(H))
    else:
        f = refc.svt_av1_compute_stats_highbd_c; f.restype = None
        f(win, ct.c_void_p(dgd.ctypes.data >> 1), ct.c_void_p(src.ctypes.data >> 1), hs, he, vs, ve, dst, sst, P(M), P(H), bd)
    return M[:win * win], H[:win ** 4]


def port_stats(port, win, dgd16, src16, hs, he, vs, ve, dst, sst, bd):
    M = np.zeros(49, np.int64); H = np.zeros(2401, np.int64)
    port.port_compute_stats.restype = None
    port.port_compute_stats(win, P(dgd16), P(src16), hs, he, vs, ve, dst, sst, P(M), P(H), bd)
    return M[:win * win], H[:win ** 4]


# ---- self-guided ---------------------------------------------------------------------------------
SGR_PARAMS = [(2, 1, 140, 3236), (2, 1, 112, 2158), (2, 1, 93, 1618), (2, 1, 80, 1438), (2, 1, 70, 1295), (2, 1, 58, 1177),
              (2, 1, 47, 1079), (2, 1, 37, 996), (2, 1, 30, 925), (2, 1, 25, 863), (0, 1, -1, 2589), (0, 1, -1, 1618),
              (0, 1, -1, 1177), (0, 1, -1, 925), (2, 0, 56, -1), (2, 0, 22, -1)]


def bptr(a, off_elems=0):
    """the reference's pixel pointer convention: uint8* for 8-bit, CONVERT_TO_BYTEPTR (addr >> 1) for uint16"""
    addr = a.ctypes.data + off_elems * a.itemsize
    return ct.c_void_p(addr if a.dtype == np.uint8 else addr >> 1)


def ref_selfguided(refc, dgd, off, w, h, stride, idx, bd):
    f0 = np.full(w * h, -12345, np.int32); f1 = np.full(w * h, -12345, np.int32)
    f = refc.svt_av1_selfguided_restoration_c; f.restype = None
    f(bptr(dgd, off), w, h, stride, P(f0), P(f1), w, idx, bd, int(dgd.dtype != np.uint8))
    return f0, f1


# svt_av1_selfguided_restoration_c keeps its 32-bit copy of the tile and its box sums in stack buffers of
# RESTORATION_PROC_UNIT_PELS = (64 + 2 * 3 + 20)^2 elements (restoration.c:681,815,926)
REF_PROC_UNIT_PELS = 90 * 90


def ref_sgr_fits(w, h):
    """whether the reference filter takes a w x h unit in one call: its box-sum rows are ((w + 6 + 3) & ~3) + 16 apart"""
    return (h + 6) * ((((w + 6) + 3) & ~3) + 16) <= REF_PROC_UNIT_PELS and (w + 6) * (h + 6) <= REF_PROC_UNIT_PELS


def ref_sgr_into(refc, dgd, off, w, h, stride, idx, bd, f0, f1, foff, fstride):
    """svt_av1_selfguided_restoration_c of the w x h block at dgd[off] into f0 / f1 at element foff, rows fstride apart"""
    assert ref_sgr_fits(w, h), (w, h)
    f = refc.svt_av1_selfguided_restoration_c; f.restype = None
    f(bptr(dgd, off), w, h, stride, P(f0, foff), P(f1, foff), fstride, idx, bd, int(dgd.dtype != np.uint8))


def ref_sgr_tiled(refc, dgd, off, w, h, stride, idx, bd, f0, f1, foff, fstride, tw=64, rows=None):
    """the reference filter of a unit of any size, as calls on sub-tiles at most tw wide whose bands start at `rows`
    (default: every 64 rows).  The box sums of a sub-tile read the real neighbouring pixels, so this equals one call on
    the whole unit as long as every band starts an even number of rows below the unit top: the r = 2 pass computes its
    coefficients on every other row, counted from the top of the call."""
    rows = list(range(0, h, 64)) if rows is None else list(rows)
    for y0, y1 in zip(rows, rows[1:] + [h]):
        for x0 in range(0, w, tw):
            ref_sgr_into(refc, dgd, off + y0 * stride + x0, min(tw, w - x0), y1 - y0, stride, idx, bd, f0, f1, foff + y0 * fstride + x0,
                         fstride)


def decode_xq(xqd, prm):
    """svt_decode_xq (restoration.c:634-645)"""
    if prm[0] == 0:
        return [0, 128 - xqd[1]]
    if prm[1] == 0:
        return [xqd[0], 0]
    return [xqd[0], 128 - xqd[0] - xqd[1]]


def port_selfguided(port, dgd16, off, w, h, stride, idx, bd):
    f0 = np.full(w * h, -12345, np.int32); f1 = np.full(w * h, -12345, np.int32)
    port.port_selfguided.restype = None
    port.port_selfguided(P(dgd16, off), w, h, stride, P(f0), P(f1), w, idx, bd)
    return f0, f1
