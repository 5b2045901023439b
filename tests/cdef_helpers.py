"""Reference-driven CDEF strength search and frame apply: replays cdef_seg_search (cdef_process.c:106-352) and
svt_av1_cdef_frame (enc_cdef.c:284-600) in Python on top of the UNMODIFIED reference functions svt_cdef_filter_fb
(cdef.c:339) and svt_aom_compute_cdef_dist_c (enc_cdef.c:129), 16-bit pixel containers; plus callers of the C
picture drivers of oracle/ref_driver.c for large pictures."""
import ctypes as ct

import numpy as np

from oracle import support as sp

BS, VL = 144, 0x7f7f


def P(a, off_elems=0):
    return ct.c_void_p(a.ctypes.data + off_elems * a.itemsize)


def make_frame(r, width, height, bd, skip_prob=0.3):
    """deblocked-recon-like and source planes (uint16 containers), + luma 8x8 skip map"""
    lim = (1 << bd) - 1
    planes_src, planes_rec = [], []
    for pli in range(3):
        w, h = (width >> (pli > 0)), (height >> (pli > 0))
        yy, xx = np.mgrid[0:h, 0:w]
        base = (np.sin(xx / 7.0) * 40 + np.cos(yy / 5.0) * 30 + (xx // 16 + yy // 16) % 2 * 50 + 100) * (lim / 255.0)
        src = np.clip(base + r.normal(0, 2 * lim / 255.0, base.shape), 0, lim).astype(np.uint16)
        rec = np.clip(src.astype(np.int32) + r.integers(-12, 13, src.shape) * (lim // 255), 0, lim).astype(np.uint16)
        planes_src.append(np.ascontiguousarray(src))
        planes_rec.append(np.ascontiguousarray(rec))
    skip = (r.random(((height + 7) // 8, (width + 7) // 8)) < skip_prob).astype(np.uint8)
    return planes_rec, planes_src, skip


def fb_list(skip, fbr, fbc):
    """svt_sb_compute_cdef_list: the non-skip 8x8s of filter block (fbr, fbc) in raster order, as (by, bx)"""
    return [(by, bx) for by in range(8) for bx in range(8)
            if fbr * 8 + by < skip.shape[0] and fbc * 8 + bx < skip.shape[1] and not skip[fbr * 8 + by, fbc * 8 + bx]]


def fill_tile(inbuf, plane, fbr, fbc, nvfb, nhfb, fbs, vsz, hsz):
    """the CDEF_BSTRIDE tile of one (filter block, plane) as cdef_seg_search builds it (cdef_process.c:211-230):
    CDEF_VERY_LARGE outside the picture, the unfiltered neighbours inside; the block starts at row 3, column 8.
    The reference copies an 8-column right border even from a neighbour only 4 chroma pixels wide, i.e. 4 pixels of
    the plane's padding; the filter taps reach 2 columns, so those never matter and stay CDEF_VERY_LARGE here."""
    inbuf[:] = VL
    yoff, xoff = 3 * (fbr != 0), 8 * (fbc != 0)
    ysize = vsz + 3 * (fbr + 1 < nvfb) + yoff
    xsize = hsz + 8 * (fbc + 1 < nhfb) + xoff
    rect = plane[fbr * fbs - yoff:fbr * fbs - yoff + ysize, fbc * fbs - xoff:fbc * fbs - xoff + xsize]
    inbuf.reshape(70, BS)[3 - yoff:3 - yoff + rect.shape[0], 8 - xoff:8 - xoff + rect.shape[1]] = rect


def ref_cdef_search(refc, rec, src, skip, width, height, bd, damping, subsampling, str_y, str_uv):
    nhfb, nvfb = (width + 63) // 64, (height + 63) // 64
    nfb, ng, cs = nhfb * nvfb, len(str_y), max(bd - 8, 0)
    mse = np.zeros((2, nfb, ng), np.uint64)
    dirs = np.zeros((nfb, 64), np.uint8)
    vars_ = np.zeros((nfb, 64), np.int32)
    ffb = refc.svt_cdef_filter_fb; ffb.restype = None
    fdist = refc.svt_aom_compute_cdef_dist_c; fdist.restype = ct.c_uint64
    inbuf = np.zeros(BS * 70, np.uint16)
    for fbr in range(nvfb):
        for fbc in range(nhfb):
            fb = fbr * nhfb + fbc
            lst = fb_list(skip, fbr, fbc)
            if not lst:
                continue
            dlist = np.array(lst, np.uint8).reshape(-1)
            dirm = np.zeros((16, 16), np.uint8); varm = np.zeros((16, 16), np.int32)
            dirinit = ct.c_int32(0)
            for pli in range(3):
                dec = 1 if pli else 0
                fbs, pw, ph = 64 >> dec, width >> dec, height >> dec
                hsz, vsz = min(fbs, pw - fbc * fbs), min(fbs, ph - fbr * fbs)
                fill_tile(inbuf, rec[pli], fbr, fbc, nvfb, nhfb, fbs, vsz, hsz)
                subs = min(subsampling, 1 if dec else 4)
                bsize = 0 if dec else 3
                for g in range(ng):
                    sv = str_uv[g] if pli else str_y[g]
                    if sv < 0:
                        mse[1, fb, g] = 1040400 * 64
                        continue
                    pri, sec = sv // 4, sv % 4
                    tmp = np.zeros(64 * 64, np.uint16)
                    ffb(None, P(tmp), 0, P(inbuf, 3 * BS + 8), dec, dec, P(dirm), ct.byref(dirinit), P(varm), pli, P(dlist), len(lst),
                        pri, sec + (sec == 3), damping, damping, cs, ct.c_uint8(subs))
                    sp = src[pli]
                    d = fdist(P(sp, fbr * fbs * sp.shape[1] + fbc * fbs), sp.shape[1], P(tmp), P(dlist), len(lst), bsize, cs, pli,
                              ct.c_uint8(subs))
                    if pli == 2:
                        mse[1, fb, g] += d * subs
                    else:
                        mse[1 if pli else 0, fb, g] = d * subs
            for (by, bx) in lst:
                dirs[fb, by * 8 + bx] = dirm[by, bx]
                vars_[fb, by * 8 + bx] = varm[by, bx]
    return mse, dirs, vars_


def ref_cdef_apply(refc, rec, skip, width, height, bd, damping, fb_idx, str_y, str_uv, out_planes, out_strides):
    """Reference-driven CDEF frame apply: replays svt_av1_cdef_frame (enc_cdef.c:284-600) on top of the UNMODIFIED
    svt_cdef_filter_fb (cdef.c:339), on tiles built from the unfiltered picture as cdef_seg_search builds them.
    out_planes: numpy arrays whose data pointer is the first pixel of each output plane (uint8 at 8 bit, else uint16),
    filled with the input by the caller; the filtered blocks are written straight into them at pitch out_strides
    (pixels).  Returns (filtered, dirs, vars): the filter blocks that were filtered and, for their non-skip 8x8s, the
    directions / variances the luma call found ([nfb][64], by * 8 + bx)."""
    nhfb, nvfb = (width + 63) // 64, (height + 63) // 64
    nfb, cs = nhfb * nvfb, max(bd - 8, 0)
    ffb = refc.svt_cdef_filter_fb; ffb.restype = None
    inbuf = np.zeros(BS * 70, np.uint16)
    dirs = np.zeros((nfb, 64), np.uint8)
    vars_ = np.zeros((nfb, 64), np.int32)
    filtered = []
    for fbr in range(nvfb):
        for fbc in range(nhfb):
            fb = fbr * nhfb + fbc
            if fb_idx[fb] < 0:  # cdef_strength == -1: the filter block is left as it is
                continue
            level, sec = str_y[fb_idx[fb]] // 4, str_y[fb_idx[fb]] % 4
            uv_level, uv_sec = str_uv[fb_idx[fb]] // 4, str_uv[fb_idx[fb]] % 4
            sec += sec == 3  # secondary strengths are {0, 1, 2, 4}
            uv_sec += uv_sec == 3
            if level == 0 and sec == 0 and uv_level == 0 and uv_sec == 0:
                continue
            lst = fb_list(skip, fbr, fbc)
            if not lst:
                continue
            filtered.append(fb)
            dlist = np.array(lst, np.uint8).reshape(-1)
            dirm = np.zeros((16, 16), np.uint8); varm = np.zeros((16, 16), np.int32)
            dirinit = ct.c_int32(0)  # the apply finds the directions itself (use_reference_cdef_fs)
            for pli in range(3):
                dec = 1 if pli else 0
                pri, sc = (uv_level, uv_sec) if pli else (level, sec)
                if pli and not (pri or sc):  # chroma runs only with a strength; luma always (it finds the directions)
                    continue
                fbs, pw, ph = 64 >> dec, width >> dec, height >> dec
                hsz, vsz = min(fbs, pw - fbc * fbs), min(fbs, ph - fbr * fbs)
                fill_tile(inbuf, rec[pli], fbr, fbc, nvfb, nhfb, fbs, vsz, hsz)
                out, os_ = out_planes[pli], out_strides[pli]
                dst = P(out, fbr * fbs * os_ + fbc * fbs)
                ffb(dst if bd == 8 else None, None if bd == 8 else dst, os_, P(inbuf, 3 * BS + 8), dec, dec, P(dirm), ct.byref(dirinit),
                    P(varm), pli, P(dlist), len(lst), pri, sc, damping, damping, cs, ct.c_uint8(1))
            for (by, bx) in lst:
                dirs[fb, by * 8 + bx] = dirm[by, bx]
                vars_[fb, by * 8 + bx] = varm[by, bx]
    return filtered, dirs, vars_


def _ref_frame(rec, src, width, height, bd, damping, subsampling):
    """CdefFrame over copies of the planes in the pixel type of the bit depth, 8 padding pixels right of every row
    (fill_tile); the copies are returned to keep them alive"""
    dt = np.uint8 if bd == 8 else np.uint16
    keep = [np.pad(p.astype(dt), ((0, 0), (0, 8))) for p in list(rec) + list(src)]
    f = sp.CdefFrame()
    f.recon_y, f.recon_cb, f.recon_cr, f.src_y, f.src_cb, f.src_cr = (k.ctypes.data for k in keep)
    f.recon_stride_y, f.recon_stride_c = keep[0].shape[1], keep[1].shape[1]
    f.src_stride_y, f.src_stride_c = keep[3].shape[1], keep[4].shape[1]
    f.width, f.height, f.bit_depth, f.damping, f.subsampling_factor, f.reserved = width, height, bd, damping, subsampling, 0
    return f, keep


def c_cdef_apply(refc, rec, skip, width, height, bd, damping, fb_idx, str_y, str_uv, out_planes, out_strides):
    """the same apply through oracle/ref_driver.c's ref_cdef_apply_frame (the producer of the committed goldens)"""
    f, keep = _ref_frame(rec, rec, width, height, bd, damping, 1)
    idx = np.ascontiguousarray(fb_idx, np.int8)
    sy, su = np.array(str_y, np.int32), np.array(str_uv, np.int32)
    refc.ref_cdef_apply_frame.restype = None
    refc.ref_cdef_apply_frame(ct.byref(f), P(skip), P(idx), P(sy), P(su), P(out_planes[0]), P(out_planes[1]), P(out_planes[2]),
                              int(out_strides[0]), int(out_strides[1]))


def c_cdef_search(refc, rec, src, skip, width, height, bd, damping, subsampling, str_y, str_uv):
    """the search through oracle/ref_driver.c's ref_cdef_search_frame: (mse, dirs, vars) as ref_cdef_search returns them"""
    nfb, ng = ((width + 63) // 64) * ((height + 63) // 64), len(str_y)
    f, keep = _ref_frame(rec, src, width, height, bd, damping, subsampling)
    sy, su = np.array(str_y, np.int32), np.array(str_uv, np.int32)
    mse = np.zeros((2, nfb, ng), np.uint64); dirs = np.zeros((nfb, 64), np.uint8); vars_ = np.zeros((nfb, 64), np.int32)
    refc.ref_cdef_search_frame.restype = None
    refc.ref_cdef_search_frame(ct.byref(f), P(skip), P(sy), P(su), ng, P(mse), P(dirs), P(vars_))
    return mse, dirs, vars_


def make_mixed_frame(r, width, height, bd, skip_prob=0.3):
    """Recon / source planes (uint16 containers) whose 16x16 luma regions (8x8 chroma) each hold one of: smooth content
    plus noise, a 0 / max checkerboard, all max (variance 0), or 0 / max stripes at one of 16 angles (every
    direction, variances past the adjust_strength cap); + a random luma 8x8 skip map"""
    lim = (1 << bd) - 1
    h16, w16 = (height + 15) // 16, (width + 15) // 16
    kind = r.integers(0, 4, (h16, w16))
    angle = r.integers(0, 16, (h16, w16)) * (np.pi / 16)
    period = r.integers(2, 6, (h16, w16))
    rec, src = [], []
    for pli in range(3):
        dec = 1 if pli else 0
        w, h = width >> dec, height >> dec
        yy, xx = np.mgrid[0:h, 0:w]
        ry, rx = (yy << dec) // 16, (xx << dec) // 16
        k, a, per = kind[ry, rx], angle[ry, rx], period[ry, rx]
        smooth = (np.sin(xx / 7.0) * 40 + np.cos(yy / 5.0) * 30 + 110) * (lim / 255.0) + r.normal(0, 6 * lim / 255.0, (h, w))
        stripes = (np.floor((xx * np.cos(a) + yy * np.sin(a)) / per) % 2) * lim
        p = np.select([k == 0, k == 1, k == 2], [smooth, ((xx + yy) & 1) * lim, np.full((h, w), lim)], stripes)
        p = np.clip(np.rint(p), 0, lim).astype(np.uint16)
        rec.append(p)
        src.append(np.clip(p.astype(np.int32) + r.integers(-3, 4, p.shape) * max(1, lim // 255), 0, lim).astype(np.uint16))
    skip = (r.random(((height + 7) // 8, (width + 7) // 8)) < skip_prob).astype(np.uint8)
    return rec, src, skip


def port_cdef_search(port, rec, src, skip, width, height, bd, damping, subsampling, str_y, str_uv):
    nfb, ng = ((width + 63) // 64) * ((height + 63) // 64), len(str_y)
    mse = np.zeros((2, nfb, ng), np.uint64); dirs = np.zeros((nfb, 64), np.uint8); vars_ = np.zeros((nfb, 64), np.int32)
    PA = ct.c_void_p * 3
    IA = ct.c_int * 3
    sy = np.array(str_y, np.int32); su = np.array(str_uv, np.int32)
    port.port_cdef_search_frame.restype = None
    port.port_cdef_search_frame(PA(*[x.ctypes.data for x in rec]), IA(*[x.shape[1] for x in rec]), PA(*[x.ctypes.data for x in src]),
                                IA(*[x.shape[1] for x in src]), width, height, bd, damping, subsampling, P(skip), P(sy), P(su), ng,
                                P(mse), P(dirs), P(vars_))
    return mse, dirs, vars_
