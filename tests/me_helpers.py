"""Reference-driven full-pel search: replays open_loop_me_fullpel_search_sblock
(motion_estimation.c:781-817) in Python on top of the UNMODIFIED reference kernels
(svt_ext_all_sad_calculation_8x8_16x16_c, svt_ext_eight_sad_calculation_32x32_64x64_c and the
1-point variants), so that the 85-PU results are produced by the reference's own update code; and the synthetic
pictures the picture-level ME checks search."""
import ctypes as ct

import numpy as np

MAX_SAD = 128 * 128 * 255


def z16(y16, x16):
    return 4 * (2 * (y16 >> 1) + (x16 >> 1)) + 2 * (y16 & 1) + (x16 & 1)


def P(a, off=0):
    return ct.c_void_p(a.ctypes.data + off)


def ref_fullpel(refc, src, src_off, ss, ref, ref_off, rs, sa_w, sa_h, org_x, org_y, sub):
    b8 = np.full(64, MAX_SAD, np.uint32); b16 = np.full(16, MAX_SAD, np.uint32)
    b32 = np.full(4, MAX_SAD, np.uint32); b64 = np.full(1, MAX_SAD, np.uint32)
    m8 = np.zeros(64, np.uint32); m16 = np.zeros(16, np.uint32); m32 = np.zeros(4, np.uint32); m64 = np.zeros(1, np.uint32)
    e16 = np.zeros(16 * 8, np.uint32); e8 = np.zeros(64 * 8, np.uint32); e32 = np.zeros(4 * 8, np.uint32)
    s16 = np.zeros(16, np.uint32); s8 = np.zeros(64, np.uint32); s32 = np.zeros(4, np.uint32)
    f_all = refc.svt_ext_all_sad_calculation_8x8_16x16_c; f_all.restype = None
    f_e32 = refc.svt_ext_eight_sad_calculation_32x32_64x64_c; f_e32.restype = None
    f_1 = refc.svt_ext_sad_calculation_8x8_16x16_c; f_1.restype = None
    f_132 = refc.svt_ext_sad_calculation_32x32_64x64_c; f_132.restype = None
    w8 = sa_w - (sa_w & 7)
    for y in range(sa_h):
        for x in range(0, w8, 8):
            mv = (((org_y + y) & 0xffff) << 16) | ((org_x + x) & 0xffff)
            f_all(P(src, src_off), ct.c_uint32(ss), P(ref, ref_off + y * rs + x), ct.c_uint32(rs), ct.c_uint32(mv), P(b8), P(b16),
                  P(m8), P(m16), P(e16), P(e8), ct.c_bool(bool(sub)))
            f_e32(P(e16), P(b32), P(b64), P(m32), P(m64), ct.c_uint32(mv), P(e32))
        for x in range(w8, sa_w):
            mv = (((org_y + y) & 0xffff) << 16) | ((org_x + x) & 0xffff)
            for blk in range(16):
                y16, x16 = blk >> 2, blk & 3
                i16 = z16(y16, x16)
                f_1(P(src, src_off + 16 * y16 * ss + 16 * x16), ct.c_uint32(ss), P(ref, ref_off + (y + 16 * y16) * rs + x + 16 * x16),
                    ct.c_uint32(rs), P(b8, 4 * 4 * i16), P(b16, 4 * i16), P(m8, 4 * 4 * i16), P(m16, 4 * i16), ct.c_uint32(mv),
                    P(s16, 4 * i16), P(s8, 4 * 4 * i16), ct.c_bool(bool(sub)))
            f_132(P(s16), P(b32), P(b64), P(m32), P(m64), ct.c_uint32(mv), P(s32))
    return np.concatenate([b64, b32, b16, b8]), np.concatenate([m64, m32, m16, m8])


def port_fullpel(port, src, src_off, ss, ref, ref_off, rs, sa_w, sa_h, org_x, org_y, sub):
    sad = np.zeros(85, np.uint32); mv = np.zeros(85, np.uint32)
    port.port_fullpel_search.restype = None
    port.port_fullpel_search(P(src, src_off), ct.c_uint32(ss), P(ref, ref_off), ct.c_uint32(rs), sa_w, sa_h, org_x, org_y, int(sub),
                             P(sad), P(mv))
    return sad, mv


def hadamard_call(lib, name, src, stride, n):
    out = np.zeros(n * n, np.int32)
    f = getattr(lib, name); f.restype = None
    if name == "port_hadamard":
        f(P(src), ct.c_ssize_t(stride), P(out), n)
    else:
        f(P(src), ct.c_ssize_t(stride), P(out))
    return out


def sequence(r, w, h, n, pan=(3, 1), noise=4.0, still_rect=None):
    """n pictures of a panning synthetic scene (optionally with a static rectangle: early-exit / stationary paths)"""
    yy, xx = np.mgrid[0:h + 160, 0:w + 160]
    base = (np.sin(xx / 13.0) * 45 + np.cos(yy / 9.0) * 35 + ((xx // 20 + yy // 28) % 2) * 70 + ((xx // 7) % 3) * 9 + 100)
    out = []
    for t in range(n):
        ox, oy = 80 + pan[0] * (t - n // 2), 80 + pan[1] * (t - n // 2)
        img = base[oy:oy + h, ox:ox + w] + r.normal(0, noise, (h, w))
        if still_rect is not None:
            x0, y0, x1, y1 = still_rect
            img[y0:y1, x0:x1] = base[80 + y0:80 + y1, 80 + x0:80 + x1] + r.normal(0, 0.6, (y1 - y0, x1 - x0))
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    return out


def case_pictures(r, w, h, n_ref, dist, content):
    """(current picture, reference pictures of list 0 then list 1) of a test_me_b64.CASES entry: nine pictures of `sequence`,
    the current one in the middle, each reference as many pictures away as its distance says (at most four)"""
    seq = sequence(r, w, h, 2 * 4 + 1, **content)
    mid = len(seq) // 2
    pick = lambda d: seq[int(np.clip(mid + np.sign(d) * min(abs(d), 4), 0, len(seq) - 1))]  # noqa: E731
    return seq[mid], [pick(dist[0][i]) for i in range(n_ref[0])] + [pick(dist[1][i]) for i in range(n_ref[1])]
