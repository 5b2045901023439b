"""Reference-driven full-pel search: replays open_loop_me_fullpel_search_sblock
(motion_estimation.c:781-817) in Python on top of the UNMODIFIED reference kernels
(svt_ext_all_sad_calculation_8x8_16x16_c, svt_ext_eight_sad_calculation_32x32_64x64_c and the
1-point variants), so that the 85-PU results are produced by the reference's own update code."""
import ctypes as ct

import numpy as np

from oracle import support as sp

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


# ---- whole-picture open-loop ME, driven on the reference kernels ------------------------------------
def i16(v):
    v &= 0xffff
    return v - 0x10000 if v & 0x8000 else v


def build_pyramid_np(full, width, height, shapes):
    """numpy restatement of svt_aom_downsample_2d_c + svt_aom_generate_padding (checked against the
    reference function in test_oracle_pins)."""
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


def pad_np(buf, pad, w, h):
    inner = buf[pad:pad + h, pad:pad + w]
    buf[:, :] = np.pad(inner, ((pad, buf.shape[0] - pad - h), (pad, buf.shape[1] - pad - w)), mode="edge")
    return buf


def hme_clip(org, origin, sa, pad, pic, round8):
    if i16(org + origin) < -pad:
        origin = i16(-pad - org)
        sa = i16(sa - (-pad - (org + origin)))
    if i16(org + origin) > pic - 1:
        origin = i16(origin - ((org + origin) - (pic - 1)))
    if i16(org + origin + sa) > pic:
        sa = max(1, i16(sa - ((org + origin + sa) - pic)))
    if round8:
        sa = sa if sa < 8 else sa & ~7
    return origin, sa


def ref_me_picture(refc, cur, refs, shapes, width, height, params, sad_fn="svt_sad_loop_kernel_c"):
    """cur/refs: lists of 3 padded numpy planes.  Returns (best_sad, best_mv, hme_centre, hme_sad)."""
    from helpers import sad_loop_call
    b64_w, b64_h = (width + 63) // 64, (height + 63) // 64
    nb = b64_w * b64_h
    R = len(refs)
    out_sad = np.zeros((R, nb, 85), np.uint32); out_mv = np.zeros((R, nb, 85), np.uint32)
    out_c = np.zeros((R, nb, 2), np.int16); out_hs = np.zeros((R, nb), np.uint64)
    curf = [p.reshape(-1) for p in cur]
    for r in range(R):
        p = params[r]
        reff = [q.reshape(-1) for q in refs[r]]
        sub = 1 if p["hme_sub_sad"] else 0
        for b in range(nb):
            bx, by = b % b64_w, b // b64_w
            prev = [(0, 0)] * 4
            lsad = [0] * 4
            for level in range(3):
                th, stride, pad, w, h = shapes[level]
                sh = 2 - level
                org_x, org_y = (bx * 64) >> sh, (by * 64) >> sh
                blk_w, blk_h = min(64, width - bx * 64) >> sh, min(64, height - by * 64) >> sh
                nxt = []
                for reg in range(4):
                    sr_w, sr_h = reg & 1, reg >> 1
                    if level == 0:
                        sa_w = (p["hme_l0_sa_w"] + 7) & ~7; sa_h = p["hme_l0_sa_h"]
                        ox = i16(-((sa_w * 2) >> 1) + sa_w * sr_w); oy = i16(-((sa_h * 2) >> 1) + sa_h * sr_h)
                        pw = ph = pad - 1
                    elif level == 1:
                        sa_w = (p["hme_l1_sa_w"] + 7) & ~7; sa_h = p["hme_l1_sa_h"]
                        ox = i16(-(sa_w >> 1) + (prev[reg][0] >> 1)); oy = i16(-(sa_h >> 1) + (prev[reg][1] >> 1))
                        pw = ph = pad - 1
                    else:
                        sa_w = (p["hme_l2_sa_w"] + 7) & ~7; sa_h = p["hme_l2_sa_h"]
                        ox = i16(-(sa_w >> 1) + prev[reg][0]); oy = i16(-(sa_h >> 1) + prev[reg][1])
                        pw = ph = 63
                    ox, sa_w = hme_clip(org_x, ox, sa_w, pw, w, True)
                    oy, sa_h = hme_clip(org_y, oy, sa_h, ph, h, False)
                    s_off = (pad + org_y) * stride + pad + org_x
                    r_off = (pad + org_y + oy) * stride + pad + org_x + ox
                    best, x, y = sad_loop_call(refc, sad_fn, curf[level], s_off, stride << sub, reff[level], r_off, stride << sub,
                                               blk_h >> sub, blk_w, stride, 0, sa_w, sa_h)
                    if sub:
                        best *= 2
                    mul = 4 if level == 0 else (2 if level == 1 else 1)
                    nxt.append((i16(i16(x + ox) * mul), i16(i16(y + oy) * mul)))
                    lsad[reg] = best
                prev = nxt
            cx, cy, cs = prev[0][0], prev[0][1], lsad[0]
            for reg in range(1, 4):
                if lsad[reg] < cs:
                    cs, cx, cy = lsad[reg], prev[reg][0], prev[reg][1]
            out_c[r, b] = (cx, cy); out_hs[r, b] = cs
            th, stride, pad, w, h = shapes[2]
            org_x, org_y = bx * 64, by * 64
            blk_w, blk_h = min(64, width - org_x), min(64, height - org_y)
            sx, sy = cx, cy
            s_off = (pad + org_y) * stride + pad + org_x
            if p["check_zero_centre"] and (sx != 0 or sy != 0):
                if i16(org_x + sx) < -63: sx = i16(-63 - org_x)
                if i16(org_x + sx) > w - 1: sx = i16(sx - ((org_x + sx) - (w - 1)))
                if i16(org_y + sy) < -63: sy = i16(-63 - org_y)
                if i16(org_y + sy) > h - 1: sy = i16(sy - ((org_y + sy) - (h - 1)))
                f = refc.svt_nxm_sad_kernel_helper_c; f.restype = ct.c_uint32
                z = f(P(curf[2], s_off), ct.c_uint32(stride * 2), P(reff[2], s_off), ct.c_uint32(stride * 2), blk_h >> 1, blk_w) << 1
                hs = f(P(curf[2], s_off), ct.c_uint32(stride * 2), P(reff[2], s_off + sy * stride + sx), ct.c_uint32(stride * 2), blk_h >> 1,
                       blk_w) << 1
                if z <= hs:
                    sx = sy = 0
            sa_w = (max(1, p["me_sa_w"]) + 7) & ~7; sa_h = max(3, p["me_sa_h"])
            ox, oy = i16(sx - (sa_w >> 1)), i16(sy - (sa_h >> 1))
            if i16(org_x + ox) < -63: ox = i16(-63 - org_x)
            if i16(org_x + ox) > width - 1: ox = i16(ox - ((org_x + ox) - (width - 1)))
            if i16(org_x + ox + sa_w) > width: sa_w = max(1, sa_w - ((org_x + ox + sa_w) - width))
            sa_w = sa_w if sa_w < 8 else sa_w & ~7
            if i16(org_y + oy) < -63: oy = i16(-63 - org_y)
            if i16(org_y + oy) > height - 1: oy = i16(oy - ((org_y + oy) - (height - 1)))
            if i16(org_y + oy + sa_h) > height: sa_h = max(1, sa_h - ((org_y + oy + sa_h) - height))
            r_off = (pad + org_y + oy) * stride + pad + org_x + ox
            sad, mv = ref_fullpel(refc, curf[2], s_off, stride, reff[2], r_off, stride, sa_w, sa_h, ox, oy, p["me_sub_sad"])
            out_sad[r, b] = sad; out_mv[r, b] = mv
    return out_sad, out_mv, out_c, out_hs


def ref_me_picture_c(refc, cur, refs, shapes, width, height, params):
    """the pthread C driver in oracle/ref_driver.c (reference kernels through the dispatch pointers)"""
    R = len(refs)
    nb = ((width + 63) // 64) * ((height + 63) // 64)
    sad = np.zeros((R, nb, 85), np.uint32); mv = np.zeros((R, nb, 85), np.uint32)
    c = np.zeros((R, nb, 2), np.int16); hs = np.zeros((R, nb), np.uint64)
    cd = sp.ref_pic_desc(cur, shapes)
    rd = (sp.MePicture * R)(*[sp.ref_pic_desc(r, shapes) for r in refs])
    pr = (sp.MeParams * R)()
    for i, p in enumerate(params):
        for k, v in p.items():
            setattr(pr[i], k, v)
    refc.ref_me_picture.restype = None
    refc.ref_me_picture(ct.byref(cd), rd, pr, R, P(sad), P(mv), P(c), P(hs))
    return sad, mv, c, hs
