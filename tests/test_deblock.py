"""K14 deblocking loop filter: the 16 T1 lpf entry points against the reference's _c functions, the whole-picture T2 call
against the reference's own svt_av1_loop_filter_frame (oracle/ref_dlf.c), and on the CPU the two claims the device design
rests on -- two whole-plane passes (every vertical edge, then every horizontal edge) give the reference's superblock-order
result, and the small AV1 tables of dlf_tables.h are the reference's."""
import ctypes as ct
import os

import numpy as np
import pytest

from helpers import rng

LPF_TAPS = (4, 6, 8, 14)

# BlockSize enumerators by (width, height)
BSIZE = {(4, 4): 0, (4, 8): 1, (8, 4): 2, (8, 8): 3, (8, 16): 4, (16, 8): 5, (16, 16): 6, (16, 32): 7, (32, 16): 8, (32, 32): 9,
         (32, 64): 10, (64, 32): 11, (64, 64): 12, (64, 128): 13, (128, 64): 14, (128, 128): 15, (4, 16): 16, (16, 4): 17,
         (8, 32): 18, (32, 8): 19, (16, 64): 20, (64, 16): 21}


class RefDlfCfg(ct.Structure):  # oracle/ref_dlf.c
    _fields_ = [(n, ct.c_int32) for n in ("width", "height", "sb_size", "bit_depth", "pixel_bytes")] + \
               [("filter_level", ct.c_int32 * 2)] + [(n, ct.c_int32) for n in ("filter_level_u", "filter_level_v", "sharpness",
                                                                                "mode_ref_delta_enabled")] + \
               [("ref_deltas", ct.c_int32 * 8), ("mode_deltas", ct.c_int32 * 2), ("segmentation_enabled", ct.c_int32),
                ("seg_lf_enabled", (ct.c_int32 * 4) * 8), ("seg_lf_data", (ct.c_int32 * 4) * 8)] + \
               [(n, ct.c_int32) for n in ("mi_rows", "mi_cols", "mi_stride", "reserved")]


DLF_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsvtav1_dlf.so")


@pytest.fixture(scope="module")
def dlfc(refc):
    """oracle/_ref/libsvtav1_dlf.so (oracle/dlf.mk): oracle/ref_dlf.c and the deblocking glue, on top of the reference
    objects refc has loaded and initialised"""
    if not os.path.exists(DLF_LIB):
        pytest.fail("oracle/_ref/libsvtav1_dlf.so is missing: build it with `python __graft_entry__.py --oracle` where the "
                    "reference sources are available")
    return ct.CDLL(DLF_LIB)


def _layout():
    from oracle.support import load_pkg_module
    return load_pkg_module("layout")


# ---- (a) T1 inputs: test/DeblockTest.cc's generator ---------------------------------------------------------------
def _deblock_input(r, limit, mask, p, i):
    """init_input: runs that step by limit - 1 along rows, then along columns; i odd = the transposed layout"""
    n = 1024
    t = np.zeros(n, np.int64)
    j = 0
    while j < n:
        val = int(r.integers(0, 256))
        if val & 0x80:
            t[j] = int(r.integers(0, 65536)); j += 1
        else:
            k = 0
            while k < (val & 0x1f) + 1 and j < n:
                k += 1
                t[j] = int(r.integers(0, 65536)) if j < 1 else (t[j - 1] + (limit - 1) if val & 0x20 else t[j - 1] - (limit - 1)) & 0xffff
                j += 1
    j = 0
    while j < n:
        val = int(r.integers(0, 256))
        if val & 0x80:
            j += 1
        else:
            k = 0
            while k < (val & 0x1f) + 1 and j < n:
                k += 1
                if j < 1:
                    t[j] = int(r.integers(0, 65536))
                else:
                    prev = t[((j - 1) % 32) * 32 + (j - 1) // 32]
                    t[(j % 32) * 32 + j // 32] = (prev + (limit - 1) if val & 0x20 else prev - (limit - 1)) & 0xffff
                j += 1
    idx = np.arange(n)
    s = t if i % 2 else t[p * (idx % p) + idx // p]
    return s & mask


@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["horizontal", "vertical"])
@pytest.mark.parametrize("taps", LPF_TAPS)
@pytest.mark.parametrize("bd", [0, 8, 10, 12], ids=["lbd", "hbd8", "hbd10", "hbd12"])
def test_lpf_t1_matches_reference(b200, refc, direction, taps, bd):
    """svt_b200_aom_{,highbd_}lpf_<dir>_<taps> == svt_aom_{,highbd_}lpf_<dir>_<taps>_c on the whole 32x32 buffer (bytes
    outside the filter's footprint must stay untouched)"""
    r = rng(taps * 100 + bd + (7 if direction == "vertical" else 0))
    hb = bd > 0
    dt = np.uint16 if hb else np.uint8
    mask = (1 << (bd if hb else 8)) - 1
    name = "svt_aom_%slpf_%s_%d_c" % ("highbd_" if hb else "", direction, taps)
    f = getattr(refc, name)
    f.restype = None
    p, start = 32, 8 + 32 * 8
    for i in range(300):
        blimit, limit, thresh = int(r.integers(0, 3 * 63 + 5)), int(r.integers(0, 64)), int(r.integers(0, 64)) >> 4
        s = _deblock_input(r, limit, mask, p, i).astype(dt)
        ref, ours = s.copy(), s.copy()
        th = [np.full(16, v, np.uint8) for v in (blimit, limit, thresh)]
        args = [ct.c_void_p(ref.ctypes.data + start * ref.itemsize), ct.c_int32(p)] + [ct.c_void_p(t.ctypes.data) for t in th]
        f(*(args + ([ct.c_int32(bd)] if hb else [])))
        b200.svt_aom_lpf(direction, taps, ours, start, p, blimit, limit, thresh, bd if hb else None)
        assert np.array_equal(ours, ref), (name, i, blimit, limit, thresh, np.flatnonzero(ours != ref)[:8])


# ---- pictures: random partitions, mode info, frame headers --------------------------------------------------------
def _partition(r, x, y, s, leaves):
    """random AV1 partition of the square at (x, y) of size s: NONE, HORZ, VERT, SPLIT, HORZ_4, VERT_4"""
    opts = ["none", "horz", "vert", "split"] + (["horz4", "vert4"] if 16 <= s <= 64 else [])
    if s == 4:
        leaves.append((x, y, 4, 4))
        return
    o = opts[int(r.integers(0, len(opts)))] if s > 8 or r.random() < 0.8 else "split"
    if o == "none":
        leaves.append((x, y, s, s))
    elif o == "horz":
        leaves += [(x, y, s, s // 2), (x, y + s // 2, s, s // 2)]
    elif o == "vert":
        leaves += [(x, y, s // 2, s), (x + s // 2, y, s // 2, s)]
    elif o == "horz4":
        leaves += [(x, y + k * s // 4, s, s // 4) for k in range(4)]
    elif o == "vert4":
        leaves += [(x + k * s // 4, y, s // 4, s) for k in range(4)]
    else:
        for k in range(4):
            _partition(r, x + (k & 1) * s // 2, y + (k >> 1) * s // 2, s // 2, leaves)


def make_mode_info(r, width, height, sb_size, skip_bias=0.5, n_seg=8):
    """mi records (rows x stride) of a random valid partition of every superblock, with random tx depth, skip,
    reference frame (0 = intra), prediction mode (GLOBALMV / GLOBAL_GLOBALMV included) and segment"""
    L = _layout()
    mi_rows, mi_cols = ((height + 7) & ~7) // 4, ((width + 7) & ~7) // 4
    mi_stride = ((mi_cols * 4 + sb_size - 1) // sb_size) * sb_size // 4
    mi = np.zeros((mi_rows, mi_stride), L.DLF_MI_DTYPE)
    for sy in range(0, mi_rows * 4, sb_size):
        for sx in range(0, mi_cols * 4, sb_size):
            leaves = []
            _partition(r, sx, sy, sb_size, leaves)
            for (x, y, w, h) in leaves:
                ref = int(r.integers(0, 8)) if r.random() < 0.7 else 0
                rec = (BSIZE[(w, h)], int(r.integers(0, 3)), int(r.random() < skip_bias), ref,
                       int(r.integers(13, 25)) if ref > 0 else int(r.integers(0, 13)), int(r.integers(0, n_seg)), (0, 0))
                mi[y // 4:(y + h) // 4, x // 4:(x + w) // 4] = rec
    return mi, mi_rows, mi_cols, mi_stride


def make_cfg(r, width, height, sb_size, bit_depth, pixel_bytes, variant, mi_rows, mi_cols, mi_stride):
    c = RefDlfCfg()
    c.width, c.height, c.sb_size, c.bit_depth, c.pixel_bytes = width, height, sb_size, bit_depth, pixel_bytes
    c.mi_rows, c.mi_cols, c.mi_stride = mi_rows, mi_cols, mi_stride
    lv = [int(v) for v in r.integers(0, 64, 4)]
    c.sharpness = (0, 3, 7, int(r.integers(0, 8)))[variant % 4]
    if variant == 1:  # luma off: nothing is filtered, chroma included
        lv[0] = lv[1] = 0
    if variant == 2:  # one luma direction off, chroma off
        lv[1], lv[3] = 0, 0
    c.filter_level[0], c.filter_level[1], c.filter_level_u, c.filter_level_v = lv
    if variant >= 3:
        c.mode_ref_delta_enabled = 1
        for i in range(8):
            c.ref_deltas[i] = int(r.integers(-20, 21))
        c.mode_deltas[0], c.mode_deltas[1] = int(r.integers(-20, 21)), int(r.integers(-20, 21))
        c.segmentation_enabled = 1
        for s in range(8):
            for k in range(4):
                c.seg_lf_enabled[s][k] = int(r.random() < 0.5)
                c.seg_lf_data[s][k] = int(r.integers(-63, 64))
    return c


def make_planes(r, width, height, pixel_bytes, bit_depth, odd_pitch):
    """three padded planes (16 pixels of padding all round, then the guard bands up to the pitch), random content"""
    dt = np.uint16 if pixel_bytes == 2 else np.uint8
    out = []
    for p in range(3):
        w, h = (width, height) if p == 0 else (width >> 1, height >> 1)
        pitch = w + 32 + (3 if odd_pitch else 0)
        base = r.integers(0, 1 << bit_depth, (h + 32, pitch))
        # piecewise-smooth content so that every filter path (flat, flat2, hev) is taken
        smooth = np.cumsum(r.integers(-2, 3, (h + 32, pitch)), axis=1) + (1 << (bit_depth - 1))
        pick = (np.arange(pitch)[None, :] // 8 + np.arange(h + 32)[:, None] // 8) % 3 == 0
        out.append(np.clip(np.where(pick, base, smooth), 0, (1 << bit_depth) - 1).astype(dt))
    return out


def ref_filter(dlfc, cfg, mi, planes, mode):
    """oracle/ref_dlf.c on copies of the planes (origin at (16, 16)) -> (planes, DlfFrame, mi records out)"""
    L = _layout()
    out = [p.copy() for p in planes]
    isz = out[0].itemsize
    frame, mi_out = L.DlfFrame(), np.zeros_like(mi)
    dlfc.ref_dlf_frame.restype = ct.c_int
    dlfc.ref_dlf_frame.argtypes = [ct.c_void_p, ct.c_void_p, ct.c_void_p, ct.c_void_p, ct.c_void_p, ct.c_int, ct.c_int, ct.c_int,
                                   ct.c_void_p, ct.c_void_p]
    ptrs = [o.ctypes.data + (16 * o.shape[1] + 16) * isz for o in out]
    rc = dlfc.ref_dlf_frame(ct.byref(cfg), mi.ctypes.data, *ptrs, out[0].shape[1], out[1].shape[1], mode, ct.byref(frame), mi_out.ctypes.data)
    assert rc == 0
    return out, frame, mi_out


SIZES = [(16, 16), (72, 72), (200, 136), (642, 362), (1920, 1080)]
FORMATS = [(8, 1), (8, 2), (10, 2), (12, 2)]  # (bit depth, pixel bytes): u8 planes, bd 8 in 16 bit, 10, 12


def _case(size, fmt, variant, sb_size, seed):
    w, h = size
    bd, pb = fmt
    r = rng(seed)
    mi, mr, mc, ms = make_mode_info(r, w, h, sb_size, skip_bias=(0.2, 0.5, 0.8, 0.5)[variant % 4])
    cfg = make_cfg(r, w, h, sb_size, bd, pb, variant, mr, mc, ms)
    planes = make_planes(r, w, h, pb, bd, odd_pitch=bool(variant & 1))
    return cfg, mi, planes


# ---- (d) CPU: two whole-plane passes == superblock order; glue round trip; tables ---------------------------------
@pytest.mark.parametrize("sb_size", [64, 128])
@pytest.mark.parametrize("fmt", FORMATS, ids=["u8", "bd8in16", "bd10", "bd12"])
@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_two_pass_equals_superblock_order(dlfc, size, fmt, sb_size):
    changed = False
    for variant in range(5):
        cfg, mi, planes = _case(size, fmt, variant, sb_size, seed=size[0] * 7 + size[1] + fmt[0] * 3 + fmt[1] + variant * 1000 + sb_size)
        sb_order, _, _ = ref_filter(dlfc, cfg, mi, planes, 0)
        two_pass, _, _ = ref_filter(dlfc, cfg, mi, planes, 1)
        for p in range(3):
            assert np.array_equal(sb_order[p], two_pass[p]), (variant, p)
        changed |= any(not np.array_equal(sb_order[p], planes[p]) for p in range(3))
    assert changed or size[0] < 72, "no case filtered anything"  # a 16x16 picture may hold a single block: no inner edge


@pytest.mark.parametrize("variant", range(5))
def test_glue_round_trip_and_tables(dlfc, variant):
    """records -> PictureControlSet -> glue gives the same records; the glue's lvl / lfthr are what
    svt_av1_loop_filter_frame_init and svt_aom_update_sharpness derive"""
    cfg, mi, planes = _case((200, 136), (10, 2), variant, 64, seed=77 + variant)
    _, frame, mi_out = ref_filter(dlfc, cfg, mi, planes, 2)
    mc = cfg.mi_cols  # the glue leaves the columns past the picture zero
    assert np.array_equal(mi_out[:, :mc].copy().view(np.uint8), mi[:, :mc].copy().view(np.uint8))
    assert (frame.width, frame.height, frame.mi_rows, frame.mi_cols, frame.mi_stride, frame.bit_depth, frame.pixel_bytes) == \
        (cfg.width, cfg.height, cfg.mi_rows, cfg.mi_cols, cfg.mi_stride, cfg.bit_depth, cfg.pixel_bytes)
    _, frame0, _ = ref_filter(dlfc, cfg, mi, planes, 0)  # the tables the frame filter itself used
    assert bytes(frame0.lvl) == bytes(frame.lvl) and bytes(frame0.lfthr) == bytes(frame.lfthr)
    # sharpness limits (the AV1 definition): lim, mblim = 2 * (lvl + 2) + lim, hev_thr = lvl >> 4
    s = cfg.sharpness
    for lvl in range(64):
        lim = lvl >> ((s > 0) + (s > 4))
        lim = max(1, min(lim, 9 - s) if s > 0 else lim)
        assert tuple(frame.lfthr[lvl]) == (2 * (lvl + 2) + lim, lim, lvl >> 4), lvl
    lvl = np.frombuffer(bytes(frame.lvl), np.uint8).reshape(3, 8, 2, 8, 2)
    if cfg.filter_level[0] or cfg.filter_level[1]:
        base = lvl[0, 0, 0, 0, 0] if not cfg.mode_ref_delta_enabled and not cfg.segmentation_enabled else None
        if base is not None:
            assert base == cfg.filter_level[0]


def test_device_tables_equal_reference(dlfc):
    """dlf_tables.h (tx depth -> tx size, 4:2:0 chroma tx size, horz / vert tx maps, 4:2:0 plane block size, block
    width / height, mode_lf_lut) entry by entry against the reference's tables"""
    dlfc.ref_dlf_table_mismatches.restype = ct.c_int
    assert dlfc.ref_dlf_table_mismatches() == 0


# ---- (b) GPU: the whole-picture call against svt_av1_loop_filter_frame ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", range(5))
@pytest.mark.parametrize("fmt", FORMATS, ids=["u8", "bd8in16", "bd10", "bd12"])
@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_loop_filter_frame_dev_matches_reference(b200, dlfc, size, fmt, variant):
    import torch
    sb_size = 128 if variant in (2, 4) else 64
    cfg, mi, planes = _case(size, fmt, variant, sb_size, seed=size[0] * 13 + size[1] + fmt[0] + fmt[1] * 5 + variant * 977)
    ref_out, frame, _ = ref_filter(dlfc, cfg, mi, planes, 0)
    tdt = torch.int16 if fmt[1] == 2 else torch.uint8
    dev = [torch.from_numpy(p.view(np.int16) if fmt[1] == 2 else p).to("cuda") for p in planes]
    d_mi = torch.from_numpy(mi.view(np.uint8).reshape(-1)).to("cuda")
    isz = planes[0].itemsize
    for p in range(3):
        frame.plane[p] = dev[p].data_ptr() + (16 * planes[p].shape[1] + 16) * isz
        frame.stride[p] = planes[p].shape[1]
    assert dev[0].dtype == tdt
    stream = torch.cuda.current_stream().cuda_stream
    assert b200.loop_filter_frame_dev(frame, d_mi.data_ptr(), stream) == 0
    torch.cuda.synchronize()
    for p in range(3):
        got = dev[p].cpu().numpy().view(planes[p].dtype)
        bad = np.argwhere(got != ref_out[p])
        assert bad.size == 0, (p, bad[:8].tolist(), int(np.count_nonzero(ref_out[p] != planes[p])))
