"""K14 deblocking filter-level search: the per-level trial SSEs of svt_b200_dlf_level_sse_dev against the reference's own
try_filter_frame steps (oracle/ref_dlf_search.c: ref_dlf_level_sse), and the claim the design rests on -- the reference's
hill-climb (search_filter_level, deblocking_filter.c:886), run over a table of one-shot trials on the unfiltered picture,
chooses what its own sequential search (svt_av1_pick_filter_level, LPF_PICK_FROM_FULL_IMAGE: ref_dlf_pick) chooses, with
the same zero_filt_sse / best_filt_sse.  On the CPU with the reference's table, on the GPU with the device's."""
import ctypes as ct
import os

import numpy as np
import pytest

from helpers import rng
from test_deblock import FORMATS, SIZES, _layout, make_cfg, make_mode_info, make_planes

DLF_SEARCH_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libsvtav1_dlf_search.so")


@pytest.fixture(scope="module")
def dlfc(refc):
    """oracle/_ref/libsvtav1_dlf_search.so (oracle/dlf_search.mk): oracle/ref_dlf_search.c and the deblocking glue, on top
    of the reference objects refc has loaded and initialised"""
    if not os.path.exists(DLF_SEARCH_LIB):
        pytest.fail("oracle/_ref/libsvtav1_dlf_search.so is missing: build it with `python __graft_entry__.py --oracle` where "
                    "the reference sources are available")
    return ct.CDLL(DLF_SEARCH_LIB)

ONLY_4X4, TX_MODE_LARGEST, TX_MODE_SELECT = 0, 1, 2
KEY_FRAME, INTER_FRAME = 0, 1
BAD_ARG = -4


class RefDlfSearch(ct.Structure):  # oracle/ref_dlf_search.c
    _fields_ = [("src", ct.c_void_p * 3), ("src_stride", ct.c_int32 * 3)] + \
               [(n, ct.c_int32) for n in ("plane_mask", "n_levels", "sharpness", "tune", "frame_type", "tx_mode",
                                          "early_exit_convergence")] + \
               [("level", ct.c_uint8 * 64), ("picked", ct.c_int32 * 4), ("zero_filt_sse", ct.c_int64), ("best_filt_sse", ct.c_int64)]


def _origin(a):
    return a.ctypes.data + (16 * a.shape[1] + 16) * a.itemsize


# ---- cases ------------------------------------------------------------------------------------------------------------
def search_case(size, fmt, variant, seed, sb_size=64):
    """(cfg, mi, recon planes, source planes, controls): a smooth source, and a recon that adds a random offset per 4x4
    block (blocking the filter can remove) -- so the climb has a real optimum -- in padded planes (odd pitch for odd
    variants, random content in the padding).  variant >= 3 adds mode / ref deltas and segment features (make_cfg)."""
    w, h = size
    bd, pb = fmt
    r = rng(seed)
    mi, mr, mc, ms = make_mode_info(r, w, h, sb_size, skip_bias=(0.2, 0.5, 0.8, 0.5)[variant % 4])
    cfg = make_cfg(r, w, h, sb_size, bd, pb, variant, mr, mc, ms)
    src = make_planes(r, w, h, pb, bd, odd_pitch=bool(variant & 1))
    top = (1 << bd) - 1
    amp = max(2, (1 << bd) >> (4 + variant % 3))
    rec = []
    for s in src:
        blocks = r.integers(-amp, amp + 1, ((s.shape[0] + 3) // 4, (s.shape[1] + 3) // 4))
        off = np.kron(blocks, np.ones((4, 4), np.int64))[:s.shape[0], :s.shape[1]]
        rec.append(np.clip(s.astype(np.int64) + off, 0, top).astype(s.dtype))
    ctl = dict(sharpness=int(r.integers(0, 8)), tune=(0, 1, 3)[variant % 3], frame_type=(KEY_FRAME, INTER_FRAME)[variant % 2],
               tx_mode=(ONLY_4X4, TX_MODE_LARGEST, TX_MODE_SELECT)[variant % 3], early_exit_convergence=(variant // 2) % 2)
    return cfg, mi, rec, src, ctl


def search_sharpness(ctl):
    """the sharpness svt_av1_pick_filter_level sets before its first try (deblocking_filter.c:1145-1148)"""
    s = min(7, max(0, ctl["sharpness"]))
    return min(7, s + 2) if ctl["frame_type"] == KEY_FRAME and ctl["tune"] in (0, 3) else s


def _search(src, ctl=None, mask=7, levels=range(64)):
    s = RefDlfSearch()
    for p in range(3):
        s.src[p] = _origin(src[p])
        s.src_stride[p] = src[p].shape[1]
    s.plane_mask = mask
    s.n_levels = len(levels)
    for i, l in enumerate(levels):
        s.level[i] = l
    for k, v in (ctl or {}).items():
        setattr(s, k, v)
    return s


def ref_level_sse(dlfc, cfg, mi, rec, src, ctl, mask=7, levels=range(64), glue=False):
    """ref_dlf_level_sse at the search's sharpness -> sse[3][n] (entries of planes outside the mask: -1), and with glue
    the (DlfFrame, DlfLevelSse, lvl tables) svt_b200_dlf_level_sse_from_pcs makes of the same search"""
    L = _layout()
    levels = list(levels)
    c = type(cfg).from_buffer_copy(cfg)
    c.sharpness = search_sharpness(ctl)
    s = _search(src, mask=mask, levels=levels)
    sse = np.full((3, len(levels)), -1, np.int64)
    frame, ls, lvl = L.DlfFrame(), L.DlfLevelSse(), np.zeros((3, len(levels), 256), np.uint8)
    f = dlfc.ref_dlf_level_sse
    f.restype = ct.c_int
    f.argtypes = [ct.c_void_p] * 5 + [ct.c_int, ct.c_int] + [ct.c_void_p] * 5
    rc = f(ct.addressof(c), mi.ctypes.data, *[_origin(p) for p in rec], rec[0].shape[1], rec[1].shape[1], ct.addressof(s),
           sse.ctypes.data, ct.addressof(frame) if glue else None, ct.addressof(ls) if glue else None, lvl.ctypes.data if glue else None)
    assert rc == 0
    return (sse, frame, ls, lvl) if glue else sse


def ref_pick(dlfc, cfg, mi, rec, src, ctl):
    """ref_dlf_pick -> (filter_level[0], filter_level[1], filter_level_u, filter_level_v), zero_filt_sse, best_filt_sse"""
    s = _search(src, ctl)
    f = dlfc.ref_dlf_pick
    f.restype = ct.c_int
    f.argtypes = [ct.c_void_p] * 5 + [ct.c_int, ct.c_int, ct.c_void_p]
    assert f(ct.addressof(cfg), mi.ctypes.data, *[_origin(p) for p in rec], rec[0].shape[1], rec[1].shape[1], ct.addressof(s)) == 0
    return tuple(s.picked), s.zero_filt_sse, s.best_filt_sse


# ---- the reference's search_filter_level, restated over a table of trial SSEs -------------------------------------------
def climb(sse, start, tx_mode, early_exit):
    """search_filter_level (deblocking_filter.c:886-1001) with try_filter_frame(level) = sse[level]: (level, tried)"""
    mid = min(max(start, 0), 63)
    step = 4 if mid < 16 else mid // 4
    tried = {mid: int(sse[mid])}
    best_err, best, direction, conv = tried[mid], mid, 0, 0
    while step > 0:
        hi, lo = min(mid + step, 63), max(mid - step, 0)
        bias = (best_err >> (15 - mid // 8)) * step
        if tx_mode != ONLY_4X4:
            bias >>= 1
        if direction <= 0 and lo != mid:
            tried.setdefault(lo, int(sse[lo]))
            if tried[lo] < best_err + bias:
                best_err = min(best_err, tried[lo])
                best = lo
        if direction >= 0 and hi != mid:
            tried.setdefault(hi, int(sse[hi]))
            if tried[hi] < best_err - bias:
                best_err, best = tried[hi], hi
        if best == mid:
            conv += 1
            step = 0 if conv == early_exit else step // 2
            direction = 0
        else:
            direction = -1 if best < mid else 1
            mid = best
    return best, tried


def pick_from_table(table, cfg, ctl):
    """svt_av1_pick_filter_level's full-image branch (deblocking_filter.c:1221-1290) for an intra picture without references,
    searching over table[plane][level]: (levels, zero_filt_sse, best_filt_sse)"""
    last = (cfg.filter_level[0], cfg.filter_level[1], cfg.filter_level_u, cfg.filter_level_v)
    y, tried = climb(table[0], (last[0] + last[1] + 1) >> 1, ctl["tx_mode"], ctl["early_exit_convergence"])
    u = v = 0
    if y:
        u = climb(table[1], last[2], ctl["tx_mode"], ctl["early_exit_convergence"])[0]
        v = climb(table[2], last[3], ctl["tx_mode"], ctl["early_exit_convergence"])[0]
    return (y, y, u, v), tried.get(0, -1), tried[y]


# ---- CPU: one-shot trials on the unfiltered picture == the reference's sequential search --------------------------------
CASES = [(size, fmt, variant) for size in SIZES for fmt in FORMATS for variant in range(6)]
CASE_IDS = ["%dx%d-bd%d-pb%d-v%d" % (s[0], s[1], f[0], f[1], v) for s, f, v in CASES]


def _case_of(size, fmt, variant):
    return search_case(size, fmt, variant, seed=size[0] * 31 + size[1] + fmt[0] * 7 + fmt[1] + variant * 1311,
                       sb_size=128 if variant == 4 else 64)


@pytest.mark.parametrize("size,fmt,variant", CASES, ids=CASE_IDS)
def test_climb_over_one_shot_table_equals_reference_pick(dlfc, size, fmt, variant):
    cfg, mi, rec, src, ctl = _case_of(size, fmt, variant)
    table = ref_level_sse(dlfc, cfg, mi, rec, src, ctl)
    assert ref_pick(dlfc, cfg, mi, rec, src, ctl) == pick_from_table(table, cfg, ctl)


def test_search_cases_cover_the_controls():
    """the CPU cases reach every sharpness, both early-exit settings, every tx_mode, both frame types, luma starts of 0
    and spread levels, and mode / ref deltas with segment features"""
    seen = {k: set() for k in ("sharpness", "early_exit_convergence", "tx_mode", "frame_type", "deltas", "start")}
    for size, fmt, variant in CASES:
        cfg, _, _, _, ctl = _case_of(size, fmt, variant)
        for k in ("early_exit_convergence", "tx_mode", "frame_type"):
            seen[k].add(ctl[k])
        seen["sharpness"].add(search_sharpness(ctl))
        seen["deltas"].add(bool(cfg.mode_ref_delta_enabled and cfg.segmentation_enabled))
        seen["start"].add((cfg.filter_level[0] + cfg.filter_level[1] + 1) >> 1 >> 4)
    assert seen["sharpness"] == set(range(8)) and seen["early_exit_convergence"] == {0, 1} and seen["tx_mode"] == {0, 1, 2}
    assert seen["frame_type"] == {0, 1} and seen["deltas"] == {False, True} and seen["start"] >= {0, 1, 2, 3}


# ---- GPU: svt_b200_dlf_level_sse_dev ---------------------------------------------------------------------------------
def _to_dev(torch, a):
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).to("cuda")


class DevCase:
    """the recon and source planes, records and glue-derived level tables of one search on the device"""

    def __init__(self, torch, frame, ls, lvl, mi, rec, src):
        self.frame, self.ls = frame, ls
        self.rec = [_to_dev(torch, p) for p in rec]
        self.src = [_to_dev(torch, p) for p in src]
        self.mi = torch.from_numpy(mi.view(np.uint8).reshape(-1)).to("cuda")
        self.lvl = torch.from_numpy(np.ascontiguousarray(lvl).reshape(-1)).to("cuda")
        isz = rec[0].itemsize
        for p in range(3):
            frame.plane[p] = self.rec[p].data_ptr() + (16 * rec[p].shape[1] + 16) * isz
            frame.stride[p] = rec[p].shape[1]
            ls.src[p] = self.src[p].data_ptr() + (16 * src[p].shape[1] + 16) * isz
            ls.src_stride[p] = src[p].shape[1]
        ls.d_lvl = self.lvl.data_ptr()

    def run(self, b200, torch, ls=None, frame=None):
        ls = ls or self.ls
        d_sse = torch.full((3 * ls.n_levels,), -1, dtype=torch.int64, device="cuda")
        rc = b200.dlf_level_sse_dev(frame or self.frame, ls, self.mi.data_ptr(), d_sse.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return rc, d_sse.cpu().numpy().reshape(3, ls.n_levels)


def _device_case(dlfc, torch, cfg, mi, rec, src, ctl, mask=7, levels=range(64)):
    sse, frame, ls, lvl = ref_level_sse(dlfc, cfg, mi, rec, src, ctl, mask=mask, levels=levels, glue=True)
    return sse, DevCase(torch, frame, ls, lvl, mi, rec, src)


@pytest.mark.gpu
@pytest.mark.parametrize("size,fmt,variant", CASES, ids=CASE_IDS)
def test_level_sse_dev_matches_reference(b200, dlfc, size, fmt, variant):
    """every level of every plane bit-exact with ref_dlf_level_sse, the recon planes untouched; then the climb over the
    device's table chooses what the reference's own search chooses"""
    import torch
    cfg, mi, rec, src, ctl = _case_of(size, fmt, variant)
    ref, dev = _device_case(dlfc, torch, cfg, mi, rec, src, ctl)
    before = [t.clone() for t in dev.rec]
    rc, got = dev.run(b200, torch)
    assert rc == 0
    bad = np.argwhere(got != ref)
    assert bad.size == 0, (bad[:8].tolist(), got[tuple(bad[0])], ref[tuple(bad[0])])
    for p in range(3):
        assert torch.equal(dev.rec[p], before[p]), p
    assert ref_pick(dlfc, cfg, mi, rec, src, ctl) == pick_from_table(got, cfg, ctl)


@pytest.mark.gpu
def test_level_lists_and_masks(b200, dlfc):
    """a short list in random order with level 0, and single planes, give the matching entries of the full list; planes
    outside the mask are not written"""
    import torch
    cfg, mi, rec, src, ctl = search_case((642, 362), (10, 2), 3, seed=4242)
    ref, dev = _device_case(dlfc, torch, cfg, mi, rec, src, ctl)
    rc, full = dev.run(b200, torch)
    assert rc == 0 and np.array_equal(full, ref)
    r = rng(99)
    for mask in (1, 2, 4, 5, 7):
        levels = [0] + [int(v) for v in r.choice(np.arange(1, 64), 6, replace=False)]
        r.shuffle(levels)
        ls = _layout().DlfLevelSse.from_buffer_copy(dev.ls)
        lvl = np.zeros((3, len(levels), 256), np.uint8)
        full_lvl = dev.lvl.cpu().numpy().reshape(3, 64, 256)
        for i, l in enumerate(levels):
            ls.level[i] = l
            lvl[:, i] = full_lvl[:, l]
        ls.n_levels, ls.plane_mask = len(levels), mask
        d_lvl = torch.from_numpy(lvl.reshape(-1)).to("cuda")
        ls.d_lvl = d_lvl.data_ptr()
        rc, got = dev.run(b200, torch, ls)
        assert rc == 0
        for p in range(3):
            want = full[p, levels] if (mask >> p) & 1 else np.full(len(levels), -1)
            assert np.array_equal(got[p], want), (mask, p, levels)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS, ids=["u8", "bd8in16", "bd10", "bd12"])
def test_chroma_with_luma_off_matches_reference(b200, dlfc, fmt):
    """with the frame's luma levels at 0 a chroma entry still filters its plane, as try_filter_frame does"""
    import torch
    cfg, mi, rec, src, ctl = search_case((200, 136), fmt, 0, seed=515 + fmt[0] + fmt[1])
    cfg.filter_level[0] = cfg.filter_level[1] = 0
    ref, dev = _device_case(dlfc, torch, cfg, mi, rec, src, ctl, mask=6)
    rc, got = dev.run(b200, torch)
    assert rc == 0 and np.array_equal(got[1:], ref[1:])
    assert all(np.any(ref[p, 1:] != ref[p, 0]) for p in (1, 2)), "no chroma entry was filtered"


@pytest.mark.gpu
def test_level_sse_dev_rejects_bad_arguments(b200, dlfc):
    import torch
    cfg, mi, rec, src, ctl = search_case((72, 72), (10, 2), 0, seed=7)
    _, dev = _device_case(dlfc, torch, cfg, mi, rec, src, ctl, levels=range(8))
    L = _layout()
    assert dev.run(b200, torch)[0] == 0

    def ls_with(**kw):
        ls = L.DlfLevelSse.from_buffer_copy(dev.ls)
        for k, v in kw.items():
            if k.startswith("level"):
                ls.level[int(k[5:])] = v
            elif k.startswith("src"):
                ls.src[int(k[3:])] = v
            else:
                setattr(ls, k, v)
        return ls

    def frame_with(**kw):
        f = L.DlfFrame.from_buffer_copy(dev.frame)
        for k, v in kw.items():
            if k.startswith("plane"):
                f.plane[int(k[5:])] = v
            else:
                setattr(f, k, v)
        return f

    for ls in (ls_with(n_levels=0), ls_with(n_levels=65), ls_with(level3=64), ls_with(plane_mask=0), ls_with(plane_mask=8),
               ls_with(src1=None), ls_with(plane_mask=1, src0=None), ls_with(d_lvl=None),
               ls_with(sse_width=0), ls_with(sse_width=80), ls_with(sse_height=80)):
        assert dev.run(b200, torch, ls)[0] == BAD_ARG
    for f in (frame_with(plane2=None), frame_with(bit_depth=9), frame_with(pixel_bytes=1), frame_with(width=0),
              frame_with(mi_rows=1), frame_with(mi_stride=1)):
        assert dev.run(b200, torch, frame=f)[0] == BAD_ARG
    assert dev.run(b200, torch, ls_with(plane_mask=1, src1=None, src2=None), frame_with(plane1=None, plane2=None))[0] == 0
