"""Synthetic "1080p preset-8 hot path" workload: the per-frame work lists the H100 T2 entry points
(and, in bench.py's reference arm, the reference's own kernels) are driven with.

One frame of work = what the reference's ME, EncDec (final encode pass), CDEF and REST process
kernels hand to the dispatched DSP functions for one 8-bit 4:2:0 picture at M8 / CRF 30 settings
(SURVEY.md 8d; search geometry from enc_mode_config.c:138-345 with qp 30, reference distance 1):

  ME     HME L0 4 regions of 16x4, L1/L2 8x3, full-pel 8x3, SUB_SAD, 2 references, every 64x64 block
  TX     residual (source - motion-compensated prediction) -> forward transform -> fp quantizer with
         quantisation matrices (PSY default) -> inverse + reconstruction (skipped for all-zero blocks, as the
         encode pass does), every luma and chroma sample once, in a 64..4 transform-size mix
  CDEF   strength search over 6 (luma, chroma) candidates on the non-skip 8x8 blocks, then apply
  REST   Wiener statistics (7x7 luma, 5x5 chroma) per restoration unit + the striped loop-restoration filter of the
         whole picture (64-row stripes offset by 8, saved deblocked / CDEF boundary lines, separable Wiener per unit)

Content follows SURVEY.md 8(d): multi-octave block noise panorama + global pan + sensor noise, seeded.
Everything here is plain numpy data preparation; it performs no DSP.
"""
import os

import numpy as np

try:
    from . import layout as dsp  # struct dtypes / geometry only: no library is loaded by this module
except ImportError:  # loaded stand-alone (bench.py's CPU reference arm must not import the product package)
    import layout as dsp

TX_W, TX_H = dsp.TX_W, dsp.TX_H

# CDEF search settings per encoder preset, from the reference's own tables for CRF 25-30, non-screen content
# (enc_mode_config.c:875-1110 + :1736-1747 CDEF search level):
#   M8: CDEF level 7 (subsampling 4);  M6 / M4: CDEF level 5 (3 + 3 strengths, every row, chroma first pass only)
PRESETS = {
    8: dict(cdef_y=[0, 4, 9, 17, 20, 35], cdef_uv=[0, 4, 8, 17, -1, 20], cdef_subsampling=4),
    6: dict(cdef_y=[0, 28, 60, 2, 30, 62], cdef_uv=[0, 28, 60, -1, -1, -1], cdef_subsampling=1),
    4: dict(cdef_y=[0, 28, 60, 2, 30, 62], cdef_uv=[0, 28, 60, -1, -1, -1], cdef_subsampling=1),
}
# The picture whose open-loop ME the workload runs: a B picture of temporal layer 3 in the default 5-layer random-access
# hierarchy, searching the reference counts the preset's MRP level tries on non-base pictures (set_mrp_ctrl,
# enc_handle.c:3376-3600: level 10 for M8 CRF, 9 for M6, 5 for M4) at picture distances 1, 2, 3(, 4).  `max_l` = the counts
# the ME result arrays are sized for (pd_process.c:3503-3519).  The MeContext controls of (preset, resolution class) are
# the reference's own derivation (svt_aom_sig_deriv_me), dumped by tools/dump_me_controls.py into me_controls.json.
ME_PICTURE = {
    8: dict(qp=30, n_ref=(2, 2), max_l=(3, 2), only_l_bwd=1, safe_limit_nref=2, gm_enabled=0),
    6: dict(qp=25, n_ref=(3, 2), max_l=(3, 2), only_l_bwd=1, safe_limit_nref=2, gm_enabled=0),
    4: dict(qp=25, n_ref=(4, 3), max_l=(4, 3), only_l_bwd=1, safe_limit_nref=0, gm_enabled=1),
}
ME_TEMPORAL_LAYER, ME_HIERARCHICAL_LEVELS, ME_IS_REF = 3, 4, 1
ME_DIST = ((-1, -2, -3, -4), (1, 2, 3, 0))  # picture-number difference of the references, list 0 (past) / list 1 (future)
# svt_aom_derive_input_resolution (sequence_control_set.c:113-131; thresholds definitions.h:2051-2056): classes 0..6
_RES_TH = (0x28500, 0x4CE00, 0xA1400, 0x16DA00, 0x535200, 0x140A000)


def input_resolution_class(width, height):
    return sum(1 for t in _RES_TH if width * height >= t)


_ME_CONTROLS = None


def me_controls(preset, width, height):
    """SvtB200MeControls field -> value for the workload's ME picture (see ME_PICTURE) at this preset / resolution class"""
    global _ME_CONTROLS
    if _ME_CONTROLS is None:
        import json
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "me_controls.json")) as f:
            _ME_CONTROLS = json.load(f)
    key = "m%d_class%d" % (preset, input_resolution_class(width, height))
    if key not in _ME_CONTROLS:
        raise KeyError("no ME controls for %s in me_controls.json: run tools/dump_me_controls.py where /root/reference exists" % key)
    return _ME_CONTROLS[key]


# BASELINE.json configs[k] -> (width, height, bit_depth, preset)
CONFIGS = {0: (640, 360, 8, 8), 1: (1920, 1080, 8, 8), 2: (1920, 1080, 10, 6), 3: (3840, 2160, 8, 8), 4: (3840, 2160, 10, 4)}
CONFIG_NAMES = {
    0: "configs[0]: 640x360 8-bit 4:2:0 synthetic hot path (the reference's CPU-runnable case; M8 search settings)",
    1: "configs[1]: 1920x1080 8-bit 4:2:0 synthetic, preset 8 CRF 30 hot path (ME 2+2 refs + TX + CDEF + Wiener), 1 frame/step",
    2: "configs[2]: 1920x1080 10-bit (HBD path) synthetic, preset 6 CRF 25 hot path, 1 frame/step",
    3: "configs[3]: 3840x2160 8-bit 4:2:0 synthetic, preset 8 hot path, 1 frame/step (frame-parallel across GPUs)",
    4: "configs[4]: 3840x2160 10-bit synthetic, preset 4, CDEF + restoration hot path, 1 frame/step",
}


def synth_sequence(width, height, n_frames, seed=20260923, bit_depth=8):
    """list of (Y, U, V) planes: uint8, or uint16 holding `bit_depth`-bit samples"""
    r = np.random.default_rng(seed)
    pw, ph = width + 64 + 3 * n_frames, height + 64 + n_frames
    pano = np.full((ph, pw), 128.0)
    for size, amp in ((64, 60), (16, 35), (4, 18), (1, 8)):
        g = r.normal(0, 1, ((ph + size - 1) // size + 1, (pw + size - 1) // size + 1))
        pano += np.kron(g, np.ones((size, size)))[:ph, :pw] * (amp / 3.0)
    frames = []
    for t in range(n_frames):
        y = pano[32 + t:32 + t + height, 32 + 3 * t:32 + 3 * t + width] + r.normal(0, 2, (height, width))
        yy = np.clip(y, 0, 255)
        c = 128 + 0.25 * (yy[0::2, 0::2] - 128)
        if bit_depth == 8:
            frames.append((yy.astype(np.uint8), np.clip(c + 3, 0, 255).astype(np.uint8), np.clip(c - 3, 0, 255).astype(np.uint8)))
        else:  # the same content with real low-order bits
            sc, mx = 1 << (bit_depth - 8), (1 << bit_depth) - 1
            frames.append(tuple(np.clip(np.rint(v * sc), 0, mx).astype(np.uint16) for v in (yy, np.clip(c + 3, 0, 255), np.clip(c - 3, 0, 255))))
    return frames


_AV1_TABLES = None


def av1_tables():
    """the reference's scan orders and quantization matrices (see tools/dump_av1_tables.py for the layout)"""
    global _AV1_TABLES
    if _AV1_TABLES is None:
        with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "av1_tables.npz")) as z:
            _AV1_TABLES = {k: z[k] for k in z.files}
    return _AV1_TABLES


def quant_tables(d_dc, d_ac):
    return {"zbin": np.array([(84 * d_dc + 64) >> 7, (84 * d_ac + 64) >> 7], np.int16),
            "round": np.array([(64 * d_dc) >> 7, (64 * d_ac) >> 7], np.int16),
            "quant": np.array([(1 << 16) // d_dc, (1 << 16) // d_ac], np.uint16).astype(np.int16),
            "quant_shift": np.array([0, 0], np.int16),
            "dequant": np.array([d_dc, d_ac], np.int16)}


class FrameWorkload:
    PAD = 16  # border of the reconstruction planes (restoration reads 3(+1) pixels beyond the picture)

    def __init__(self, width=1920, height=1080, seed=20260923, bit_depth=8, preset=8):
        assert width % 8 == 0 and height % 8 == 0 and bit_depth in (8, 10) and preset in PRESETS
        self.width, self.height, self.bit_depth, self.preset = width, height, bit_depth, preset
        self.me_picture = ME_PICTURE[preset]
        self.n_ref = self.me_picture["n_ref"]          # (list 0, list 1) reference pictures searched
        self.n_refs = self.n_ref[0] + self.n_ref[1]
        self.me_controls = me_controls(preset, width, height)
        self.pixel_bytes = 1 if bit_depth == 8 else 2
        self.pixel_dtype = np.uint8 if bit_depth == 8 else np.uint16
        self._set_pictures(seed)
        self.me_shapes = dsp.me_plane_shapes(width, height)
        self.me_n_pu = 85 if self.me_controls["enable_me_8x8"] else 21  # square PUs that carry ME candidates (enable_me_16x16 is always on)
        self.plane_dims = [(width, height), (width // 2, height // 2), (width // 2, height // 2)]
        self._build_tx_items()
        self._build_cdef()
        self._build_rest()

    @classmethod
    def from_config(cls, k, seed=20260923):
        w, h, bd, preset = CONFIGS[k]
        return cls(w, h, seed=seed, bit_depth=bd, preset=preset)

    def me_luma(self, planes):
        """the 8-bit luma open-loop ME searches: the picture itself, or the 8 MSBs of a 10-bit picture (the
        reference keeps that plane for every input, pic_analysis / EbPaReferenceObject)"""
        return planes[0] if self.bit_depth == 8 else (planes[0] >> (self.bit_depth - 8)).astype(np.uint8)

    def _set_pictures(self, seed):
        self.seed = seed
        back, fwd = max(-d for d in ME_DIST[0][:self.n_ref[0]]), max((0,) + ME_DIST[1][:self.n_ref[1]])
        seq = synth_sequence(self.width, self.height, back + fwd + 1, seed, self.bit_depth)
        self.cur = seq[back]
        # reference pictures in the order the ME call takes them: list 0 (nearest past first), then list 1 (nearest future first)
        self.refs = [seq[back + d] for d in ME_DIST[0][:self.n_ref[0]]] + [seq[back + d] for d in ME_DIST[1][:self.n_ref[1]]]
        # prediction = the previous picture displaced by the sequence's global motion (the panorama pans (3, 1) luma
        # pixels per frame): an integer-pel motion-compensated inter prediction, edge-clamped like a padded reference.
        # Luma residual = the sensor noise of the two pictures; chroma keeps the half-pel mismatch of its (1.5, 0.5) motion.
        self.pred = [self._shift(self.refs[0][p], *((3, 1) if p == 0 else (2, 1))) for p in range(3)]
        self.residual = [self.cur[p].astype(np.int16) - self.pred[p].astype(np.int16) for p in range(3)]

    @staticmethod
    def _shift(plane, dx, dy):
        h, w = plane.shape
        ys = np.clip(np.arange(h) + dy, 0, h - 1)
        xs = np.clip(np.arange(w) + dx, 0, w - 1)
        return np.ascontiguousarray(plane[np.ix_(ys, xs)])

    def with_seed(self, seed):
        """the same work lists (they do not depend on the content) over another synthetic sequence"""
        import copy
        w = copy.copy(self)
        w._set_pictures(seed)
        return w

    # -- planes as flat buffers ---------------------------------------------------------------------
    def flat_offsets(self, itemsize_elems=1):
        off, o = [], 0
        for (w, h) in self.plane_dims:
            off.append(o)
            o += w * h
        return off, o

    def padded_shape(self, p):
        w, h = self.plane_dims[p]
        return h + 2 * self.PAD, (w + 2 * self.PAD + 15) & ~15

    def padded_offsets(self):
        off, o = [], 0
        for p in range(3):
            th, st = self.padded_shape(p)
            off.append(o)
            o += th * st
        return off, o

    # -- transform / quant / inverse work lists ---------------------------------------------------------
    def _build_tx_items(self):
        W, H = self.width, self.height
        res_off, _ = self.flat_offsets()
        rec_off, _ = self.padded_offsets()
        pattern = [4] * 2 + [3] * 6 + [2] * 8 + [1] * 3 + [0] * 1
        types_small = [0] * 7 + [3, 9, 10]
        fwd, inv, qnt = [], [], []
        coef_pos = 0
        sizes_used = set()
        k = 0
        for sby in range(0, H, 64):
            for sbx in range(0, W, 64):
                sz_l = pattern[k % len(pattern)]
                k += 1
                if sby + 64 > H or sbx + 64 > W:
                    sz_l = 1  # partial superblock: 8x8 luma / 4x4 chroma tiles the remainder exactly
                for p in range(3):
                    dec = 1 if p else 0
                    sz = sz_l if p == 0 else max(sz_l - 1, 0)
                    bw, bh = TX_W[sz], TX_H[sz]
                    pw, ph = self.plane_dims[p]
                    x0, y0 = sbx >> dec, sby >> dec
                    x1, y1 = min(x0 + (64 >> dec), pw), min(y0 + (64 >> dec), ph)
                    th, st = self.padded_shape(p)
                    j = 0
                    for y in range(y0, y1, bh):
                        for x in range(x0, x1, bw):
                            if y + bh > ph or x + bw > pw:
                                continue
                            ty = types_small[(k + j) % len(types_small)] if max(bw, bh) <= 16 else 0
                            j += 1
                            n = min(bw, 32) * min(bh, 32)
                            fwd.append((res_off[p] + y * pw + x, coef_pos, pw, sz, ty, 1))
                            rpos = rec_off[p] + (self.PAD + y) * st + self.PAD + x
                            inv.append((coef_pos, rpos, rpos, st, st, sz, ty, self.bit_depth, 0, 0))
                            qnt.append((coef_pos, sz, ty, int(p > 0)))
                            coef_pos += n
                            sizes_used.add(sz)
        self.fwd_items = np.array(fwd, dtype=dsp.FWD_ITEM_DTYPE)
        self.inv_items = np.array(inv, dtype=dsp.INV_ITEM_DTYPE)
        self.n_coeffs = coef_pos
        # scan orders and quantization matrices: the reference's own tables (av1_tables.npz, dumped from the compiled reference by
        # tools/dump_av1_tables.py).  One entry per (tx_size, tx_type) / (plane type, tx_size) in use.  QM levels as the encoder
        # derives them for qindex 120 with its default --qm-min 2 --qm-max 15 / --chroma-qm-min 8 --chroma-qm-max 15
        # (aom_get_qmlevel, md_config_process.c:189; defaults enc_settings.c:1058-1062)
        tb = av1_tables()
        self.qindex = 120
        self.qm_level = (2 + (self.qindex * (15 + 1 - 2)) // 256, 8 + (self.qindex * (15 + 1 - 8)) // 256)
        scan_parts, iscan_parts, qm_parts, scan_off, qm_off = [], [], [], {}, {}
        so = qo = 0
        for sz, ty in sorted({(s_, t_) for _, s_, t_, _ in qnt}):
            n, o = int(tb["scan_len"][sz]), int(tb["scan_off"][sz, ty])
            assert n == min(TX_W[sz], 32) * min(TX_H[sz], 32)
            scan_off[sz, ty] = so
            scan_parts.append(tb["scan"][o:o + n])
            iscan_parts.append(tb["iscan"][o:o + n])
            so += n
        for sz, pt in sorted({(s_, c_) for _, s_, _, c_ in qnt}):
            n, o = int(tb["scan_len"][sz]), int(tb["qm_off"][sz])
            qm_off[sz, pt] = (qo, qo + n)
            qm_parts += [tb["qm"][self.qm_level[pt], pt, o:o + n], tb["iqm"][self.qm_level[pt], pt, o:o + n]]
            qo += 2 * n
        self.scan_table = np.ascontiguousarray(np.concatenate(scan_parts), np.int16)
        self.iscan_table = np.ascontiguousarray(np.concatenate(iscan_parts), np.int16)
        self.qm_table = np.ascontiguousarray(np.concatenate(qm_parts), np.uint8)
        t = quant_tables(52 << (self.bit_depth - 8), 61 << (self.bit_depth - 8))  # dc/ac step of qindex ~120, scaled with the bit depth
        q = np.zeros(len(qnt), dtype=dsp.QUANT_ITEM_DTYPE)
        cp = np.array([c for c, _, _, _ in qnt], np.uint64)
        szs = np.array([s for _, s, _, _ in qnt])
        q["coeff_off"] = q["q_off"] = q["dq_off"] = cp
        q["scan_off"] = [scan_off[s_, t_] for _, s_, t_, _ in qnt]
        q["qm_off"] = [qm_off[s_, c_][0] for _, s_, _, c_ in qnt]
        q["iqm_off"] = [qm_off[s_, c_][1] for _, s_, _, c_ in qnt]
        q["n_coeffs"] = [min(TX_W[s], 32) * min(TX_H[s], 32) for s in szs]
        for name in ("zbin", "round", "quant", "quant_shift", "dequant"):
            q[name] = t[name]
        q["mode"] = dsp.QUANT_FP_LBD if self.bit_depth == 8 else dsp.QUANT_FP_HBD
        # log_scale of av1_get_tx_scale: 0 up to 256 coefficients... 1 for 512/1024, 2 for 64x64-class
        q["log_scale"] = [2 if TX_W[s] * TX_H[s] > 1024 else (1 if TX_W[s] * TX_H[s] > 256 else 0) for s in szs]
        self.quant_items = q
        # batch order of the transform calls: by team class, then (tx_size, tx_type) so that teams sharing a warp agree
        cls = np.array([dsp.txfm_team_class(int(s)) for s in self.fwd_items["tx_size"]])
        order = np.lexsort((self.fwd_items["tx_type"], self.fwd_items["tx_size"], cls))
        self.fwd_items = self.fwd_items[order]
        self.inv_items = self.inv_items[order]
        self.quant_items = self.quant_items[order]  # same block order everywhere (eobs[i] belongs to block i)
        trio = np.zeros(len(order), dtype=dsp.TRIO_ITEM_DTYPE)  # the fused call takes the three items side by side
        trio["fwd"], trio["quant"], trio["inv"] = self.fwd_items, self.quant_items, self.inv_items
        self.trio_items = trio
        self.tx_class_counts = [int((cls == c).sum()) for c in range(dsp.TXFM_CLASSES)]

    # -- CDEF ---------------------------------------------------------------------------------------------
    def _build_cdef(self):
        r = np.random.default_rng(11)
        self.skip8x8 = (r.random(((self.height + 7) // 8, (self.width + 7) // 8)) < 0.10).astype(np.uint8)
        ps = PRESETS[self.preset]
        self.cdef_str_y = np.array(ps["cdef_y"], np.int32)
        self.cdef_str_uv = np.array(ps["cdef_uv"], np.int32)
        self.cdef_damping = 3 + (120 >> 6)
        self.cdef_subsampling = ps["cdef_subsampling"]  # CdefSearchControls.subsampling_factor of the preset's search level
        nfb = ((self.width + 63) // 64) * ((self.height + 63) // 64)
        self.cdef_fb_idx = (np.arange(nfb) % 4).astype(np.int8)
        self.cdef_apply_y = np.array([4, 9, 17, 0], np.int32)
        self.cdef_apply_uv = np.array([4, 8, 0, 0], np.int32)

    # -- restoration ------------------------------------------------------------------------------------------
    @staticmethod
    def lr_unit_ranges(size, unit_size, off):
        """[(start, end)] of the restoration units along one dimension: units of `unit_size`, the last one absorbs a
        remainder below 1.5 units (foreach_rest_unit_in_tile, restoration.c:1247-1294); with off > 0 (rows) every unit is
        shifted up by the 8-luma-row stripe offset"""
        n = max((size + (unit_size >> 1)) // unit_size, 1)
        out = []
        for i in range(n):
            s0 = max(0, i * unit_size - off)
            e0 = size if i == n - 1 else (i + 1) * unit_size - off
            out.append((s0, e0))
        return out

    def _build_rest(self):
        r = np.random.default_rng(13)
        rec_off, _ = self.padded_offsets()
        src_off, _ = self.flat_offsets()
        stats, self.lr_units, self.lr_unit_size = [], [], []
        for p in range(3):
            pw, ph = self.plane_dims[p]
            th, st = self.padded_shape(p)
            ru = 256 if p == 0 else 128
            win = 7 if p == 0 else 5
            cols, rows = self.lr_unit_ranges(pw, ru, 0), self.lr_unit_ranges(ph, ru, 8 >> (1 if p else 0))
            units = np.zeros(len(rows) * len(cols), dtype=dsp.LR_UNIT_DTYPE)
            k = 0
            for (y0, y1) in rows:
                for (x0, x1) in cols:
                    # search_wiener_seg: statistics over the unit's limits (restoration_pick.c:1281-1330)
                    stats.append((rec_off[p] + self.PAD * st + self.PAD, src_off[p], st, pw, x0, x1, y0, y1, win, 0))
                    t0, t1, t2 = int(r.integers(-5, 11)), int(r.integers(-23, 9)), int(r.integers(-17, 47))
                    taps = np.array([t0, t1, t2, -2 * (t0 + t1 + t2), t2, t1, t0, 0], np.int16)
                    if p:
                        taps[0] = taps[6] = 0  # chroma uses the 5-tap window
                        taps[3] = -2 * (taps[1] + taps[2])
                    units["restoration_type"][k] = 1  # RESTORE_WIENER (the self-guided filter is off at these presets, SURVEY F8)
                    units["hfilter"][k] = taps
                    units["vfilter"][k] = taps
                    k += 1
            self.lr_units.append(units)
            self.lr_unit_size.append(ru)
        self.stats_items = np.array(stats, dtype=dsp.STATS_ITEM_DTYPE)

    def lr_num_stripes(self, p):
        ss = 1 if p else 0
        return (self.plane_dims[p][1] + (8 >> ss) + (64 >> ss) - 1) // (64 >> ss)

    def lr_boundary_stride(self, p):
        return (self.plane_dims[p][0] + 8 + 31) & ~31

    # -- algorithmic bytes per frame (SURVEY.md 8d) -----------------------------------------------------------
    def algorithmic_bytes(self):
        """SURVEY 8(d) figures, per call of the frame pipeline (bpp = bytes per pixel)"""
        W, H, R, bpp = self.width, self.height, self.n_refs, self.pixel_bytes
        n64 = ((W + 63) // 64) * ((H + 63) // 64)
        N = int(1.5 * W * H)  # samples = transform coefficients of the final pass
        calls = {
            "me_pyramid": int(1.3125 * W * H),                                    # full-res read + the two decimated levels written
            "me_search": int((1 + R) * 1.3125 * W * H + n64 * R * 85 * 8),        # every pyramid read once + SAD/MV per reference out
            "fwd_txfm": 6 * N, "quant": 12 * N, "inv_txfm": (4 + 2 * bpp) * N,    # (22 + 2 bpp) N in total
            "txfm_trio": (22 + 2 * bpp) * N,                                      # SURVEY 8(d)'s figure for the unfused chain
            # what the FUSED call has to move: source + prediction in, qcoeff + dqcoeff (4N each) + recon out
            "txfm_trio_fused_min": (8 + 3 * bpp) * N,    # source + prediction in, qcoeff + dqcoeff + recon out
            "pack_levels": 6 * N,                                                 # upper bound: every level read (4 B) and written (<= 4 B) once more
            "cdef_search": int(2 * bpp * N + n64 * 2 * len(self.cdef_str_y) * 8),  # recon + source in, mse out
            "cdef_apply": 2 * bpp * N,                                            # recon in, filtered out
            "rest_extend": 0,
            "wiener_stats": int(2 * bpp * N + len(self.stats_items) * (49 + 2401) * 8),
            "lr_boundaries": 0,                                                   # 4 lines per 64-row stripe: ~6 % of a plane, not counted
            "wiener_filter": 2 * bpp * N,
        }
        stage_of = {"me_pyramid": "me", "me_search": "me", "txfm_trio": "tx", "pack_levels": "tx", "cdef_search": "cdef",
                    "cdef_apply": "cdef", "lr_boundaries": "rest", "rest_extend": "rest", "wiener_stats": "rest", "wiener_filter": "rest"}
        out = dict(calls)
        for st in ("me", "tx", "cdef", "rest"):
            out[st] = sum(v for k, v in calls.items() if stage_of.get(k) == st)
        return out

    def wiener_stats_macs(self):
        """multiply-accumulates of compute_stats: (win^2 (win^2 + 1) / 2 + win^2) per pixel (SURVEY 8d)"""
        tot = 0
        for it in self.stats_items:
            win = int(it["wiener_win"])
            w2 = win * win
            tot += (int(it["h_end"]) - int(it["h_start"])) * (int(it["v_end"]) - int(it["v_start"])) * (w2 * (w2 + 1) // 2 + w2)
        return tot
