"""The C ABI's data layout (include/svt_b200.h), described once: one ctypes.Structure per `typedef struct SvtB200*`, named
after the C type without `SvtB200`, with the header's fields in the header's order (natural alignment, pointers as
c_void_p); the numpy dtypes of the T2 work items derived from those; the reference's enumerator values and the plane
geometry of the ME pyramid.  tests/test_host_logic.py checks every field of every class against the compiled header.
No library is loaded here -- the module is shared by the product's host mirror (dsp.py), the synthetic workload
(workload.py) and, loaded stand-alone, by the CPU checkers of the tests and bench.py's CPU reference arm, which must not
map libsvtav1_b200.so."""
import ctypes as ct

import numpy as np


def _same(ctype, *names):
    return [(n, ctype) for n in names]


# ---- K1/K3 SAD search -----------------------------------------------------------------------------------------------
class SadSearchItem(ct.Structure):
    _fields_ = [("src_off", ct.c_uint64), ("ref_off", ct.c_uint64), ("src_stride", ct.c_uint32), ("ref_stride", ct.c_uint32),
                ("ref_step", ct.c_uint32), ("block_w", ct.c_uint16), ("block_h", ct.c_uint16), ("sa_w", ct.c_int16),
                ("sa_h", ct.c_int16), ("skip_search_line", ct.c_uint16), ("reserved", ct.c_uint16)]


class SadSearchResult(ct.Structure):
    _fields_ = [("best_sad", ct.c_uint32), ("x", ct.c_int16), ("y", ct.c_int16)]


SAD_ITEM_DTYPE = np.dtype(SadSearchItem)
SAD_RESULT_DTYPE = np.dtype(SadSearchResult)

# ---- K5/K6 transforms, K7 quantisation ------------------------------------------------------------------------------
TX_W = [4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64]
TX_H = [4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16]
TX_NAME = ["%dx%d" % (w, h) for w, h in zip(TX_W, TX_H)]
TXFM_CLASSES = 5  # SVT_B200_TXFM_CLASSES

def txfm_team_class(tx_size):
    """log2(max(W, H)) - 2: the order key of the transform batch calls (svt_b200_txfm_team_class)."""
    return {4: 0, 8: 1, 16: 2, 32: 3, 64: 4}[max(TX_W[tx_size], TX_H[tx_size])]


class FwdTxfmItem(ct.Structure):
    _fields_ = [("src_off", ct.c_uint64), ("dst_off", ct.c_uint64), ("src_stride", ct.c_uint32), ("tx_size", ct.c_uint8),
                ("tx_type", ct.c_uint8), ("reserved", ct.c_uint16)]


class InvTxfmItem(ct.Structure):
    _fields_ = _same(ct.c_uint64, "coef_off", "pred_off", "recon_off") + _same(ct.c_uint32, "pred_stride", "recon_stride") + \
               _same(ct.c_uint8, "tx_size", "tx_type", "bd", "reserved") + [("reserved2", ct.c_uint32)]


QUANT_B_LBD, QUANT_B_HBD, QUANT_FP_LBD, QUANT_FP_HBD = 0, 1, 2, 3
NO_QM = 0xffffffff


class QuantItem(ct.Structure):
    _fields_ = _same(ct.c_uint64, "coeff_off", "q_off", "dq_off") + _same(ct.c_uint32, "scan_off", "qm_off", "iqm_off", "n_coeffs") + \
               _same(ct.c_int16 * 2, "zbin", "round", "quant", "quant_shift", "dequant") + \
               [("mode", ct.c_uint8), ("log_scale", ct.c_uint8), ("reserved", ct.c_uint16)]


class TrioItem(ct.Structure):  # the fused call takes the three items side by side
    _fields_ = [("fwd", FwdTxfmItem), ("quant", QuantItem), ("inv", InvTxfmItem)]


class ResidualPlane(ct.Structure):
    _fields_ = _same(ct.c_uint64, "src_off", "pred_off", "res_off") + \
               _same(ct.c_int32, "src_stride", "pred_stride", "res_stride", "w", "h", "reserved")


class ResidualPlanes(ct.Structure):
    _fields_ = [("p", ResidualPlane * 3)]


FWD_ITEM_DTYPE = np.dtype(FwdTxfmItem)
INV_ITEM_DTYPE = np.dtype(InvTxfmItem)
QUANT_ITEM_DTYPE = np.dtype(QuantItem)
TRIO_ITEM_DTYPE = np.dtype(TrioItem)

# ---- K4 Hadamard / SATD, K2 full-pel search -------------------------------------------------------------------------
class Buf2D(ct.Structure):  # == the reference's Buf2D
    _fields_ = [("buf", ct.c_void_p), ("buf0", ct.c_void_p), ("width", ct.c_int), ("height", ct.c_int), ("stride", ct.c_int)]


class HadamardItem(ct.Structure):
    _fields_ = [("src_off", ct.c_uint64), ("coeff_off", ct.c_uint64), ("src_stride", ct.c_uint32), ("size", ct.c_uint32)]


class FullpelItem(ct.Structure):
    _fields_ = [("src_off", ct.c_uint64), ("ref_off", ct.c_uint64), ("src_stride", ct.c_uint32), ("ref_stride", ct.c_uint32)] + \
               _same(ct.c_int16, "sa_w", "sa_h", "org_x", "org_y") + [("sub_sad", ct.c_uint8), ("seeded", ct.c_uint8)] + \
               [("seed_x", ct.c_int16), ("seed_y", ct.c_int16), ("reserved", ct.c_uint8 * 2)]


HADAMARD_ITEM_DTYPE = np.dtype(HadamardItem)
FULLPEL_ITEM_DTYPE = np.dtype(FullpelItem)

# ---- K8 CDEF --------------------------------------------------------------------------------------------------------
class CdefList(ct.Structure):  # == the reference's CdefList
    _fields_ = [("by", ct.c_uint8), ("bx", ct.c_uint8)]


class CdefFrame(ct.Structure):
    _fields_ = _same(ct.c_void_p, "recon_y", "recon_cb", "recon_cr", "src_y", "src_cb", "src_cr") + \
               _same(ct.c_int32, "recon_stride_y", "recon_stride_c", "src_stride_y", "src_stride_c", "width", "height", "bit_depth",
                     "damping", "subsampling_factor", "reserved")


# ---- K14 deblocking loop filter ---------------------------------------------------------------------------------------
class DlfMi(ct.Structure):
    _fields_ = _same(ct.c_uint8, "bsize", "tx_depth", "skip") + [("ref_frame0", ct.c_int8), ("mode", ct.c_uint8), ("segment_id", ct.c_uint8),
                                                                 ("reserved", ct.c_uint8 * 2)]


class DlfFrame(ct.Structure):
    _fields_ = [("plane", ct.c_void_p * 3), ("stride", ct.c_int32 * 3)] + \
               _same(ct.c_int32, "width", "height", "mi_rows", "mi_cols", "mi_stride", "bit_depth", "pixel_bytes") + \
               [("filter_level", ct.c_int32 * 2)] + _same(ct.c_int32, "filter_level_u", "filter_level_v", "reserved") + \
               [("lvl", ct.c_uint8 * 2 * 8 * 2 * 8 * 3), ("lfthr", ct.c_uint8 * 3 * 64), ("reserved2", ct.c_uint8 * 4)]


class DlfLevelSse(ct.Structure):
    _fields_ = [("src", ct.c_void_p * 3), ("src_stride", ct.c_int32 * 3)] + \
               _same(ct.c_int32, "sse_width", "sse_height", "plane_mask", "n_levels") + \
               [("level", ct.c_uint8 * 64), ("reserved", ct.c_uint8 * 4), ("d_lvl", ct.c_void_p)]


DLF_MI_DTYPE = np.dtype(DlfMi)


# ---- K9/K11 Wiener filter + statistics, K10/K12 self-guided filter, a13 loop-restoration drivers --------------------
class ConvolveParams(ct.Structure):  # == the reference's ConvolveParams
    _fields_ = [("ref", ct.c_int32), ("do_average", ct.c_int32), ("dst", ct.c_void_p)] + \
               _same(ct.c_int32, "dst_stride", "round_0", "round_1", "plane", "is_compound", "use_jnt_comp_avg", "fwd_offset",
                     "bck_offset", "use_dist_wtd_comp_avg")


class WienerUnit(ct.Structure):
    _fields_ = [("src_off", ct.c_uint64), ("dst_off", ct.c_uint64), ("src_stride", ct.c_int32), ("dst_stride", ct.c_int32),
                ("w", ct.c_uint16), ("h", ct.c_uint16), ("reserved", ct.c_uint32), ("hfilter", ct.c_int16 * 8), ("vfilter", ct.c_int16 * 8)]


class StatsItem(ct.Structure):
    _fields_ = [("dgd_off", ct.c_uint64), ("src_off", ct.c_uint64)] + \
               _same(ct.c_int32, "dgd_stride", "src_stride", "h_start", "h_end", "v_start", "v_end", "wiener_win", "reserved")


class SgrUnit(ct.Structure):
    _fields_ = _same(ct.c_uint64, "dgd_off", "flt0_off", "flt1_off") + [("dgd_stride", ct.c_int32), ("flt_stride", ct.c_int32)] + \
               _same(ct.c_uint16, "w", "h", "params_idx", "reserved")


class LrPlane(ct.Structure):
    _fields_ = _same(ct.c_void_p, "deblocked", "cdef", "dst", "src", "boundary_above", "boundary_below") + \
               _same(ct.c_int32, "stride_deblocked", "stride_cdef", "stride_dst", "stride_src", "boundary_stride", "width", "height",
                     "ss_x", "ss_y", "unit_size", "frame_restoration_type")


class LrUnitInfo(ct.Structure):
    _fields_ = [("restoration_type", ct.c_int32), ("sgr_ep", ct.c_int32), ("sgr_xqd", ct.c_int32 * 2), ("hfilter", ct.c_int16 * 8),
                ("vfilter", ct.c_int16 * 8)]


WIENER_UNIT_DTYPE = np.dtype(WienerUnit)
STATS_ITEM_DTYPE = np.dtype(StatsItem)
SGR_UNIT_DTYPE = np.dtype(SgrUnit)
LR_UNIT_DTYPE = np.dtype(LrUnitInfo)

# ---- K13 + T2 open-loop ME ------------------------------------------------------------------------------------------
ME_PAD = (16, 32, 72)  # padding of the 1/16, 1/4 and full luma planes (the reference uses 16 / 32 / 64+)


def me_plane_shapes(width, height):
    """[(h_total, w_total, org, w, h)] for levels 0 (1/16), 1 (1/4), 2 (full); strides are 16-byte multiples"""
    out = []
    for lvl in range(3):
        w, h, pad = width >> (2 - lvl), height >> (2 - lvl), ME_PAD[lvl]
        stride = (w + 2 * pad + 15) & ~15
        out.append((h + 2 * pad, stride, pad, w, h))
    return out

SAD_SIZES = [(128, 128), (128, 64), (64, 128), (64, 64), (64, 32), (64, 16), (32, 64), (32, 32), (32, 16), (32, 8), (16, 64), (16, 32), (16, 16), (16, 8), (16, 4), (8, 32), (8, 16), (8, 8), (8, 4), (4, 16), (4, 8), (4, 4)]  # (width, height) of the svt_aom_sadMxN family


class MePicture(ct.Structure):
    _fields_ = [("plane", ct.c_void_p * 3)] + _same(ct.c_int32 * 3, "stride", "org_x", "org_y", "width", "height") + \
               [("reserved", ct.c_int32 * 2)]


class PlaneExtent(ct.Structure):
    _fields_ = [("buf", ct.c_void_p)] + _same(ct.c_int32, "stride", "w", "h", "org_x", "org_y", "pixel_bytes")


# SvtB200MeControls: the MeContext controls after svt_aom_sig_deriv_me, flattened; (name, int32 count)
ME_CONTROL_FIELDS = [("n_list", 1), ("n_ref", 2), ("temporal_layer_index", 1), ("is_ref", 1), ("hierarchical_levels", 1), ("dist", 8),
                     ("enable_hme", 1), ("enable_l0", 1), ("enable_l1", 1), ("enable_l2", 1), ("hme_sub_sad", 1), ("me_sub_sad", 1),
                     ("hme_l0_min_w", 1), ("hme_l0_min_h", 1), ("hme_l0_max_w", 1), ("hme_l0_max_h", 1), ("hme_l1_w", 1), ("hme_l1_h", 1),
                     ("hme_l2_w", 1), ("hme_l2_h", 1), ("me_min_w", 1), ("me_min_h", 1), ("me_max_w", 1), ("me_max_h", 1),
                     ("prehme_enable", 1), ("prehme_sa", 8), ("prehme_skip_search_line", 1), ("prehme_l1_early_exit", 1),
                     ("prune_enable", 1), ("prune_hme_th", 1), ("prune_me_th", 1), ("zz_sad_th", 1), ("zz_sad_pct", 1), ("phme_sad_th", 1),
                     ("phme_sad_pct", 1), ("sr_enable", 1), ("sr_mv_length_th", 1), ("sr_stationary_hme_sad_abs_th", 1),
                     ("sr_stationary_divisor", 1), ("sr_hme_sad_abs_th", 1), ("sr_low_hme_sad_divisor", 1), ("sr_distance_based_hme_resizing", 1),
                     ("var_enable", 1), ("var_div4_th", 1), ("var_div2_th", 1), ("var_mult2_th", 1),
                     ("mvsa_enable", 1), ("mvsa_nearest_ref_only", 1), ("mvsa_mv_size_th", 1), ("mvsa_multiplier", 1),
                     ("reduce_hme_l0_sr_th_min", 1), ("reduce_hme_l0_sr_th_max", 1),
                     ("me_early_exit_th", 1), ("me_safe_limit_zz_th", 1), ("prev_me_stage_based_exit_th", 1), ("prune_me_candidates_th", 1),
                     ("use_best_unipred_cand_only", 1), ("similar_brightness_refs", 1), ("only_l_bwd", 1), ("enable_me_8x8", 1),
                     ("enable_me_16x16", 1), ("max_cand", 1), ("max_refs", 1), ("max_l0", 1), ("gm_enabled", 1),
                     ("gm_use_distance_based_active_th", 1), ("resolution_le_480p", 1), ("reserved", 5)]


class MeControls(ct.Structure):  # the 2-D arrays of the header (dist, prehme_sa) are flat here
    _fields_ = [(n, ct.c_int32 if k == 1 else ct.c_int32 * k) for n, k in ME_CONTROL_FIELDS]

    @classmethod
    def from_dict(cls, d):
        """d: field -> int (or a flat list for the array fields), e.g. the reference's derivation dumped by tools/dump_me_controls.py"""
        c = cls()
        for n, k in ME_CONTROL_FIELDS:
            if n == "reserved" or n not in d:
                continue
            if k == 1:
                setattr(c, n, int(d[n]))
            else:
                for i, v in enumerate(d[n]):
                    getattr(c, n)[i] = int(v)
        return c

    def as_dict(self):
        return {n: (int(getattr(self, n)) if k == 1 else [int(v) for v in getattr(self, n)]) for n, k in ME_CONTROL_FIELDS if n != "reserved"}


class MeB64Results(ct.Structure):  # device pointers
    _fields_ = _same(ct.c_void_p, "total_me_candidate_index", "me_candidate_array", "me_mv_array", "distortion", "flags", "do_ref",
                     "hme_centre", "zz_sad", "best_sad", "best_mv")


# golden-fixture / comparison names of the ME outputs -> MeB64Results field (best_sad / best_mv are undefined for pruned references: not compared whole)
ME_OUTPUT_NAMES = {"me_total": "total_me_candidate_index", "me_cand": "me_candidate_array", "me_mvs": "me_mv_array", "me_dist": "distortion",
                   "me_flags": "flags", "me_do_ref": "do_ref", "me_centre": "hme_centre", "me_zz": "zz_sad"}
