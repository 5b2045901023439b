"""GPU parity of the complete open-loop ME driver at the shapes its HME stages cut into warp jobs differently: more than
five references (every pre-HME and HME stage has more jobs than the CTA has warps), partial last block column and row
(the narrow-block search path and clipped windows), and the 1080p preset-8 picture, whose 200-row pre-HME strips are cut
into row slices and clipped at the bottom of the picture.  The comparison is the one of test_me_b64."""
import pytest

import me_helpers as mh
import test_me_b64 as base
from helpers import rng
from oracle import support as sp

pytestmark = pytest.mark.gpu

CASES = [
    # name, W, H, preset, n_ref, poc distances, temporal layer, is_ref, extra cfg, content
    ("m4_nonbase_4p3_partial", 456, 328, 4, (4, 3), ((-1, -2, -3, -4), (1, 2, 3, 0)), 3, 0, dict(max_l=(4, 3), only_l_bwd=0),
     dict(pan=(0, 0), noise=20.0)),
    ("m6_ref_3p2", 384, 256, 6, (3, 2), ((-2, -4, -6, 0), (2, 4, 0, 0)), 2, 1, dict(max_l=(3, 2)), dict(pan=(1, 0), noise=14.0)),
    ("m8_1080p_2p2", 1920, 1080, 8, (2, 2), ((-1, -2, 0, 0), (1, 2, 0, 0)), 3, 0, {}, dict(pan=(4, 2), still_rect=(512, 256, 1400, 800))),
]

HME_WARPS = 8  # warps of a me_b64_hme_kernel CTA


def reference(b200, refc, case):
    """(controls dict, reference outputs) of a case, built as test_me_b64 builds them"""
    name, W, H, preset, n_ref, dist, tl, is_ref, extra, content = case
    refc.ref_set_tier(0)
    r = rng(500 + len(name))
    shapes = b200.me_plane_shapes(W, H)
    cur_full, fulls = mh.case_pictures(r, W, H, n_ref, dist, content)
    cur_np = sp.build_pyramid_np(cur_full, W, H, shapes)
    refs_np = [sp.build_pyramid_np(f, W, H, shapes) for f in fulls]
    cfg = sp.me_b64_cfg(preset=preset, n_ref=n_ref, poc_dist=dist, temporal_layer_index=tl, is_ref=is_ref, **extra)
    ctrl, want = sp.ref_me_b64_picture(refc, cur_np, refs_np, shapes, cfg)
    return ctrl.as_dict(), want


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_me_b64_stages_match_reference_driver(b200, refc, case):
    base.test_me_b64_matches_reference_driver(b200, refc, case)
    # the case must exercise what it is there for
    name, W, H = case[0], case[1], case[2]
    cd, want = reference(b200, refc, case)
    live = want["do_ref"].reshape(want["do_ref"].shape[0], -1).sum(axis=1)  # references still searched after every pruning
    if name == "m4_nonbase_4p3_partial":
        # partial last block column and row; the column's 1/16- and 1/4-resolution blocks are neither 16, 32 nor 64 wide
        assert W % 64 and H % 64 and (W % 64) >> 2 not in (16, 32, 64) and (W % 64) >> 1 not in (16, 32, 64)
        # blocks with at least three references searched through HME: 12 or more (reference, region) jobs per level, for 8 warps
        assert (live * 4 > HME_WARPS).any()
    if name == "m6_ref_3p2":
        assert cd["prehme_enable"] and (live * 4 > HME_WARPS).any()
    if name == "m8_1080p_2p2":
        # band 0 of the distance-2 references: an 8 x 200 strip (cut into row slices), line skipping on, 56-row last block row
        f = (2 * 5) // 8 + 1
        assert cd["prehme_enable"] and cd["prehme_skip_search_line"] and H % 64 == 56
        assert min(cd["prehme_sa"][1] * f, cd["prehme_sa"][3]) == 200
