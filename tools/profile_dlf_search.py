"""Time svt_b200_dlf_level_sse_dev, the trial SSEs of the deblocking filter-level search (one launch after a memset).

Cases: 1080p 8-bit, 1080p 10-bit, 2160p 10-bit, 4:2:0, on tests/test_deblock_search.py's generator (random valid
partition of 64x64 superblocks, smooth source, recon = source + a random offset per 4x4 block), no mode / ref deltas or
segment features, so each level's table is that level everywhere.  Two level sets: all three planes x 64 levels (every
trial any search could make), and luma x 5 levels (one hill-climb step and its neighbours).  Reports the median of CUDA-event
times of --calls calls after warm-up and the bytes the call must read at least (recon + source of the evaluated planes,
once), and prints the card, its power limit and max SM clock in the same run.  With oracle/_ref/libsvtav1_dlf_search.so present
it also times the reference's own svt_av1_pick_filter_level (ref_dlf_pick: the whole search, sequential tries of
whole-plane filter + SSE + restore) once per case on one host core.
Usage: python tools/profile_dlf_search.py [--calls N] [--no-host]"""
import ctypes as ct
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
DLF_LIB = os.path.join(ROOT, "oracle", "_ref", "libsvtav1_dlf_search.so")


def main():
    import torch
    import svt_av1_psy_b200 as pkg
    from test_deblock_search import ref_pick, search_case, search_sharpness
    calls = int(sys.argv[sys.argv.index("--calls") + 1]) if "--calls" in sys.argv else 200
    host = "--no-host" not in sys.argv and os.path.exists(DLF_LIB)
    if host:
        import oracle  # noqa: F401  (loads and initialises the reference objects the checker library links to)
        dlfc = ct.CDLL(DLF_LIB)
    pkg.init(0)
    d = pkg.dsp
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": smi.stdout.strip()}))
    st = torch.cuda.current_stream()
    for (w, h, bd) in ((1920, 1080, 8), (1920, 1080, 10), (3840, 2160, 10)):
        pb = 1 if bd == 8 else 2
        cfg, mi, rec, src, ctl = search_case((w, h), (bd, pb), 0, seed=w + bd)
        assert not cfg.mode_ref_delta_enabled and not cfg.segmentation_enabled
        f = d.DlfFrame()
        f.width, f.height, f.mi_rows, f.mi_cols, f.mi_stride, f.bit_depth, f.pixel_bytes = w, h, cfg.mi_rows, cfg.mi_cols, cfg.mi_stride, bd, pb
        s = search_sharpness(ctl)
        for l in range(64):  # the AV1 sharpness limits: lim, mblim = 2 * (lvl + 2) + lim, hev_thr = lvl >> 4
            lim = l >> ((s > 0) + (s > 4))
            lim = max(1, min(lim, 9 - s) if s > 0 else lim)
            f.lfthr[l][0], f.lfthr[l][1], f.lfthr[l][2] = 2 * (l + 2) + lim, lim, l >> 4
        dev = [torch.from_numpy(p.view(np.int16) if pb == 2 else p).to("cuda") for p in rec + src]
        ls = d.DlfLevelSse()
        for p in range(3):
            f.plane[p] = dev[p].data_ptr() + (16 * rec[p].shape[1] + 16) * pb
            f.stride[p] = rec[p].shape[1]
            ls.src[p] = dev[3 + p].data_ptr() + (16 * src[p].shape[1] + 16) * pb
            ls.src_stride[p] = src[p].shape[1]
        ls.sse_width, ls.sse_height = (w + 7) & ~7, (h + 7) & ~7
        d_mi = torch.from_numpy(mi.view(np.uint8).reshape(-1)).to("cuda")
        d_sse = torch.zeros(3 * 64, dtype=torch.int64, device="cuda")
        for name, mask, levels in (("3 planes x 64 levels", 7, list(range(64))), ("luma x 5 levels", 1, [24, 26, 28, 30, 32])):
            ls.plane_mask, ls.n_levels = mask, len(levels)
            lvl = np.zeros((3, len(levels), 256), np.uint8)
            for i, l in enumerate(levels):
                ls.level[i] = l
                lvl[:, i] = l
            d_lvl = torch.from_numpy(lvl.reshape(-1)).to("cuda")
            ls.d_lvl = d_lvl.data_ptr()
            for _ in range(20):
                assert d.dlf_level_sse_dev(f, ls, d_mi.data_ptr(), d_sse.data_ptr(), st.cuda_stream) == 0
            times = []
            for _ in range(calls):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                d.dlf_level_sse_dev(f, ls, d_mi.data_ptr(), d_sse.data_ptr(), st.cuda_stream)
                e1.record(st)
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            med = float(np.median(times))
            pixels = w * h * (1 if mask == 1 else 1.5)
            nbytes = int(2 * pixels * pb)
            print(json.dumps({"case": "%dx%d %d-bit" % (w, h, bd), "levels": name, "median_ms": round(med, 4), "calls": calls,
                              "us_per_plane_level": round(1000 * med / (len(levels) * (1 if mask == 1 else 3)), 2),
                              "min_bytes": nbytes, "gbs": round(nbytes / med / 1e6, 1)}))
        if host:
            t0 = time.perf_counter()
            picked, _, _ = ref_pick(dlfc, cfg, mi, rec, src, ctl)
            print(json.dumps({"case": "%dx%d %d-bit" % (w, h, bd), "host_ref_pick_ms": round(1000 * (time.perf_counter() - t0), 1),
                              "picked": list(picked), "host": "one core, reference C path (oracle/_ref)"}))
    pkg.shutdown()


if __name__ == "__main__":
    main()
