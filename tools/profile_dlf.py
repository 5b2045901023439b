"""Time svt_b200_loop_filter_frame_dev (two launches: all vertical edges, then all horizontal edges of the three planes).

Cases: 1080p 8-bit, 1080p 10-bit, 2160p 10-bit, 4:2:0, on a random valid partition of 64x64 superblocks (tests/test_deblock.py's
generator) with luma levels 32 / 28, chroma 20 / 16, sharpness 0.  Reports the median of >= 1000 calls timed with CUDA
events after warm-up, the algorithmic bytes (2 passes x read + write of 1.5 * W * H pixels) and their fraction of the
H100 SXM's 3.35 TB/s.  The filter is integer arithmetic with data-dependent branches per 4-pixel segment: expect it to be
bound by instructions and latency, not by HBM bandwidth.  Prints one JSON line per case plus the card, its power limit
and max SM clock.  Usage: python tools/profile_dlf.py [--calls N]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import torch
    import svt_av1_psy_b200 as pkg
    from test_deblock import make_mode_info
    from helpers import rng
    calls = int(sys.argv[sys.argv.index("--calls") + 1]) if "--calls" in sys.argv else 1000
    pkg.init(0)
    d = pkg.dsp
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": smi.stdout.strip()}))
    for (w, h, bd) in ((1920, 1080, 8), (1920, 1080, 10), (3840, 2160, 10)):
        r = rng(w + bd)
        mi, mr, mc, ms = make_mode_info(r, w, h, 64)
        pb = 1 if bd == 8 else 2
        f = d.DlfFrame()
        f.width, f.height, f.mi_rows, f.mi_cols, f.mi_stride, f.bit_depth, f.pixel_bytes = w, h, mr, mc, ms, bd, pb
        f.filter_level[0], f.filter_level[1], f.filter_level_u, f.filter_level_v = 32, 28, 20, 16
        lvl = np.zeros((3, 8, 2, 8, 2), np.uint8)
        lvl[0, :, 0], lvl[0, :, 1], lvl[1], lvl[2] = 32, 28, 20, 16
        ct_lvl = (type(f.lvl)).from_buffer_copy(lvl.tobytes())
        f.lvl = ct_lvl
        for l in range(64):  # sharpness 0: lim = max(1, l), mblim = 2 * (l + 2) + lim, hev_thr = l >> 4
            lim = max(1, l)
            f.lfthr[l][0], f.lfthr[l][1], f.lfthr[l][2] = 2 * (l + 2) + lim, lim, l >> 4
        dt = torch.uint8 if pb == 1 else torch.int16
        planes = []
        for p in range(3):
            pw, ph = (w, h) if p == 0 else (w // 2, h // 2)
            t = torch.randint(0, 1 << (bd - 1), (ph + 32, pw + 32), dtype=torch.int32, device="cuda").to(dt)
            planes.append(t)
            f.plane[p] = t.data_ptr() + (16 * t.shape[1] + 16) * pb
            f.stride[p] = t.shape[1]
        d_mi = torch.from_numpy(mi.view(np.uint8).reshape(-1)).to("cuda")
        st = torch.cuda.current_stream()
        for _ in range(50):
            assert d.loop_filter_frame_dev(f, d_mi.data_ptr(), st.cuda_stream) == 0
        times = []
        for _ in range(calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            d.loop_filter_frame_dev(f, d_mi.data_ptr(), st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        med = float(np.median(times))
        nbytes = 2 * 2 * int(1.5 * w * h) * pb
        print(json.dumps({"case": "%dx%d %d-bit" % (w, h, bd), "median_ms": round(med, 4), "calls": calls, "algorithmic_bytes": nbytes,
                          "gbs": round(nbytes / med / 1e6, 1), "frac_of_3350_gbs": round(nbytes / med / 1e6 / 3350.0, 4)}))
    pkg.shutdown()


if __name__ == "__main__":
    main()
