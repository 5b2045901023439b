"""Time svt_b200_picture_statistics_dev (the picture-analysis statistics of one picture) on the GPU next to the reference's
svt_aom_gathering_picture_statistics on one host core (C path, oracle/_ref/libsvtav1_pa_stats.so), at 1080p and 2160p, with
the encoder's default controls (BLOCK_MEAN_PREC_SUB, 8x8 variances on, 4 x 4 regions, decim_step 4) and scene-change
sampling (decim_step 1).

    python tools/profile_pa_stats.py [--calls 300] [--warmup 50]

Device: the median of per-call CUDA-event times after warm-up.  The calls of a batch are queued behind a sleeping kernel, so that
the GPU runs them back to back and the events time the device, not the host's enqueue rate.  Also timed: the call with both parts off, which runs only
the one-CTA reduction kernel (the second launch of every call).  Host: the median of --host-calls runs of the reference
function (with the oracle's pcs set-up around it).  Bytes: what the call must read -- W*H/2 of the full plane (every other
row) + (W/4 * H/4) / decim^2 of the 1/16 plane.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
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


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--host-calls", type=int, default=5)
    args = ap.parse_args()
    import torch
    import svt_av1_psy_b200 as pkg
    import test_pa_stats as tp
    from oracle import support as sp
    dsp = pkg.dsp
    pkg.init(0)
    import oracle
    pa = oracle.load("pa_stats")
    if pa is not None:
        pa.ref_pa_stats.argtypes = [ct.c_void_p] * 4
        pa.ref_pa_stats.restype = ct.c_int
    print("gpu:", gpu_info())
    for W, H in ((1920, 1080), (3840, 2160)):
        planes, shapes = tp.picture(W, H, "random", 7)
        dplanes = [torch.from_numpy(p).cuda() for p in planes]
        pic = tp._desc(dsp, dplanes, shapes)
        for label, kw in (("default d=4", dict()), ("scd d=1", dict(scd=1)), ("reduction only", dict(var=0, hist=0))):
            c = tp.cfg(**kw)
            ctl = dsp.PaStatsControls(c.calculate_variance, c.block_mean_calc_prec, 1, c.calc_hist, 1 if c.scene_change_detection else 4, 4, 4, 0)
            rc, out = dsp.picture_statistics_dev(pic, ctl, torch)
            assert rc == 0
            res = dsp.PaStatsResults(*[out[n].data_ptr() for n, _ in dsp.PaStatsResults._fields_])
            call = lambda: dsp.lib.svt_b200_picture_statistics_dev(ct.byref(pic), ct.byref(ctl), ct.byref(res), None)  # noqa: E731
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.calls)]
            for i0 in range(0, args.calls, 100):
                torch.cuda._sleep(50_000_000)  # ~25 ms at 1980 MHz: longer than queueing 100 calls takes
                for a, b in ev[i0:i0 + 100]:
                    a.record()
                    call()
                    b.record()
                torch.cuda.synchronize()
            dev_us = float(np.median([a.elapsed_time(b) for a, b in ev]) * 1e3)
            host_us = None
            if pa is not None and label != "reduction only":
                ts = []
                for _ in range(args.host_calls):
                    o = tp.sentinel_outputs(((W + 63) // 64) * ((H + 63) // 64), 4, 4)
                    d = sp.ref_pic_desc(planes, shapes)
                    t0 = time.perf_counter()
                    pa.ref_pa_stats(ct.byref(d), ct.byref(c), None, ct.byref(tp._out_struct(o)))
                    ts.append(time.perf_counter() - t0)
                host_us = float(np.median(ts) * 1e6)
            dec = 1 if c.scene_change_detection else 4
            nbytes = (W * H // 2 if c.calculate_variance else 0) + ((W // 4) * (H // 4) // (dec * dec) if c.calc_hist else 0)
            row = dict(size="%dx%d" % (W, H), controls=label, device_us=round(dev_us, 2), host_ref_us=None if host_us is None else round(host_us, 1),
                       bytes=nbytes, gbps=round(nbytes / dev_us / 1e3, 1) if nbytes else None)
            print(json.dumps(row))


if __name__ == "__main__":
    main()
