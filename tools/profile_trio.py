#!/usr/bin/env python3
"""Per-class timing of the transform kernel (txfm_kernel<Chain / Forward / Inverse, 4..64>) and the bench figures next to it.

    python tools/profile_trio.py [--configs 1 2] [--steps 20] [--out DIR] [--kernels me_b64 fullpel_search]
    python tools/profile_trio.py --bench-runs 3 --bench-trees . ../other_checkout [--bench-config 1]

Profile mode: frames of each configuration through the hot path with every call in order on one stream, under
torch.profiler (CUDA activities); one line per trio kernel -- name, grid, launches, mean us -- and the other calls'
kernels summed per call, with the card's name and power limit; then the separate calls (residual, forward, quantise,
inverse) on the same frame, one line per forward and inverse kernel.  With --kernels, one line per kernel whose name
contains one of the given strings, in place of the trio lines (e.g. `--kernels me_b64 fullpel_search` splits the
me_search call).  The traces go to DIR (default: a temporary directory).  Bench mode: `bench.py --gpus 1 --steps 3000 --warmup 50 --no-cpu-baseline` run alternately from each
tree, `value` and `calls_ms` printed per run.  The two modes are separate processes: the profiler slows the host."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown card (%s)" % e


def profile(configs, steps, out_dir, kernels=None):
    sys.path.insert(0, ROOT)
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    import svt_av1_psy_b200 as pkg
    from svt_av1_psy_b200.pipeline import FramePipeline
    from svt_av1_psy_b200.workload import FrameWorkload

    if not torch.cuda.is_available():
        raise SystemExit("profile_trio: no CUDA device")
    pkg.init(0)
    print("card: %s" % card())
    for cfg in configs:
        fp = FramePipeline(FrameWorkload.from_config(cfg), torch)
        ev = [torch.cuda.Event() for _ in range(len(FramePipeline.CALLS) + 1)]
        for _ in range(5):  # warm every shape (module loads, smem attributes)
            fp.step(ev)
        torch.cuda.synchronize()
        trace = os.path.join(out_dir, "trio_config%d.pt.trace.json" % cfg)
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                fp.step(ev)  # with events: the calls run one after the other on the current stream
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        kern = kernel_times(trace)
        print("config %d: %d profiled steps" % (cfg, steps))
        if kernels:
            for k in kernels:
                print_classes(kern, k)
            sys.stdout.flush()
            continue
        print_classes(kern, "txfm_kernel<Chain")
        per = {}
        for (s, g), (n, t) in kern.items():
            base = s.split("<")[0]
            p = per.setdefault(base, [0, 0.0])
            p[0] += n
            p[1] += t
        print("  all kernels, summed per name (us per step):")
        for base, (n, t) in sorted(per.items(), key=lambda x: -x[1][1]):
            print("    %-40s %8.2f" % (base, t / steps))
        # the separate calls on the frame the steps left behind, in order on one stream
        s = torch.cuda.current_stream().cuda_stream
        calls = (fp.call_residual, fp.call_fwd_txfm, fp.call_quant, fp.call_inv_txfm)
        for c in calls:
            c(s)
        torch.cuda.synchronize()
        trace = os.path.join(out_dir, "separate_config%d.pt.trace.json" % cfg)
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                for c in calls:
                    c(s)
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        kern = kernel_times(trace)
        print("config %d: separate calls, %d profiled rounds" % (cfg, steps))
        print_classes(kern, "txfm_kernel<Forward")
        print_classes(kern, "txfm_kernel<Inverse")
        sys.stdout.flush()


def kernel_times(trace):
    """(short name, grid) -> [launches, total us] of the kernels in a chrome trace"""
    kern = {}
    for e in json.load(open(trace))["traceEvents"]:
        if e.get("cat") != "kernel":
            continue
        name = e["name"]
        short = name.split("(")[0].replace("void ", "").replace("b200::", "") or name[:60]
        grid = tuple(e.get("args", {}).get("grid", ()))
        k = kern.setdefault((short, grid), [0, 0.0])
        k[0] += 1
        k[1] += float(e["dur"])
    return kern


def print_classes(kern, pattern):
    rows = sorted(((s, g, n, t) for (s, g), (n, t) in kern.items() if pattern in s), key=lambda x: -x[3] / x[2])
    for s, g, n, t in rows:
        print("  %-60s grid=%-14s launches=%-5d mean=%8.2f us" % (s, "x".join(map(str, g)), n, t / n))


def bench(trees, runs, config, steps, warmup):
    print("card: %s" % card())
    res = {t: [] for t in trees}
    for i in range(runs):
        for t in trees:
            cmd = [sys.executable, os.path.join(t, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
                   "--no-cpu-baseline", "--config", str(config)]
            r = subprocess.run(cmd, capture_output=True, text=True, cwd=t)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            if r.returncode != 0 or not line:
                print("run %d %s: FAILED rc=%d\n%s" % (i, t, r.returncode, r.stderr[-3000:]))
                continue
            j = json.loads(line[-1])
            res[t].append(j["value"])
            calls = {k: v for k, v in j.get("calls_ms", {}).items()}
            print("config %d run %d %-20s value=%.1f calls_ms=%s" % (config, i, t, j["value"], json.dumps(calls)))
            sys.stdout.flush()
    for t in trees:
        v = sorted(res[t])
        print("config %d %-20s values=%s median=%s" % (config, t, v, v[len(v) // 2] if v else None))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for the profiler traces (default: a temporary directory)")
    ap.add_argument("--kernels", nargs="+", default=None,
                    help="profile mode: print only the kernels whose names contain one of these strings (default: the trio)")
    ap.add_argument("--bench-runs", type=int, default=0)
    ap.add_argument("--bench-trees", nargs="+", default=[ROOT])
    ap.add_argument("--bench-config", type=int, default=1)
    ap.add_argument("--bench-steps", type=int, default=3000)
    ap.add_argument("--bench-warmup", type=int, default=50)
    a = ap.parse_args()
    if a.bench_runs:
        bench([os.path.abspath(t) for t in a.bench_trees], a.bench_runs, a.bench_config, a.bench_steps, a.bench_warmup)
        return
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        profile(a.configs, a.steps, a.out, a.kernels)
    else:
        with tempfile.TemporaryDirectory() as d:
            profile(a.configs, a.steps, d, a.kernels)


if __name__ == "__main__":
    main()
