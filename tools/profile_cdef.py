#!/usr/bin/env python3
"""Where the CDEF strength search's time goes: the phase split of its CTAs, and its SASS.

    python tools/profile_cdef.py --phases [--configs 1 2 4] [--steps 20] [--build-dir DIR]
    python tools/profile_cdef.py --sass

Phase mode: the library is built a second time, into DIR (default: a temporary directory), with B200_CDEF_PHASES=1, so
that thread 0 of every search CTA sums the clock64() cycles of each phase (cdef.cu, cdef_phase): table, block list,
staging, segment pass 0 (the block's direction), pass 1 (direction 0), shuffle combine and source moments, the wait
for the CTA's other segments, and the distortion warps.  Frames of each configuration run through the hot path; the
cycles per item (luma, chroma pair) and each phase's share are printed with the card's name and power limit.  A DIR
that already holds that build is reused.  Kernel times are `tools/profile_trio.py --kernels cdef_`.

SASS mode: the instruction histogram of `cdef_search_kernel` in the library as built, per pixel type."""
import argparse
import collections
import ctypes
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ("table", "list", "staging", "pass 0", "pass 1", "combine", "wait", "distortion")


def phase_build(dest):
    """a copy of the package, the header and the build script in dest, built with B200_CDEF_PHASES=1"""
    for d in ("svt-av1-psy_b200", "svt_av1_psy_b200", "include"):
        if not os.path.isdir(os.path.join(dest, d)):
            shutil.copytree(os.path.join(ROOT, d), os.path.join(dest, d),
                            ignore=shutil.ignore_patterns("build", "*.so", "__pycache__"))
    shutil.copy(os.path.join(ROOT, "__graft_entry__.py"), dest)
    sys.path.insert(0, dest)
    import __graft_entry__ as g
    assert os.path.dirname(os.path.abspath(g.__file__)) == os.path.abspath(dest)
    g.NVCC_FLAGS.append("-DB200_CDEF_PHASES=1")
    g.build_cuda()


def phases(configs, steps, dest):
    phase_build(dest)
    import torch
    import svt_av1_psy_b200 as pkg
    from svt_av1_psy_b200.pipeline import FramePipeline
    from svt_av1_psy_b200.workload import FrameWorkload
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from profile_trio import card

    if not torch.cuda.is_available():
        raise SystemExit("profile_cdef: no CUDA device")
    pkg.init(0)
    read = pkg.lib.svt_b200_cdef_phases_read
    read.argtypes = [ctypes.c_void_p]
    read.restype = ctypes.c_int
    buf = (ctypes.c_ulonglong * (2 * (len(PHASES) + 1)))()
    print("card: %s" % card())
    for cfg in configs:
        fp = FramePipeline(FrameWorkload.from_config(cfg), torch)
        ev = [torch.cuda.Event() for _ in range(len(FramePipeline.CALLS) + 1)]
        for _ in range(5):
            fp.step(ev)
        torch.cuda.synchronize()
        assert read(buf) == 0
        for _ in range(steps):
            fp.step(ev)  # the calls one after the other: the search runs alone on the GPU
        torch.cuda.synchronize()
        assert read(buf) == 0
        v = list(buf)
        print("config %d: %d steps, thread-0 cycles per item" % (cfg, steps))
        for it, name in ((0, "luma"), (1, "chroma pair")):
            row = v[it * (len(PHASES) + 1):(it + 1) * (len(PHASES) + 1)]
            n = max(row[-1], 1)
            tot = sum(row[:-1])
            print("  %-12s items=%-7d total=%8.0f  " % (name, row[-1] // steps, tot / n) +
                  "  ".join("%s %.0f (%.1f%%)" % (p, c / n, 100.0 * c / max(tot, 1)) for p, c in zip(PHASES, row[:-1])))
        sys.stdout.flush()


def sass():
    lib = os.path.join(ROOT, "svt-av1-psy_b200", "libsvtav1_b200.so")
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True, check=True).stdout
    func, hist = None, collections.OrderedDict()
    for ln in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            func = m.group(1) if "cdef_search_kernel" in m.group(1) else None
            if func:
                hist[func] = collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", ln)
        if func and m:
            hist[func][m.group(1)] += 1
    for f, h in hist.items():
        print("%s: %d instructions" % (f, sum(h.values())))
        for op, n in h.most_common(40):
            print("  %-28s %d" % (op, n))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--phases", action="store_true")
    ap.add_argument("--sass", action="store_true")
    ap.add_argument("--configs", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--build-dir", default=None, help="where the B200_CDEF_PHASES build goes (default: a temporary directory)")
    a = ap.parse_args()
    if a.sass:
        sass()
    if a.phases:
        if a.build_dir:
            os.makedirs(a.build_dir, exist_ok=True)
            phases(a.configs, a.steps, os.path.abspath(a.build_dir))
        else:
            with tempfile.TemporaryDirectory() as d:
                phases(a.configs, a.steps, d)


if __name__ == "__main__":
    main()
