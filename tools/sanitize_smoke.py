#!/usr/bin/env python3
"""One small frame (384x256, 8-bit then 10-bit) through the T2 pipeline, for `compute-sanitizer --tool memcheck|racecheck python
tools/sanitize_smoke.py` on a GPU box (no oracle involved: this only drives the product library)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import svt_av1_psy_b200 as pkg  # noqa: E402
from svt_av1_psy_b200.pipeline import FramePipeline  # noqa: E402
from svt_av1_psy_b200.workload import FrameWorkload  # noqa: E402

pkg.init(0)
for bd in (8, 10):  # 8-bit: IMMA statistics, u8 TMA maps; 10-bit: lag-sum statistics, u16 planes
    fp = FramePipeline(FrameWorkload(384, 256, bit_depth=bd), torch)
    fp.load_inputs()
    fp.step()
    fp.read_outputs()
    fp.read_levels()
    torch.cuda.synchronize()
    print("done", bd, int(fp.final.sum()), int(fp.qcoeff.abs().sum()))
