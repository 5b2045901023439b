#!/usr/bin/env python3
"""The open-loop ME call alone (pyramid + complete driver) for `compute-sanitizer --tool memcheck|racecheck python
tools/sanitize_me.py`: preset 8 (4 references) and preset 4 (7 references: every pre-HME and HME stage of
me_b64_hme_kernel has more warp jobs than the CTA has warps).  Drives only the product library."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import svt_av1_psy_b200 as pkg  # noqa: E402
from svt_av1_psy_b200.pipeline import FramePipeline  # noqa: E402
from svt_av1_psy_b200.workload import FrameWorkload  # noqa: E402

pkg.init(0)
for preset in (8, 4):
    fp = FramePipeline(FrameWorkload(384, 256, preset=preset), torch)
    fp.load_inputs()
    s = torch.cuda.current_stream().cuda_stream
    fp.call_me_pyramid(s)
    fp.call_me_search(s)
    torch.cuda.synchronize()
    print("done preset", preset, "refs", fp.wl.n_refs, int(fp.me["distortion"].to(torch.int64).sum()), int(fp.me["total_me_candidate_index"].sum()))
