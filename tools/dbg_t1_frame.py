#!/usr/bin/env python3
"""debug helper: one reference frame step with the H100 T1 pointers installed (REF_TRACE=1 prints the stage)"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle
from oracle.frame_ref import RefFrame, load_workload_module
enc = oracle.load("enc")
assert enc is not None, "libsvtav1_enc.so: " + oracle.BUILD_HINT
enc.ref_set_tier(0)
assert enc.svt_b200_install_rtcd(0) == 0
enc.ref_set_threads(int(sys.argv[3]) if len(sys.argv) > 3 else 1)
wl = load_workload_module().FrameWorkload(384, 256, bit_depth=int(sys.argv[1]), preset=int(sys.argv[2]))
fr = RefFrame(wl, enc)
fr.step()
print("step ok")
