#!/usr/bin/env python3
"""debug helper: encode with only some kernel groups of the H100 tier installed (SVT_B200_RTCD_GROUPS) and compare with the C path"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import test_rtcd_binding as t
cfg = dict(w=640, h=360, n=int(sys.argv[2]) if len(sys.argv) > 2 else 4, bd=int(sys.argv[1]), preset=int(sys.argv[3]) if len(sys.argv) > 3 else 8, crf=30, lp=8)
c = t._encode(False, **cfg)
print("C", c)
for g in (1, 2, 4, 8, 16, 32, 64, 128):
    os.environ["SVT_B200_RTCD_GROUPS"] = str(g)
    r = t._encode(True, **cfg)
    print("group", g, "SAME" if r["sha256"] == c["sha256"] else "DIFF", r["bytes"], r["launches"], r["seconds"])
