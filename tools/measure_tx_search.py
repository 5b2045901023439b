#!/usr/bin/env python3
"""Dev-time measurement (needs oracle/_ref/libsvtav1_enc.so, i.e. /root/reference): encode the synthetic sequence of
workload.synth_sequence with the UNMODIFIED reference encoder (C path) and read the transform call counters of
oracle/enc_counters.c.  Prints SURVEY.md 8(d)'s mode-decision search factor

    k = sum of N over svt_aom_estimate_transform calls / (1.5 * W * H * frames)

plus the same ratio for the inverse transform, and the call mix per transform size.  The numbers go into DESIGN.md and
FrameWorkload.TX_SEARCH_K.  Usage: measure_tx_search.py [W H frames preset crf]"""
import ctypes as ct
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from oracle.frame_ref import load_workload_module  # noqa: E402

W, H, N, PRESET, CRF = ([int(a) for a in sys.argv[1:6]] + [1920, 1080, 17, 8, 30][len(sys.argv) - 1:])[:5]
lib = oracle.load("enc")
assert lib is not None, "libsvtav1_enc.so: " + oracle.BUILD_HINT
lib.ref_encode.restype = ct.c_int64
lib.ref_encode.argtypes = [ct.c_void_p] + [ct.c_int] * 8 + [ct.c_void_p, ct.c_int64, ct.c_void_p]
lib.ref_counters_read.restype = ct.c_int
lib.ref_counters_read.argtypes = [ct.POINTER(ct.c_uint64), ct.c_int]

wlm = load_workload_module()
frames = wlm.synth_sequence(W, H, N)
yuv = np.concatenate([p.reshape(-1) for f in frames for p in f])
out = np.zeros(64 << 20, np.uint8)
npk = ct.c_int32()
lib.ref_counters_reset()
size = lib.ref_encode(yuv.ctypes.data, W, H, N, 8, PRESET, CRF, os.cpu_count(), -1, out.ctypes.data, out.size, ct.byref(npk))
assert size > 0, size
c = (ct.c_uint64 * 64)()
n = lib.ref_counters_read(c, 64)
samples = 1.5 * W * H * N
names = ["4X4", "8X8", "16X16", "32X32", "64X64", "4X8", "8X4", "8X16", "16X8", "16X32", "32X16", "32X64", "64X32", "4X16", "16X4", "8X32", "32X8",
         "16X64", "64X16"]
print(json.dumps({"width": W, "height": H, "frames": N, "preset": PRESET, "crf": CRF, "bitstream_bytes": int(size),
                  "fwd_calls_per_frame": c[0] / N, "k_fwd": c[1] / samples, "k_fwd_shaped_outputs": c[2] / samples,
                  "inv_calls_per_frame": c[3] / N, "k_inv": c[4] / samples, "inv_eob0_calls_per_frame": c[5] / N,
                  "fwd_calls_by_size_per_frame": {names[i]: round(c[6 + i] / N, 1) for i in range(19) if c[6 + i]}}, indent=1))
