#!/usr/bin/env python3
"""Spread of warp finish times in the hot window reduce, on the bench's ring (512 fields x 1 Mi f64, W = 1000, survey stream).

Needs a library built with -DGPUD_EXPERIMENT_FINISH (every warp of the hot launch records %globaltimer at entry and exit and
the number of windows it reduced):

  tools/build_variant.sh finish -DGPUD_EXPERIMENT_FINISH
  python tools/exp_warp_finish.py build/libgpud_finish.so [reps]

Prints one JSON line per launch: the launch's span (first warp start -> last warp end), the warp end times relative to the first
start (min / median / p99 / max), the time the GPU runs with some warps already gone (last end - median end, last end - first end),
the windows per warp, and the library's event time of the reduce.
"""
import ctypes as C
import json
import os
import sys

if len(sys.argv) < 2:
    sys.exit(__doc__)
os.environ["GPUD_B200_LIB"] = os.path.abspath(sys.argv[1])
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import gpud_b200 as g
import synth_device as sd

F, CAP, W = 512, 1 << 20, 1000
SEED = 0x67707564
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
MAXW = 4096

ctx = g.Context([0])
ring = g.Ring(ctx, F, CAP, W, thresholds=sd.thresholds("survey", F, CAP, SEED))
sd.fill_ring(ring, "survey", F, CAP, SEED, torch.device("cuda", 0))
L = ring._L
L.gpud_exp_warp_finish.restype = C.c_int32
L.gpud_exp_warp_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
buf = np.zeros((MAXW, 3), dtype=np.uint64)
for _ in range(3):
    ring.reduce()
ctx._check(L.gpud_exp_warp_finish(ring._h, C.c_void_p(buf.ctypes.data), MAXW))
for _ in range(reps):
    ring.reduce()
    ctx._check(L.gpud_exp_warp_finish(ring._h, C.c_void_p(buf.ctypes.data), MAXW))
    rec = buf[buf[:, 1] != 0].astype(np.int64)
    t0 = rec[:, 0].min()
    end_us = (rec[:, 1] - t0) / 1e3
    start_us = (rec[:, 0] - t0) / 1e3
    n = rec[:, 2]
    print(json.dumps({"warps": int(len(rec)), "span_us": float(end_us.max()),
                      "end_us": {"min": float(end_us.min()), "median": float(np.median(end_us)), "p99": float(np.percentile(end_us, 99)),
                                 "max": float(end_us.max())},
                      "tail_after_median_us": float(end_us.max() - np.median(end_us)), "tail_after_first_us": float(end_us.max() - end_us.min()),
                      "start_us_max": float(start_us.max()),
                      "windows_per_warp": {"min": int(n.min()), "max": int(n.max()), "sum": int(n.sum())},
                      "us_per_window_median": float(np.median(end_us / np.maximum(n, 1))),
                      "reduce_kernel_ms": float(ring.kernel_ms()[0])}))
ring.close()
ctx.close()
