#!/usr/bin/env python3
"""Time windows handles over chosen fields (gpud_ring_windows_open_fields, DESIGN.md §2 "Field selection") against the all-field
handle of the same span and hop on the same ring.  Every field handle's answer is checked in the same run against the matching rows
of its all-field twin, all six outputs bit for bit.

  live      BASELINE configs[1]: 64 fields x 1 M samples (10 kHz x 100 s), W = 1000.  One live second = push 10 000 uint32 poll rows
            + reduce a span-600 / hop-10 handle (the p99 of the last minute, every second) + sync, over 1 field, alternated round by
            round with the same over all 64 fields.  Wall time per live second and the handle's device time (gpud_ring_windows_stats).
  catch_up  512 fields x 1 Mi samples (the survey stream of tests/synth_device.py), W = 1000: the first reduce of a handle over a full
            ring at span 10 and span 600, over 1, 8, 64 and 512 fields (every 512 / n-th field) and over all fields through the
            all-field handle, in alternating order.  Each repeat refills the ring with another seed (a loss and a restart for every
            handle).
Prints one JSON line with the card, its power limit and its top SM clock, read in the same run.  Writes nothing in the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

OPS = ("min", "max", "mean", "ema", "p99", "n_over")


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "n": len(xs)}


def check_rows(h, twin):
    """h's history equals twin's rows h.fields(), bit for bit in all six outputs, over the windows both hold"""
    first, nxt, _ = twin.counts()
    assert h.counts()[:2] == (first, nxt)
    rows = h.fields()
    for k in OPS:
        a, b = h.read(k, first, nxt - first), twin.read(k, first, nxt - first)[rows]
        assert np.array_equal(a.view(np.uint64) if k != "n_over" else a, b.view(np.uint64) if k != "n_over" else b), k


def live(g, ctx, torch, sd, rounds, secs):
    F, N, W = 64, 1000000, 1000
    stream = torch.cuda.Stream()
    rows = torch.randint(30, 90, (10000, F), dtype=torch.int32).pin_memory()
    r = g.Ring(ctx, F, N, W, thresholds=sd.thresholds("survey", F, N, 1))
    r.set_stream(stream.cuda_stream)
    hs = {"1_field": r.windows(600, 0, hop=10, fields=[17]), "64_fields": r.windows(600, 0, hop=10)}
    sd.fill_ring(r, "survey", F, N, 1, torch.device("cuda:0"), chunk=1 << 17)
    for h in hs.values():
        h.reduce()
    r.sync()
    walls = {k: [] for k in hs}
    dev = {k: [] for k in hs}
    for i in range(2 * rounds):
        kind = tuple(hs)[i % 2]
        other = tuple(hs)[1 - i % 2]
        for _ in range(secs):
            t0 = time.perf_counter()
            r.push_raw_ptr(rows.data_ptr(), 10000, g.DTYPES["uint32"])
            assert hs[kind].reduce()[0] == 1
            r.sync()
            walls[kind].append((time.perf_counter() - t0) * 1e3)
            dev[kind].append(hs[kind].stats()[0])
            hs[other].reduce()                          # the twin keeps up, untimed
            r.sync()
        check_rows(hs["1_field"], hs["64_fields"])
    for h in hs.values():
        h.close()
    r.close()
    return {"workload": "64 fields x 1 M samples, W = 1000; one live second = push 10 000 uint32 rows + a span-600 / hop-10 reduce "
                        "(a 600 000-sample p99 window every second) + sync, over 1 field or all 64, alternated by rounds",
            "live_second_ms": {k: spread(v) for k, v in walls.items()}, "device_ms": {k: spread(v) for k, v in dev.items()}}


def catch_up(g, ctx, torch, sd, repeat):
    F, CAP, W = 512, 1 << 20, 1000
    dev = torch.device("cuda:0")
    r = g.Ring(ctx, F, CAP, W, thresholds=sd.thresholds("survey", F, CAP, 1))
    hs = {}
    for span in (10, 600):
        hs["span%d_all" % span] = r.windows(span, 1)
        for n in (1, 8, 64, 512):
            hs["span%d_%d" % (span, n)] = r.windows(span, 1, fields=list(range(0, F, F // n)))
    sd.fill_ring(r, "survey", F, CAP, 1, dev)
    for h in hs.values():                                 # warm-up: every kernel and every scratch buffer once
        h.reduce()
    r.sync()
    ms = {k: [] for k in hs}
    L_max = 600 * W
    for i in range(repeat):
        pad = (-(r.counts()[0] + CAP)) % L_max            # the refill ends on a window boundary of both spans
        if pad:
            z = torch.zeros((pad, F), dtype=torch.float64, device=dev)
            r.push_device(z.data_ptr(), pad)
            r.sync()
            del z
        sd.fill_ring(r, "survey", F, CAP, 2 + i, dev)
        kinds = list(hs)
        if i % 2:
            kinds.reverse()
        for k in kinds:
            hs[k].reduce()
            r.sync()
            ms[k].append(hs[k].stats()[0])
        for k, h in hs.items():
            if not k.endswith("_all"):
                check_rows(h, hs[k.split("_")[0] + "_all"])
    for h in hs.values():
        h.close()
    r.close()
    return {"workload": "512 fields x 1 Mi samples (survey stream), W = 1000: first reduce of a handle over a full ring, tumbling "
                        "span 10 and span 600, over n fields (every 512 / n-th) or all fields, in alternating order",
            "device_ms": {k: spread(v) for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--secs", type=int, default=20)
    ap.add_argument("--repeat", type=int, default=6)
    a = ap.parse_args()
    import torch
    import gpud_b200 as g
    import synth_device as sd
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    ctx = g.Context([0])
    out = {"card": card, "live": live(g, ctx, torch, sd, a.rounds, a.secs), "catch_up": catch_up(g, ctx, torch, sd, a.repeat)}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
