#!/usr/bin/env python3
"""Time gpud_box_query_create_fields (the box query over chosen fields) against the all-field query, with simulated ranks as in
bench_ring_box_dist.py: every ring on one device, each driven by its own query, stepped in lockstep, the all-gather device-to-device
copies into one receive buffer.  The transport's own time (NCCL over NVLink, gloo) is therefore NOT measured: what is reported is the
largest rank's device time inside the query (gpud_box_query_stats; median / min / max over the runs), the rounds and the bytes each rank
sends, each field query alternated with the all-field query.
  box     8 rings of 64 fields x 1 M samples, W = 1000: the box p99 of the last minute, one set of 8 ranges, one per ring; 1 / 8 / 64 fields.
  survey  the 512 fields x 1 Mi survey stream (tests/synth_device.py) split over 8 rings of CAP / 8: 100 sets of 100 random ranges of
          1 - 10 000 samples from random rings; 1 / 8 / 64 / 512 fields.
Every field answer is checked bit for bit, in all six outputs, against the all-field query's rows in the same run, and every rank's
against rank 0's.  Prints one JSON line with the card and its power limit, read in the same run.  Writes nothing in the tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_ring_ranges import spread       # noqa: E402

OPS = ("min", "max", "mean", "ema", "p99", "n_over")


def lockstep(g, torch, rings, args, fields):
    """one query per ring, stepped together: (rank 0's result, per-rank stats)"""
    from gpud_b200.dist import _DevBytes
    qs = [g.BoxQuery(r, k, len(rings), *args, fields=fields) for k, r in enumerate(rings)]
    outs, buf = [q.step() for q in qs], None
    while outs[0][1]:
        nb = outs[0][1]
        assert all(o[1] == nb for o in outs)
        buf = torch.empty(len(qs) * nb, dtype=torch.uint8, device="cuda:0")
        for k, (ptr, _) in enumerate(outs):
            buf[k * nb:(k + 1) * nb].copy_(torch.as_tensor(_DevBytes(ptr, nb), device="cuda:0"))
        torch.cuda.synchronize()
        outs = [q.step(buf.data_ptr()) for q in qs]
    res = [q.result() for q in qs]
    for r in res[1:]:
        for k in r:
            assert np.array_equal(r[k].view(np.uint8), res[0][k].view(np.uint8)), k
    stats = [q.stats() for q in qs]
    for q in qs:
        q.close()
    return res[0], stats


def measure(g, torch, rings, args, lists, repeat):
    """per field count: the field query and the all-field query alternated, every field answer against the all-field rows"""
    out = {}
    for name, fields in lists.items():
        ms, info = {"fields": [], "all_fields": []}, {}
        for i in range(repeat):
            got = {}
            for kind in (("fields", "all_fields") if i % 2 == 0 else ("all_fields", "fields")):
                res, st = lockstep(g, torch, rings, args, fields if kind == "fields" else None)
                got[kind] = res
                ms[kind].append(max(s["device_ms"] for s in st))
                info[kind] = {"rounds": st[0]["rounds"], "bytes_sent_per_rank": max(s["bytes_sent"] for s in st)}
            for op in OPS:
                assert np.array_equal(got["fields"][op].view(np.uint8), got["all_fields"][op][fields].view(np.uint8)), (name, op)
        out[name] = {"device_ms": {k: spread(v) for k, v in ms.items()}, **{k + "_exchange": v for k, v in info.items()}}
    return out


def box(g, ctx, torch, sd, repeat):
    R, F, N, W, MIN = 8, 64, 1000000, 1000, 60000
    thr = sd.thresholds("survey", F, N, 1)
    rings = []
    for k in range(R):
        r = g.Ring(ctx, F, N, W, thresholds=thr)
        sd.fill_ring(r, "survey", F, N, 1 + k, torch.device("cuda:0"), chunk=1 << 17)
        rings.append(r)
    totals = [r.counts()[0] for r in rings]
    args = (np.arange(R, dtype=np.int32), np.array([t - MIN for t in totals], dtype=np.int64), np.full(R, MIN, dtype=np.int64),
            np.array([0, R], dtype=np.int64))
    lists = {"1": [F // 2], "8": list(range(3, F, 8)), "64": list(range(F))}
    out = measure(g, torch, rings, args, lists, repeat)
    for r in rings:
        r.close()
    return {"workload": "8 rings of 64 fields x 1 M samples, W = 1000: the box p99 of the last minute, one set of 8 ranges of 60 000", **out}


def survey(g, ctx, torch, sd, repeat, rng):
    n, F, CAP, W = 8, 512, 1 << 20, 1000
    C = CAP // n
    thr = sd.thresholds("survey", F, CAP, 1)
    rings = [g.Ring(ctx, F, C, W, thresholds=thr) for _ in range(n)]
    t0 = 0
    for x, m in sd.chunks("survey", F, CAP, C, 1, torch.device("cuda:0")):
        x = x.contiguous()
        torch.cuda.current_stream().synchronize()
        rings[t0 // C].push_device(x.data_ptr(), m)
        rings[t0 // C].sync()
        t0 += m
    per, n_sets = 100, 100
    length = rng.integers(1, 10001, n_sets * per).astype(np.int64)
    ro = rng.integers(0, n, n_sets * per).astype(np.int32)
    first = (rng.random(n_sets * per) * (C - length + 1)).astype(np.int64)
    set_off = np.arange(0, n_sets * per + 1, per, dtype=np.int64)
    lists = {"1": [300], "8": list(range(7, F, 64)), "64": list(range(5, F, 8)), "512": list(range(F))}
    out = measure(g, torch, rings, (ro, first, length, set_off), lists, repeat)
    for r in rings:
        r.close()
    return {"workload": "512 fields x 1 Mi survey stream split over 8 rings of CAP / 8, W = 1000: 100 sets of 100 random ranges of 1 - 10 000 "
                        "samples from random rings", **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=6)
    a = ap.parse_args()
    import torch
    import gpud_b200 as g
    import synth_device as sd
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    ctx = g.Context([0])
    out = {"card": card, "transport": "not measured (simulated ranks on one device)", "box": box(g, ctx, torch, sd, a.repeat),
           "survey": survey(g, ctx, torch, sd, a.repeat, np.random.default_rng(2026))}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
