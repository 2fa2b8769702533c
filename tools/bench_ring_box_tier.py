#!/usr/bin/env python3
"""Measure box range sets that reach into the rings' tiers (DESIGN.md §2 "Box sets", "Tier") on BASELINE configs[1]: 8 rings of 64
fields, CAP = 1 000 000, W = 1000, each with a 512 MB tier, on one GPU, fed NVML-like uint32 gauges (tools/bench_ring_checkpoint.py's)
at 10 000 rows per live second until every tier is full.  Ring k's rows come from a pool of P chunks of 50 s held on the device (chunk
c of ring k is pool[(c + k) % P]), pushed with gpud_ring_push_device, so that filling eight tiers takes seconds and the oracle can
rebuild any range on the host.

Queries, each one set of 8 ranges (one per ring, the same seconds): the box p99 of 30 s ending 5 minutes back, of the last 10 minutes
(INTEGRATION.md's example), and of the last 30 minutes.  For each: device ms of the home ring's gpud_ring_ranges_stats (the whole call)
and its decode (gpud_ring_tier_stats), median and spread over --runs, alternated in the same run with the 8 one-ring calls
(gpud_ring_reduce_ranges) over the same ranges, whose device and decode ms are summed.  Every box answer is checked in the same run
against the C oracle on the concatenated samples (min / max / p99 / n_over bit for bit, mean and EMA within oracle/SPEC.md's tolerance)
on the fields named in the output.  Prints one JSON line with the card and its power limit, read in the same run.  Writes nothing in
the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

RATE = 10_000
CHUNK = 50 * RATE


def spread(xs):
    q = np.percentile(xs, [10, 50, 90])
    return {"median": statistics.median(xs), "p10": float(q[0]), "p90": float(q[2]), "min": min(xs), "max": max(xs), "n": len(xs)}


def samples(pool, k, first, n, fields):
    """ring k's samples [first, first + n) of `fields`, [len(fields)][n] f64, rebuilt from the pool"""
    out = np.empty((len(fields), n), dtype=np.float64)
    a = first
    while a < first + n:
        c, o = divmod(a, CHUNK)
        m = min(CHUNK - o, first + n - a)
        out[:, a - first:a - first + m] = pool[(c + k) % len(pool)][o:o + m, fields].T
        a += m
    return out


def check(got, pool, firsts, n, thr, alpha, fields):
    from oracle import coracle
    x = np.concatenate([samples(pool, k, f, n, fields) for k, f in enumerate(firsts)], axis=1)
    want = coracle.windows_fields(np.ascontiguousarray(x), x.shape[1], thr[fields], alpha)
    for key in ("min", "max", "p99"):
        assert np.array_equal(got[key][fields, 0].view(np.uint64), want[key][:, 0].view(np.uint64)), key
    assert np.array_equal(got["n_over"][fields, 0], want["n_over"][:, 0].astype(np.uint32)), "n_over"
    for key in ("mean", "ema"):
        a, b = got[key][fields, 0], want[key][:, 0]
        assert np.all(np.abs(a - b) <= 1e-6 * np.maximum(np.abs(b), np.abs(x).max(axis=1))), key


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", type=int, default=8)
    ap.add_argument("--tier-mb", type=int, default=512)
    ap.add_argument("--max-seconds", type=int, default=2600, help="live seconds pushed at most while the tiers fill")
    ap.add_argument("--pool", type=int, default=4, help="distinct 50 s chunks the rings' rows come from")
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    import torch
    import gpud_b200 as g
    from bench_ring_checkpoint import nvml_rows
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    ctx = g.Context([0])
    F, cap, W, alpha = 64, 1_000_000, 1000, 0.01
    thr = np.array([(46.0, 350000.0, 1980.0, 50.0)[f % 4] for f in range(F)])
    pool = [nvml_rows(F, CHUNK, 2000 + i) for i in range(a.pool)]
    dpool = [torch.from_numpy(p.astype(np.float64)).cuda() for p in pool]
    torch.cuda.synchronize()
    rings = [g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha) for _ in range(a.rings)]
    for r in rings:
        r.tier_open(a.tier_mb << 20)
    total = 0
    while total < a.max_seconds * RATE:
        c = total // CHUNK
        for k, r in enumerate(rings):
            t = dpool[(c + k) % a.pool]
            r.push_device(t.data_ptr(), CHUNK)
        total += CHUNK
        if total >= 1900 * RATE and all(r.tier_counts()[0] > 0 for r in rings):   # every tier full: it has begun to evict
            break
    for r in rings:
        r.sync()
    counts = [r.tier_counts() for r in rings]
    reach = [min(total - cap, c[0]) for c in counts]
    out = {"card": card, "rings": a.rings, "F": F, "cap": cap, "rate": RATE, "tier_bytes": a.tier_mb << 20, "seconds_pushed": total / RATE,
           "tier_history_s": [(c[1] - c[0]) / RATE for c in counts], "reach_s": [(total - lo) / RATE for lo in reach],
           "rows_lost": [c[3] for c in counts], "tiers_full": all(c[0] > 0 for c in counts)}
    queries = [("box_30s_ending_5min_back", total - 330 * RATE, 30 * RATE, np.arange(16)),
               ("box_last_10min", total - 600 * RATE, 600 * RATE, np.arange(4)),
               ("box_last_30min", total - 1800 * RATE, 1800 * RATE, np.arange(1))]
    home = rings[0]
    for name, first, n, fields in queries:
        if first < max(reach):
            out[name] = "beyond the tiers' reach"
            continue
        firsts = [first] * a.rings
        ring_of = np.arange(a.rings, dtype=np.int32)
        set_off = np.array([0, a.rings], dtype=np.int64)
        box_ms, box_dec, one_ms, one_dec = [], [], [], []
        got = None
        for run in range(a.runs + 1):                   # run 0 warms both up and is not kept
            order = ("box", "one") if run % 2 else ("one", "box")
            for what in order:
                if what == "box":
                    got = g.rings_reduce_range_sets(rings, ring_of, firsts, [n] * a.rings, set_off)
                    ms, dec = home.ranges_stats()[0], home.tier_stats()[1]
                    if run:
                        box_ms.append(ms)
                        box_dec.append(dec)
                else:
                    ms = dec = 0.0
                    for r in rings:
                        r.reduce_ranges([first], [n])
                        ms += r.ranges_stats()[0]
                        dec += r.tier_stats()[1]
                    if run:
                        one_ms.append(ms)
                        one_dec.append(dec)
        check(got, pool, firsts, n, thr, alpha, fields)
        out[name] = {"seconds": n / RATE, "samples_per_field": n * a.rings,
                     "box_device_ms": spread(box_ms), "box_decode_ms": spread(box_dec),
                     "one_ring_calls_summed_device_ms": spread(one_ms), "one_ring_calls_summed_decode_ms": spread(one_dec),
                     "box_over_one_ring_sum": statistics.median(box_ms) / statistics.median(one_ms),
                     "checked": "oracle, fields %d..%d" % (fields[0], fields[-1])}
    for r in rings:
        r.close()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
