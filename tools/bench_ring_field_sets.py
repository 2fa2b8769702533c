#!/usr/bin/env python3
"""Time range sets over chosen fields (gpud_rings_reduce_range_sets_fields, DESIGN.md §2 "Field selection") against the all-field call
(gpud_rings_reduce_range_sets) over the same rings, ranges and sets, alternated run by run.  Every field answer is checked in the same
run against the matching columns of the all-field answer, all six outputs bit for bit.

  survey  512 fields x 1 Mi samples (the survey stream of tests/synth_device.py), W = 1000: 100 sets of 100 random ranges of 1 - 10 000
          samples (tools/bench_ring_range_sets.py's shape), over 1 field, 8 contiguous, 8 spread (every 64th), 64 contiguous and all
          512 in order.
  tier    BASELINE configs[1] live: rings of 64 fields, CAP = 1 000 000, W = 1000, a 512 MB tier each, fed NVML-like uint32 gauges at
          10 000 rows per second until every tier is full (tools/bench_ring_box_tier.py's feed): a 30-minute range and 30 s ending 5
          minutes back on ring 0, and the same seconds as one box set over every ring, for 1 field against all 64.
  live    one live second on ring 0 of the tier shape: push 10 000 uint32 rows, then the last minute's p99 of one field, alternated
          second by second with the same push + the all-field call.
Device ms come from gpud_ring_ranges_stats (the whole call) and, tiered, gpud_ring_tier_stats (its decode), as median and spread over
the runs.  Prints one JSON line with the card, its power limit and its top SM clock, read in the same run.  Writes nothing in the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_ring_box_tier import CHUNK, RATE, spread   # noqa: E402

OPS = ("min", "max", "mean", "ema", "p99", "n_over")


def same_cols(got, full, fields):
    for k in OPS:
        a, b = got[k], full[k][np.asarray(fields)]
        assert np.array_equal(a.view(np.uint64) if k != "n_over" else a, b.view(np.uint64) if k != "n_over" else b), k


def g_error():
    import gpud_b200 as g
    return g.GpudError


def alternate(call_fields, call_all, fields, runs, home):
    """runs of (field call, all-field call) in alternating order after one warm-up pair: device ms and decode ms of each"""
    ms = {"fields": [], "all": []}
    dec = {"fields": [], "all": []}
    for run in range(runs + 1):
        order = ("fields", "all") if run % 2 else ("all", "fields")
        got = {}
        for what in order:
            got[what] = call_fields() if what == "fields" else call_all()
            if run:
                ms[what].append(home.ranges_stats()[0])
                try:
                    dec[what].append(home.tier_stats()[1])
                except g_error():                    # an untiered ring decodes nothing
                    dec[what].append(0.0)
        same_cols(got["fields"], got["all"], fields)
    return ms, dec


def survey(g, ctx, torch, sd, runs, rng):
    F, CAP, W = 512, 1 << 20, 1000
    thr = sd.thresholds("survey", F, CAP, 1)
    r = g.Ring(ctx, F, CAP, W, thresholds=thr)
    sd.fill_ring(r, "survey", F, CAP, 1, torch.device("cuda:0"))
    length = rng.integers(1, 10001, 100 * 100).astype(np.int64)
    first = (rng.random(100 * 100) * (CAP - length + 1)).astype(np.int64)
    set_off = np.arange(0, 100 * 100 + 1, 100, dtype=np.int64)
    lists = {"1": [100], "8_contiguous": list(range(64, 72)), "8_spread": list(range(0, F, 64)), "64_contiguous": list(range(128, 192)),
             "512_in_order": list(range(F))}
    out = {"workload": "512 fields x 1 Mi samples (survey stream), W = 1000: 100 sets of 100 random ranges of 1 - 10 000 samples",
           "samples_per_field": int(length.sum())}
    for name, fields in lists.items():
        ms, _ = alternate(lambda: r.reduce_range_sets(first, length, set_off, fields=fields), lambda: r.reduce_range_sets(first, length, set_off),
                          fields, runs, r)
        out[name] = {"n_fields": len(fields), "fields_device_ms": spread(ms["fields"]), "all_device_ms": spread(ms["all"]),
                     "ratio_of_medians": spread(ms["fields"])["median"] / spread(ms["all"])["median"]}
    r.close()
    return out


def tiered(g, ctx, torch, n_rings, tier_mb, runs, secs):
    from bench_ring_checkpoint import nvml_rows
    F, cap, W, alpha = 64, 1_000_000, 1000, 0.01
    thr = np.array([(46.0, 350000.0, 1980.0, 50.0)[f % 4] for f in range(F)])
    pool = [torch.from_numpy(nvml_rows(F, CHUNK, 2000 + i).astype(np.float64)).cuda() for i in range(4)]
    torch.cuda.synchronize()
    rings = [g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha) for _ in range(n_rings)]
    for r in rings:
        r.tier_open(tier_mb << 20)
    total = 0
    while total < 2600 * RATE:
        c = total // CHUNK
        for k, r in enumerate(rings):
            r.push_device(pool[(c + k) % len(pool)].data_ptr(), CHUNK)
        total += CHUNK
        if total >= 1900 * RATE and all(r.tier_counts()[0] > 0 for r in rings):
            break
    for r in rings:
        r.sync()
    reach = max(min(total - cap, r.tier_counts()[0]) for r in rings)
    out = {"workload": "configs[1] live: %d rings of 64 fields x 1 M samples, W = 1000, %d MB tier each, full" % (n_rings, tier_mb),
           "seconds_pushed": total / RATE, "reach_s": (total - reach) / RATE}
    home, fields = rings[0], [1]
    for name, first, n in (("last_30min", total - 1800 * RATE, 1800 * RATE), ("30s_ending_5min_back", total - 330 * RATE, 30 * RATE)):
        if first < reach:
            out[name] = "beyond the tiers' reach"
            continue
        one = alternate(lambda: home.reduce_ranges([first], [n], fields=fields), lambda: home.reduce_ranges([first], [n]), fields, runs, home)
        ro, so = np.arange(n_rings, dtype=np.int32), np.array([0, n_rings], dtype=np.int64)
        box = alternate(lambda: g.rings_reduce_range_sets(rings, ro, [first] * n_rings, [n] * n_rings, so, fields=fields),
                        lambda: g.rings_reduce_range_sets(rings, ro, [first] * n_rings, [n] * n_rings, so), fields, runs, home)
        out[name] = {"one_ring": {"1_field_device_ms": spread(one[0]["fields"]), "64_fields_device_ms": spread(one[0]["all"]),
                                  "1_field_decode_ms": spread(one[1]["fields"]), "64_fields_decode_ms": spread(one[1]["all"])},
                     "box_sets": {"1_field_device_ms": spread(box[0]["fields"]), "64_fields_device_ms": spread(box[0]["all"]),
                                  "1_field_decode_ms": spread(box[1]["fields"]), "64_fields_decode_ms": spread(box[1]["all"])}}
    # one live second: push 10 000 uint32 rows, then the last minute's p99 of one field (or of every field), alternated
    rows = torch.randint(30, 90, (RATE, F), dtype=torch.int32).pin_memory()
    walls = {"fields": [], "all": []}
    dev = {"fields": [], "all": []}
    for i in range(2 * secs):
        what = ("fields", "all")[i % 2]
        t0 = time.perf_counter()
        home.push_raw_ptr(rows.data_ptr(), RATE, g.DTYPES["uint32"])
        t = home.counts()[0]
        got = home.reduce_ranges([t - 60 * RATE], [60 * RATE], fields=fields if what == "fields" else None)
        walls[what].append((time.perf_counter() - t0) * 1e3)
        dev[what].append(home.ranges_stats()[0])
        if what == "fields":
            same_cols(got, home.reduce_ranges([t - 60 * RATE], [60 * RATE]), fields)
    out["live_second"] = {"workload": "ring 0: push 10 000 uint32 rows + the last minute of 1 field or of all 64, alternated",
                          "wall_ms": {k: spread(v) for k, v in walls.items()}, "device_ms": {k: spread(v) for k, v in dev.items()}}
    for r in rings:
        r.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=6)
    ap.add_argument("--rings", type=int, default=8)
    ap.add_argument("--tier-mb", type=int, default=512)
    ap.add_argument("--secs", type=int, default=30)
    a = ap.parse_args()
    import torch
    import gpud_b200 as g
    import synth_device as sd
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()
    ctx = g.Context([0])
    out = {"card": card, "survey": survey(g, ctx, torch, sd, a.runs, np.random.default_rng(2026)),
           "tier": tiered(g, ctx, torch, a.rings, a.tier_mb, a.runs, a.secs)}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
