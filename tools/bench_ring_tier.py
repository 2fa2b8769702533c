#!/usr/bin/env python3
"""Measure the ring's tier (DESIGN.md §2 "Tier") on BASELINE configs[1] live: 64 fields, CAP = 1 000 000, W = 1000, NVML-like uint32
rows (tools/bench_ring_checkpoint.py's gauges) pushed raw at 10 000 rows per live second, into a ring with a 512 MB tier and into an
untiered twin, alternated second by second.

Reports: host ms per live second of push (+ encode on the tiered ring) to the end of its device work, both rings, median and spread;
the tier's bytes per sample and the seconds of history it holds; device ms (gpud_ring_ranges_stats, decode included, and the decode
alone) of a 30 s range ending 5 minutes back and of one 30-minute range (or the longest range the tier holds, if it holds less); and
the tier bytes per sample of the survey stream (BASELINE configs[3], tests/synth_device.py).  Every range answer is checked in the
same run against the C oracle on the kept rows: min / max / p99 / n_over bit for bit, mean and EMA within oracle/SPEC.md's tolerance.
Prints one JSON line with the card and its power limit, read in the same run.  Writes nothing in the tree.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

RATE = 10_000


def spread(xs):
    q = np.percentile(xs, [10, 50, 90])
    return {"median": statistics.median(xs), "p10": float(q[0]), "p90": float(q[2]), "min": min(xs), "max": max(xs), "n": len(xs)}


def check(got, x, thr, alpha, fields):
    """the range's answer for `fields` against the oracle on its rows x [len(fields)][n] (f64)"""
    from oracle import coracle
    want = coracle.windows_fields(np.ascontiguousarray(x), x.shape[1], thr[fields], alpha)
    for k in ("min", "max", "p99"):
        assert np.array_equal(got[k][fields, 0].view(np.uint64), want[k][:, 0].view(np.uint64)), k
    assert np.array_equal(got["n_over"][fields, 0], want["n_over"][:, 0].astype(np.uint32)), "n_over"
    for k in ("mean", "ema"):
        a, b = got[k][fields, 0], want[k][:, 0]
        assert np.all(np.abs(a - b) <= 1e-6 * np.maximum(np.abs(b), np.abs(x).max(axis=1))), k


def range_ms(r, first, n, runs):
    ms, dec, got = [], [], None
    for _ in range(runs):
        got = r.reduce_ranges([first], [n])
        ms.append(r.ranges_stats()[0])
        dec.append(r.tier_stats()[1])
    return got, spread(ms), spread(dec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=int, default=2200, help="live seconds pushed")
    ap.add_argument("--tier-mb", type=int, default=512)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--survey", type=int, default=1)
    a = ap.parse_args()
    import gpud_b200 as g
    from bench_ring_checkpoint import nvml_rows
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    ctx = g.Context([0])
    F, cap, W, alpha = 64, 1_000_000, 1000, 0.01
    thr = np.array([(46.0, 350000.0, 1980.0, 50.0)[f % 4] for f in range(F)])
    tier_bytes = a.tier_mb << 20
    rt = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha)
    ru = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha)
    rt.tier_open(tier_bytes)
    S = a.seconds
    total = S * RATE
    # kept rows for the oracle: every field of the 30 s ending 5 minutes back, fields 0..3 of the last 30 minutes
    near0 = total - 330 * RATE
    far0 = max(0, total - 1800 * RATE)
    near = np.empty((330 * RATE - 300 * RATE, F), dtype=np.uint32) if S >= 330 else None
    far = np.empty((total - far0, 4), dtype=np.uint32)
    chunk = 100 * RATE
    t_tier, t_plain = [], []
    for c0 in range(0, total, chunk):
        rows = nvml_rows(F, min(chunk, total - c0), 1000 + c0 // chunk)
        lo_, hi_ = max(c0, far0), min(c0 + len(rows), total)
        if hi_ > lo_:
            far[lo_ - far0:hi_ - far0] = rows[lo_ - c0:hi_ - c0, :4]
        if near is not None:
            lo_, hi_ = max(c0, near0), min(c0 + len(rows), near0 + len(near))
            if hi_ > lo_:
                near[lo_ - near0:hi_ - near0] = rows[lo_ - c0:hi_ - c0]
        for s0 in range(0, len(rows), RATE):
            sec = np.ascontiguousarray(rows[s0:s0 + RATE])
            order = ((rt, t_tier), (ru, t_plain)) if (c0 + s0) // RATE % 2 == 0 else ((ru, t_plain), (rt, t_tier))
            for r, acc in order:
                t = time.perf_counter()
                r.push_raw(sec)
                r.sync()
                acc.append((time.perf_counter() - t) * 1e3)
        del rows
    first, nxt, used, lost = rt.tier_counts()
    enc, _, blocks = rt.tier_stats()
    out = {"card": card, "F": F, "cap": cap, "rate": RATE, "seconds_pushed": S, "tier_bytes": tier_bytes,
           "push_ms_per_live_second_tiered": spread(t_tier[10:]), "push_ms_per_live_second_untiered": spread(t_plain[10:]),
           "tier_first_sample": first, "tier_next_sample": nxt, "tier_bytes_used": used, "rows_lost": lost,
           "tier_bytes_per_sample": used / ((nxt - first) * F), "tier_history_s": (nxt - first) / RATE,
           "reach_s": (total - min(first, total - cap)) / RATE, "full": first > 0, "last_encode_device_ms": enc, "last_encode_blocks": blocks}
    lo = min(first, total - cap)
    if near is not None and near0 >= lo:
        got, ms, dec = range_ms(rt, near0, 30 * RATE, a.runs)
        check(got, near.T.astype(np.float64), thr, alpha, np.arange(F))
        out["range_30s_5min_back"] = {"device_ms": ms, "decode_ms": dec, "checked": "oracle, all fields"}
    n = min(1800 * RATE, total - lo)
    got, ms, dec = range_ms(rt, total - n, n, a.runs)
    check(got, far[len(far) - n:].T.astype(np.float64), thr, alpha, np.arange(4))
    out["range_long"] = {"seconds": n / RATE, "device_ms": ms, "decode_ms": dec, "checked": "oracle, fields 0..3"}
    rt.close()
    ru.close()
    if a.survey:
        import synth_device as SD
        Fs, caps = 512, 1 << 20
        r = g.Ring(ctx, Fs, caps, 1000)
        SD.fill_ring(r, "survey", Fs, caps, 5, "cuda")
        r.tier_open(1 << 30)
        f0, f1, u, _ = r.tier_counts()
        out["survey_tier_bytes_per_sample"] = u / ((f1 - f0) * Fs)
        out["survey_rows_held"] = (f1 - f0) // 1024
        r.close()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
