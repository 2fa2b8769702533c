#!/usr/bin/env python3
"""Measure tier checkpoints (DESIGN.md "Ring tier checkpoint format") on BASELINE configs[1] live: 64 fields, CAP = 1 000 000,
W = 1000, NVML-like uint32 rows (tools/bench_ring_checkpoint.py's gauges) pushed raw at 10 000 rows per live second into a ring with a
full 512 MB tier.  A full tier checkpoint is written 11 minutes before the end, then a tier delta after every further live minute.

Reports: the full tier checkpoint at the end (bytes, device ms of its export and check pass, host ms into pageable and pinned
memory), the one-minute tier deltas (bytes, device and host ms), and the restore of the base plus its 10 deltas into a new ring after
its own ring checkpoint (device ms of the check pass and load, host ms).  Every round trip is checked in the same run: the restored
tier's counts equal the original's, its full tier checkpoint equals the original's byte for byte (so every held row does, but for
the offset word), and a 30 s range ending 5 minutes back equals the original's bit for bit and the C oracle (min / max / p99 / n_over
bit for bit, mean and EMA within oracle/SPEC.md's tolerance).  Prints one JSON line with the card and its power limit, read in the
same run.  Writes nothing in the tree.
"""
import argparse
import ctypes as C
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

RATE = 10_000
CHUNK = 10 * RATE                       # rows per push: well below CAP - 1024, so no row is ever lost


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=int, default=2200, help="live seconds pushed (the tier fills after about 1900)")
    ap.add_argument("--tier-mb", type=int, default=512)
    ap.add_argument("--deltas", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import gpud_b200 as g
    from bench_ring_checkpoint import nvml_rows
    from bench_ring_tier import check, spread
    import ring_tier_ckpt as TK
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    L = g.lib()
    ctx = g.Context([0])
    F, cap, W, alpha = 64, 1_000_000, 1000, 0.01
    thr = np.array([(46.0, 350000.0, 1980.0, 50.0)[f % 4] for f in range(F)])
    tier_bytes = a.tier_mb << 20
    S, total = a.seconds, a.seconds * RATE
    base_at = total - (a.deltas + 1) * 60 * RATE
    marks = {base_at + 60 * RATE * (i + 1): i for i in range(a.deltas)}       # the end of minute i after the base: delta i
    near0 = total - 330 * RATE
    near = np.empty((30 * RATE, F), dtype=np.uint32)
    rt = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha)
    rt.tier_open(tier_bytes)
    chain, delta_ms, delta_dev = [], [], []
    pos = 0
    while pos < total:
        n = min(CHUNK, total - pos, *[m - pos for m in list(marks) + [base_at] if m > pos])
        rows = nvml_rows(F, n, 1000 + pos // CHUNK)
        lo_, hi_ = max(pos, near0), min(pos + n, near0 + len(near))
        if hi_ > lo_:
            near[lo_ - near0:hi_ - near0] = rows[lo_ - pos:hi_ - pos]
        rt.push_raw(rows)
        pos += n
        if pos == base_at:
            chain.append(rt.tier_checkpoint())
        elif pos in marks:
            t = time.perf_counter()
            chain.append(rt.tier_checkpoint_delta())
            delta_ms.append((time.perf_counter() - t) * 1e3)
            delta_dev.append(rt.tier_checkpoint_stats()[0])
    first, nxt, used, lost = rt.tier_counts()
    assert lost == 0
    out = {"card": card, "F": F, "cap": cap, "rate": RATE, "seconds_pushed": S, "tier_bytes": tier_bytes, "tier_bytes_used": used,
           "tier_history_s": (nxt - first) / RATE, "tier_full": first > 0}
    # the full tier checkpoint at the end, into pageable and pinned memory
    bound = rt.tier_checkpoint_bound()
    page = bytearray(bound)
    p = C.c_void_p()
    assert L.gpud_host_alloc(bound, C.byref(p)) == 0
    pinned = np.frombuffer((C.c_char * bound).from_address(p.value), dtype=np.uint8)
    full = None
    for kind, buf in (("pageable", page), ("pinned", pinned)):
        host, dev = [], []
        for _ in range(a.runs):
            t = time.perf_counter()
            n = rt.tier_checkpoint(out=buf)
            host.append((time.perf_counter() - t) * 1e3)
            dev.append(rt.tier_checkpoint_stats()[0])
            blob = bytes(memoryview(buf)[:n])
            assert full is None or blob == full, kind
            full = blob
        out["full_" + kind] = {"host_ms": spread(host), "device_ms": spread(dev)}
    out["full_bytes"] = len(full)
    out["full_rows"] = rt.tier_checkpoint_stats()[2]
    out["delta_1min"] = {"bytes": spread([len(b) for b in chain[1:]]), "host_ms": spread(delta_ms), "device_ms": spread(delta_dev),
                         "rows": spread([TK.header(b)["next"] - TK.header(b)["from"] for b in chain[1:]])}
    ring_blob = rt.checkpoint()
    want = rt.reduce_ranges([near0], [30 * RATE])
    check(want, near.T.astype(np.float64), thr, alpha, np.arange(F))
    # restore of the base plus its deltas, each into a new ring after the ring's own restore
    host, dev = [], []
    for run in range(a.runs):
        r2 = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha)
        r2.restore(ring_blob)
        t = time.perf_counter()
        r2.tier_restore(tier_bytes, chain)
        host.append((time.perf_counter() - t) * 1e3)
        dev.append(r2.tier_checkpoint_stats()[1])
        if run == 0:
            assert r2.tier_counts() == rt.tier_counts()
            assert r2.tier_checkpoint() == full, "restored tier blob"
            got = r2.reduce_ranges([near0], [30 * RATE])
            for k in got:
                assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)), k
            check(got, near.T.astype(np.float64), thr, alpha, np.arange(F))
        r2.close()
    out["restore_base_plus_%d_deltas" % a.deltas] = {"chain_bytes": sum(len(b) for b in chain), "host_ms": spread(host), "device_ms": spread(dev),
                                                     "checked": "tier counts, full tier blob byte for byte, 30 s range 5 min back vs original and oracle"}
    L.gpud_host_free(p)
    rt.close()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
