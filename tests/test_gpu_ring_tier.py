"""The ring's tier on the GPU (DESIGN.md §2 "Tier").  Ranges and range sets that reach into the tier against an untiered ring large
enough to hold every sample (all six outputs bit for bit) and against the C oracle (min / max / p99 / n_over bit for bit, mean and
EMA within oracle/SPEC.md's tolerance), on NVML-like uint32 rows pushed raw (INT blocks) and f64 fields with noise, infinities and NaN (RAW blocks): wholly in the tier,
straddling its boundary with the ring, wholly in the ring, 1 sample, <= 1024, > 1024 and > CAP.  Every row's bytes against the host
model (tests/ring_tier.py), its placement and tier_counts after every push against the model's, refusals before the tier with
nothing written, every push entry point and raw dtype giving the same bytes, a tiered ring's reduce, handles and checkpoints equal to
an untiered twin's, and forced small field groups giving the same answers.  The range path's routes on the decoded ring, wide rows,
natural field groups and capacities that are not a multiple of 1024 are test_gpu_tier_paths.py's.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import ring_tier as T
import mean_ema_ref as R
from test_gpu_ring_ranges import OPS, _fields, _thr
from test_gpu_window_paths import _check

pytestmark = pytest.mark.gpu
ROW = T.ROW


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx, g.lib()
    ctx.close()


def _nvml(F, n, rng):
    """NVML-like uint32 gauges: temperatures, clocks, power in mW, utilisation, a byte counter: [n][F]"""
    cols = []
    for f in range(F):
        kind = f % 4
        if kind == 0:
            c = 40 + np.cumsum(rng.integers(-1, 2, n)) % 40
        elif kind == 1:
            c = 1980 - 15 * rng.integers(0, 3, n)
        elif kind == 2:
            c = 350000 + np.cumsum(rng.integers(-2000, 2001, n))
        else:
            c = np.cumsum(rng.integers(0, 1 << 12, n))
        cols.append(np.asarray(c % (1 << 32), dtype=np.uint32))
    return np.ascontiguousarray(np.stack(cols, axis=1))


def _push_all(r, rows, chunks):
    a = 0
    for n in chunks:
        if a >= len(rows):
            break
        r.push_raw(rows[a:a + n]) if rows.dtype != np.float64 else r.push(rows[a:a + n])
        a += n


def _cases(total, cap, lo, rng):
    """ranges wholly in the tier, straddling, wholly in the ring; 1, <= 1024, > 1024, > CAP samples"""
    ring0 = total - cap
    out = [(lo, 1), (lo, ROW), (lo + 3, 1500), (ring0 - 700, 1400), (ring0 - 1, 2), (ring0 - 5000, 5000 + cap // 2), (ring0, cap),
           (total - 1, 1), (total - 1000, 1000), (lo, total - lo), (lo + 1, min(3 * cap, total - lo - 1)), (ring0 - 2 * cap, 2 * cap + 77)]
    for _ in range(12):
        n = int(rng.choice([1, 31, 1024, 1025, 4000, cap + 5]))
        n = min(n, total - lo)
        out.append((int(rng.integers(lo, total - n + 1)), n))
    return [(f, n) for f, n in out if f >= lo and n >= 1 and f + n <= total]


def _oracle(x, first, length, set_off, thr, alpha):
    cols = []
    for s in range(len(set_off) - 1):
        c = np.concatenate([x[:, f:f + n] for f, n in zip(first[set_off[s]:set_off[s + 1]], length[set_off[s]:set_off[s + 1]])], axis=1)
        cols.append(R.windows_fields(np.ascontiguousarray(c), c.shape[1], thr, alpha))
    return {k: np.concatenate([c[k] for c in cols], axis=1) for k in cols[0]}


def _bitwise(a, b, keys=OPS):
    return all(np.array_equal(a[k].view(np.uint64 if k != "n_over" else np.uint32), b[k].view(np.uint64 if k != "n_over" else np.uint32)) for k in keys)


@pytest.mark.parametrize("kind,cap", [("nvml", 16384), ("noise", 8192), ("nvml", 65536)])
def test_ranges_against_large_ring_and_oracle(env, kind, cap):
    g, ctx, _ = env
    F, W, alpha = 8, 1000, 0.01
    rng = np.random.default_rng(cap + len(kind))
    total = 12 * cap + 777
    if kind == "nvml":
        rows = _nvml(F, total, rng)
        x = rows.T.astype(np.float64)
    else:
        x = _fields(F, total, rng)
        rows = np.ascontiguousarray(x.T)
    thr = np.array([np.median(x[f][np.isfinite(x[f])]) if np.isfinite(x[f]).any() else 0.0 for f in range(F)])
    if kind == "noise":
        thr = _thr(x)
    r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha)
    big = g.Ring(ctx, F, 1 << 20, W, thresholds=thr, ema_alpha=alpha)
    r.tier_open(20 * cap * F)
    chunks = [int(c) for c in rng.choice([1, 100, 1023, 1024, 5000, cap // 2], 4000)]
    _push_all(r, rows, chunks)
    _push_all(big, rows, chunks)
    assert r.counts()[0] == total
    t0, t1, used, lost = r.tier_counts()
    assert lost == 0 and t1 == (total // ROW) * ROW and 0 < used <= 20 * cap * F
    lo = min(total - cap, t0)
    assert lo < total - cap                          # the tier reaches before the ring
    cases = _cases(total, cap, lo, rng)
    first = np.array([f for f, _ in cases], dtype=np.int64)
    length = np.array([n for _, n in cases], dtype=np.int64)
    got = r.reduce_ranges(first, length)
    want = big.reduce_ranges(first, length)
    _check(got, _oracle(x, first, length, np.arange(len(first) + 1), thr, alpha))
    assert _bitwise(got, want)                     # mean and EMA too: tiles follow the concatenated samples, not their columns
    ms, _, _ = r.ranges_stats()
    enc, dec, blocks = r.tier_stats()
    assert ms > 0 and dec > 0 and enc > 0
    assert blocks["int"] + blocks["raw"] > 0 and (blocks["int"] > 0 or kind == "noise")
    # sets: mixed ring and tier pieces, a set wholly in the ring, one across the boundary, permuted and repeated ranges
    order = rng.permutation(len(cases))
    sf, sl = first[order], length[order]
    set_off = np.array(sorted({0, len(sf)} | set(rng.integers(1, len(sf), 6).tolist())), dtype=np.int64)
    got = r.reduce_range_sets(sf, sl, set_off)
    want = big.reduce_range_sets(sf, sl, set_off)
    _check(got, _oracle(x, sf, sl, set_off, thr, alpha))
    assert _bitwise(got, want)
    # small field groups give the same answers, bit for bit
    for G in (1, 3):
        r.tier_group(G)
        assert _bitwise(r.reduce_range_sets(sf, sl, set_off), got)
    r.tier_group(0)
    r.close()
    big.close()


def test_row_bytes_placement_and_counts(env):
    """a small tier that evicts and wraps: every row's bytes and offset and tier_counts after every push, against the host model"""
    g, ctx, _ = env
    F, cap = 3, 4096
    rng = np.random.default_rng(5)
    total = 90 * ROW + 300
    rows = _nvml(F, total, rng)
    rows[40 * ROW:60 * ROW, 1] = rng.integers(0, 1 << 31, (20 * ROW,))   # wide rows in the middle
    bits = rows.T.astype(np.float64).view(np.uint64)
    sizes = [T.row_bytes(bits[:, k * ROW:(k + 1) * ROW]) for k in range(total // ROW)]
    tier_bytes = 4 * T.max_row_bytes(F) // 3
    r = g.Ring(ctx, F, cap, 100, thresholds=np.full(F, 1000.0), ema_alpha=0.01)
    pre = 2500
    r.push_raw(rows[:pre])
    r.tier_open(tier_bytes)
    m = T.Tier(cap, F, tier_bytes, pre)
    m.settle(sizes)
    a = pre
    pushes = [1, 1023, 1024, 1500, cap - 1023, 7, cap - 1022, 3000, cap, 2 * cap]
    k = 0
    while a < total:
        n = min(pushes[k % len(pushes)], total - a)
        k += 1
        r.push_raw(rows[a:a + n])
        a += n
        m.push(n, sizes)
        assert r.tier_counts() == (m.first * ROW, m.next * ROW, m.used, m.lost), (a, n)
        for row, off, _ in m.rows:
            img = r.tier_row(row)
            assert img == T.row_image(bits[:, row * ROW:(row + 1) * ROW], row, off), row
    assert m.lost > 0 and any(o == 0 for o in m.row_off.values() if o is not None)
    # a range before the tier's first sample, or in lost rows, is refused with nothing written
    L = g.lib()
    t0 = r.tier_counts()[0]
    lo = min(total - cap, t0)
    f64 = np.full((5, F, 1), 7.0)
    nov = np.full((F, 1), 7, dtype=np.uint32)
    for f, n in ((lo - 1, 1), (0, 10), (lo, total - lo + 1)):
        fa, la = np.array([f], dtype=np.int64), np.array([n], dtype=np.int64)
        rc = L.gpud_ring_reduce_ranges(r._h, C.c_void_p(fa.ctypes.data), C.c_void_p(la.ctypes.data), 1, C.c_void_p(f64.ctypes.data),
                                       C.c_void_p(nov.ctypes.data))
        assert rc == -1 and (f64 == 7.0).all() and (nov == 7).all()
    so = np.array([0, 1], dtype=np.int64)
    fa, la = np.array([lo - 1], dtype=np.int64), np.array([5], dtype=np.int64)
    rc = L.gpud_ring_reduce_range_sets(r._h, C.c_void_p(fa.ctypes.data), C.c_void_p(la.ctypes.data), 1, C.c_void_p(so.ctypes.data), 1,
                                       C.c_void_p(f64.ctypes.data), C.c_void_p(nov.ctypes.data))
    assert rc == -1 and (f64 == 7.0).all()
    got = r.reduce_ranges([lo], [total - lo])
    want = R.windows_fields(np.ascontiguousarray(rows.T[:, lo:].astype(np.float64)), total - lo, np.full(F, 1000.0), 0.01)
    _check(got, want)
    r.close()


def test_open_refusals(env):
    g, ctx, _ = env
    r = g.Ring(ctx, 2, 2046, 100)
    with pytest.raises(g.GpudError) as e:
        r.tier_open(1 << 20)
    assert e.value.code == -1
    r.close()
    r = g.Ring(ctx, 2, 4096, 100)
    with pytest.raises(g.GpudError) as e:
        r.tier_open(T.max_row_bytes(2) - 1)
    assert e.value.code == -1
    r.tier_open(T.max_row_bytes(2))
    with pytest.raises(g.GpudError) as e:
        r.tier_open(1 << 20)
    assert e.value.code == -6
    r.close()


def test_entry_points_and_dtypes(env):
    import torch
    g, ctx, _ = env
    F, cap = 4, 8192
    rng = np.random.default_rng(11)
    n = 9 * ROW + 17
    base = rng.integers(0, 200, (n, F)).astype(np.uint8)
    rings = []
    for how in ("push", "device", "u8", "u16", "i16", "u32", "i32", "f32", "i64", "u64"):
        r = g.Ring(ctx, F, cap, 100)
        r.tier_open(1 << 20)
        for a in range(0, n, 3001):
            part = base[a:a + 3001]
            if how == "push":
                r.push(part.astype(np.float64))
            elif how == "device":
                t = torch.from_numpy(part.astype(np.float64)).cuda()
                r.push_device(t.data_ptr(), part.shape[0])
                torch.cuda.synchronize()
            else:
                dt = {"u8": np.uint8, "u16": np.uint16, "i16": np.int16, "u32": np.uint32, "i32": np.int32, "f32": np.float32, "i64": np.int64,
                      "u64": np.uint64}[how]
                r.push_raw(part.astype(dt))
        rings.append(r)
    ref = [rings[0].tier_row(k) for k in range(9)]
    for r in rings:
        assert r.tier_counts()[:2] == (0, 9 * ROW)
        assert [r.tier_row(k) for k in range(9)] == ref
    x = base.T.astype(np.float64).view(np.uint64)
    assert ref[4] == T.row_image(x[:, 4 * ROW:5 * ROW], 4, int.from_bytes(ref[4][8:16], "little"))
    for r in rings:
        r.close()


def test_twin_invariance(env):
    """a tiered ring's reduce, stream and windows histories, counts, and full and delta checkpoint bytes equal an untiered twin's"""
    g, ctx, _ = env
    F, cap, W = 6, 16384, 1000
    rng = np.random.default_rng(3)
    x = _fields(F, 7 * cap + 123, rng)
    thr = _thr(x)
    a = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=0.02)
    b = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=0.02)
    a.tier_open(8 * cap * F)
    for r in (a, b):
        r.stream_open()
    wa, wb = a.windows(3, hop=1), b.windows(3, hop=1)
    pos, blobs = 0, []
    for step, n in enumerate((5000, cap - 1023, 1, 2 * cap, 777, 30000, cap, 4000)):
        part = np.ascontiguousarray(x[:, pos:pos + n].T)
        pos += n
        for r in (a, b):
            r.push(part)
        assert a.stream_reduce() == b.stream_reduce()
        assert wa.reduce() == wb.reduce()
        assert a.counts() == b.counts()
        assert _bitwise(a.reduce_all(), b.reduce_all())
        if step == 2:
            blobs.append((a.checkpoint(), b.checkpoint()))
        elif step > 2:
            blobs.append((a.checkpoint_delta(), b.checkpoint_delta()))
    for ba, bb in blobs:
        assert ba == bb
    assert a.stream_counts() == b.stream_counts() and wa.counts() == wb.counts()
    f0, f1, _ = a.stream_counts()
    for op in OPS:
        assert np.array_equal(a.stream_read(op, f0, f1 - f0).view(np.uint8), b.stream_read(op, f0, f1 - f0).view(np.uint8))
        h0, h1, _ = wa.counts()
        assert np.array_equal(wa.read(op, h0, h1 - h0).view(np.uint8), wb.read(op, h0, h1 - h0).view(np.uint8))
    # ranges wholly in the ring: the same launches and results as the twin
    first, length = [pos - cap, pos - 50], [cap, 50]
    assert _bitwise(a.reduce_ranges(first, length), b.reduce_ranges(first, length))
    # a restored ring has no tier, and restore refuses a tiered ring
    c = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=0.02)
    c.tier_open(8 * cap * F)
    with pytest.raises(g.GpudError) as e:
        c.restore(blobs[0][0])
    assert e.value.code == -6
    for r in (a, b, c):
        r.close()
