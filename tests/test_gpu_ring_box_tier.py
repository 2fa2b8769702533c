"""gpud_rings_reduce_range_sets over rings whose tiers it reaches into (DESIGN.md §2 "Box sets", "Tier").  2, 5 and 8 rings on NVML-like
uint32 rows pushed raw (INT blocks) and f64 fields with noise, infinities and NaN (RAW blocks): a tier that reaches before its ring, an
untiered ring, a tier shorter than its ring and one that wraps its byte ring.  Sets from test_gpu_ring_box_sets._mixed's generators made
to reach back: singletons per ring, many 1-sample ranges, joins at 1/31/32/33/1023/1024/1025 between rings and across the tier/ring
boundary, the partial newest row, every ring whole from its reach.  Every answer equals the same call over untiered twins that hold every
sample (all six outputs bit for bit) and the C oracle (min / max / p99 / n_over bit for bit, mean and EMA within oracle/SPEC.md's
tolerance); singleton sets equal their ring's reduce_ranges; nothing of the other rings changes; forced field groups and an untiered home
ring give the same bits.  Calls with no tier set equal the same call on untiered rings of the same CAP, routes and scratch included.  A
set spread over two tiered rings, its data built against its strided sample, takes every route the segment model predicts.  Refusals at
every ring's reach +-1 write nothing and name the ring and the range.  The same on two devices when the machine has them.  Run on an
H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import ring_box_tier as B
import ring_tier as T
import test_segment_paths_model as M
import test_tier_paths_model as TM
from test_gpu_ring_box_sets import _n_gpus, _sets, _want
from test_gpu_ring_ranges import OPS, _alpha, _fields, _thr
from test_gpu_ring_tier import _bitwise, _nvml
from test_gpu_segment_paths import _check_scratch, _scratch
from test_gpu_window_paths import _check

pytestmark = pytest.mark.gpu
ROW = T.ROW


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    L = g.lib()
    L.gpudh_ring_segment_scratch.restype = C.c_int32
    L.gpudh_ring_segment_scratch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64)]
    yield g, ctx, L
    ctx.close()


KINDS = ("long", "none", "short", "wrap")   # ring k's tier: reaches before the ring, none, shorter than the ring, wraps its byte ring


def _tier_bytes(kind, F, cap, total, data):
    row = T.max_row_bytes(F)
    if kind == "long":
        return row * (total // ROW + 2)
    if kind == "short":
        return row                                  # a few coded rows: fewer than the ring holds
    return row * (cap // ROW + 8) if data == "noise" else 3 * row   # "wrap": more rows than the ring, evicting


def _build(g, ctx, devs, data, W, q, alpha, cap=1 << 14, F=8, kinds=None, twin_cap=None):
    """rings on devs (tiers by KINDS, or kinds), their samples x [F][total] from push-order sample 0, and untiered twins that hold every
    sample (capacity twin_cap, default large enough)"""
    n = len(devs)
    kinds = kinds or [KINDS[k % 4] for k in range(n)]
    rng = np.random.default_rng([n, W, q[0], len(data)])
    totals = [(12 * cap + 777, 5 * cap + 3, 9 * cap + 3 * ROW, 7 * cap + 500)[k % 4] + 1000 * (k // 4) for k in range(n)]
    xs, raws = [], []
    for t in totals:
        if data == "nvml":
            rows = _nvml(F, t, rng)
            raws.append(rows)
            xs.append(rows.T.astype(np.float64))
        else:
            x = _fields(F, t, rng)
            xs.append(x)
            raws.append(np.ascontiguousarray(x.T))
    x0 = xs[0]
    if data == "nvml":
        thr = np.array([np.median(x0[f]) for f in range(F)])
    else:
        thr = _thr(x0)
    twin_cap = twin_cap or 1 << 18
    rings, twins = [], []
    for k, d in enumerate(devs):
        r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1], dev=d)
        tw = g.Ring(ctx, F, twin_cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1], dev=d)
        if kinds[k] != "none":
            r.tier_open(_tier_bytes(kinds[k], F, cap, totals[k], data))
        for a in range(0, totals[k], 5000):             # pushes well below CAP - 1023: the tier codes every row before it is overwritten
            part = raws[k][a:a + 5000]
            for rr in (r, tw):
                rr.push_raw(part) if data == "nvml" else rr.push(part)
        rings.append(r)
        twins.append(tw)
    return rings, twins, xs, thr, totals, kinds


def _reach(rings, cap):
    """per ring: (lo_k, first sample the ring holds, total)"""
    out = []
    for r in rings:
        total = r.counts()[0]
        held = total - min(total, cap)
        lo = min(held, r.tier_counts()[0]) if _tiered(r) else held
        out.append((lo, held, total))
    return out


def _tiered(r):
    import gpud_b200 as g
    try:
        r.tier_counts()
        return True
    except g.GpudError:
        return False


def _mixed_sets(rng, reach):
    n = len(reach)

    def pick(k, m, tier=False):
        lo, held, total = reach[k]
        m = min(m, total - lo)
        hi = held - 1 if tier and lo < held else total - m
        return (k, int(rng.integers(lo, max(lo, min(hi, total - m)) + 1)), m)

    def anyring(m, tier=False):
        return pick(int(rng.integers(0, n)), m, tier)
    sets = []
    for k in range(n):                                                  # singletons per ring: short, one tile, long; in the tier and not
        for m in (1, 33, 1025, 40000):
            sets.append([pick(k, m, tier=True)])
            sets.append([pick(k, m)])
    sets.append([anyring(1, tier=True) for _ in range(700)])            # many 1-sample ranges over every ring: short
    sets.append([anyring(1, tier=bool(i % 2)) for i in range(3000)])    # ... and long, a join at every sample
    for cut in (1, 31, 32, 33, 1023, 1024, 1025):                       # joins between rings, from a tier into a ring
        a, b = (0, 1) if cut % 2 else (n - 1, 0)
        sets.append([pick(a, cut, tier=True), pick(b, 3000), anyring(700, tier=True)])
    for k in range(n):
        lo, held, total = reach[k]
        if lo < held:                                                   # across the tier/ring boundary, then a join into another tier
            f0 = max(lo, held - 1023)
            sets.append([(k, f0, min(2048, total - f0)), pick((k + 1) % n, 1025, tier=True)])
        end = (total // ROW) * ROW                                      # into the partial newest row
        sets.append([(k, end - 3, total - end + 3), anyring(50, tier=True)])
    sets.append([(k, reach[k][0], reach[k][2] - reach[k][0]) for k in range(n)])   # every ring whole from its reach: the box
    sets.append([anyring(400, tier=True), anyring(400), anyring(400, tier=True)])
    order = rng.permutation(len(sets))
    return [sets[i] for i in order]


def _ring_state(r):
    st = [r.counts()]
    if _tiered(r):
        st += [r.tier_counts(), r.tier_stats()]
    try:
        st.append(r.ranges_stats())
    except Exception:
        st.append(None)
    return st


def _close(*groups):
    for grp in groups:
        for r in grp:
            r.close()


def _mixed(g, ctx, L, devs, data, W, q, alpha, groups=False):
    rings, twins, xs, thr, totals, kinds = _build(g, ctx, devs, data, W, q, alpha)
    try:
        reach = _reach(rings, 1 << 14)
        assert any(lo < held for lo, held, _ in reach)
        rng = np.random.default_rng([len(devs), W])
        sets = _mixed_sets(rng, reach)
        ring_of, first, length, set_off = _sets(sets)
        for r in rings[1:]:                                             # give every ring a ranges_stats of its own to compare
            r.reduce_ranges([r.counts()[0] - 10], [10])
        before = [_ring_state(r) for r in rings[1:]]
        got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
        ms, n_radix, why = rings[0].ranges_stats()
        assert ms > 0 and n_radix == sum(why.values())
        if kinds[0] != "none":
            assert rings[0].tier_stats()[1] > 0                        # the home ring's decode time is the call's
        assert [_ring_state(r) for r in rings[1:]] == before            # nothing of the other rings changed
        want = g.rings_reduce_range_sets(twins, ring_of, first, length, set_off)
        assert _bitwise(got, want)
        _check(got, _want(xs, [0] * len(xs), ring_of, first, length, set_off, thr, _alpha(W, alpha), q))
        if groups:
            for G in (1, 3, rings[0].F - 1):                            # forced field groups on the tiered home ring
                rings[0].tier_group(G)
                try:
                    assert _bitwise(g.rings_reduce_range_sets(rings, ring_of, first, length, set_off), got), G
                finally:
                    rings[0].tier_group(0)
            # an untiered home ring (ring 1) with tiered others: the same sets, the same bits
            perm = [1, 0] + list(range(2, len(rings)))
            inv = np.argsort(perm)
            got_u = g.rings_reduce_range_sets([rings[i] for i in perm], inv[ring_of], first, length, set_off)
            assert _bitwise(got_u, got)
        # singleton sets: their own ring's reduce_ranges, all six outputs bit for bit; a one-ring call is that ring's reduce_range_sets
        gb = {k: got[k] for k in OPS}
        for k in range(len(rings)):
            idx = [i for i, s in enumerate(sets) if len(s) == 1 and s[0][0] == k]
            own = rings[k].reduce_ranges([sets[i][0][1] for i in idx], [sets[i][0][2] for i in idx])
            assert _bitwise({op: gb[op][:, idx] for op in OPS}, own), k
        k = next(i for i, kd in enumerate(kinds) if kd != "none")
        mine = [i for i, s in enumerate(sets) if all(p[0] == k for p in s)]
        s1 = [[(0, f, m) for _, f, m in sets[i]] for i in mine]
        ro1, f1, l1, so1 = _sets(s1)
        assert _bitwise(g.rings_reduce_range_sets([rings[k]], ro1, f1, l1, so1), rings[k].reduce_range_sets(f1, l1, so1))
    finally:
        _close(rings, twins)


@pytest.mark.parametrize("n_rings,data,W,q,alpha", [(2, "nvml", 1000, (0, 0), 0.0), (5, "noise", 999, (999, 1000), 0.9999),
                                                     (8, "nvml", 1, (1, 2), 0.0), (5, "nvml", 1000, (99, 100), 0.01)])
def test_mixed_sets_against_twins_and_oracle(env, n_rings, data, W, q, alpha):
    g, ctx, L = env
    _mixed(g, ctx, L, [0] * n_rings, data, W, q, alpha, groups=n_rings == 5)


def test_calls_without_tier_sets_are_unchanged(env):
    """sets wholly in the rings: the same answers, open count, reasons and segment-select scratch as the same call on untiered rings
    of the same CAP"""
    g, ctx, L = env
    cap = 1 << 14
    rings, same, xs, thr, totals, kinds = _build(g, ctx, [0] * 4, "noise", 1000, (99, 100), 0.0, twin_cap=cap)
    try:
        rng = np.random.default_rng(8)
        sets = []
        for _ in range(30):
            parts = []
            for _ in range(int(rng.integers(1, 4))):
                k = int(rng.integers(0, 4))
                m = int(rng.choice([1, 500, 1025, 5000, cap]))
                parts.append((k, int(rng.integers(totals[k] - cap, totals[k] - m + 1)), m))
            sets.append(parts)
        ring_of, first, length, set_off = _sets(sets)
        got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
        st, scr = rings[0].ranges_stats()[1:], _scratch(L, rings[0])
        want = g.rings_reduce_range_sets(same, ring_of, first, length, set_off)
        assert _bitwise(got, want)
        assert st == same[0].ranges_stats()[1:]
        s2 = _scratch(L, same[0])
        for a, b in zip(scr, s2):
            assert np.array_equal(a, b)
    finally:
        _close(rings, same)


def test_routes_of_a_set_over_two_tiers(env):
    """test_gpu_tier_paths.test_sets_of_pieces_in_the_tier with its six pieces alternating between two tiered rings (given twice): every
    reason, pivot, list fill and class count the segment model predicts from the set's strided sample, a NaN field among them"""
    g, ctx, L = env
    pieces, pos, k, built = TM.sets_layout()
    F, cap, total, q = len(built), TM.SETS_CAP, TM.SETS_TOTAL, TM.SETS_Q
    xs = [np.random.default_rng(5 + kr).normal(60.0 + 10 * kr, 3.0, (F, total)) for kr in range(2)]
    for f, (_, xf) in enumerate(built):
        for j, ((p, ln), a) in enumerate(zip(pieces, TM.SETS_CUTS[:-1])):
            xs[j % 2][f, p:p + ln] = xf[a:a + ln]
    thr = np.full(F, 60.0)
    rings, twins = [], []
    try:
        for kr in range(2):
            r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
            tw = g.Ring(ctx, F, 1 << 17, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
            r.tier_open(T.max_row_bytes(F) * (total // ROW + 2))
            rings.append(r)
            twins.append(tw)
            for a in range(0, total, 8192):
                part = np.ascontiguousarray(xs[kr][:, a:a + 8192].T)
                r.push(part)
                tw.push(part)
        one = [(j % 2, p, ln) for j, (p, ln) in enumerate(pieces)]
        ring_of, first, length, set_off = _sets([one, one])
        route = B.split([total, total], cap, [(0, total // ROW)] * 2, ring_of, first, length, set_off)[0]
        assert route == [1, 1]
        got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
        _, n_open, why = rings[0].ranges_stats()
        scr = _scratch(L, rings[0])
        assert _bitwise(got, g.rings_reduce_range_sets(twins, ring_of, first, length, set_off))
    finally:
        _close(rings, twins)
    _check(got, _want(xs, [0, 0], ring_of, first, length, set_off, thr, _alpha(1000, 0.0), q))
    expect = {}
    for rt, _ in built:
        if rt in M.OPEN:
            expect[rt] = expect.get(rt, 0) + 2
    assert expect and why == expect and n_open == sum(expect.values()), (why, expect)
    geo = TM.sets_geo(pos, k)
    nt = -(-TM.SETS_N // M.TILE)
    models = {}
    for f, (_, xf) in enumerate(built):
        m = M.model_segment(xf, geo)
        for j in range(2):
            models[f * 2 + j, f * 2 * nt + j * nt] = m
    _check_scratch(scr, models, 2 * F, 2 * F * nt)


def test_refusals(env):
    """each ring's reach: lo_k - 1 and a range past total_k refused with the output untouched and the ring and the range named (its
    reach for a tiered ring); lo_k and total_k taken; every ring's counts, tier counts, tier stats and ranges stats read the same"""
    g, ctx, L = env
    cap = 1 << 14
    rings, twins, xs, thr, totals, kinds = _build(g, ctx, [0] * 3, "nvml", 1000, (99, 100), 0.0, kinds=["long", "none", "short"])
    try:
        reach = _reach(rings, cap)
        F = rings[0].F
        for r in rings:
            r.reduce_ranges([r.counts()[0] - 10], [10])

        def call(ro, f, n):
            ro, f, n = (np.ascontiguousarray(a, dt) for a, dt in ((ro, np.int32), (f, np.int64), (n, np.int64)))
            so = np.array([0, len(f)], np.int64)
            out, nov = np.full((5, F, 1), 7.0), np.full((F, 1), 7, np.uint32)
            hs = (C.c_void_p * 3)(*[r._h.value for r in rings])
            rc = L.gpud_rings_reduce_range_sets(C.cast(hs, C.c_void_p), 3, C.c_void_p(ro.ctypes.data), C.c_void_p(f.ctypes.data),
                                                C.c_void_p(n.ctypes.data), len(f), C.c_void_p(so.ctypes.data), 1, C.c_void_p(out.ctypes.data),
                                                C.c_void_p(nov.ctypes.data))
            return rc, bool(np.all(out == 7.0) and np.all(nov == 7))

        def last_error():
            buf = C.create_string_buffer(512)
            L.gpud_last_error(ctx._h, buf, 512)
            return buf.value.decode()
        for k, (lo, held, total) in enumerate(reach):
            others = [j for j in range(3) if j != k]
            for f, n, ok in ((lo - 1, 5, False), (lo, 5, True), (total - 7, 8, False), (total - 7, 7, True)):
                ro = [k] + others
                fs = [f] + [reach[j][2] - 10 for j in others]
                ns = [n] + [10] * 2
                before = [_ring_state(r) for r in rings]
                rc, clean = call(ro, fs, ns)
                if ok:
                    assert rc == 0 and not clean, (k, f, n)
                    continue
                err = last_error()
                assert rc == -1 and clean, (k, f, n)
                assert "range 0" in err and ("ring %d" % k) in err and ("[%d, +%d)" % (f, n)) in err, err
                if kinds[k] != "none":
                    assert "reach [%d, %d)" % (lo, total) in err, err
                else:
                    assert "(pushed %d, held %d)" % (total, min(total, cap)) in err, err
                assert [_ring_state(r) for r in rings] == before, (k, f, n)   # nothing of any ring reads differently
        assert reach[0][0] < reach[0][1] and reach[2][0] == reach[2][1]   # a tier before its ring, and one shorter than its ring
    finally:
        _close(rings, twins)


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("devs", [(0, 1), (1, 0, 1, 0)])
def test_two_devices(devs):
    """rings on two devices: other rings' coded rows decoded on the home device through the peer mapping"""
    import gpud_b200 as g
    ctx = g.Context([0, 1])
    try:
        _mixed(g, ctx, g.lib(), list(devs), "nvml", 1000, (0, 0), 0.0)
    finally:
        ctx.close()
