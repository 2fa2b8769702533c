"""gpud_rings_reduce_range_sets_fields (DESIGN.md §2 "Field selection"): range sets over the fields a caller names.  Column g of every
answer is row fields[g] of gpud_rings_reduce_range_sets over the same rings, ranges and sets, all six outputs bit for bit, and the C
oracle on that field (min / max / p99 / n_over bit for bit, mean / EMA within mean_ema_ref's budget).  Covered: one field (first,
last, middle), unsorted and repeated lists, every field in order (the whole parent output, pivots and stats) and reversed; short sets,
long streamed tiles, tiles across joins and sets over 2 and 5 rings, with the segment select's pivots, list fill and class counts equal
to the parent's for the named fields' segments; every radix-select reason forced on a named field; an unnamed +NaN field never read;
tiered rings of every kind with named fields spanning a forced small field group; every refusal with nothing written and the argument
named, and the parent's refusals kept; reduce results and open handles unchanged.  The same on two devices when the machine has two
GPUs.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import range_cases as RC
import test_segment_paths_model as M
from test_gpu_ring_box_sets import _n_gpus, _sets, _state, _want
from test_gpu_ring_box_tier import _build, _close, _mixed_sets, _reach
from test_gpu_ring_range_sets import _push
from test_gpu_ring_ranges import OPS, _alpha, _fields, _thr
from test_gpu_ring_tier import _bitwise
from test_gpu_segment_paths import _scratch
from test_gpu_window_paths import _check

pytestmark = pytest.mark.gpu
E_INVALID = -1


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


def _cols(got, parent, fields):
    """got's row g is parent's row fields[g], all six outputs bit for bit"""
    return _bitwise(got, {k: parent[k][np.asarray(fields)] for k in OPS})


def _sub(want, fields):
    return {k: v[np.asarray(fields)] for k, v in want.items()}


def _scratch_cols(scr, parent_scr, fields, F):
    """the named fields' segments of the field call's last segment select equal the parent's: pivots, fill, class counts"""
    piv, fill, cls = scr
    ppiv, pfill, pcls = parent_scr
    nf = len(fields)
    n_long, rows = len(fill) // nf, len(cls) // nf
    assert len(pfill) == F * n_long and len(pcls) == F * rows
    idx = np.concatenate([np.arange(f * n_long, (f + 1) * n_long) for f in fields])
    ridx = np.concatenate([np.arange(f * rows, (f + 1) * rows) for f in fields])
    assert np.array_equal(piv, ppiv[idx]) and np.array_equal(fill, pfill[idx]) and np.array_equal(cls, pcls[ridx])


def _rings(g, ctx, n_rings, F, cap, W, q, alpha, seed, dev=None):
    rng = np.random.default_rng(seed)
    totals = [(3 * cap + 54321, cap - 12345, cap, 2 * cap + 1)[k % 4] + 1000 * (k // 4) for k in range(n_rings)]
    xs_all = [_fields(F, t, rng) for t in totals]
    thr = _thr(xs_all[0])
    rings = []
    for k in range(n_rings):
        r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1], dev=(dev[k] if dev else 0))
        _push(r, xs_all[k])
        rings.append(r)
    olds = [max(0, t - cap) for t in totals]
    return rings, [x[:, o:] for x, o in zip(xs_all, olds)], olds, totals, thr, rng


def _route_sets(rng, n_rings, olds, totals):
    """short sets, single long ranges (strided sample and sample ring), tiles across joins, sets over every ring"""
    def pick(k, n):
        return (k, int(rng.integers(olds[k], totals[k] - n + 1)), n)

    def anyring(n):
        return pick(int(rng.integers(0, n_rings)), n)
    sets = [[pick(0, n)] for n in (1, 33, 1024, 1025, 5000, 70000)]
    sets += [[anyring(10), anyring(20), anyring(30)], [anyring(1) for _ in range(2000)]]
    for cut in (1, 31, 1023, 1024, 1025):
        sets.append([anyring(cut), anyring(3000), anyring(700)])
    sets.append([(k, olds[k], totals[k] - olds[k]) for k in range(n_rings)])
    return sets


def _field_lists(F):
    return [[0], [F - 1], [F // 2], [5, 2, F - 1, 0], [3, 3, 7, 3], list(range(F)), list(range(F))[::-1]]


def test_field_lists_on_one_ring(env):
    """every kind of field list over one ring's sets: the parent's columns; all fields in order: the parent's output, open count,
    reasons and scratch; Ring.reduce_ranges(fields=...) is the same call over one range per set"""
    g, ctx, L = env
    F, cap = 16, 1 << 17
    rings, xs, olds, totals, thr, rng = _rings(g, ctx, 1, F, cap, 1000, (99, 100), 0.0, 11)
    r = rings[0]
    try:
        sets = _route_sets(rng, 1, olds, totals)
        _, first, length, set_off = _sets(sets)
        parent = r.reduce_range_sets(first, length, set_off)
        pst, pscr = r.ranges_stats()[1:], _scratch(L, r)
        for fields in _field_lists(F):
            got = r.reduce_range_sets(first, length, set_off, fields=fields)
            assert _cols(got, parent, fields), fields
            _scratch_cols(_scratch(L, r), pscr, fields, F)
            if fields == list(range(F)):
                assert _bitwise(got, parent) and r.ranges_stats()[1:] == pst
        singles = [i for i, s in enumerate(sets) if len(s) == 1]
        fs = [F - 1, 4]
        got = r.reduce_ranges([sets[i][0][1] for i in singles], [sets[i][0][2] for i in singles], fields=fs)
        assert _cols(got, {k: parent[k][:, singles] for k in OPS}, fs)
    finally:
        r.close()


@pytest.mark.parametrize("n_rings,W,q,alpha", [(1, 1000, (0, 0), 0.0), (2, 999, (999, 1000), 0.9999), (5, 1, (1, 2), 0.0)])
def test_routes_on_named_fields(env, n_rings, W, q, alpha):
    """short sets, long streamed tiles, tiles across joins and sets over every ring: the parent's columns, its scratch for the named
    fields' segments, and the oracle"""
    g, ctx, L = env
    F, cap = 8, 1 << 17
    rings, xs, olds, totals, thr, rng = _rings(g, ctx, n_rings, F, cap, W, q, alpha, n_rings)
    try:
        ring_of, first, length, set_off = _sets(_route_sets(rng, n_rings, olds, totals))
        parent = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
        pscr = _scratch(L, rings[0])
        fields = [6, 1, 1, 3]
        got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off, fields=fields)
        assert _cols(got, parent, fields)
        _scratch_cols(_scratch(L, rings[0]), pscr, fields, F)
        u = sorted(set(fields))
        _check(_sub(got, [fields.index(f) for f in u]), _want([x[u] for x in xs], olds, ring_of, first, length, set_off, thr[u], _alpha(W, alpha), q))
    finally:
        _close(rings)


@pytest.mark.parametrize("q,reasons", [((99, 100), ("above", "below", "nan", "overflow")), ((0, 1), ("below", "nan", "pivots"))])
def test_radix_reasons_on_named_fields(env, q, reasons):
    """one field per generator of tests/range_cases.py, its data built against the set's strided sample over pieces in two rings: each
    forced reason reported for the named fields alone, every column the parent's (the two quantiles force every GPUD_RANGE_OPEN_*
    reason of a sampled segment between them)"""
    g, ctx, L = env
    cap, n = 1 << 18, 200001
    S = min(RC.SAMPLE_MAX, max(64, n // 32))
    pos = np.arange(S, dtype=np.int64) * (n // S) + (n // S) // 2
    k = RC.k_from_top(n, *q)
    built = []
    for i, (name, fn, route) in enumerate(RC.GENERATORS):
        lay = RC.Layout(n, pos, k, np.random.default_rng([i, n, 9]))
        xf = fn(lay)
        if xf is not None:
            built.append((route(lay) if callable(route) else route, xf))
    F = len(built)
    totals = [cap + cap // 2 + 1, cap - 5]
    cuts = [0, 1, 1057, n // 3, n // 3 + 1024, n - 31, n]
    pieces, cur = [], list(totals)
    for j, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        cur[j % 2] -= b - a
        pieces.append((j % 2, cur[j % 2], b - a))
    xs = [np.random.default_rng(5 + kr).normal(60.0, 3.0, (F, t)) for kr, t in enumerate(totals)]
    for f, (_, xf) in enumerate(built):
        for (kr, p, ln), a in zip(pieces, cuts[:-1]):
            xs[kr][f, p:p + ln] = xf[a:a + ln]
    rings = []
    try:
        for kr in range(2):
            r = g.Ring(ctx, F, cap, 1000, thresholds=np.full(F, 60.0), q_num=q[0], q_den=q[1])
            _push(r, xs[kr], 1 << 18)
            rings.append(r)
        ring_of, first, length, set_off = _sets([pieces, pieces])
        parent = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
        opened = [f for f, (rt, _) in enumerate(built) if rt in M.OPEN]
        assert {built[f][0] for f in opened} == set(reasons)
        for fields in [[f] for f in opened] + [list(range(F))[::-1], opened[::2] + [0]]:
            got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off, fields=fields)
            _, n_radix, why = rings[0].ranges_stats()
            expect = {}
            for f in fields:
                if built[f][0] in M.OPEN:
                    expect[built[f][0]] = expect.get(built[f][0], 0) + 2
            assert why == expect and n_radix == sum(expect.values()), (fields, why, expect)
            assert _cols(got, parent, fields), fields
    finally:
        _close(rings)


def test_unnamed_fields_are_never_read(env):
    """a +NaN in field 1 opens GPUD_RANGE_OPEN_NAN in the parent call; a call that does not name field 1 opens nothing"""
    g, ctx, L = env
    F, cap, n = 4, 1 << 18, 200000
    x = np.random.default_rng(2).normal(60.0, 3.0, (F, n))
    x[1, n // 2] = np.nan
    r = g.Ring(ctx, F, cap, 1000, thresholds=np.full(F, 60.0))
    try:
        _push(r, x)
        parent = r.reduce_ranges([0, 1000], [n, n - 1000])
        assert r.ranges_stats()[2] == {"nan": 2}
        got = r.reduce_ranges([0, 1000], [n, n - 1000], fields=[3, 0, 2])
        assert r.ranges_stats()[1:] == (0, {})
        assert _cols(got, parent, [3, 0, 2])
    finally:
        r.close()


@pytest.mark.parametrize("n_rings,data", [(4, "nvml"), (5, "noise")])
def test_tiers_on_named_fields(env, n_rings, data):
    """rings whose tiers reach before the ring, none, shorter than the ring and wrapping: named fields spanning a forced group of 2
    decode alone and give the untiered twins' columns bit for bit; the home ring's decode time reports the call"""
    g, ctx, L = env
    rings, twins, xs, thr, totals, kinds = _build(g, ctx, [0] * n_rings, data, 1000, (99, 100), 0.0)
    try:
        sets = _mixed_sets(np.random.default_rng([n_rings, 7]), _reach(rings, 1 << 14))
        ring_of, first, length, set_off = _sets(sets)
        want = g.rings_reduce_range_sets(twins, ring_of, first, length, set_off)
        for G in (0, 2):
            rings[0].tier_group(G)
            try:
                for fields in ([5, 0, 7, 7, 2], [rings[0].F - 1], list(range(rings[0].F))):
                    got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off, fields=fields)
                    assert rings[0].tier_stats()[1] > 0
                    assert _cols(got, want, fields), (G, fields)
            finally:
                rings[0].tier_group(0)
    finally:
        _close(rings, twins)


def test_refusals(env):
    """each refusal of a field list writes nothing into sentinel-filled outputs and names the argument; the parent's refusals stay;
    the home ring's ranges stats, reduce results and open handles read the same"""
    g, ctx, L = env
    F, cap, W = 3, 1 << 17, 64
    thr = np.array([1.0, 2.0, 3.0])
    rings, spans = [], []
    for t in (150000, 70000):
        r = g.Ring(ctx, F, cap, W, thresholds=thr)
        span = r.windows(2)
        r.push(np.arange(3 * t, dtype=np.float64).reshape(t, 3))
        span.reduce()
        r.reduce()
        r.reduce_range(0)
        rings.append(r)
        spans.append(span)
    other = g.Ring(ctx, F, cap, W, thresholds=np.array([1.0, 2.0, 4.0]))
    other.push(np.ones((70000, F)))
    ring_of = np.array([0, 1, 0], np.int32)
    first = np.array([150000 - 100, 100, 149000], np.int64)
    length = np.array([100, 2000, 5], np.int64)
    so = np.array([0, 2, 3], np.int64)

    def call(rs, fields, nf=None, f=first, n=length, s=so, ns=None, out=None):
        fa = None if fields is None else np.ascontiguousarray(fields, np.int32)
        nf = len(fields) if nf is None else nf
        ns = len(s) - 1 if ns is None else ns
        if out is None:
            out = (np.full((5, max(nf, 1), max(ns, 1)), 7.0), np.full((max(nf, 1), max(ns, 1)), 7, np.uint32))
        f, n, s = (np.ascontiguousarray(a, np.int64) for a in (f, n, s))
        hs = (C.c_void_p * len(rs))(*[r._h.value for r in rs])
        rc = L.gpud_rings_reduce_range_sets_fields(C.cast(hs, C.c_void_p), len(rs), C.c_void_p(ring_of.ctypes.data),
                                                   None if fa is None else C.c_void_p(fa.ctypes.data), nf, C.c_void_p(f.ctypes.data),
                                                   C.c_void_p(n.ctypes.data), len(f), C.c_void_p(s.ctypes.data), ns,
                                                   C.c_void_p(out[0].ctypes.data), C.c_void_p(out[1].ctypes.data))
        return rc, bool(np.all(out[0] == out[0].flat[0]) and np.all(out[1] == out[1].flat[0]))

    def last_error():
        buf = C.create_string_buffer(512)
        L.gpud_last_error(ctx._h, buf, 512)
        return buf.value.decode()
    try:
        assert call(rings, [2, 0])[0] == 0
        states = [_state(r, s) for r, s in zip(rings, spans)]
        rstats = rings[0].ranges_stats()
        for fields, nf, what in ((None, 2, "fields is NULL"), ([0], 0, "n_fields is 0"), ([0, -1], None, "fields[1] is -1"),
                                 ([0, 1, 3], None, "fields[2] is 3")):
            rc, clean = call(rings, fields, nf)
            assert rc == E_INVALID and clean and what in last_error(), (fields, nf, last_error())
        # the segment limit counts the named fields: 2 x (2^23 + 1) sets; zero-filled outputs of that size, never written
        ns = (1 << 23) + 1
        big = (np.zeros((5, 2, ns)), np.zeros((2, ns), np.uint32))
        rc, clean = call(rings, [0, 0], ns=ns, out=big)
        assert rc == E_INVALID and clean and not big[0].any() and "GPUD_RANGES_MAX_SEGMENTS" in last_error()
        del big
        assert call(rings, [0], f=[0, 100, 149000])[0] == E_INVALID and "range 0" in last_error()   # before ring 0's oldest sample
        assert call(rings, [0], n=[100, 0, 5]) == (E_INVALID, True)                                # an empty range
        assert call(rings, [0], s=[0, 2, 2]) == (E_INVALID, True)                                  # set_off[n_sets] != n_ranges
        assert call(rings, [0], s=[0, 0, 3])[0] == E_INVALID and "set 0" in last_error()           # an empty set
        rc, clean = call([rings[0], other], [1])
        assert rc == E_INVALID and clean and "thresholds" in last_error() and "ring 1" in last_error()
        assert call(rings, [0], ns=0) == (0, True)                                                 # n_sets = 0 touches nothing
        assert rings[0].ranges_stats() == rstats
        for r, s, st in zip(rings, spans, states):
            now = _state(r, s)
            for a, b in zip(now[:2], st[:2]):
                for k in OPS:
                    assert np.array_equal(a[k], b[k]), k
            assert now[2:] == st[2:]
        # a call that runs leaves reduce results and handles as they were
        assert call(rings, [1, 1, 2])[0] == 0
        for r, s, st in zip(rings, spans, states):
            now = _state(r, s)
            for a, b in zip(now[:2], st[:2]):
                for k in OPS:
                    assert np.array_equal(a[k], b[k]), k
            assert now[2:] == st[2:]
    finally:
        _close(rings + [other])


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
def test_two_devices():
    """rings on two devices, read through the peer mapping over the named fields only"""
    import gpud_b200 as g
    ctx = g.Context([0, 1])
    try:
        rings, xs, olds, totals, thr, rng = _rings(g, ctx, 2, 8, 1 << 17, 1000, (99, 100), 0.0, 21, dev=[0, 1])
        ring_of, first, length, set_off = _sets(_route_sets(rng, 2, olds, totals))
        parent = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
        got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off, fields=[7, 2, 2])
        assert _cols(got, parent, [7, 2, 2])
        _close(rings)
    finally:
        ctx.close()
