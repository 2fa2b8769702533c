"""gpud_rings_reduce_range_sets (DESIGN.md §2 "Box sets") against the C oracle: sets whose ranges lie in 2 to 8 rings of one config,
with different totals (some wrapped, some not).  Every set is compared with mean_ema_ref.windows_fields on its ranges' samples
concatenated in the order given, W = their total: min / max / p99 / n_over bit for bit, mean and EMA within oracle/SPEC.md's tolerance.
Covered: short and long sets, tiles across a join of two rings, singleton sets in every ring (equal to that ring's reduce_ranges in all
six outputs, and its pivots taken from that ring's own sample ring), one-ring calls (equal to reduce_range_sets), sets cut across rings that hold
the same pushed data (equal to the uncut range bit for bit) in a call of three batches, every radix-select reason forced in a set spread
over two rings, and every refusal with nothing written and nothing the call does not own reading differently.  The same on rings of
two devices when the machine has two GPUs (skipped otherwise).  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import range_cases as RC
import test_segment_paths_model as M
import mean_ema_ref as R
from test_gpu_ring_range_sets import _bits, _push
from test_gpu_ring_ranges import OPS, _alpha, _fields, _thr
from test_gpu_segment_paths import _scratch
from test_gpu_window_paths import _check

pytestmark = pytest.mark.gpu


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


def _want(xs, olds, ring_of, first, length, set_off, thr, alpha, q):
    """the oracle on each set's concatenated samples (ring k holds xs[k] from push-order sample olds[k] on), [F][n_sets]"""
    cols = []
    for s in range(len(set_off) - 1):
        c = np.concatenate([xs[k][:, f - olds[k]:f - olds[k] + n] for k, f, n in
                            zip(ring_of[set_off[s]:set_off[s + 1]], first[set_off[s]:set_off[s + 1]], length[set_off[s]:set_off[s + 1]])], axis=1)
        cols.append(R.windows_fields(np.ascontiguousarray(c), c.shape[1], thr, alpha, q[0], q[1]))
    return {k: np.concatenate([c[k] for c in cols], axis=1) for k in cols[0]}


def _sets(sets):
    """[[(ring, first, len), ...], ...] -> ring_of, first, length, set_off"""
    ring_of = np.array([k for s in sets for k, _, _ in s], dtype=np.int32)
    first = np.array([f for s in sets for _, f, _ in s], dtype=np.int64)
    length = np.array([n for s in sets for _, _, n in s], dtype=np.int64)
    return ring_of, first, length, np.cumsum([0] + [len(s) for s in sets]).astype(np.int64)


def _mixed(g, ctx, devs, W, q, alpha):
    """rings on devs (rings[0] the home ring), random sets over all of them, checked against the oracle and reduce_ranges"""
    n_rings, F, cap = len(devs), 8, 1 << 17
    rng = np.random.default_rng([n_rings, W, q[0]])
    totals = [(3 * cap + 54321, cap - 12345, cap, 2 * cap + 1)[k % 4] + 1000 * (k // 4) for k in range(n_rings)]   # wrapped and not
    xs_all = [_fields(F, t, rng) for t in totals]
    thr = _thr(xs_all[0])
    rings = []
    for k, d in enumerate(devs):
        r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1], dev=d)
        _push(r, xs_all[k])
        rings.append(r)
    olds = [max(0, t - cap) for t in totals]
    xs = [x[:, o:] for x, o in zip(xs_all, olds)]

    def pick(k, n):
        return int(rng.integers(olds[k], totals[k] - n + 1))

    def anyring(n):
        k = int(rng.integers(0, n_rings))
        return (k, pick(k, n), n)
    sets = []
    for k in range(n_rings):                                          # singleton sets in every ring: short, one tile, the sample ring
        for n in (1, 33, 1025, 70000):
            sets.append([(k, pick(k, n), n)])
    sets.append([anyring(1) for _ in range(700)])                     # many 1-sample ranges over every ring: short
    sets.append([anyring(1) for _ in range(3000)])                    # ... and long, a join at every sample
    for cut in (1, 31, 32, 33, 500, 1023, 1024, 1025, 2047, 2049):   # a join between two rings at lane 0 / 31 / mid-row / a tile edge +-1
        a, b = (0, 1) if cut % 2 else (n_rings - 1, 0)
        sets.append([(a, pick(a, cut), cut), (b, pick(b, 3000), 3000), anyring(700)])
    for k in range(n_rings):                                          # pieces across each wrapped ring's physical end
        end = (totals[k] // cap) * cap
        if totals[k] > cap and end - 300 >= olds[k] and end + 300 <= totals[k]:
            sets.append([(k, end - 300, 600), ((k + 1) % n_rings, pick((k + 1) % n_rings, 2500), 2500)])
    sets.append([(k, olds[k], totals[k] - olds[k]) for k in range(n_rings)])   # every ring whole: the box
    sets.append([anyring(10), anyring(20), anyring(30)])              # a short set of three
    sets.append([anyring(400), anyring(400), anyring(400)])           # short pieces, long set
    order = rng.permutation(len(sets))
    sets = [sets[i] for i in order]
    ring_of, first, length, set_off = _sets(sets)
    got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
    _check(got, _want(xs, olds, ring_of, first, length, set_off, thr, _alpha(W, alpha), q))
    ms, n_radix, why = rings[0].ranges_stats()                        # the home ring reports the call
    assert ms > 0 and n_radix == sum(why.values())
    # singleton sets: their own ring's reduce_ranges, all six outputs bit for bit
    gb = _bits(got)
    for k in range(n_rings):
        idx = [i for i, s in enumerate(sets) if len(s) == 1 and s[0][0] == k]
        b = _bits(rings[k].reduce_ranges([sets[i][0][1] for i in idx], [sets[i][0][2] for i in idx]))
        for op in OPS:
            assert np.array_equal(gb[op][:, idx], b[op]), (k, op)
    for r in rings:
        r.close()


@pytest.mark.parametrize("n_rings,W,q,alpha", [(2, 1000, (0, 0), 0.0), (5, 999, (999, 1000), 0.9999), (8, 1, (1, 2), 0.0)])
def test_mixed_sets_against_oracle(env, n_rings, W, q, alpha):
    g, ctx = env
    _mixed(g, ctx, [0] * n_rings, W, q, alpha)


def test_one_ring_calls(env):
    """a call of one ring, and a call whose ranges all lie in one ring that is not the home ring, equal reduce_range_sets on that ring"""
    g, ctx = env
    F, cap = 8, 1 << 16
    rng = np.random.default_rng(4)
    rings, totals = [], [cap + 999, 3 * cap + 1, cap // 3]
    thr = np.full(F, 60.0)
    for t in totals:
        r = g.Ring(ctx, F, cap, 100, thresholds=thr)
        _push(r, _fields(F, t, rng))
        rings.append(r)
    for k, r in enumerate(rings):
        lo, hi = max(0, totals[k] - cap), totals[k]
        sets = [[(int(rng.integers(lo, hi - n + 1)), n) for n in rng.integers(1, min(5000, hi - lo), int(rng.integers(1, 5)))] for _ in range(40)]
        first = np.array([f for s in sets for f, _ in s], dtype=np.int64)
        length = np.array([n for s in sets for _, n in s], dtype=np.int64)
        set_off = np.cumsum([0] + [len(s) for s in sets]).astype(np.int64)
        want = _bits(r.reduce_range_sets(first, length, set_off))
        alone = _bits(g.rings_reduce_range_sets([r], np.zeros(len(first)), first, length, set_off))
        order = [rings[0], r] + [o for o in rings[1:] if o is not r] if k else rings   # ring k > 0 as slot 1 of a call homed on ring 0
        slot = 1 if k else 0
        mixed = _bits(g.rings_reduce_range_sets(order, np.full(len(first), slot), first, length, set_off))
        for op in OPS:
            assert np.array_equal(alone[op], want[op]), (k, op)
            assert np.array_equal(mixed[op], want[op]), (k, op)
    for r in rings:
        r.close()


def test_cuts_across_rings_and_three_batches(env):
    """two rings that hold the same pushed data: sets cut at random points into pieces that alternate between them read exactly like the
    uncut range of one ring, all six outputs bit for bit.  64 fields x 140 sets of 1 Mi samples take three batches of the long route."""
    g, ctx = env
    F, cap = 64, 1 << 20
    rng = np.random.default_rng(3)
    total = cap + 12345
    rings = [g.Ring(ctx, F, cap, 1000, thresholds=np.full(F, 60.0)) for _ in range(2)]
    for a in range(0, total, 1 << 18):
        rows = rng.normal(60.0, 3.0, (min(1 << 18, total - a), F)).astype(np.float32)
        for r in rings:
            r.push(rows)
    lo = total - cap
    sets, whole = [], []
    for i in range(140):
        a = int(rng.integers(lo, total - cap + 1)) if rng.random() < 0.2 else lo
        b = np.concatenate([[0], np.sort(rng.choice(np.arange(1, cap), 3, replace=False)), [cap]])
        sets.append([((i + j) % 2, a + int(b[j]), int(b[j + 1] - b[j])) for j in range(4)])
        whole.append((a, cap))
    ring_of, first, length, set_off = _sets(sets)
    got = _bits(g.rings_reduce_range_sets(rings, ring_of, first, length, set_off))
    want = _bits(rings[0].reduce_ranges([w[0] for w in whole], [w[1] for w in whole]))
    for op in OPS:
        assert np.array_equal(got[op], want[op]), op
    # wrapped, pieces across the physical end and joins of the two rings at a tile edge +-1
    rows = rng.normal(60.0, 3.0, (cap // 2 + 777, F)).astype(np.float32)
    for r in rings:
        r.push(rows)
    total += cap // 2 + 777
    a = (total // cap) * cap - 5000
    sets = [[(1, a, 1023), (0, a + 1023, 2), (1, a + 1025, 50000)], [(0, a, 4000), (1, a + 4000, 2000), (0, a + 6000, 1)],
            [(1, a + 1, 1024), (0, a + 1025, 70000)]]
    ring_of, first, length, set_off = _sets(sets)
    got = _bits(g.rings_reduce_range_sets(rings, ring_of, first, length, set_off))
    want = _bits(rings[0].reduce_ranges([s[0][1] for s in sets], [sum(n for _, _, n in s) for s in sets]))
    for op in OPS:
        assert np.array_equal(got[op], want[op]), op
    for r in rings:
        r.close()


@pytest.mark.parametrize("cap,n", [(1 << 20, 1 << 20), (1 << 18, 200001)])
def test_radix_reasons_across_rings(env, cap, n):
    """one set per field generator of tests/range_cases.py, its data built against the set's strided pivot sample over the concatenation
    and its pieces spread over two rings of different totals: exact whatever the route, with the generator's reason reported"""
    g, ctx = env
    q = (99, 100)
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
    totals = [cap + cap // 2 + 1, cap - 5]                             # ring 0 wrapped, ring 1 not
    olds = [totals[0] - cap, 0]
    cuts = [0, 1, 1057, n // 3, n // 3 + 1024, n - 31, n]
    pieces, cur = [], list(totals)
    for j, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        kr = j % 2
        cur[kr] -= b - a
        pieces.append((kr, cur[kr], b - a))
    assert cur[0] >= olds[0] and cur[1] >= olds[1]
    xs = [np.random.default_rng(5 + kr).normal(60.0, 3.0, (F, t)) for kr, t in enumerate(totals)]
    for f, (_, xf) in enumerate(built):
        for (kr, p, ln), a in zip(pieces, cuts[:-1]):
            xs[kr][f, p:p + ln] = xf[a:a + ln]
    thr = np.full(F, 60.0)
    rings = []
    for kr in range(2):
        r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
        _push(r, xs[kr], 1 << 18)
        rings.append(r)
    ring_of, first, length, set_off = _sets([pieces, pieces])
    got = g.rings_reduce_range_sets(rings, ring_of, first, length, set_off)
    _, n_radix, why = rings[0].ranges_stats()
    for r in rings:
        r.close()
    held = [x[:, o:] for x, o in zip(xs, olds)]
    _check(got, _want(held, olds, ring_of, first, length, set_off, thr, _alpha(1000, 0.0), q))
    expect = {}
    for route, _ in built:
        if route in M.OPEN:
            expect[route] = expect.get(route, 0) + 2
    assert why == expect and n_radix == sum(expect.values()), (why, expect)


def _state(r, span):
    c = span.counts()
    return ({k: r.read(k).view(np.uint8).copy() for k in OPS}, {k: span.read(k, c[0], c[1] - c[0]).view(np.uint8).copy() for k in OPS}, c,
            r.result_ptr("p99"), r.range_stats())


def test_refusals(env):
    """every refusal: GPUD_E_INVALID, nothing written, and every ring's reads, handles and stats (the home ring's ranges stats too)
    reading the same"""
    g, ctx = env
    F, cap, W = 3, 1 << 17, 64
    thr = np.array([1.0, 2.0, 3.0])
    totals = [150000, 70000, 140000]                                  # every reduce_range samples (>= 64 Ki held)
    rings, spans, states = [], [], []
    for t in totals:
        r = g.Ring(ctx, F, cap, W, thresholds=thr)
        span = r.windows(2)
        r.push(np.arange(3 * t, dtype=np.float64).reshape(t, 3))
        span.reduce()
        r.reduce()
        r.reduce_range(0)
        r.reduce_ranges([t - 100], [100])
        rings.append(r)
        spans.append(span)
    states = [_state(r, s) for r, s in zip(rings, spans)]
    rstats = [r.ranges_stats() for r in rings]
    others = [g.Ring(ctx, 4, cap, W), g.Ring(ctx, F, cap, 32, thresholds=thr), g.Ring(ctx, F, 2 * cap, W, thresholds=thr),
              g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=0.5), g.Ring(ctx, F, cap, W, thresholds=thr, q_num=1, q_den=2),
              g.Ring(ctx, F, cap, W, thresholds=np.array([1.0, 2.0, np.nextafter(3.0, 4.0)]))]   # n_fields, window, capacity, alpha, q, thr
    ctx2 = g.Context([0])
    foreign = g.Ring(ctx2, F, cap, W, thresholds=thr)
    for o in others + [foreign]:
        o.push(np.ones((totals[2], o.F)))                             # range 2 is valid in each: only the config or the ctx refuses
    L = rings[0]._L
    lo = [max(0, t - cap) for t in totals]
    ring_of = np.array([0, 1, 2], np.int32)
    first = np.array([lo[0], lo[1] + 10, totals[2] - 5], np.int64)
    length = np.array([100, 2000, 5], np.int64)
    so = np.array([0, 2, 3], np.int64)

    def call(rs, ro, f, n, s):
        ro, f, n, s = (np.ascontiguousarray(a, dt) for a, dt in ((ro, np.int32), (f, np.int64), (n, np.int64), (s, np.int64)))
        ns = len(s) - 1
        out, nov = np.full((5, F, max(ns, 1)), 7.0), np.full((F, max(ns, 1)), 7, np.uint32)
        hs = (C.c_void_p * len(rs))(*[r._h.value if r is not None else None for r in rs])
        rc = L.gpud_rings_reduce_range_sets(C.cast(hs, C.c_void_p), len(rs), C.c_void_p(ro.ctypes.data), C.c_void_p(f.ctypes.data),
                                            C.c_void_p(n.ctypes.data), len(f), C.c_void_p(s.ctypes.data), ns, C.c_void_p(out.ctypes.data),
                                            C.c_void_p(nov.ctypes.data))
        return rc, np.all(out == 7.0) and np.all(nov == 7)

    def last_error():
        buf = C.create_string_buffer(512)
        L.gpud_last_error(ctx._h, buf, 512)
        return buf.value.decode()

    assert call(rings, ring_of, first, length, so)[0] == 0
    rstats[0] = rings[0].ranges_stats()                               # the home ring reports the call that ran
    bad = [
        (rings, [0, 3, 2], first, length, so),                        # ring_of outside the call
        (rings, [0, -1, 2], first, length, so),
        (rings, [0, 0, 2], first, length, so),                        # [lo1 + 10, +2000) is not in ring 0 (before its oldest)
        (rings, [0, 1, 1], first, length, so),                        # [total2 - 5, +5) is past ring 1's newest sample
        (rings, ring_of, first, [100, 0, 5], so),                     # an empty range
        (rings, ring_of, first, length, [1, 2, 3]),                   # set_off[0] != 0
        (rings, ring_of, first, length, [0, 2]),                      # set_off[n_sets] != n_ranges
        (rings, ring_of, first, length, [0, 2, 2, 3]),                # an empty set
        (rings[:2] + [None], ring_of, first, length, so),             # a NULL ring
        ([], ring_of, first, length, so),                             # no ring
    ]
    for rs, ro, f, n, s in bad:
        rc, clean = call(rs, ro, f, n, s)
        assert rc == -1 and clean, (len(rs), ro, f, n, s)             # GPUD_E_INVALID, nothing written
    # the same call with ring 2 replaced by one whose every range is valid: refused for its ctx or the config field that differs alone
    twin = g.Ring(ctx, F, cap, W, thresholds=thr)
    twin.push(np.ones((totals[2], F)))
    assert call(rings[:2] + [twin], ring_of, first, length, so) == (0, False)   # it runs and writes
    rstats[0] = rings[0].ranges_stats()
    for o, what in [(foreign, "another ctx")] + list(zip(others, ("n_fields", "window", "capacity", "ema_alpha", "quantile", "thresholds"))):
        rc, clean = call(rings[:2] + [o], ring_of, first, length, so)
        assert rc == -1 and clean and what in last_error() and "ring 2" in last_error(), (what, last_error())
    reps = (1 << 32) // 2000 + 1                                      # m_s > UINT32_MAX over two rings
    rc, clean = call(rings, np.arange(reps) % 2, np.where(np.arange(reps) % 2, lo[1], lo[0]), np.full(reps, 2000), [0, reps])
    assert rc == -1 and clean
    for r, s, st, rs in zip(rings, spans, states, rstats):
        now = _state(r, s)
        for a, b in zip(now[:2], st[:2]):
            for k in OPS:
                assert np.array_equal(a[k], b[k]), k
        assert now[2:] == st[2:]
        assert r.ranges_stats() == rs
    for r in rings + others + [foreign, twin]:
        r.close()
    ctx2.close()


def test_singleton_pivots_from_its_own_ring(env):
    """a set of one long range in a ring other than the home ring takes its pivots from that ring's sample ring: the pivots, list fill
    and radix reasons of the call equal those of that ring's own reduce_ranges (the home ring holds other data, so its sample ring
    would give other pivots, while the exact answer could not tell)"""
    g, ctx = env
    L = g.lib()
    L.gpudh_ring_segment_scratch.restype = C.c_int32
    L.gpudh_ring_segment_scratch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64)]
    F, cap = 4, 1 << 17
    rng = np.random.default_rng(12)
    thr = np.full(F, 30.0)
    rings = []
    for k, (mu, t) in enumerate([(60.0, cap + 777), (20.0, 2 * cap + 5)]):
        r = g.Ring(ctx, F, cap, 1000, thresholds=thr)
        _push(r, rng.normal(mu, 3.0 + k, (F, t)))
        rings.append(r)
    t1 = rings[1].counts()[0]
    first, n = t1 - 100000, 100000                                    # 100 000 >> 4 = 6250 sample-ring slots: the sample ring's rule
    box = _bits(g.rings_reduce_range_sets(rings, [1], [first], [n], [0, 1]))
    box_scr, box_stats = _scratch(L, rings[0]), rings[0].ranges_stats()[1:]
    own = _bits(rings[1].reduce_ranges([first], [n]))
    own_scr, own_stats = _scratch(L, rings[1]), rings[1].ranges_stats()[1:]
    for op in OPS:
        assert np.array_equal(box[op], own[op]), op
    assert np.array_equal(box_scr[0], own_scr[0]) and np.array_equal(box_scr[1], own_scr[1])   # pivots and list fill
    assert box_stats == own_stats
    for r in rings:
        r.close()


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("devs", [(0, 1), (1, 0, 1, 0)])
def test_two_devices_against_oracle(devs):
    """rings on two devices, read by the home device's kernels through the peer mapping"""
    import gpud_b200 as g
    ctx = g.Context([0, 1])
    try:
        _mixed(g, ctx, list(devs), 1000, (0, 0), 0.0)
    finally:
        ctx.close()
