"""gpud_ring_reduce_range_sets against the C oracle.  Every set of a call is compared with mean_ema_ref.windows_fields run on its
ranges' samples concatenated in the order given, with W = their total and the ring's alpha: min / max / p99 / n_over bit for bit, mean
and EMA within oracle/SPEC.md's tolerance.  Covered: singleton sets (equal to gpud_ring_reduce_ranges in all six outputs), sets of
many 1-sample ranges short and long, joins at lane 0 / 31, mid-row and at a tile edge +-1, pieces across the physical end of a wrapped
ring, overlapping and repeated ranges with more samples than CAP, permuted sets, mixed short and long sets, a call of three batches,
W = 1000 / 1 / 999 with quantiles other than 99/100, alpha = 0.9999, the data fields of the ranges test, every radix-select reason forced
in a multi-range set with data built against its pivots (tests/range_cases.py), its pivots, list fill and class counts against the
model, and every refusal with nothing written and the ring's other results and handles reading the same.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import range_cases as RC
import test_segment_paths_model as M
import mean_ema_ref as R
from test_gpu_ring_ranges import OPS, _alpha, _fields, _thr
from test_gpu_segment_paths import _check_scratch, _scratch
from test_gpu_window_paths import _check

pytestmark = pytest.mark.gpu


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


def _concat(x, oldest, first, length, set_off, s):
    return np.concatenate([x[:, f - oldest:f - oldest + n] for f, n in zip(first[set_off[s]:set_off[s + 1]], length[set_off[s]:set_off[s + 1]])],
                          axis=1)


def _want(x, oldest, first, length, set_off, thr, alpha, q):
    """the oracle on each set's concatenated samples, stacked into [F][n_sets]"""
    cols = []
    for s in range(len(set_off) - 1):
        c = _concat(x, oldest, first, length, set_off, s)
        cols.append(R.windows_fields(np.ascontiguousarray(c), c.shape[1], thr, alpha, q[0], q[1]))
    return {k: np.concatenate([c[k] for c in cols], axis=1) for k in cols[0]}


def _sets(pieces):
    """[[(first, len), ...], ...] -> first, length, set_off"""
    first = np.array([f for s in pieces for f, _ in s], dtype=np.int64)
    length = np.array([n for s in pieces for _, n in s], dtype=np.int64)
    return first, length, np.cumsum([0] + [len(s) for s in pieces]).astype(np.int64)


def _push(r, x, chunk=100000):
    for a in range(0, x.shape[1], chunk):
        r.push(np.ascontiguousarray(x[:, a:a + chunk].T))


def _bits(d):
    return {k: d[k].view(np.uint64 if k != "n_over" else np.uint32) for k in OPS}


@pytest.mark.parametrize("W,q,alpha", [(1000, (0, 0), 0.0), (1, (1, 2), 0.0), (999, (999, 1000), 0.9999), (1000, (1, 100), 0.0)])
def test_sets_against_oracle(env, W, q, alpha):
    g, ctx, _ = env
    F, cap = 8, 1 << 17
    total = 3 * cap + 54321                                          # wrapped three times, the head at an odd column
    rng = np.random.default_rng(W + q[0])
    x = _fields(F, total, rng)
    thr = _thr(x)
    r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1])
    _push(r, x)
    lo = total - cap
    end = (total // cap) * cap                                       # push-order number of the sample at physical column 0
    pick = lambda n: int(rng.integers(lo, total - n + 1))           # noqa: E731
    sets = []
    for n in (1, 33, 1024, 1025, 70000):                             # singleton sets, short and long
        sets.append([(pick(n), n)])
    sets.append([(pick(1), 1) for _ in range(700)])                  # many 1-sample ranges: short
    sets.append([(pick(1), 1) for _ in range(3000)])                 # ... and long, a join at every sample
    for cut in (1, 31, 32, 33, 500, 1023, 1024, 1025, 2047, 2049):  # a join at lane 0 / 31 / mid-row / a tile edge +-1
        sets.append([(pick(cut), cut), (pick(3000), 3000), (pick(700), 700)])
    sets.append([(end - 300, 600), (end - 2000, 2500), (lo, 10)])    # pieces across the physical end
    sets.append([(lo, cap), (lo + 5, cap - 5), (total - 100, 100)])  # overlapping and repeated: m_s > CAP
    sets.append([(pick(10), 10), (pick(20), 20), (pick(30), 30)])    # a short set of three
    sets.append([(pick(400), 400), (pick(400), 400), (pick(400), 400)])   # short pieces, long set
    order = rng.permutation(len(sets))                               # mixed short and long, any order
    sets = [sets[i] for i in order]
    first, length, set_off = _sets(sets)
    got = r.reduce_range_sets(first, length, set_off)
    _check(got, _want(x[:, lo:], lo, first, length, set_off, thr, _alpha(W, alpha), q))
    ms, n_radix, why = r.ranges_stats()
    assert ms > 0 and n_radix == sum(why.values())
    # singleton sets: gpud_ring_reduce_ranges' answer, all six outputs bit for bit
    single = [i for i, s in enumerate(sets) if len(s) == 1]
    b = r.reduce_ranges([sets[i][0][0] for i in single], [sets[i][0][1] for i in single])
    gb, bb = _bits(got), _bits(b)
    for k in OPS:
        assert np.array_equal(gb[k][:, single], bb[k]), k
    # a permuted set: min, max, p99 and n_over unchanged, the EMA (and the mean's last bits) follow the new order
    multi = [s for s in sets if len(s) > 2]
    perm = [[s[i] for i in rng.permutation(len(s))] for s in multi]
    f0, l0, o0 = _sets(multi)
    f1, l1, o1 = _sets(perm)
    a0, a1 = r.reduce_range_sets(f0, l0, o0), r.reduce_range_sets(f1, l1, o1)
    b0, b1 = _bits(a0), _bits(a1)
    for k in ("min", "max", "p99", "n_over"):
        assert np.array_equal(b0[k], b1[k]), k
    _check(a1, _want(x[:, lo:], lo, f1, l1, o1, thr, _alpha(W, alpha), q))
    r.close()


def test_contiguous_splits_and_three_batches(env):
    """sets whose ranges cut one contiguous stretch at random points (tiles cross the joins anywhere) read exactly like that stretch
    as one range: all six outputs equal gpud_ring_reduce_ranges' bit for bit.  64 fields x 140 sets of 1 Mi samples need three
    batches of the long route."""
    g, ctx, _ = env
    F, cap = 64, 1 << 20
    rng = np.random.default_rng(3)
    total = cap + 12345
    r = g.Ring(ctx, F, cap, 1000, thresholds=np.full(F, 60.0))
    for a in range(0, total, 1 << 18):
        n = min(1 << 18, total - a)
        r.push(rng.normal(60.0, 3.0, (n, F)).astype(np.float32))
    lo = total - cap
    sets, whole = [], []
    for _ in range(140):
        a = int(rng.integers(lo, total - cap + 1)) if rng.random() < 0.2 else lo
        cuts = np.sort(rng.choice(np.arange(1, cap), 3, replace=False))
        b = np.concatenate([[0], cuts, [cap]])
        sets.append([(a + int(b[i]), int(b[i + 1] - b[i])) for i in range(4)])
        whole.append((a, cap))
    first, length, set_off = _sets(sets)
    got = _bits(r.reduce_range_sets(first, length, set_off))
    want = _bits(r.reduce_ranges([w[0] for w in whole], [w[1] for w in whole]))
    for k in OPS:
        assert np.array_equal(got[k], want[k]), k
    # the same on a wrapped ring, with pieces across the physical end and joins at a tile edge +-1
    r.push(rng.normal(60.0, 3.0, (cap // 2 + 777, F)).astype(np.float32))
    total += cap // 2 + 777
    end = (total // cap) * cap
    a = end - 5000
    sets = [[(a, 1023), (a + 1023, 2), (a + 1025, 50000)], [(a, 4000), (a + 4000, 2000), (a + 6000, 1)], [(a + 1, 1024), (a + 1025, 70000)]]
    first, length, set_off = _sets(sets)
    got = _bits(r.reduce_range_sets(first, length, set_off))
    want = _bits(r.reduce_ranges([s[0][0] for s in sets], [sum(n for _, n in s) for s in sets]))
    for k in OPS:
        assert np.array_equal(got[k], want[k]), k
    r.close()


@pytest.mark.parametrize("cap,n", [(1 << 20, 1 << 20), (1 << 18, 200001)])
def test_radix_reasons(env, cap, n):
    """one set of several ranges per field generator of tests/range_cases.py, its data built against the set's strided pivot sample
    over the concatenation (S = clamp(n / 32, 64, 8192)): the answer is exact whatever the route, the segments the pass cannot settle are
    reported under the generator's reason, and the pivots, list fill and class counts are the model's"""
    g, ctx, L = env
    q = (99, 100)
    S = min(RC.SAMPLE_MAX, max(64, n // 32))
    stride = n // S
    pos = np.arange(S, dtype=np.int64) * stride + stride // 2
    k = RC.k_from_top(n, *q)
    built = []
    for i, (name, fn, route) in enumerate(RC.GENERATORS):
        Lay = RC.Layout(n, pos, k, np.random.default_rng([i, n, 7]))
        xf = fn(Lay)
        if xf is not None:
            built.append((route(Lay) if callable(route) else route, xf))
    F = len(built)
    # the set's pieces: a wrapped ring, pieces in reverse push order, one across the physical end, cuts at odd places
    total = cap + cap // 2 + 1
    oldest = total - cap
    cuts = [0, 1, 1057, n // 3, n // 3 + 1024, n - 31, n]
    pieces, cur = [], total
    for a, b in zip(cuts[:-1], cuts[1:]):
        cur -= b - a
        pieces.append((cur, b - a))
    assert cur >= oldest
    x = np.random.default_rng(5).normal(60.0, 3.0, (F, total))
    for f, (_, xf) in enumerate(built):
        for (p, ln), a in zip(pieces, cuts[:-1]):
            x[f, p:p + ln] = xf[a:a + ln]
    thr = np.full(F, 60.0)
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    _push(r, x, 1 << 18)
    first, length, set_off = _sets([pieces, pieces])                   # twice: each copy is its own segment
    got = r.reduce_range_sets(first, length, set_off)
    _, n_radix, why = r.ranges_stats()
    scr = _scratch(L, r)
    r.close()
    xs = x[:, oldest:]
    _check(got, _want(xs, oldest, first, length, set_off, thr, _alpha(1000, 0.0), q))
    expect = {}
    for route, _ in built:
        if route in M.OPEN:
            expect[route] = expect.get(route, 0) + 2
    assert why == expect and n_radix == sum(expect.values()), (why, expect)
    geo = dict(n=n, start=0, k=k, src="strided", pos=pos, lcap=M.seg_list_cap(n, S, k))
    nt = -(-n // M.TILE)
    models = {}
    for f, (_, xf) in enumerate(built):
        m = M.model_segment(xf, geo)
        for j in range(2):
            models[f * 2 + j, f * 2 * nt + j * nt] = m
    _check_scratch(scr, models, 2 * F, 2 * F * nt)


def test_arguments(env):
    g, ctx, _ = env
    F, cap = 3, 1 << 17
    r = g.Ring(ctx, F, cap, 64)
    L = r._L
    with pytest.raises(g.GpudError):
        r.reduce_range_sets([0], [1], [0, 1])                         # an empty ring holds no range
    assert r.reduce_range_sets([], [], [0])["min"].shape == (F, 0)   # nothing to do
    span = r.windows(2)
    total = 150000
    lo = total - cap
    x = np.arange(3 * total, dtype=np.float64).reshape(total, 3)
    r.push(x)                                                        # holds samples [lo, total)
    span.reduce()
    r.reduce()
    red = {k: r.read(k) for k in OPS}
    r.reduce_range(0)
    stats0 = r.range_stats()
    c0 = span.counts()
    hist0 = {k: span.read(k, c0[0], c0[1] - c0[0]) for k in OPS}
    ptr0 = r.result_ptr("p99")
    ranges0 = r.reduce_ranges([lo], [2000])
    rstats0 = r.ranges_stats()
    first = np.array([lo, lo + 100, total - 10], dtype=np.int64)
    lens = np.array([10, 20, 10], dtype=np.int64)
    bad = [
        (first, lens, [1, 2, 3]),                                    # set_off[0] != 0
        (first, lens, [0, 2]),                                       # set_off[n_sets] != n_ranges
        (first, lens, [0, 2, 2, 3]),                                 # an empty set
        (first, lens, [0, 3, 2, 3]),
        (first, np.array([10, 0, 10]), [0, 2, 3]),                   # an empty range
        (np.array([lo - 1, lo + 100, total - 10]), lens, [0, 2, 3]),   # no longer in the ring
        (first, np.array([10, 20, 11]), [0, 2, 3]),                  # past the newest sample
    ]
    for f, n, so in bad:
        so = np.array(so, dtype=np.int64)
        ns = len(so) - 1
        out = np.full((5, F, ns), 7.0)
        nov = np.full((F, ns), 7, dtype=np.uint32)
        rc = L.gpud_ring_reduce_range_sets(r._h, C.c_void_p(f.ctypes.data), C.c_void_p(n.ctypes.data), len(f), C.c_void_p(so.ctypes.data), ns,
                                           C.c_void_p(out.ctypes.data), C.c_void_p(nov.ctypes.data))
        assert rc == -1 and np.all(out == 7.0) and np.all(nov == 7), (f, n, so)   # GPUD_E_INVALID, nothing written
    # m_s > UINT32_MAX: one set of the same 100 000 samples 42 950 times
    reps = (1 << 32) // 100000 + 1
    ff, nn, so = np.full(reps, lo, np.int64), np.full(reps, 100000, np.int64), np.array([0, reps], np.int64)
    out = np.full((5, F, 1), 7.0)
    nov = np.full((F, 1), 7, dtype=np.uint32)
    assert L.gpud_ring_reduce_range_sets(r._h, C.c_void_p(ff.ctypes.data), C.c_void_p(nn.ctypes.data), reps, C.c_void_p(so.ctypes.data), 1,
                                         C.c_void_p(out.ctypes.data), C.c_void_p(nov.ctypes.data)) == -1
    assert np.all(out == 7.0) and np.all(nov == 7)
    # F x n_sets above GPUD_RANGES_MAX_SEGMENTS, n_sets = 0
    big = (1 << 24) // F + 1
    one = np.ones(1, np.int64)
    assert L.gpud_ring_reduce_range_sets(r._h, C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), 1, C.c_void_p(one.ctypes.data), big,
                                         C.c_void_p(out.ctypes.data), C.c_void_p(nov.ctypes.data)) == -1
    assert L.gpud_ring_reduce_range_sets(r._h, None, None, 0, None, 0, None, None) == 0
    # nothing the call does not own reads differently after the refusals, and after calls that ran
    assert r.ranges_stats() == rstats0
    got = r.reduce_range_sets([lo, total - 1, lo], [4096, 1, 1], [0, 2, 3])
    assert got["max"][0, 0] == x[total - 1, 0] and got["min"][0, 0] == x[lo, 0] and got["max"][2, 1] == x[lo, 2]
    assert np.array_equal(_bits(r.reduce_ranges([lo], [2000]))["p99"], _bits(ranges0)["p99"])
    for k in OPS:
        assert np.array_equal(r.read(k).view(np.uint8), red[k].view(np.uint8)), k
        assert np.array_equal(span.read(k, c0[0], c0[1] - c0[0]).view(np.uint8), hist0[k].view(np.uint8)), k
    assert span.counts() == c0
    assert r.result_ptr("p99") == ptr0
    assert r.range_stats() == stats0
    r.close()
