"""gpud_ring_reduce_ranges against the C oracle.  Every range of a call is compared with mean_ema_ref.windows_fields run on that
range's own samples with W = its length and the ring's alpha: min / max / p99 / n_over bit for bit (the C oracle's), mean and EMA
within the rounding budget of their extended-precision reference.  Lengths on both sides of 1024 (the short route and the long
one), 64 Ki and the whole ring, ranges across the physical end after the ring has wrapped several times, overlapping, duplicate and unsorted ranges in one call, W = 1000 / 1 / 999 with quantiles
other than 99/100, fields of constants, signed zeros, infinities, NaN of both signs, monotone counters and ties, alpha = 0.9999 through
+inf and -inf, and every radix-select reason, forced with data built against the long route's pivots (tests/range_cases.py).
Cross-checks: gpud_ring_reduce_range, span and hop handles, gpud_ring_reduce's tumbling windows, and that none of them, nor
gpud_ring_range_stats, reads differently after the call.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import range_cases as RC
import mean_ema_ref as R
from test_gpu_window_paths import _check

pytestmark = pytest.mark.gpu

OPS = ("min", "max", "mean", "ema", "p99", "n_over")


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


def _alpha(W, alpha):
    return alpha if alpha > 0 else min(2.0 / (W + 1.0), 0.9999)


def _want(x, first0, firsts, lens, thr, alpha, q):
    """the reference on each range's own samples (x holds samples first0 ..), stacked into [F][n]"""
    cols = [R.windows_fields(x[:, f - first0:f - first0 + n], int(n), thr, alpha, q[0], q[1]) for f, n in zip(firsts, lens)]
    return {k: np.concatenate([c[k] for c in cols], axis=1) for k in cols[0]}


def _fields(F, n, rng):
    """per field, in turn: a gauge, a constant, signed zeros, a monotone counter, integer ties, a gauge with +-inf and NaN of both signs,
    +inf early then a gauge, -inf then a gauge"""
    xs = []
    for f in range(F):
        kind = f % 8
        if kind == 0:
            x = rng.normal(60.0, 3.0, n)
        elif kind == 1:
            x = np.full(n, 42.5)
        elif kind == 2:
            x = rng.choice(np.array([-0.0, 0.0, -1.0, 1.0]), n, p=[0.45, 0.45, 0.05, 0.05])
        elif kind == 3:
            x = np.cumsum(rng.integers(0, 3, n)).astype(np.float64) + 2.0 ** 53 - 2.0 ** 40   # a u64 counter as float64
        elif kind == 4:
            x = rng.integers(55, 58, n).astype(np.float64)
        elif kind == 5:
            x = rng.normal(60.0, 3.0, n)
            idx = rng.choice(n, 40, replace=False)
            x[idx[:10]] = np.inf
            x[idx[10:20]] = -np.inf
            x[idx[20:30]] = RC.NEG_NAN
            x[idx[30:35]] = RC.POS_NAN
            x[idx[35:]] = np.nan
        elif kind == 6:
            x = rng.normal(60.0, 3.0, n)
            x[rng.choice(n, n // 5000 + 1, replace=False)] = np.inf
        else:
            x = rng.normal(60.0, 3.0, n)
            x[rng.choice(n, n // 5000 + 1, replace=False)] = -np.inf
        xs.append(x)
    return np.stack(xs)


def _thr(x):
    return np.array([(np.inf, 60.0, 0.0, x[f, 0], 56.0, 61.0, -np.inf, np.nan)[f % 8] for f in range(x.shape[0])])


@pytest.mark.parametrize("W,q,alpha", [(1000, (0, 0), 0.0), (1, (1, 2), 0.0), (999, (999, 1000), 0.9999), (1000, (1, 100), 0.0)])
def test_lengths_positions_and_data(env, W, q, alpha):
    g, ctx = env
    F, cap = 8, 1 << 17
    total = 3 * cap + 54321                                          # wrapped three times, the head at an odd column
    rng = np.random.default_rng(W + q[0])
    x = _fields(F, total, rng)
    thr = _thr(x)
    r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1])
    for a in range(0, total, 100000):
        r.push(np.ascontiguousarray(x[:, a:a + 100000].T))
    lo = total - cap
    end_col = (total // cap) * cap                                   # push-order number of the sample at physical column 0
    lens, firsts = [], []
    for n in (1, 2, 31, 32, 33, 1023, 1024, 1025, 4095, 65535, 65536, 65537, cap):
        lens += [n, n]
        firsts += [int(rng.integers(lo, total - n + 1)), total - n]  # anywhere, and the newest n
        if n < cap:
            lens.append(n)
            firsts.append(end_col - n // 2 - 1)                      # across the physical end of the ring
    lens += [cap, 1, 5000, 5000, 2000]
    firsts += [lo, lo, firsts[3], firsts[3], firsts[3] + 1000]      # the oldest samples, duplicates and overlaps
    order = rng.permutation(len(lens))                               # any order
    firsts, lens = np.array(firsts)[order], np.array(lens)[order]
    got = r.reduce_ranges(firsts, lens)
    want = _want(x[:, lo:], lo, firsts, lens, thr, _alpha(W, alpha), q)
    _check(got, want)
    ms, n_radix, why = r.ranges_stats()
    assert ms > 0 and n_radix == sum(why.values())
    r.close()


def _positions(cap, start, n):
    """chronological positions of the long route's pivot sample: the sample ring when 2048 of its slots fall into the range, else
    S = clamp(n / 32, 64, 8192) strided reads (gpud_ring_segments' rule)"""
    if RC.sample_source(cap, n) == "ring":
        return RC.sample_positions(cap, start, n)[1]
    S = min(RC.SAMPLE_MAX, max(64, n // 32))
    stride = n // S
    return np.arange(S, dtype=np.int64) * stride + stride // 2


OPEN = {"above", "below", "overflow", "nan", "pivots"}


@pytest.mark.parametrize("cap,n,at", [(1 << 20, 1 << 20, 0), (1 << 20, 300001, 777777), (1 << 18, 200001, 200000)])
def test_radix_reasons(env, cap, n, at):
    """one long range per call at physical column `at` (the last case wraps), a field per generator of tests/range_cases.py built
    against this range's pivot sample: the answer is exact whatever the route, and the segments the pass cannot settle are reported
    under the generator's reason"""
    g, ctx = env
    q = (99, 100)
    pos = _positions(cap, at, n)
    k = RC.k_from_top(n, *q)
    built = []
    for i, (name, fn, route) in enumerate(RC.GENERATORS):
        L = RC.Layout(n, pos, k, np.random.default_rng([i, n]))
        xf = fn(L)
        if xf is not None:
            built.append((route(L) if callable(route) else route, xf))
    F = len(built)
    first = cap + at                                                 # sample `first` lands on column `at`, the ring has wrapped
    total = first + n
    x = np.random.default_rng(5).normal(60.0, 3.0, (F, total))
    for f, (_, xf) in enumerate(built):
        x[f, first:] = xf
    thr = np.full(F, 60.0)
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    r.push(np.ascontiguousarray(x.T))
    got = r.reduce_ranges([first, first], [n, n])                  # twice: each copy is its own segment
    want = _want(x[:, first:], first, [first, first], [n, n], thr, _alpha(1000, 0.0), q)
    _check(got, want)
    _, n_radix, why = r.ranges_stats()
    expect = {}
    for route, _ in built:
        if route in OPEN:
            expect[route] = expect.get(route, 0) + 2
    assert why == expect and n_radix == sum(expect.values()), (why, expect)
    r.close()


def test_cross_checks(env):
    g, ctx = env
    F, cap, W = 8, 1 << 17, 1000
    rng = np.random.default_rng(11)
    total = 2 * cap + 4321
    x = _fields(F, total, rng)
    thr = _thr(x)
    r = g.Ring(ctx, F, cap, W, thresholds=thr)
    span = r.windows(10)                                             # L = 10 000
    hop = r.windows(20, hop=5)                                       # L = 20 000 every 5 000
    small = r.windows(1)
    for a in range(0, total, 50000):
        r.push(np.ascontiguousarray(x[:, a:a + 50000].T))
        span.reduce(); hop.reduce(); small.reduce()
    # the newest n samples: gpud_ring_reduce_range's answer
    for n in (500, 1024, 5000, 100000, cap):
        a = r.reduce_range(n)
        b = r.reduce_ranges([total - n], [n])
        for k in ("min", "max", "p99"):
            assert np.array_equal(a[k].view(np.uint64), b[k][:, 0].view(np.uint64)), (n, k)
        assert np.array_equal(a["n_over"], b["n_over"][:, 0])
    # a handle's windows
    for h in (span, hop, small):
        first, nxt, _ = h.counts()
        first = max(first, -(-(total - cap) // h.P))                 # the history outlives the ring: the windows still in it
        ks = np.arange(first, nxt)
        assert len(ks) > 2
        b = r.reduce_ranges(ks * h.P, np.full(len(ks), h.L))
        for k in ("min", "max", "p99", "n_over"):
            assert np.array_equal(h.read(k, first, nxt - first).view(np.uint64 if k != "n_over" else np.uint32),
                                  b[k].view(np.uint64 if k != "n_over" else np.uint32)), (h.L, h.P, k)
        want = _want(x, 0, ks * h.P, np.full(len(ks), h.L), thr, _alpha(W, 0.0), (0, 0))
        R.check_mean_ema({"mean": h.read("mean", first, nxt - first)}, want, keys=("mean",), what=("handle", h.L, h.P))
        R.check_mean_ema(b, want, keys=("mean",), what=("ranges", h.L, h.P))
    # the ring's tumbling windows
    r.reduce()
    red = {k: r.read(k) for k in OPS}
    _, count, nw = r.counts()
    o = total - count
    firsts = o + np.arange(nw) * W
    lens = np.minimum(W, total - firsts)
    b = r.reduce_ranges(firsts, lens)
    for k in ("min", "max", "p99", "n_over"):
        assert np.array_equal(red[k].view(np.uint64 if k != "n_over" else np.uint32), b[k].view(np.uint64 if k != "n_over" else np.uint32)), k
    # nothing the call does not own reads differently after it
    r.reduce_range(0)
    stats0 = r.range_stats()
    hist0 = {k: span.read(k, *span.counts()[:1], span.counts()[1] - span.counts()[0]) for k in OPS}
    counts0 = [h.counts() for h in (span, hop, small)]
    ptr0 = r.result_ptr("p99")
    r.reduce_ranges([o, total - 70000, o + 3], [cap, 70000, 999])
    for k in OPS:
        assert np.array_equal(r.read(k).view(np.uint8), red[k].view(np.uint8)), k
        first, nxt, _ = span.counts()
        assert np.array_equal(span.read(k, first, nxt - first).view(np.uint8), hist0[k].view(np.uint8)), k
    assert [h.counts() for h in (span, hop, small)] == counts0
    assert r.result_ptr("p99") == ptr0
    assert r.range_stats() == stats0
    r.close()


def test_arguments(env):
    g, ctx = env
    F, cap = 3, 4096
    r = g.Ring(ctx, F, cap, 64)
    L = r._L
    with pytest.raises(g.GpudError):
        r.ranges_stats()                                             # no call yet
    with pytest.raises(g.GpudError):
        r.reduce_ranges([0], [1])                                    # an empty ring holds no range
    assert r.reduce_ranges([], [])["min"].shape == (F, 0)            # nothing to do
    x = np.arange(3 * 5000, dtype=np.float64).reshape(5000, 3)
    r.push(x)                                                        # holds samples [904, 5000)
    for f, n in ((904, 0), (903, 2), (5000, 1), (4990, 11), (-1, 1)):
        first = np.array([904, f], dtype=np.int64)
        lens = np.array([10, n], dtype=np.int64)
        out = np.full((5, F, 2), 7.0)
        nov = np.full((F, 2), 7, dtype=np.uint32)
        rc = L.gpud_ring_reduce_ranges(r._h, C.c_void_p(first.ctypes.data), C.c_void_p(lens.ctypes.data), 2, C.c_void_p(out.ctypes.data),
                                       C.c_void_p(nov.ctypes.data))
        assert rc == -1 and np.all(out == 7.0) and np.all(nov == 7), (f, n)   # GPUD_E_INVALID, nothing written
    assert L.gpud_ring_reduce_ranges(r._h, None, None, 0, None, None) == 0
    big = (1 << 24) // F + 1
    one, zero = np.ones(1, np.int64), np.zeros(1, np.int64)
    assert L.gpud_ring_reduce_ranges(r._h, C.c_void_p(zero.ctypes.data), C.c_void_p(one.ctypes.data), big, C.c_void_p(out.ctypes.data),
                                     C.c_void_p(nov.ctypes.data)) == -1   # F x n_ranges above GPUD_RANGES_MAX_SEGMENTS, checked first
    got = r.reduce_ranges([904, 4999], [4096, 1])
    assert got["max"][0, 0] == x[4999, 0] and got["min"][0, 0] == x[904, 0] and got["min"][2, 1] == x[4999, 2]
    r.close()
