"""Stream windows of any span (gpud_ring_windows_*) against the C oracle.  The whole pushed stream is kept on the host; after each
reduce every window of the handle's history is compared with mean_ema_ref.windows_fields with W = L = span x W, run over the
stream from the history's EMA seed on: min / max / p99 / n_over bit for bit, mean and EMA within their rounding budget.
Spans 1, 2, 10, 600 and L = CAP; W = 1000, 1024, 999, 7 and 1, so that both the window kernel (L <= 1024) and the segment select
(L > 1024) run, on odd starts too; push sizes around L and CAP with windows that wrap the physical end, loss and eviction; the EMA
over many calls (alpha = 0.9999 through +inf); segments built to hit every route of the select and every reason it hands a segment
to the radix select; several handles on one ring next to the ring's other reduces; a span-1 handle against gpud_ring_stream_*.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import mean_ema_ref as R
from test_gpu_window_paths import _check
from test_gpu_ring_stream import _stream, _thresholds
import range_cases as RC
import test_ring_windows_model as WM

pytestmark = pytest.mark.gpu

OPS = ("min", "max", "mean", "ema", "p99", "n_over")


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


class WRun:
    """a ring fed from a host stream [F][n] and one windows handle on it, checked against the oracle"""

    def __init__(self, g, ctx, x, W, cap, thr, span, alpha=0.0, history=0, q=(0, 0)):
        self.g, self.x, self.W, self.cap, self.thr, self.alpha, self.q = g, x, W, cap, thr, alpha, q
        self.L = span * W
        self.H = history if history > 0 else -(-cap // self.L)
        self.r = g.Ring(ctx, x.shape[0], cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1])
        self.pos = 0
        self.h = self.r.windows(span, history)
        assert self.h.counts() == (0, 0, 0)
        self.seed_w = 0

    def push(self, n):
        assert self.pos + n <= self.x.shape[1]
        self.r.push(np.ascontiguousarray(self.x[:, self.pos:self.pos + n].T))
        self.pos += n

    def reduce(self, check=True):
        first0, next0, lost0 = self.h.counts()
        n_new, n_lost = self.h.reduce()
        first, nxt, lost = self.h.counts()
        reducible = -(-max(0, self.pos - self.cap) // self.L)
        assert n_lost == max(0, reducible - next0) and lost == lost0 + n_lost
        assert nxt == self.pos // self.L and n_new == nxt - max(next0, reducible)
        if n_lost:
            self.seed_w = nxt - n_new
            assert first == max(self.seed_w, nxt - self.H)
        if check:
            self.check()
        return n_new, n_lost

    def check(self):
        first, nxt, _ = self.h.counts()
        if nxt == first:
            return
        a = self.seed_w * self.L
        xs = self.x[:, a:nxt * self.L]
        alpha = self.alpha if self.alpha > 0 else min(2.0 / (self.W + 1.0), 0.9999)   # the ring's alpha, not the default for W = L
        want = R.windows_fields(xs, self.L, self.thr, alpha, self.q[0], self.q[1])
        want = {k: v[:, first - self.seed_w:] for k, v in want.items()}
        got = {k: self.h.read(k, first, nxt - first) for k in OPS}
        _check(got, want)

    def close(self):
        self.h.close()
        self.r.close()


# (W, CAP, span): spans 1, 2, 10, 600 and L = CAP on the window kernel's shapes; CAP not a multiple of L so windows wrap
SHAPES = [(1000, 20500, 1), (1000, 20500, 2), (1000, 20500, 10), (1024, 20600, 10), (999, 20500, 3), (7, 9000, 600),
          (1, 9000, 600), (1, 9000, 2000), (1000, 10000, 10), (7, 8400, 1200)]


@pytest.mark.parametrize("W,cap,span", SHAPES, ids=["W%d-cap%d-span%d" % s for s in SHAPES])
def test_push_sizes(env, W, cap, span):
    """push sizes 1, L-1, L, L+1, 3L+7, CAP-L, CAP and more than CAP, a reduce after every push, then after several pushes"""
    g, ctx = env
    L = W * span
    sizes = [1, max(1, L - 1), L, L + 1, 3 * L + 7, max(1, cap - L), cap, cap + L + 1, L + 1, 2 * L]
    several = [[L - 1, 2], [L + 3, max(1, cap - L)], [1] * 3, [cap + L]]
    n = sum(sizes) + sum(sum(s) for s in several) + 4 * L
    x = _stream(6, W, -(-n // W), seed=W + span)
    run = WRun(g, ctx, x, W, cap, _thresholds(x, np.random.default_rng(span)), span)
    try:
        lost = 0
        for s in sizes:
            run.push(s)
            lost += run.reduce()[1]
        for group in several:
            for s in group:
                run.push(s)
            lost += run.reduce()[1]
        assert lost > 0
        assert run.h.counts()[2] == lost
        if L > 1024:
            ms, n_open, why = run.h.stats()
            assert ms > 0 and n_open == sum(why.values())
    finally:
        run.close()


def test_window_of_a_whole_ring(env):
    """L = CAP: a window is reducible only from the push that completes it until the next push"""
    g, ctx = env
    W, cap = 1000, 10000
    x = _stream(4, W, 80, seed=5)
    run = WRun(g, ctx, x, W, cap, _thresholds(x, np.random.default_rng(5)), 10)
    try:
        run.push(cap)
        assert run.reduce() == (1, 0)
        run.push(cap // 2)
        run.push(cap // 2)
        assert run.reduce() == (1, 0)                    # window 1 completed by the last push: still wholly in the ring
        run.push(cap)
        run.push(1)                                      # window 2 completed, then its first sample left the ring
        assert run.reduce() == (0, 1)
        assert run.h.counts() == (3, 3, 1)
        run.push(cap - 1)
        assert run.reduce() == (1, 0)
        assert run.h.counts() == (3, 4, 1)
    finally:
        run.close()


@pytest.mark.parametrize("alpha", [0.0, 0.9999])
def test_ema_carried_over_many_calls(env, alpha):
    """40 reduces of 1 .. 3L samples each on a span-10 handle: the EMA runs on from the stored state over the sub-window partials.
    alpha = 0.9999 makes the scan's weights 0 (the guarded scan), and field 1's +inf keeps its EMA infinite from there on"""
    g, ctx = env
    W, cap, span = 1000, 60000, 10
    L = W * span
    rng = np.random.default_rng(17)
    pushes = rng.integers(1, 3 * L, 40)
    n = int(pushes.sum()) + L
    x = 60.0 + rng.normal(0.0, 3.0, (4, n))
    x[1, 3 * L + 17] = np.inf
    x[2] = np.round(x[2])
    run = WRun(g, ctx, x, W, cap, np.array([60.0, 61.0, np.nan, -np.inf]), span, alpha)
    try:
        for p in pushes:
            run.push(int(p))
            run.reduce()
        assert run.seed_w == 0
        first, nxt, _ = run.h.counts()
        assert nxt - first >= 5
        ema = run.h.read("ema", first, nxt - first)
        assert np.isposinf(ema[1]).all()
    finally:
        run.close()


OPEN = ("nan", "pivots", "above", "below", "overflow")


@pytest.mark.parametrize("q", [(99, 100), (1, 100), (1, 2)], ids=["p99", "p1", "p50"])
def test_segment_routes(env, q):
    """one field per route generator of tests/range_cases.py, each of its windows built for the segment's strided sample
    (S = L / 32): the answer is exact on every route, and the segments handed to the radix select are exactly the ones the model
    of tests/test_ring_windows_model.py sends there, with their reasons (gpud_ring_windows_stats)"""
    g, ctx = env
    W, span, cap = 1000, 20, 100000
    L = W * span
    assert RC.smp_shift(cap) == 4 and (L >> 4) < 2048        # the strided source
    pos = WM.seg_sample(L)
    k = RC.k_from_top(L, q[0], q[1])
    cap_list = WM.seg_list_cap(L, len(pos), k)
    n_win = 4
    rng = np.random.default_rng(q[0] * 7 + q[1])
    rows, want = [], {}
    for name, gen, _ in WM.GENERATORS:
        segs = [WM.build_segment(name, gen, L, k, rng) for _ in range(n_win)]
        if any(sg is None for sg in segs):
            continue
        rows.append(np.concatenate(segs))
        for sg in segs:
            route = WM.seg_route(sg, pos, k, cap_list)[0]
            if route in OPEN:
                want[route] = want.get(route, 0) + 1
    assert want
    x = np.stack(rows)
    run = WRun(g, ctx, x, W, cap, np.full(x.shape[0], 55.0), span, q=q)
    try:
        run.push(x.shape[1] // 3 + 11)
        run.reduce()
        run.push(x.shape[1] - run.pos)
        run.reduce()
        assert run.h.counts()[:2] == (0, n_win)
        # a handle opened now reduces all the windows in one call: the reasons of every segment
        h2 = run.r.windows(span)
        assert h2.reduce() == (n_win, 0)
        ms, n_open, why = h2.stats()
        assert why == want and n_open == sum(want.values()), (why, want)
        for key in ("min", "max", "mean", "p99", "n_over"):              # the EMA scans ran over other call boundaries
            assert h2.read(key, 0, n_win).tobytes() == run.h.read(key, 0, n_win).tobytes(), key
        h2.close()
    finally:
        run.close()


def test_handles_and_other_reduces(env):
    """two handles (spans 2 and 10) on a ring with stream windows, interleaved with gpud_ring_stream_*, gpud_ring_reduce and
    gpud_ring_reduce_range: each of those gives bit for bit what a ring without the handles gives, and the handles match the oracle"""
    g, ctx = env
    W, cap = 1000, 40500
    x = _stream(8, W, 240, seed=31)
    thr = _thresholds(x, np.random.default_rng(31))
    a = WRun(g, ctx, x, W, cap, thr, 2)
    h10 = Side(a, 10)
    a.r.stream_open()
    b = g.Ring(ctx, x.shape[0], cap, W, thresholds=thr)
    b.stream_open()
    try:
        pos = 0
        for i, n in enumerate([W + 1, 3 * W, 12 * W + 3, cap + W, W - 1, 25 * W, 5 * W + 11, 70 * W]):
            chunk = np.ascontiguousarray(x[:, pos:pos + n].T)
            a.push(n)
            b.push(chunk)
            pos += n
            a.reduce(check=(i % 2 == 0))
            h10.reduce(check=(i % 2 == 1))
            assert a.r.stream_reduce() == b.stream_reduce()
            ga, gb = a.r.reduce_all(), b.reduce_all()
            h10.reduce(check=False)
            ra, rb = a.r.reduce_range(3 * W + 7), b.reduce_range(3 * W + 7)
            wa, wb = a.r.reduce_range(0), b.reduce_range(0)
            a.reduce(check=False)
            assert b.stream_counts() == a.r.stream_counts()
            f, nx, _ = a.r.stream_counts()
            sa = {k: a.r.stream_read(k, f, nx - f) for k in OPS}
            sb = {k: b.stream_read(k, f, nx - f) for k in OPS}
            for got, want in ((ga, gb), (ra, rb), (wa, wb), (sa, sb)):
                for key in OPS:
                    u, v = np.asarray(got[key]), np.asarray(want[key])
                    assert u.shape == v.shape and u.tobytes() == v.tobytes(), (i, key)
        a.check()
        h10.check()
        assert h10.h.counts()[2] > 0
    finally:
        h10.h.close()
        a.close()
        b.close()


class Side(WRun):
    """a second handle on a WRun's ring, following its pushes"""

    def __init__(self, main, span):
        self.main, self.g, self.x, self.W, self.cap, self.thr, self.alpha, self.q = main, main.g, main.x, main.W, main.cap, main.thr, main.alpha, main.q
        self.L = span * main.W
        self.H = -(-main.cap // self.L)
        self.r = main.r
        self.h = main.r.windows(span)
        assert self.h.counts() == (0, 0, 0) and main.pos == 0
        self.seed_w = 0

    @property
    def pos(self):
        return self.main.pos


def test_span_one_is_the_stream(env):
    """a span-1 handle gives bit for bit what gpud_ring_stream_* gives on the same ring, counts and every aggregate"""
    g, ctx = env
    W, cap = 999, 8492
    x = _stream(6, W, 60, seed=41)
    r = g.Ring(ctx, 6, cap, W, thresholds=_thresholds(x, np.random.default_rng(41)), ema_alpha=0.3)
    r.stream_open(5)
    h = r.windows(1, 5)
    try:
        pos = 0
        for n in (1, W, 3 * W + 5, cap + 2 * W, 7, 2 * W - 1, 9 * W):
            r.push(np.ascontiguousarray(x[:, pos:pos + n].T))
            pos += n
            assert h.reduce() == r.stream_reduce()
            assert h.counts() == r.stream_counts()
            f, nx, _ = h.counts()
            for key in OPS:
                assert h.read(key, f, nx - f).tobytes() == r.stream_read(key, f, nx - f).tobytes(), key
            if nx > 0:
                assert h.stats()[1:] == (0, {})
    finally:
        h.close()
        r.close()


def test_bad_arguments(env):
    """span 0, L > CAP, reads outside the history, a short buffer, stats before the first reduce; the ring frees open handles"""
    g, ctx = env
    W, cap = 1000, 10500
    r = g.Ring(ctx, 3, cap, W)
    try:
        for span in (0, -1, 11):
            with pytest.raises(g.GpudError) as e:
                r.windows(span)
            assert e.value.code == -1
        h = r.windows(2, 3)
        with pytest.raises(g.GpudError) as e:
            h.stats()
        assert e.value.code == -6
        r.push(np.ones((9 * W, 3)))
        assert h.reduce() == (4, 0)
        assert h.counts() == (1, 4, 0)
        for a, n in ((0, 1), (0, 4), (3, 2), (4, 1)):
            with pytest.raises(g.GpudError) as e:
                h.read("p99", a, n)
            assert e.value.code == -1
        assert h.read("n_over", 4, 0).shape == (3, 0)
        out = np.empty((3, 2))
        assert r._L.gpud_ring_windows_read(h._h, 0, 1, 3, out.ctypes.data, out.nbytes) == -4
        assert r._L.gpud_ring_windows_open(r._h, 1, 0, None) == -1
        h.close()
        h2 = r.windows(3)                                # left open: gpud_ring_destroy frees it
        h2.reduce()
    finally:
        r.close()
