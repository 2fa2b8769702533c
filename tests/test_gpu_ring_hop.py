"""Hopping stream windows (gpud_ring_windows_open_hop) against the C oracle.  The whole pushed stream is kept on the host; after each
reduce every window of the handle's history is compared with mean_ema_ref.windows_fields: min / max / p99 / n_over bit for bit
and the mean within its rounding budget from W = L run on each window's own samples, the EMA within budget from W = P run
over the stream from the handle's EMA seed on, read at the windows' ends.  Shapes with L <= 1024 (the window kernel) and L > 1024
(the segment select), P <= 1024 and P > 1024, CAP not a multiple of L or P, hop = span; pushes of 1, P - 1, P, L, CAP and more;
loss, restart and eviction; alpha = 0.9999 through +inf and -inf; the select's radix reasons through the stats; and cross-checks
against tumbling handles, gpud_ring_reduce_range, and a ring without handles.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import mean_ema_ref as R
from test_gpu_window_paths import _check
from test_gpu_ring_stream import _stream, _thresholds
import test_ring_windows_model as WM

pytestmark = pytest.mark.gpu

OPS = ("min", "max", "mean", "ema", "p99", "n_over")
AGG = ("min", "max", "mean", "p99", "n_over")


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


class HRun:
    """a ring fed from a host stream [F][n] and one hopping handle on it (or on `ring`, a ring another HRun feeds), checked
    against the oracle"""

    def __init__(self, g, ctx, x, W, cap, thr, span, hop, alpha=0.0, history=0, q=(0, 0), main=None):
        self.g, self.x, self.W, self.cap, self.thr, self.alpha, self.q = g, x, W, cap, thr, alpha, q
        self.L, self.P, self.p = span * W, hop * W, span // hop
        self.H = history if history > 0 else -(-cap // self.P)
        self.main = main
        self.r = main.r if main else g.Ring(ctx, x.shape[0], cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1])
        self._pos = 0
        self.h = self.r.windows(span, history, hop=hop)
        assert self.h.hop == hop and self.h.P == self.P
        self.seed_w = self.h.counts()[0]

    @property
    def pos(self):
        return self.main.pos if self.main else self._pos

    def push(self, n):
        assert self.main is None and self._pos + n <= self.x.shape[1]
        self.r.push(np.ascontiguousarray(self.x[:, self._pos:self._pos + n].T))
        self._pos += n

    def reduce(self, check=True):
        first0, next0, lost0 = self.h.counts()
        n_new, n_lost = self.h.reduce()
        first, nxt, lost = self.h.counts()
        reducible = -(-max(0, self.pos - self.cap) // self.P)
        complete = 0 if self.pos < self.L else (self.pos - self.L) // self.P + 1
        assert n_lost == max(0, reducible - next0) and lost == lost0 + n_lost
        assert nxt == complete and n_new == nxt - max(next0, reducible)
        if n_lost:
            self.seed_w = nxt - n_new
            assert first == max(self.seed_w, nxt - self.H)
        assert nxt - first <= self.H
        if check:
            self.check()
        return n_new, n_lost

    def want(self, first, nxt):
        alpha = self.alpha if self.alpha > 0 else min(2.0 / (self.W + 1.0), 0.9999)   # the ring's alpha
        xs = np.concatenate([self.x[:, k * self.P:k * self.P + self.L] for k in range(first, nxt)], axis=1)
        want = R.windows_fields(xs, self.L, self.thr, alpha, self.q[0], self.q[1])
        src = self.x[:, self.seed_w * self.P:(nxt - 1) * self.P + self.L]
        ema = R.windows_fields(src, self.P, self.thr, alpha, self.q[0], self.q[1])
        ends = [k - self.seed_w + self.p - 1 for k in range(first, nxt)]
        for key in ("ema", "ema_err", "ema_exempt"):
            want[key] = ema[key][:, ends]
        return want, src

    def check(self):
        first, nxt, _ = self.h.counts()
        if nxt == first:
            return
        want, src = self.want(first, nxt)
        got = {k: self.h.read(k, first, nxt - first) for k in OPS}
        _check(got, want)

    def close(self):
        self.h.close()
        if self.main is None:
            self.r.close()


# (W, CAP, span, hop, history): L <= 1024 and L > 1024, P <= 1024 (Wq = P) and P > 1024 (Wq = W g), odd W, CAP a multiple of
# neither L nor P, hop = span, histories shorter than a reduce's new windows (eviction)
SHAPES = [(1000, 20500, 10, 1, 0), (1000, 655002, 600, 10, 3), (1000, 655002, 600, 60, 2), (999, 20500, 6, 2, 0), (7, 9002, 1200, 3, 0),
          (1, 9000, 2000, 1000, 0), (1000, 20500, 10, 10, 0), (10, 2054, 60, 6, 0), (7, 3002, 100, 25, 4), (100, 4102, 10, 1, 7),
          (1000, 20500, 10, 5, 2)]


@pytest.mark.parametrize("W,cap,span,hop,history", SHAPES, ids=["W%d-cap%d-s%d-h%d-H%d" % s for s in SHAPES])
def test_push_sizes(env, W, cap, span, hop, history):
    """push sizes 1, P-1, P, L, CAP, more than CAP and a few in between, a reduce after every push, then after several pushes"""
    g, ctx = env
    L, P = W * span, W * hop
    sizes = [1, max(1, P - 1), P, L, L + 1, 2 * P + 3, cap, cap + P + 1, max(1, P - 1), L]
    several = [[P - 1, 2], [L + 3, max(1, cap - L)], [1] * 3, [cap + L]]
    n = sum(sizes) + sum(sum(s) for s in several) + 2 * L
    F = 2 if L > 100000 else 5
    x = _stream(F, W, -(-n // W), seed=W + span + hop)
    run = HRun(g, ctx, x, W, cap, _thresholds(x, np.random.default_rng(span + hop)), span, hop, history=history)
    try:
        lost = 0
        for s in sizes:
            run.push(s)
            lost += run.reduce()[1]
        for group in several:
            for s in group:
                run.push(s)
            lost += run.reduce()[1]
        assert lost > 0 and run.h.counts()[2] == lost
        ms, n_open, why = run.h.stats()
        assert ms > 0 and n_open == sum(why.values())
        if L <= 1024:
            assert (n_open, why) == (0, {})
    finally:
        run.close()


@pytest.mark.parametrize("alpha", [0.0, 0.9999])
def test_ema_over_many_calls(env, alpha):
    """40 reduces of 1 .. 3L samples on a span-10 / hop-2 handle: the EMA runs on from the stored state, sampled every P.
    alpha = 0.9999 makes the scan's weights 0 (the guarded scan); field 1's +inf keeps its EMA infinite, field 3's -inf too"""
    g, ctx = env
    W, cap, span, hop = 1000, 60000, 10, 2
    L = W * span
    rng = np.random.default_rng(23)
    pushes = rng.integers(1, 3 * L, 40)
    n = int(pushes.sum()) + L
    x = 60.0 + rng.normal(0.0, 3.0, (4, n))
    x[1, 3 * L + 17] = np.inf
    x[3, 2 * L + 5] = -np.inf
    x[2] = np.round(x[2])
    run = HRun(g, ctx, x, W, cap, np.array([60.0, 61.0, np.nan, -np.inf]), span, hop, alpha)
    try:
        for p in pushes:
            run.push(int(p))
            run.reduce()
        assert run.seed_w == 0
        first, nxt, _ = run.h.counts()
        assert nxt - first >= 5
        ema = run.h.read("ema", first, nxt - first)
        assert np.isposinf(ema[1]).all() and np.isneginf(ema[3]).all()
    finally:
        run.close()


def test_loss_and_restart(env):
    """windows lost while no reduce runs: the history restarts at the first reducible window and the EMA is re-seeded there; a
    restart with nothing to reduce re-seeds at the next reduce"""
    g, ctx = env
    W, cap, span, hop = 100, 5002, 20, 4
    L, P = W * span, W * hop
    x = _stream(4, W, 400, seed=3)
    run = HRun(g, ctx, x, W, cap, _thresholds(x, np.random.default_rng(3)), span, hop)
    try:
        run.push(2 * L)
        assert run.reduce() == ((2 * L - L) // P + 1, 0)
        run.push(2 * cap)
        n_new, n_lost = run.reduce()
        assert n_lost > 0 and n_new > 0
        run.push(cap + 1)                                  # loses windows; the newest may not be complete yet
        run.push(L // 2)
        run.reduce()
        for n in (P - 1, 1, L, P):
            run.push(n)
            run.reduce()
        assert run.h.counts()[2] > 0
    finally:
        run.close()


def test_hop_equals_span_is_tumbling(env):
    """hop = span through gpud_ring_windows_open_hop is gpud_ring_windows_open, bit for bit, on the same ring"""
    g, ctx = env
    W, cap = 999, 20500
    x = _stream(5, W, 120, seed=7)
    r = g.Ring(ctx, 5, cap, W, thresholds=_thresholds(x, np.random.default_rng(7)), ema_alpha=0.2)
    hs = [(r.windows(6, 4, hop=6), r.windows(6, 4)), (r.windows(1, 0, hop=1), r.windows(1))]
    try:
        pos = 0
        for n in (1, W, 6 * W + 5, cap + 2 * W, 7, 12 * W - 1, 30 * W):
            r.push(np.ascontiguousarray(x[:, pos:pos + n].T))
            pos += n
            for a, b in hs:
                assert a.reduce() == b.reduce() and a.counts() == b.counts()
                f, nx, _ = a.counts()
                for key in OPS:
                    assert a.read(key, f, nx - f).tobytes() == b.read(key, f, nx - f).tobytes(), key
    finally:
        for a, b in hs:
            a.close()
            b.close()
        r.close()


@pytest.mark.parametrize("W,span,hop,cap", [(1000, 10, 1, 30500), (1000, 600, 60, 655002), (10, 60, 6, 2054)])
def test_against_tumbling_and_range(env, W, span, hop, cap):
    """on one ring: window j p of a hopping handle is window j of a tumbling handle of the same span, bit for bit in min / max /
    mean / p99 / n_over; after a push that ends a window, its min / max / p99 / n_over are gpud_ring_reduce_range(L)'s"""
    g, ctx = env
    L, P, p = W * span, W * hop, span // hop
    F = 3
    x = _stream(F, W, -(-(3 * cap + 4 * L) // W), seed=span)
    thr = _thresholds(x, np.random.default_rng(span))
    r = g.Ring(ctx, F, cap, W, thresholds=thr)
    hh, ht = r.windows(span, 0, hop=hop), r.windows(span, 0)
    try:
        pos = 0
        for n in (L, P, 3 * P + 1, L - 1 - P, cap - P, P):
            r.push(np.ascontiguousarray(x[:, pos:pos + n].T))
            pos += n
            hh.reduce()
            ht.reduce()
            f, nx, _ = hh.counts()
            ft, nt, _ = ht.counts()
            for j in range(max(ft, -(-f // p)), nt):
                for key in AGG:
                    assert hh.read(key, j * p, 1).tobytes() == ht.read(key, j, 1).tobytes(), (j, key)
            if nx > f and (nx - 1) * P + L == pos:          # this push ended window nx - 1: the newest L samples
                rr = r.reduce_range(L)
                for key in ("min", "max", "p99", "n_over"):
                    assert hh.read(key, nx - 1, 1)[:, 0].tobytes() == np.asarray(rr[key]).tobytes(), key
    finally:
        hh.close()
        ht.close()
        r.close()


def test_other_reduces_unchanged(env):
    """hopping handles (L <= 1024 and L > 1024) on a ring with stream windows, interleaved with gpud_ring_stream_*, gpud_ring_reduce
    and gpud_ring_reduce_range: each gives bit for bit what a ring without the handles gives, and the handles match the oracle"""
    g, ctx = env
    W, cap = 100, 40502
    x = _stream(6, W, 2400, seed=31)
    thr = _thresholds(x, np.random.default_rng(31))
    a = HRun(g, ctx, x, W, cap, thr, 30, 3)
    side = HRun(g, ctx, x, W, cap, thr, 8, 2, main=a)
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
            side.reduce(check=(i % 2 == 1))
            assert a.r.stream_reduce() == b.stream_reduce()
            ga, gb = a.r.reduce_all(), b.reduce_all()
            ra, rb = a.r.reduce_range(3 * W + 7), b.reduce_range(3 * W + 7)
            assert b.stream_counts() == a.r.stream_counts()
            f, nx, _ = a.r.stream_counts()
            sa = {k: a.r.stream_read(k, f, nx - f) for k in OPS}
            sb = {k: b.stream_read(k, f, nx - f) for k in OPS}
            for got, want in ((ga, gb), (ra, rb), (sa, sb)):
                for key in OPS:
                    u, v = np.asarray(got[key]), np.asarray(want[key])
                    assert u.shape == v.shape and u.tobytes() == v.tobytes(), (i, key)
        a.check()
        side.check()
    finally:
        side.close()
        a.close()
        b.close()


OPEN = ("nan", "pivots", "above", "below", "overflow")


def test_segment_reasons(env):
    """the segments of tests/test_ring_windows_model.py's routes, one window each, on a span-20 / hop-10 handle: the windows j p are
    the built segments, so the reduce's stats (summed over its phases) reach every reason the model sends a segment to the radix
    select for, at least as often; every window, the ones between the built segments too, is exact"""
    g, ctx = env
    W, span, hop, cap = 1000, 20, 10, 100000
    L = W * span
    q = (99, 100)
    pos = WM.seg_sample(L)
    k = WM.RC.k_from_top(L, q[0], q[1])
    cap_list = WM.seg_list_cap(L, len(pos), k)
    n_win = 4
    rng = np.random.default_rng(5)
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
    run = HRun(g, ctx, x, W, cap, np.full(x.shape[0], 55.0), span, hop, q=q)
    try:
        run.push(x.shape[1])
        n_new, _ = run.reduce()
        assert n_new == (n_win - 1) * (span // hop) + 1
        ms, n_open, why = run.h.stats()
        assert n_open == sum(why.values()) and all(why.get(r, 0) >= c for r, c in want.items()), (why, want)
        ht = run.r.windows(span)
        assert ht.reduce() == (n_win, 0)
        for j in range(n_win):
            for key in AGG:
                assert run.h.read(key, j * 2, 1).tobytes() == ht.read(key, j, 1).tobytes(), (j, key)
        ht.close()
    finally:
        run.close()


def test_bad_arguments(env):
    """hop 0, negative, above span or not dividing it, L > CAP; the default history; handles left open are freed by the ring"""
    g, ctx = env
    W, cap = 1000, 10500
    r = g.Ring(ctx, 3, cap, W)
    try:
        for span, hop in ((6, 0), (6, -2), (6, 7), (6, 4), (11, 1), (0, 0)):
            with pytest.raises(g.GpudError) as e:
                r.windows(span, hop=hop)
            assert e.value.code == -1, (span, hop)
        assert r._L.gpud_ring_windows_open_hop(r._h, 6, 3, 0, None) == -1
        h = r.windows(6, hop=2)
        assert h.hop == 2 and h.span == 6
        r.push(np.ones((cap, 3)))
        n_new, _ = h.reduce()
        assert n_new == (cap - 6 * W) // (2 * W) + 1
        assert h.counts() == (0, n_new, 0)                 # default history ceil(CAP / P) holds them all
        assert (h.read("p99", 0, n_new) == 1.0).all()
        h2 = r.windows(4, 3, hop=1)                        # left open: gpud_ring_destroy frees it
        h2.reduce()
    finally:
        r.close()
