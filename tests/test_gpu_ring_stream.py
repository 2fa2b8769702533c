"""Stream windows of the ring against the C oracle.  The whole pushed stream is kept on the host; after each stream reduce every
window of the history is compared with mean_ema_ref.windows_fields run over the stream from the history's EMA seed (the window
the stream was opened or last restarted at) on: min / max / p99 / n_over bit for bit, mean and EMA within their rounding
budget.  Push sizes around W and CAP (and past CAP, which loses windows), the window loop's instantiations (W = 1000, 1024,
960, 999, 1, 7) with windows that wrap the physical end of the ring, the EMA carried over many calls (also at alpha = 0.9999
through an infinite sample), eviction past the history, and the ring's other reduces left exactly as they are.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import mean_ema_ref as R
from test_gpu_window_paths import _check
import window_cases as WC

pytestmark = pytest.mark.gpu

OPS = ("min", "max", "mean", "ema", "p99", "n_over")


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


def _stream(F, W, n_windows, seed):
    """[F][n_windows * W] chronological samples.  W >= 32: one window of tests/window_cases.py's kinds per stream window (wide
    kinds in every fourth field); shorter windows: ties, signed zeros, integers and, in every fourth field, infinities and NaN"""
    if W >= 32:
        shape = dict(W=W, count=n_windows * W, tail={})
        return np.stack([WC.field_content(shape, f, 99, 100, seed) for f in range(F)])
    rng = np.random.default_rng(seed)
    pool = np.array([0.0, -0.0, 1.0, -1.0, 45.3, 45.3, 100.0, WC.SUBNORMAL])
    x = np.where(rng.random((F, n_windows * W)) < 0.5, 60.0 + rng.normal(0.0, 3.0, (F, n_windows * W)),
                 pool[rng.integers(0, len(pool), (F, n_windows * W))])
    for f in range(3, F, 4):
        x[f, rng.integers(0, x.shape[1], 3)] = [np.inf, WC.POS_NAN, WC.NEG_NAN]
    return x


def _thresholds(x, rng):
    """per field a random pick: +inf, -inf, NaN, one of the field's samples (the compare is a strict >), a gauge level"""
    pick = [np.inf, -np.inf, np.nan, None, 60.0]
    thr = np.empty(x.shape[0])
    for f in range(x.shape[0]):
        v = pick[int(rng.integers(0, len(pick)))]
        thr[f] = x[f, int(rng.integers(0, x.shape[1]))] if v is None else v
    return thr


class Run:
    """a ring fed from a host stream, its stream windows checked against the oracle"""

    def __init__(self, g, ctx, x, W, cap, thr, alpha=0.0, history=0):
        self.g, self.x, self.W, self.cap, self.thr, self.alpha = g, x, W, cap, thr, alpha
        self.history = history
        self.H = history if history > 0 else -(-cap // W)
        self.r = g.Ring(ctx, x.shape[0], cap, W, thresholds=thr, ema_alpha=alpha)
        self.pos = 0
        self.seed_w = None

    def push(self, n):
        assert self.pos + n <= self.x.shape[1]
        self.r.push(np.ascontiguousarray(self.x[:, self.pos:self.pos + n].T))
        self.pos += n

    def open(self):
        self.r.stream_open(self.history)
        first, nxt, lost = self.r.stream_counts()
        assert first == nxt == -(-max(0, self.pos - self.cap) // self.W) and lost == 0
        self.seed_w = first

    def reduce(self, check=True):
        first0, next0, lost0 = self.r.stream_counts()
        n_new, n_lost = self.r.stream_reduce()
        first, nxt, lost = self.r.stream_counts()
        reducible = -(-max(0, self.pos - self.cap) // self.W)
        assert n_lost == max(0, reducible - next0) and lost == lost0 + n_lost
        assert nxt == self.pos // self.W and n_new == nxt - max(next0, reducible)
        if n_lost:
            self.seed_w = nxt - n_new                    # the history restarts, and the EMA is re-seeded, at the first reducible window
            assert first == max(self.seed_w, nxt - self.H)
        if check:
            self.check()
        return n_new, n_lost

    def check(self):
        first, nxt, _ = self.r.stream_counts()
        if nxt == first:
            return
        a = self.seed_w * self.W
        want = R.windows_fields(self.x[:, a:nxt * self.W], self.W, self.thr, self.alpha)
        want = {k: v[:, first - self.seed_w:] for k, v in want.items()}
        got = {k: self.r.stream_read(k, first, nxt - first) for k in OPS}
        _check(got, want)

    def close(self):
        self.r.close()


def _run(env, x, W, cap, thr, alpha=0.0, history=0):
    g, ctx = env
    return Run(g, ctx, x, W, cap, thr, alpha, history)


# (W, CAP): the window loop's instantiations, with a CAP that W does not divide, so stream windows wrap the physical end
SHAPES = [(1000, 8500), (1024, 8704), (960, 8160), (999, 8492), (1, 10), (7, 60)]


@pytest.mark.parametrize("W,cap", SHAPES, ids=["W%d" % s[0] for s in SHAPES])
def test_push_sizes(env, W, cap):
    """push sizes 1, W-1, W, W+1, 7W+3, CAP-W, CAP and more than CAP, a reduce after every push, then after several pushes"""
    sizes = [1, max(1, W - 1), W, W + 1, 7 * W + 3, cap - W, cap, cap + 3 * W + 1, W + 1, 2 * W]
    several = [[W - 1, 2], [7 * W + 3, cap - W], [1] * 5, [cap + W]]
    n = sum(sizes) + sum(sum(s) for s in several) + 8 * W
    x = _stream(8, W, -(-n // W), seed=W)
    run = _run(env, x, W, cap, _thresholds(x, np.random.default_rng(W)))
    try:
        run.open()
        lost = 0
        for s in sizes:
            run.push(s)
            lost += run.reduce()[1]
        for group in several:
            for s in group:
                run.push(s)
            lost += run.reduce()[1]
        assert lost > 0                                  # the pushes past CAP lost windows
        assert run.r.stream_counts()[2] == lost
    finally:
        run.close()


@pytest.mark.parametrize("alpha", [0.0, 0.9999])
def test_ema_carried_over_many_calls(env, alpha):
    """60 stream reduces of 1 .. 2W samples each: the EMA runs on from the stored state every time.  alpha = 0.9999 makes every
    decay weight of the scan 0 (the guarded carry), and field 1's +inf must keep its EMA infinite from there on"""
    W, cap = 1000, 8000
    rng = np.random.default_rng(7)
    pushes = rng.integers(1, 2 * W, 60)
    n = int(pushes.sum()) + W
    x = 60.0 + rng.normal(0.0, 3.0, (4, n))
    x[1, 5 * W + 17] = np.inf
    x[2] = np.round(x[2])                                # an integer gauge
    run = _run(env, x, W, cap, np.array([60.0, 61.0, np.nan, -np.inf]), alpha)
    try:
        run.open()
        for k, p in enumerate(pushes):
            run.push(int(p))
            run.reduce()
        assert run.seed_w == 0 and run.r.stream_counts()[1] >= 50
        first, nxt, _ = run.r.stream_counts()
        ema = run.r.stream_read("ema", first, nxt - first)
        assert np.isposinf(ema[1]).all()
    finally:
        run.close()


def test_loss_restarts_the_history(env):
    """a push of more than the ring holds since the last reduce: the complete windows that left the ring are counted as lost,
    the history is cleared and restarts at the first window still in the ring, with the EMA re-seeded there"""
    W, cap = 1000, 8000
    x = _stream(6, W, 40, seed=3)
    run = _run(env, x, W, cap, _thresholds(x, np.random.default_rng(3)))
    try:
        run.open()
        run.push(5 * W + 300)
        assert run.reduce() == (5, 0)
        run.push(cap + 2 * W + 500)                      # samples 5300 .. 15799 pushed; the ring keeps 7800 .. 15799
        n_new, n_lost = run.reduce()
        assert (n_lost, n_new) == (3, 7)                 # windows 5, 6, 7 lost; 8 .. 14 reduced
        first, nxt, lost = run.r.stream_counts()
        assert (first, nxt, lost) == (8, 15, 3) and run.seed_w == 8
        with pytest.raises(run.g.GpudError):
            run.r.stream_read("min", 4, 1)               # the old history is gone
        run.push(3 * W)
        assert run.reduce() == (3, 0)
    finally:
        run.close()


def test_eviction_reads_and_open_after_wrap(env):
    """a history of 3 windows: a catch-up over a whole ring writes only the newest 3; reads outside [first, next) fail; an open
    after the ring has wrapped starts at the first whole window; the calls' order is enforced"""
    g, ctx = env
    W, cap = 1024, 8704
    x = _stream(5, W, 40, seed=11)
    run = _run(env, x, W, cap, _thresholds(x, np.random.default_rng(11)), history=3)
    try:
        with pytest.raises(g.GpudError) as e:
            run.r.stream_reduce()
        assert e.value.code == -6
        run.push(2 * cap + 333)                          # wrapped: oldest sample 9037, first whole window 9
        run.open()
        assert run.seed_w == 9
        with pytest.raises(g.GpudError) as e:
            run.r.stream_open(3)
        assert e.value.code == -6
        run.push(100)                                    # windows 9 .. 16 complete, all still in the ring: 8 new for 3 slots
        assert run.reduce() == (8, 0)
        first, nxt, _ = run.r.stream_counts()
        assert (first, nxt) == (14, 17)
        for a, n in ((13, 1), (13, 2), (16, 2), (17, 1), (0, 3)):
            with pytest.raises(g.GpudError) as e:
                run.r.stream_read("p99", a, n)
            assert e.value.code == -1
        assert run.r.stream_read("n_over", 17, 0).shape == (5, 0)
        out = np.empty((5, 2))
        rc = run.r._L.gpud_ring_stream_read(run.r._h, 0, 14, 3, out.ctypes.data, out.nbytes)
        assert rc == -4                                  # too small a buffer
        for k in range(4):                               # eviction one window at a time: slots wrap around the 3
            run.push(W)
            assert run.reduce()[0] == 1
            assert run.r.stream_counts()[:2] == (15 + k, 18 + k)
    finally:
        run.close()


def test_other_reduces_unchanged(env):
    """interleaved with stream reduces, gpud_ring_reduce + gpud_ring_read and gpud_ring_reduce_range give bit for bit what the
    same ring gives without stream windows"""
    g, ctx = env
    W, cap = 1000, 8500
    x = _stream(8, W, 60, seed=21)
    thr = _thresholds(x, np.random.default_rng(21))
    a = _run(env, x, W, cap, thr)
    b = _run(env, x, W, cap, thr)
    try:
        a.open()
        for k, n in enumerate([W + 1, 3 * W, 7 * W + 3, cap + W, W - 1, 2 * W, 5 * W + 11]):
            a.push(n)
            b.push(n)
            a.reduce(check=(k % 2 == 0))
            ga, gb = a.r.reduce_all(), b.r.reduce_all()
            a.reduce(check=False)
            ra, rb = a.r.reduce_range(3 * W + 7), b.r.reduce_range(3 * W + 7)
            for got, want in ((ga, gb), (ra, rb)):
                for key in OPS:
                    u, v = np.asarray(got[key]), np.asarray(want[key])
                    assert u.shape == v.shape and u.tobytes() == v.tobytes(), (k, key)
        a.check()
    finally:
        a.close()
        b.close()
