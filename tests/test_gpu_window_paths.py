"""The window reduce against the C oracle on windows built for each branch of its order-statistic cascade (window_cases.py), in
rings shaped so that every compiled copy of the window loop runs: <1,15,0>, <1,16,0>, <1,-1,0>, <0,-1,0> and the tail loop inside
the aligned kernels (the window that wraps the physical end of the ring and the trailing partial window).  The rings are large
enough for the work cursor to hand out runs of 8 windows, and the window kinds cycle along each field, so every run changes branch
from one window to the next while reusing the warp's candidate list, row list and scratch.  Also: the EMA carry with infinities
and decay weights that underflow to 0.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from oracle import pyoracle as O
import mean_ema_ref as R
from test_window_paths_model import dispatch
import window_cases as WC

pytestmark = pytest.mark.gpu

CTAS_PER_SM, WARPS_PER_CTA = 2, 8            # k_window_reduce's persistent grid (kCtasPerSM, kWarpsPerBlock in ring.cu)


@pytest.fixture(scope="module")
def env():
    import torch
    import gpud_b200 as g
    ctx = g.Context([0])
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    yield g, ctx, sm
    ctx.close()


def _persistent_warps(sm, reserve, units):
    """the warps launch_one starts: kCtasPerSM CTAs per SM less the reserve, no more than the units need"""
    return WARPS_PER_CTA * max(1, min((units + WARPS_PER_CTA - 1) // WARPS_PER_CTA, sm * CTAS_PER_SM - reserve))


def _check(got, want):
    """min / max / p99 / n_over bit for bit; mean and EMA within the budget of mean_ema_ref.py, infinities and NaN where the reference
    has them.  Returns the worst error-to-budget ratio."""
    for k in ("min", "max", "p99"):
        bad = np.argwhere(got[k].view(np.uint64) != want[k].view(np.uint64))
        assert bad.size == 0, (k, bad[:5].tolist(), got[k][tuple(bad[0])], want[k][tuple(bad[0])])
    bad = np.argwhere(got["n_over"].astype(np.uint64) != want["n_over"].astype(np.uint64))
    assert bad.size == 0, ("n_over", bad[:5].tolist())
    return R.check_mean_ema(got, want)


def _thresholds(x):
    """per field, in turn: +inf, -inf, NaN, a value that is one of the field's samples (the compare is a strict >), a gauge level"""
    F = x.shape[0]
    thr = np.empty(F)
    for f in range(F):
        thr[f] = (np.inf, -np.inf, np.nan, x[f, x.shape[1] // 2], 60.0)[f % 5]
    return thr


def _run_ring(env, shape, q_num, q_den, seed=0):
    g, ctx, sm = env
    W, cap, count, start = shape["W"], shape["cap"], shape["count"], shape["start"]
    nw = (count + W - 1) // W
    assert dispatch(start, W, count, cap) == (shape["inst"], shape["tail"]), shape["name"]
    reserve = sm - 1                                       # a small persistent grid: fewer fields give every warp several runs
    warps = _persistent_warps(sm, reserve, 1 << 30)
    F = max(4, -(-5 * warps // nw))                        # units (field x window) >= 4 x warps x 1.25
    assert F * nw >= 5 * _persistent_warps(sm, reserve, F * nw)
    x = np.stack([WC.field_content(shape, f, q_num, q_den, seed) for f in range(F)])    # [F][count], chronological
    thr = _thresholds(x)
    r = g.Ring(ctx, F, cap, W, thresholds=thr, q_num=q_num, q_den=q_den)
    try:
        r.set_cta_reserve(reserve)
        if start:                                          # a filler prefix of `start` samples puts the oldest sample at column start
            assert count == cap
            r.push(np.ascontiguousarray(np.tile(np.arange(start, dtype=np.float64)[:, None], (1, F))))
        r.push(np.ascontiguousarray(x.T))
        total = start + count
        assert r.counts() == (total, count, nw)
        got = r.reduce_all()
    finally:
        r.close()
    want = R.windows_fields(x, W, thr, 0.0, q_num, q_den)
    _check(got, want)


@pytest.mark.parametrize("shape", WC.RING_SHAPES, ids=[s["name"] for s in WC.RING_SHAPES])
@pytest.mark.parametrize("k", [11, 33])
def test_ring_shapes(env, shape, k):
    """every copy of the window loop on every window kind; k = 11 is the default p99 of W = 1000, k = 33 the first rank past the
    k <= 32 guards (the bit search)"""
    W = shape["W"]
    q_num, q_den = (W - k + 1, W) if W >= k else (0, 1)
    _run_ring(env, shape, q_num, q_den, seed=k)


SWEEP = [(1000 - k + 1, 1000, k) for k in range(1, 35)] + [(1, 2, 501), (0, 1, 1000)]     # q = (W - k + 1) / W, median, minimum


@pytest.mark.parametrize("q_num,q_den,k", SWEEP, ids=["k%d" % s[2] for s in SWEEP])
def test_quantile_sweep(env, q_num, q_den, k):
    """k = 1 .. 34, the median and the minimum (k = m) on the hot instantiation with a wrap window and a partial last window"""
    assert 1000 - O.quantile_rank(1000, q_num, q_den) + 1 == k
    shape = next(s for s in WC.RING_SHAPES if s["name"] == "w1000_tail")
    _run_ring(env, shape, q_num, q_den, seed=100 + k)


# ------------------------------------------------------------------------------------------------ EMA with infinities
def _ema_fields(W, n, rng):
    x = 60.0 + rng.normal(0.0, 3.0, (4, n))
    x[0, min(W // 2, n - 1)] = np.inf            # +inf in window 0
    x[1, 0] = np.inf                             # +inf at x[0], the carry's starting value
    x[2, int(n * 0.8)] = -np.inf                 # -inf late in the ring
    x[3, int(n * 0.1)] = np.inf                  # +inf, then -inf: NaN from there on
    x[3, int(n * 0.6)] = -np.inf
    return x


@pytest.mark.parametrize("alpha", [0.01, 0.5, 0.9, 0.9999])
@pytest.mark.parametrize("W,nw", [(1000, 260), (7, 300)])
def test_ema_carry_keeps_infinities(env, alpha, W, nw):
    """(1-alpha)^W and its powers underflow to 0 (alpha = 0.5, W = 1000: from d^2 on); an infinite EMA must stay infinite all the
    same, as in the recurrence e_t = alpha x_t + (1-alpha) e_(t-1), and +inf followed by -inf is NaN"""
    g, ctx, _ = env
    n = W * nw
    x = _ema_fields(W, n, np.random.default_rng(int(alpha * 1e4) + W))
    thr = np.full(4, 60.0)
    r = g.Ring(ctx, 4, n, W, thresholds=thr, ema_alpha=alpha)
    try:
        r.push(np.ascontiguousarray(x.T))
        got = r.reduce_all()
    finally:
        r.close()
    want = R.windows_fields(x, W, thr, alpha)
    assert np.isposinf(want["ema"][0]).all() and np.isposinf(want["ema"][1]).all() and np.isnan(want["ema"][3, -1])
    R.check_mean_ema(got, want, keys=("ema",), what=(alpha, W))


def test_range_ema_carry_keeps_infinities(env):
    """reduce_range runs the same carry over 1024-sample windows: at alpha = 0.9 every decay weight is 0"""
    g, ctx, _ = env
    F, cap, W, n = 2, 8192, 1000, 5000
    x = 60.0 + np.random.default_rng(5).normal(0.0, 3.0, (10000, F))
    x[10000 - n + 100, 0] = np.inf
    x[10000 - n + 2000, 1] = -np.inf
    thr = np.full(F, 60.0)
    r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=0.9)
    try:
        r.push(x)
        got = r.reduce_range(n)
    finally:
        r.close()
    for f, want in ((0, np.inf), (1, -np.inf)):
        assert O.window_aggregates(x[-n:, f], n, thr[f], 0.9)["ema"][0] == want
        assert got["ema"][f] == want, (f, got["ema"][f])
