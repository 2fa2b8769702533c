"""Mean and EMA, route by route, against the extended-precision reference and its rounding budget (mean_ema_ref.py), on data built so
that the slips those routes can make move an output by many budgets (mean_ema_cases.py; test_mean_ema_ref_model.py checks that on
the CPU): large distinct values on both sides of every tile, piece, ring and window join and of the physical end, a mean away from
zero, and a small alpha (mean_ema_cases.ALPHA) so the EMA reaches back over the whole range.  Routes: the window reduce (full
windows, the wrap window, the partial last window; the EMA carry plain and guarded), gpud_ring_reduce_range (W = CAP and last_n),
gpud_ring_reduce_ranges (short, tiled long, and long ranges whose pivots come from the sample ring, up to 2.2 M samples), range sets
with joins at 1 / 1023 / 1024 / 1025, box sets over 2 and 8 rings, the box query over simulated ranks (EMA partials composed across
ranks), stream and hop windows with the EMA carried across calls, and ranges and box sets that reach back into the tier
(the configs[1] shape for the ranges, marks at the tier/ring boundary).  Each test records its worst error-to-budget ratio
(`worst_ratio`).  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import mean_ema_cases as MC
import mean_ema_ref as R
import ring_tier as T
from test_gpu_ring_box_dist import _lockstep
from test_gpu_ring_box_sets import _sets as _box_sets
from test_gpu_ring_hop import HRun
from test_gpu_ring_range_sets import _sets

pytestmark = pytest.mark.gpu
OPS = ("min", "max", "mean", "ema", "p99", "n_over")


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


def _check(got, want, record_property, what=""):
    for k in ("min", "max", "p99"):
        assert np.array_equal(np.asarray(got[k]).view(np.uint64), np.asarray(want[k]).view(np.uint64)), (what, k)
    worst = R.check_mean_ema(got, want, what=what)
    record_property("worst_ratio", worst)
    return worst


def _push(r, x, chunk=1 << 18):
    for a in range(0, x.shape[1], chunk):
        r.push(np.ascontiguousarray(x[:, a:a + chunk].T))


# ------------------------------------------------------------------------------------------------ the window reduce
@pytest.mark.parametrize("alpha", [MC.ALPHA, 0.5], ids=["plain_carry", "guarded_carry"])
def test_window_reduce(env, alpha, record_property):
    """W = 1000 over a ring whose oldest sample sits at column 20250: full windows (sum * inv_w), the window across the physical end
    and the partial last window of 500; alpha = 0.5 makes (1 - alpha)^(128 W) underflow, so the carry takes its guarded variant"""
    g, ctx = env
    W, cap, start, joins, ends = MC.window_layout()
    F = 3
    x = np.stack([MC.series(cap, joins, [1, f], ends) for f in range(F)])
    r = g.Ring(ctx, F, cap, W, thresholds=np.zeros(F), ema_alpha=alpha)
    try:
        r.push(np.zeros((start, F)))
        r.push(np.ascontiguousarray(x.T))
        got = r.reduce_all()
    finally:
        r.close()
    _check(got, R.windows_fields(x, W, np.zeros(F), alpha), record_property)


# ------------------------------------------------------------------------------------------------ reduce_range
@pytest.mark.parametrize("last_n", [0, 300001])
def test_reduce_range(env, last_n, record_property):
    """the whole ring (W = CAP, the sampled single pass and its finish's sum / n) and the newest 300001 samples, on a wrapped ring"""
    g, ctx = env
    cap, total, n, joins, ends = MC.range_layout(last_n)
    F = 2
    x = np.stack([MC.series(total, joins, [2, f], ends) for f in range(F)])
    r = g.Ring(ctx, F, cap, 1000, thresholds=np.zeros(F), ema_alpha=MC.ALPHA)
    try:
        _push(r, x)
        got = r.reduce_range(last_n)
    finally:
        r.close()
    _check(got, R.select(R.windows_fields(x[:, total - n:], n, np.zeros(F), MC.ALPHA), (slice(None), 0)), record_property)


# ------------------------------------------------------------------------------------------------ reduce_ranges
def test_reduce_ranges(env, record_property):
    """short ranges (one warp each) and tiled long ranges in one call, some across the physical end, and one long range of 2.2 M
    samples whose pivots come from the sample ring"""
    g, ctx = env
    cap, total, ranges, joins, ends = MC.ranges_layout()
    F = 2
    x = np.stack([MC.series(total, joins, [3, f], ends) for f in range(F)])
    r = g.Ring(ctx, F, cap, 1000, thresholds=np.zeros(F), ema_alpha=MC.ALPHA)
    try:
        _push(r, x)
        firsts, lens = [f for f, _ in ranges], [n for _, n in ranges]
        got = r.reduce_ranges(firsts, lens)
    finally:
        r.close()
    cols = [R.windows_fields(x[:, f:f + n], int(n), np.zeros(F), MC.ALPHA) for f, n in ranges]
    _check(got, {k: np.concatenate([c[k] for c in cols], axis=1) for k in cols[0]}, record_property)


# ------------------------------------------------------------------------------------------------ range sets
def test_range_sets(env, record_property):
    """a long set whose joins fall at 1, 1023, 1024 and 1025 samples and inside later tiles, and a short set with a piece across
    the physical end"""
    g, ctx = env
    cap, total, sets, joins, ends = MC.sets_layout()
    F = 2
    x = np.stack([MC.series(total, joins, [4, f], ends) for f in range(F)])
    r = g.Ring(ctx, F, cap, 1000, thresholds=np.zeros(F), ema_alpha=MC.ALPHA)
    try:
        _push(r, x)
        got = r.reduce_range_sets(*_sets(sets))
    finally:
        r.close()
    cols = [np.concatenate([x[:, a:a + n] for a, n in s], axis=1) for s in sets]
    want = R.stack([R.select(R.windows_fields(c, c.shape[1], np.zeros(F), MC.ALPHA), (slice(None), 0)) for c in cols])
    _check(got, want, record_property)


# ------------------------------------------------------------------------------------------------ box sets and the box query
def _box(g, ctx, n_rings, seed):
    cap, totals, sets, joins, ends = MC.box_layout(n_rings, seed)
    F = 2
    xs = [np.stack([MC.series(totals[k], joins[k], [5, seed, k, f], ends[k]) for f in range(F)]) for k in range(n_rings)]
    rings = [g.Ring(ctx, F, cap, 1000, thresholds=np.zeros(F), ema_alpha=MC.ALPHA) for _ in range(n_rings)]
    for r, x in zip(rings, xs):
        _push(r, x)
    cols = [np.concatenate([xs[k][:, a:a + n] for k, a, n in s], axis=1) for s in sets]
    want = R.stack([R.select(R.windows_fields(c, c.shape[1], np.zeros(F), MC.ALPHA), (slice(None), 0)) for c in cols])
    return rings, _box_sets(sets), want


@pytest.mark.parametrize("n_rings", [2, 8])
def test_box_sets(env, n_rings, record_property):
    """sets whose pieces lie in 2 or 8 rings of one process: short sets, long sets with a tile across each ring join"""
    g, ctx = env
    rings, args, want = _box(g, ctx, n_rings, n_rings)
    try:
        got = g.rings_reduce_range_sets(rings, *args)
    finally:
        for r in rings:
            r.close()
    _check(got, want, record_property)


@pytest.mark.parametrize("n_rings", [2, 4])
def test_box_query_ranks(env, n_rings, record_property):
    """the same sets through gpud_box_query, one simulated rank per ring: each rank's piece partials composed over the set in order"""
    g, ctx = env
    rings, args, want = _box(g, ctx, n_rings, 10 + n_rings)
    try:
        qs, got, _ = _lockstep(g, rings, *args)
        for q in qs:
            q.close()
    finally:
        for r in rings:
            r.close()
    _check({k: got[k].view(np.float64) if k != "n_over" else got[k] for k in OPS}, want, record_property)


# ------------------------------------------------------------------------------------------------ stream and hop windows
@pytest.mark.parametrize("span,hop", [(1, 1), (10, 10), (600, 10), (20, 4)])
def test_stream_and_hop_windows(env, span, hop, record_property):
    """handles whose windows are reduced over several calls: the EMA state carried from one call's last window to the next"""
    g, ctx = env
    W, cap, n, joins, ends = MC.stream_layout(span, hop)
    F = 2
    x = np.stack([MC.series(n, joins, [6, span, hop, f], ends) for f in range(F)])
    run = HRun(g, ctx, x, W, cap, np.zeros(F), span, hop, alpha=MC.ALPHA)
    worst = 0.0
    try:
        for step in (1, W - 1, span * W + 7, cap // 3, cap // 2, n):
            run.push(min(step, n - run.pos))
            run.reduce(check=False)
            first, nxt, _ = run.h.counts()
            if nxt > first:
                want, _ = run.want(first, nxt)
                got = {k: run.h.read(k, first, nxt - first) for k in OPS}
                worst = max(worst, _check(got, want, lambda *a: None, what=(span, hop, step)))
            if run.pos == n:
                break
    finally:
        run.close()
    record_property("worst_ratio", worst)


# ------------------------------------------------------------------------------------------------ the tier
def _tiered(g, ctx, F, cap, total):
    r = g.Ring(ctx, F, cap, 1000, thresholds=np.zeros(F), ema_alpha=MC.ALPHA)
    r.tier_open(T.max_row_bytes(F) * (total // T.ROW + 2))          # room for every block row: the tier loses nothing
    return r


def test_tier_ranges(env, record_property):
    """64 fields, CAP = 10^6 (natural field groups): the newest 2.2 M samples, most decoded from the tier, a range across the
    tier/ring boundary and one wholly in the tier"""
    g, ctx = env
    F, cap, total, ranges, joins, ends = MC.tier_layout()
    x = np.stack([MC.series(total, joins, [7, f], ends) for f in range(F)])
    r = _tiered(g, ctx, F, cap, total)
    try:
        _push(r, x, chunk=1 << 17)                                   # pushes well below CAP: the tier codes every row
        t0, _, _, lost = r.tier_counts()
        assert t0 == 0 and lost == 0
        got = r.reduce_ranges([f for f, _ in ranges], [n for _, n in ranges])
        assert r.tier_stats()[1] > 0                                  # the call decoded from the tier
    finally:
        r.close()
    cols = [R.windows_fields(x[:, f:f + n], int(n), np.zeros(F), MC.ALPHA) for f, n in ranges]
    _check(got, {k: np.concatenate([c[k] for c in cols], axis=1) for k in cols[0]}, record_property)


def test_box_tier_sets(env, record_property):
    """sets over two tiered rings whose pieces lie in each tier, across each tier/ring boundary and in each ring"""
    g, ctx = env
    cap, totals, sets, joins, ends = MC.box_tier_layout()
    F = 8
    xs = [np.stack([MC.series(totals[k], joins[k], [8, k, f], ends[k]) for f in range(F)]) for k in range(2)]
    rings = [_tiered(g, ctx, F, cap, t) for t in totals]
    try:
        for r, x in zip(rings, xs):
            _push(r, x, chunk=1 << 14)
            assert r.tier_counts()[0] == 0
        got = g.rings_reduce_range_sets(rings, *_box_sets(sets))
    finally:
        for r in rings:
            r.close()
    cols = [np.concatenate([xs[k][:, a:a + n] for k, a, n in s], axis=1) for s in sets]
    want = R.stack([R.select(R.windows_fields(c, c.shape[1], np.zeros(F), MC.ALPHA), (slice(None), 0)) for c in cols])
    _check(got, want, record_property)
