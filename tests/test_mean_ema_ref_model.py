"""The mean / EMA reference and its budget (mean_ema_ref.py), on the CPU: the reference against 300-bit arithmetic; the budget never
too tight for legitimate f64 code (the C oracle's sequential sums on every window kind and on ranges up to 2.2 M samples, and numpy
emulations of the device's schemes from DESIGN.md: tile means times m folded, the lane-strided Horner with q64 = (1 - alpha)^64, the
decayed scan over window partials with pow(d_full, t + 1) and d_last, the piece composition (1 - alpha)^len); and the route tests'
data (mean_ema_cases.py) sensitive: every slip the routes could make moves an output by at least 10 budgets.  Long ranges are checked
at a sample of their joins (every 97th or 211th, and the last ones): a dropped or repeated sample moves the mean by the same amount
wherever it lies, and the marks make every join's sample far from the mean.  The guarded carry's case (alpha = 0.5) is checked for
the slips it can show: its carry decays to nothing within a window, so a late seed or a decay off by one is the plain carry's case."""
import mpmath
import numpy as np
import pytest

import mean_ema_cases as MC
import mean_ema_ref as R
import window_cases as WC
from oracle import coracle

POS_NAN, NEG_NAN = WC.POS_NAN, WC.NEG_NAN


# ------------------------------------------------------------------------------------------------ the reference against exact arithmetic
def _exact(x, W, alpha):
    """300-bit mean and EMA of every window (NaN / inf by IEEE rules, taken from the recurrence itself)"""
    mpmath.mp.prec = 300
    a, b = mpmath.mpf(alpha), mpmath.mpf(1.0 - alpha)
    n = x.size
    means, emas = [], []
    e = mpmath.mpf(x[0])
    for t in range(n):
        e = a * mpmath.mpf(x[t]) + b * e
        if t % W == W - 1 or t == n - 1:
            w = x[t - t % W:t + 1]
            s = mpmath.fsum([mpmath.mpf(v) for v in w])
            means.append(s / len(w))
            emas.append(e)
    return means, emas


def _close(ref, exact, rel=2.0 ** -53 + 2.0 ** -60):
    """the f64 reference is the exact value rounded to nearest (u = 2^-53 relative), up to the long double's own 2^-60"""
    if mpmath.isnan(exact):
        return np.isnan(ref)
    if mpmath.isinf(exact):
        return ref == float(exact)
    return abs(mpmath.mpf(float(ref)) - exact) <= rel * abs(exact) + mpmath.mpf(2) ** -1074


SMALL = [
    ("one sample", np.array([3.25]), 1, 0.0),
    ("seed only windows", np.array([5.0, -7.0, 11.0]), 1, 0.3),
    ("alpha 0.9999", 60.0 + np.random.default_rng(1).normal(0, 3, 300), 7, 0.9999),
    ("alpha of W = 2^20", 60.0 + np.random.default_rng(2).normal(0, 3, 3000), 1000, 2.0 / (2 ** 20 + 1.0)),
    ("signed zeros", np.array([0.0, -0.0, -0.0, 0.0, -0.0]), 2, 0.5),
    ("subnormals", np.array([5e-324, -5e-324, 2.2e-308, 1e-310, -1e-320, 5e-324]), 3, 0.01),
    ("+inf", np.array([1.0, 2.0, np.inf, 3.0, 4.0]), 2, 0.1),
    ("-inf first", np.array([-np.inf, 2.0, 3.0, 4.0]), 3, 0.1),
    ("+inf then -inf", np.array([1.0, np.inf, 2.0, -np.inf, 5.0, 6.0]), 2, 0.2),
    ("+NaN", np.array([1.0, 2.0, POS_NAN, 3.0]), 2, 0.1),
    ("-NaN", np.array([NEG_NAN, 2.0, 3.0]), 1, 0.1),
    ("offset 1e12", 1e12 + np.random.default_rng(3).normal(0, 1, 2000), 500, 0.001),
    ("zero mean +-1e6", np.random.default_rng(4).choice([-1e6, 1e6], 2000) + np.random.default_rng(5).normal(0, 1, 2000), 400, 0.01),
]


@pytest.mark.parametrize("name,x,W,alpha", SMALL, ids=[s[0] for s in SMALL])
def test_reference_against_300_bits(name, x, W, alpha):
    want = R.windows_fields(x[None, :], W, np.zeros(1), alpha)
    means, emas = _exact(x, W, R.ema_alpha(W, alpha))
    for w, (m, e) in enumerate(zip(means, emas)):
        assert _close(want["mean"][0, w], m), (name, "mean", w, want["mean"][0, w], m)
        assert _close(want["ema"][0, w], e), (name, "ema", w, want["ema"][0, w], e)
    assert not R.exempt_any(want)


def test_infinite_ema_follows_the_recurrence():
    """SPEC.md: an infinite EMA stays infinite however small the decay weights get, and +inf then -inf is NaN"""
    x = np.full(5000, 60.0)
    x[10] = np.inf
    y = x.copy()
    y[4000] = -np.inf
    want = R.windows_fields(np.stack([x, y]), 100, np.zeros(2), 0.5)
    assert np.isposinf(want["ema"][0, 1:]).all() and np.isposinf(want["ema"][1, 1:40]).all() and np.isnan(want["ema"][1, 40:]).all()


def test_exemptions_are_named_cases_only():
    """the mask covers a mean whose positive samples sum past DBL_MAX and the EMA from a window with two samples above DBL_MAX / 8"""
    x = np.full((3, 3000), 60.0)
    x[0, 10] = x[0, 20] = WC.DBL_MAX                              # window 0's mean overflows an f64 sum
    x[1, 1500] = x[1, 1600] = WC.DBL_MAX / 4                        # window 1 holds two samples above DBL_MAX / 8
    x[2, 100] = WC.DBL_MAX                                          # one such sample: neither
    want = R.windows_fields(x, 1000, np.zeros(3))
    assert want["mean_exempt"].tolist() == [[True, False, False], [False, False, False], [False, False, False]]
    assert want["ema_exempt"].tolist() == [[True, True, True], [False, True, True], [False, False, False]]
    # there the former rule holds against the f64 oracle: its overflowed mean of window 0 (+inf) passes, a finite answer does not
    f64 = coracle.windows_fields(x, 1000, np.zeros(3))
    assert np.isposinf(f64["mean"][0, 0]) and np.isposinf(want["mean"][0, 0])
    R.check_mean_ema(f64, want)
    bad = {k: v.copy() for k, v in f64.items()}
    bad["mean"][0, 0] = WC.DBL_MAX / 500
    with pytest.raises(AssertionError):
        R.check_mean_ema(bad, want)


# ------------------------------------------------------------------------------------------------ the budget holds for legitimate f64 code
def test_oracle_within_budget_on_every_window_kind():
    """the C oracle's sequential f64 sums on every window_cases kind, after a gauge prefix; only the DBL_MAX, infinity and NaN kinds
    may carry exempt outputs"""
    worst = 0.0
    for i, kind in enumerate(WC.KINDS):
        x = np.concatenate([60.0 + np.random.default_rng(i).normal(0, 3, 3000)] + [WC.window(kind, 1000, 11, s) for s in range(20)])[None]
        want = R.windows_fields(x, 1000, np.zeros(1))
        worst = max(worst, R.check_mean_ema(coracle.windows_fields(x, 1000, np.zeros(1)), want, what=kind))
        if R.exempt_any(want):
            assert kind in ("ext_dbl_max", "ext_inf", "ext_pos_nan", "ext_neg_nan", "ext_all_neg_nan"), kind
    assert worst < 0.7, worst


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 65537, 300001, 2_200_000])
def test_oracle_within_budget_on_long_ranges(n):
    """one window of the whole range at the ring's alpha, and at alpha = 1e-6 (the EMA reaches back over the whole range)"""
    rng = np.random.default_rng(n)
    x = np.stack([60.0 + rng.normal(0, 3, n), rng.normal(0, 1e6, n), 1e12 + rng.normal(0, 1, n)])
    for alpha in (2.0 / 1001.0, 1e-6):
        want = R.windows_fields(x, n, np.zeros(3), alpha)
        r = R.check_mean_ema(coracle.windows_fields(x, n, np.zeros(3), alpha), want, what=(n, alpha))
        assert r < 0.5, (n, alpha, r)


# f64 emulations of the device schemes (DESIGN.md): numpy has no fma, so each fma is a multiply and an add - one rounding more than
# the device, which only makes the emulation's error larger.
def _tile_mean(x, tile=MC.TILE):
    """tile sums, tile means S_t / m_t, folded back as mean_t * m_t in tile order, divided by n (select.cu, box_query.cu)"""
    n = x.size
    s = 0.0
    for a in range(0, n, tile):
        w = x[a:a + tile]
        s += float(np.sum(w)) / w.size * w.size
    return s / n


def _pw(alpha):
    return {e: (1.0 - alpha) ** e for e in range(-63, 64)}


def _horner_partial(w, alpha, q64):
    """the window kernel's EMA partial of one window of m <= 1024 samples: lane l runs es = es * q64 + x over its samples
    t = 64 j + 2 l + h, then weighs the last pair with pw[m - 1 - 64 (J - 1) - 2 l - h], the lanes are summed as a tree, times alpha"""
    m = w.size
    J = (m + 63) // 64
    pw = _pw(alpha)
    lanes = np.zeros(32)
    for lane in range(32):
        es = [0.0, 0.0]
        for j in range(J):
            for h in (0, 1):
                t = 64 * j + 2 * lane + h
                es[h] = es[h] * q64 + (w[t] if t < m else 0.0)
        eb = m - 1 - 64 * (J - 1) - 2 * lane
        lanes[lane] = es[0] * pw[eb] + es[1] * pw[eb - 1]
    while lanes.size > 1:
        lanes = lanes[:lanes.size // 2] + lanes[lanes.size // 2:]
    return float(lanes[0]) * alpha


def _decayed_scan(P, d_full, d_last, seed):
    """k_ema_carry: rows of 128 partials, an inclusive decayed Kogge-Stone scan inside each warp of 32 (weights d^(2^i) by squaring),
    the preceding warps' totals carried with d^32 and applied with d^(lane + 1), the row's incoming carry with pow(d, t + 1); the last
    window folded in with d_last"""
    n = len(P) - 1
    dp = [d_full]
    for i in range(1, 6):
        dp.append(dp[-1] * dp[-1])
    out = np.empty(n + 1)
    carry = seed
    for row in range(0, n, 128):
        s = np.array([P[row + t] if row + t < n else 0.0 for t in range(128)])
        for i in range(5):
            sh = np.concatenate([np.zeros(1 << i), s[:-(1 << i)]])
            lane = np.arange(128) % 32
            s = np.where(lane >= (1 << i), dp[i] * sh + s, s)
        warp_tot = [s[32 * v + 31] for v in range(4)]
        for t in range(128):
            wid, lane = t // 32, t % 32
            pre = 0.0
            for v in range(wid):
                pre = dp[5] * pre + warp_tot[v]
            e = d_full ** (lane + 1) * pre + s[t]
            e = d_full ** (t + 1) * carry + e
            if row + t < n:
                out[row + t] = e
        carry = out[min(n, row + 128) - 1]
    out[n] = d_last * (carry if n else seed) + P[n]
    return out


def _device_ema(x, W, alpha):
    """window partials by the Horner scheme, then the carry scan: the EMA at every window's end (gpud_ring_reduce)"""
    q64 = (1.0 - alpha) ** 64
    P = [_horner_partial(x[a:a + W], alpha, q64) for a in range(0, x.size, W)]
    m_last = x.size - (len(P) - 1) * W
    return _decayed_scan(P, (1.0 - alpha) ** W, (1.0 - alpha) ** m_last, x[0])


@pytest.mark.parametrize("alpha,n", [(2.0 / 1001.0, 64500), (1e-6, 300 * 1024 + 517), (0.9999, 20000), (2.0 / (2 ** 20 + 1), 200 * 1024)])
def test_device_schemes_within_budget(alpha, n):
    """the window reduce's EMA (W = 1000) and the long ranges' (W = 1024 tiles, d_last for the last one), and the tile-mean fold"""
    rng = np.random.default_rng(n)
    for x in (60.0 + rng.normal(0, 3, n), rng.normal(0, 1e6, n), MC.series(n, range(0, n, 1024), [n], [n])):
        for W in (1000, MC.TILE):
            want = R.windows_fields(x[None], W, np.zeros(1), alpha)
            e = _device_ema(x, W, alpha)
            r = R.check_mean_ema({"ema": e[None]}, want, keys=("ema",))
            assert r < 0.5, (alpha, n, W, r)
        whole = R.windows_fields(x[None], n, np.zeros(1), alpha)
        assert R.check_mean_ema({"mean": np.array([[_tile_mean(x)]])}, whole, keys=("mean",)) < 0.5


def test_piece_composition_within_budget():
    """a set's EMA composed over its pieces in order, e = (1 - alpha)^len e + P_piece, each piece's partial itself composed over its
    tiles (k_box_summarize / k_box_fold)"""
    rng = np.random.default_rng(9)
    lens = [1, 1022, 1, 1, 50000, 1, 250000, 3000, 1025]
    c = np.concatenate([MC.series(n, [0, n], [7, i]) for i, n in enumerate(lens)])
    for alpha in (1e-6, 2.0 / 1001.0, 0.3):
        q64 = (1.0 - alpha) ** 64
        e = c[0]
        a = 0
        for n in lens:
            P = 0.0
            for t in range(0, n, MC.TILE):
                w = c[a + t:a + min(n, t + MC.TILE)]
                P = (1.0 - alpha) ** w.size * P + _horner_partial(w, alpha, q64)
            e = (1.0 - alpha) ** n * e + P
            a += n
        want = R.windows_fields(c[None], c.size, np.zeros(1), alpha)
        assert R.check_mean_ema({"ema": np.array([[e]])}, want, keys=("ema",)) < 0.5, alpha
    assert rng is not None


# ------------------------------------------------------------------------------------------------ the route tests' data is sensitive
def _sensitive(c, alpha, joins, decay_starts=(), **kw):
    moved = MC.budgets_moved(c, alpha, joins, decay_starts, **kw)
    weak = {k: v for k, v in moved.items() if not v >= 10.0}
    assert not weak, weak
    return min(moved.values())


def test_window_layout_sensitive():
    W, cap, start, joins, ends = MC.window_layout()
    x = MC.series(cap, joins, [1, 0], ends)
    for w in (0, 1, 44, 63, 64):                                    # first, a full one, the wrap window, the partial last one
        a, b = w * W, min(cap, (w + 1) * W)
        _sensitive(x[a:b], MC.ALPHA, [j - a for j in joins if a < j < b])


def test_window_layout_sensitive_guarded():
    """alpha = 0.5: the mean's slips, a sample dropped or repeated at a join, and the last two samples swapped"""
    W, cap, start, joins, ends = MC.window_layout()
    x = MC.series(cap, joins, [1, 0], ends)
    for w in (0, 44, 64):
        a, b = w * W, min(cap, (w + 1) * W)
        _sensitive(x[a:b], 0.5, [j - a for j in joins if a < j < b], seed=False)


@pytest.mark.parametrize("span,hop", [(1, 1), (10, 10), (600, 10), (20, 4)])
def test_stream_layout_sensitive(span, hop):
    """each window's mean over its own samples; its EMA over the stream from the handle's seed (sample 0)"""
    W, cap, n, joins, ends = MC.stream_layout(span, hop)
    x = MC.series(n, joins, [6, span, hop, 0], ends)
    L, P = span * W, hop * W
    last = (n - L) // P
    for k in (0, last // 2, last):
        a = k * P
        _sensitive(x[a:a + L], MC.ALPHA, [j - a for j in joins if a < j < a + L][::37], outputs=("mean",))
        _sensitive(x[:a + L], MC.ALPHA, (), outputs=("ema",))


def test_tier_layout_sensitive():
    F, cap, total, ranges, joins, ends = MC.tier_layout()
    x = MC.series(total, joins, [7, 0], ends)
    held = total - cap
    for f, n in ranges:
        rel = sorted({j - f for j in joins if f < j < f + n})
        at_boundary = [held - f] if f < held < f + n else []
        _sensitive(x[f:f + n], MC.ALPHA, rel[::211] + rel[-2:] + at_boundary, MC.tile_starts(n))


def test_box_tier_layout_sensitive():
    cap, totals, sets, joins, ends = MC.box_tier_layout()
    xs = [MC.series(totals[k], joins[k], [8, k, 0], ends[k]) for k in range(2)]
    for s in sets:
        c = np.concatenate([xs[k][a:a + n] for k, a, n in s])
        sj = MC.set_joins([n for _, _, n in s])
        inner = []                                                  # each ring's tier/ring boundary inside a piece
        for (k, a, n), off in zip(s, [0] + sj):
            if a < totals[k] - cap < a + n:
                inner.append(off + totals[k] - cap - a)
        ends_far = [a for a, e in zip([0] + sj, sj + [c.size]) if c.size - e >= 5000]
        _sensitive(c, MC.ALPHA, sj + inner, [p for p in ends_far if p > 0])


@pytest.mark.parametrize("last_n", [0, 300001])
def test_range_layout_sensitive(last_n):
    cap, total, n, joins, ends = MC.range_layout(last_n)
    x = MC.series(total, joins, [2, 0], ends)
    c = x[total - n:]
    rel = [j - (total - n) for j in joins if total - n < j < total]
    _sensitive(c, MC.ALPHA, rel[::97] + rel[-3:], MC.tile_starts(n))


def test_ranges_layout_sensitive():
    cap, total, ranges, joins, ends = MC.ranges_layout()
    x = MC.series(total, joins, [3, 0], ends)
    for f, n in ranges:
        rel = [j - f for j in joins if f < j < f + n]
        _sensitive(x[f:f + n], MC.ALPHA, rel[::211] + rel[-2:], MC.tile_starts(n))


def test_sets_layout_sensitive():
    cap, total, sets, joins, ends = MC.sets_layout()
    x = MC.series(total, joins, [4, 0], ends)
    for s in sets:
        c = np.concatenate([x[a:a + n] for a, n in s])
        sj = MC.set_joins([n for _, n in s])
        ends_far = [a for a, e in zip([0] + sj, sj + [c.size]) if c.size - e >= 5000]
        _sensitive(c, MC.ALPHA, sj, [p for p in ends_far if p > 0] + MC.tile_starts(c.size)[-1:])


@pytest.mark.parametrize("n_rings,seed", [(2, 2), (8, 8), (2, 12), (4, 14)])
def test_box_layout_sensitive(n_rings, seed):
    """the box sets' (seed = n_rings) and the box query's (seed = 10 + n_rings) layouts"""
    cap, totals, sets, joins, ends = MC.box_layout(n_rings, seed)
    xs = [MC.series(totals[k], joins[k], [5, seed, k, 0], ends[k]) for k in range(n_rings)]
    for s in sets:
        c = np.concatenate([xs[k][a:a + n] for k, a, n in s])
        sj = MC.set_joins([n for _, _, n in s])
        ends_far = [a for a, e in zip([0] + sj, sj + [c.size]) if c.size - e >= 5000]
        _sensitive(c, MC.ALPHA, sj, [p for p in ends_far if p > 0])
