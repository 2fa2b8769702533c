"""Fields aimed at each route of the whole-range order statistic (gpud_ring_reduce_range: k_range_pivots, the RANGE pass of
k_window_reduce, k_range_finish and the radix select of gpud_b200/csrc/select.cu), and the ring shapes that reach both sample
sources.  Shared by test_range_paths_model.py (numpy model of the routes) and test_gpu_range_paths.py (the kernels against it).

A sampled range (n >= 64 Ki) takes its pivots from S sample keys: hi is the rh-th largest, lo the rl-th largest, with
rh = floor(r0 - d), rl = ceil(r0 + d), r0 = p S, d = 5 sqrt(S p (1 - p)) + 2, p = k / n for the rank k from the top; rh < 1 makes hi
+inf and rl > S makes lo -inf.  A generator knows which chronological positions the sample reads, so it can put chosen values at
chosen sample ranks and the rank k of the whole range where it wants it.  Every generator returns one chronological field of n
float64 samples, or None when its route cannot be built at this (n, S, k)."""
import math
from fractions import Fraction

import numpy as np

SAMPLED_MIN = 65536          # kSampledMin (select.cu)
LIST_CAP = 65536             # kListCap (select.cu)
SAMPLE_MAX = 8192            # GPUD_RANGE_SAMPLE_MAX (internal.h)
POS_NAN = np.array([0x7FFFFFFFFFFFFFFF], dtype=np.uint64).view(np.float64)[0]    # the largest totalOrder key
NEG_NAN = np.array([0xFFFFFFFFFFFFFFFF], dtype=np.uint64).view(np.float64)[0]    # the smallest key (0)


# ------------------------------------------------------------------------------------------------ where the sample comes from
def smp_shift(cap):
    """gpud_ring_create: the smallest s with ceil(cap / 2^s) <= 8192 sample slots"""
    s = 0
    while (cap + (1 << s) - 1) >> s > SAMPLE_MAX:
        s += 1
    return s


def range_start(cap, pushed, n):
    """physical column of the oldest sample of the newest n (gpud_ring_reduce_range)"""
    count = min(pushed, cap)
    start = (0 if pushed <= cap else pushed % cap) + (count - n)
    return start - cap if start >= cap else start


def sample_source(cap, n):
    """'ring' when k_range_pivots reads the sample ring, else 'strided' (gpud_ring_reduce_range's use_ring_sample)"""
    return "ring" if (n >> smp_shift(cap)) >= 2048 else "strided"


def sample_positions(cap, start, n):
    """(source, chronological positions in [0, n) that k_range_pivots samples).
    sample ring: slot sl mirrors column col = sl 2^s + 2^(s-1); it is used when col < cap and (col - start) mod cap < n.
    strided: S = min(8192, n / 8) reads at j stride + stride / 2, stride = n / S."""
    src = sample_source(cap, n)
    if src == "ring":
        s = smp_shift(cap)
        slots = (cap + (1 << s) - 1) >> s
        col = (np.arange(slots, dtype=np.int64) << s) + ((1 << s) >> 1)
        c = (col - start) % cap
        return src, np.sort(c[(col < cap) & (c < n)])
    S = min(SAMPLE_MAX, n // 8)
    stride = n // S
    return src, np.arange(S, dtype=np.int64) * stride + stride // 2


def fma(a, b, c):
    """a * b + c rounded once, as the device's fma.rn.f64"""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def pivot_ranks(n, k, S):
    """(rh, rl) of k_range_pivots, unclamped; d is one fma on the device (nvcc contracts 5 sqrt(.) + 2)"""
    pr = float(k) / float(n)
    r0 = pr * float(S)
    d = fma(math.sqrt(r0 * (1.0 - pr)), 5.0, 2.0)
    return math.floor(r0 - d), math.ceil(r0 + d)


def k_from_top(n, q_num, q_den):
    r = (n * q_num + q_den - 1) // q_den
    return n - max(1, min(n, r)) + 1


# ------------------------------------------------------------------------------------------------ building a field from levels
class Layout:
    """what a generator needs to place values: n, the sample positions, S, U = n - S, the rank k and the pivot ranks
    (rhc, rlc clamped into [1, S]; top: hi = +inf, bot: lo = -inf)"""

    def __init__(self, n, pos, k, rng):
        self.n, self.pos, self.k, self.rng = n, pos, k, rng
        self.S = len(pos)
        self.U = n - self.S
        self.rh, self.rl = pivot_ranks(n, k, self.S)
        self.top, self.bot = self.rh < 1, self.rl > self.S
        self.rhc, self.rlc = max(1, min(self.S, self.rh)), max(1, min(self.S, self.rl))

    def build(self, levels):
        """levels, in descending value order: (values, n_in_sample, n_elsewhere).  values is a float (a tie) or (a, b): distinct
        values spread over [a, b).  Values are shuffled within the sample positions and within the rest."""
        S, U = self.S, self.U
        cs = [lv[1] for lv in levels]
        cu = [lv[2] for lv in levels]
        if min(cs + cu) < 0 or sum(cs) != S or sum(cu) != U:
            return None
        def fill(counts):
            parts = []
            for (v, _, _), c in zip(levels, counts):
                if isinstance(v, tuple):
                    parts.append(np.sort(self.rng.uniform(v[0], v[1], c))[::-1])
                else:
                    parts.append(np.full(c, v))
            vals = np.concatenate(parts) if parts else np.empty(0)
            return self.rng.permutation(vals)
        x = np.empty(self.n)
        mask = np.zeros(self.n, dtype=bool)
        mask[self.pos] = True
        x[mask] = fill(cs)
        x[~mask] = fill(cu)
        return x


GAUGE = (50.0, 70.0)


def gen_list(L):
    """a continuous gauge: the pivots hold and the ~2 d n / S keys between them fit the list"""
    return L.build([(GAUGE, L.S, L.U)])


def _ties_hi(L, edge):
    """a tie V = 60 covers sample ranks rh..rl (lo = hi = V, all_equal; or hi = V over lo = -inf) and the range's rank k.  edge: k is
    the last copy of V (k == above + equal)."""
    if L.top:                                            # hi = +inf: rank k must be a +inf
        m = L.k if edge else L.k + 2
        return L.build([(np.inf, 0, m), (GAUGE, L.S, L.U - m)])
    a_s = L.rhc - 1
    a_u = max(0, L.k - 1 - a_s) // 2
    e_s = L.S - a_s if L.bot else L.rlc - a_s + (L.S - L.rlc) // 2
    need = L.k - a_s - a_u - e_s                         # copies of V the rest must hold for rank k to be one
    if need < 0 and edge:
        return None
    e_u = max(0, need) if edge else max(0, need) + (L.U - a_u - max(0, need)) // 2
    return L.build([((61.0, 66.0), a_s, a_u), (60.0, e_s, e_u), ((50.0, 59.0), L.S - a_s - e_s, L.U - a_u - e_u)])


def gen_hi(L):
    return _ties_hi(L, False)


def gen_hi_edge(L):
    return _ties_hi(L, True)


def _ties_lo(L, edge):
    """integer ties: hi = 61 (or +inf), lo = 60, nothing strictly between, rank k a copy of 60; lo = -inf: rank k a -inf.
    edge: k is the last copy of lo (k == above + equal hi + inside + equal lo)"""
    if L.bot:
        m = L.n - L.k + 1 if edge else L.n - L.k + 3
        return L.build([(GAUGE, L.S, L.U - m), (-np.inf, 0, m)])
    if L.top:
        a_s, h_s = 0, 0                                  # nothing may sit above the rl-th sample key
        v_s = L.rlc + (L.S - L.rlc) // 2
    else:
        a_s, h_s = L.rhc - 1, L.rlc - L.rhc
        v_s = max(1, (L.S - L.rlc + 1) // 2)
    if a_s + h_s >= L.k:
        return None
    a_u = (L.k - 1 - a_s - h_s) // 2
    need = L.k - a_s - h_s - a_u - v_s
    if need < 0 and edge:
        return None
    v_u = max(0, need) if edge else max(0, need) + (L.U - a_u - max(0, need)) // 2
    b_s, b_u = L.S - a_s - h_s - v_s, L.U - a_u - v_u
    return L.build([((62.0, 66.0), a_s, a_u), (61.0, h_s, 0), (60.0, v_s, v_u), ((50.0, 59.0), b_s, b_u)])


def gen_lo(L):
    return _ties_lo(L, False)


def gen_lo_edge(L):
    return _ties_lo(L, True)


def gen_above(L):
    """the sampled positions low, the rest high: far more keys lie above hi than the sample promised"""
    if L.top or L.k > L.U + L.rhc - 1:
        return None
    return L.build([((10.0, 11.0), 0, L.U), ((0.0, 1.0), L.S, 0)])


def gen_below(L):
    """the sampled positions high, the rest low; with lo = -inf (the minimum wanted) a few -NaN below everything"""
    if L.bot:
        m = L.n - L.k + 3
        return L.build([(GAUGE, L.S, L.U - m), (NEG_NAN, 0, m)])
    if L.k <= L.rlc:
        return None
    return L.build([((10.0, 11.0), L.S, 0), ((0.0, 1.0), 0, L.U)])


def gen_overflow(L):
    """the sample split +-1e6 between the pivot ranks, the rest in (-1, 1): everything else lies between the pivots"""
    if L.U <= LIST_CAP or L.k > L.U + L.rlc - 1:
        return None
    mid = (L.rhc + L.rlc) // 2
    return L.build([((1e6, 2e6), mid, 0), ((-1.0, 1.0), 0, L.U), ((-2e6, -1e6), L.S - mid, 0)])


def gen_nan(L):
    """one +NaN at a position the sample does not read"""
    return L.build([(POS_NAN, 0, 1), (GAUGE, L.S, L.U - 1)])


def gen_pivots(L):
    """-NaN at every sampled position with lo = -inf: the upper pivot (-NaN, key 0) lies below the lower one"""
    if not L.bot or L.top:
        return None
    return L.build([(GAUGE, 0, L.U), (NEG_NAN, L.S, 0)])


def gen_const(L):
    return L.build([(42.0, L.S, L.U)])


def _zeros(L, hi_zero, k_at):
    """signed zeros at the pivots.  hi_zero '+0': hi = +0 over lo = -0 (k_at 'pos' or 'neg'), or lo = hi = +0 ('below': rank k
    is a -0, which as a double is >= +0 but as a key lies below it).  hi_zero '-0': lo = hi = -0 with +0 only where the sample
    does not look (each +0 is flagged by the double compare and counted above on its key)."""
    if L.top or L.bot:
        return None
    a_s = L.rhc - 1
    up, un = (1.0, 2.0), (-2.0, -1.0)
    if hi_zero == "-0":
        z_s = L.rlc - a_s + (L.S - L.rlc) // 2
        p_u = max(1, (L.k - 1 - a_s) // 2)
        if a_s + p_u >= L.k:
            return None
        z_u = max(0, L.k - a_s - p_u - z_s) + (L.U - p_u - max(0, L.k - a_s - p_u - z_s)) // 2
        return L.build([(up, a_s, 0), (0.0, 0, p_u), (-0.0, z_s, z_u), (un, L.S - a_s - z_s, L.U - p_u - z_u)])
    if k_at == "below":
        p_s, z_s = L.rlc - a_s, L.S - L.rlc
        if a_s + p_s >= L.k or z_s < 1:
            return None
        z_u = max(0, L.k - a_s - p_s - z_s) + (L.U - max(0, L.k - a_s - p_s - z_s)) // 2
        return L.build([(up, a_s, 0), (0.0, p_s, 0), (-0.0, z_s, z_u), (un, 0, L.U - z_u)])
    p_s, z_s = L.rlc - 1 - a_s, max(1, (L.S - L.rlc + 1) // 2)
    if k_at == "pos":
        a_u = max(0, L.k - 1 - a_s) // 2
        p_u = max(0, L.k - a_s - a_u - p_s) + 1
    else:
        if a_s + p_s >= L.k:
            return None
        a_u, p_u = 0, 0
    need = L.k - a_s - a_u - p_s - p_u - z_s
    z_u = max(0, need) + (L.U - a_u - p_u - max(0, need)) // 2
    return L.build([(up, a_s, a_u), (0.0, p_s, p_u), (-0.0, z_s, z_u), (un, L.S - a_s - p_s - z_s, L.U - a_u - p_u - z_u)])


def gen_zero_hi(L):
    return _zeros(L, "+0", "pos")


def gen_zero_lo(L):
    return _zeros(L, "+0", "neg")


def gen_zero_below(L):
    return _zeros(L, "+0", "below")


def gen_zero_hi_neg(L):
    return _zeros(L, "-0", None)


def gen_specials(L):
    """a gauge with +-inf and -NaN of two payloads sprinkled where the sample does not look"""
    x = L.build([(GAUGE, L.S, L.U)])
    rest = np.setdiff1d(np.arange(L.n), L.pos)
    pick = L.rng.choice(rest, 12, replace=False)
    x[pick[:4]] = np.inf
    x[pick[4:8]] = -np.inf
    x[pick[8:10]] = NEG_NAN
    x[pick[10:]] = np.array([0xFFF8000000000001], dtype=np.uint64).view(np.float64)[0]
    return x


def route_specials(L):
    """four +inf answer a rank k <= 4 under hi = +inf, four -NaN the minimum"""
    return "below" if L.k > L.n - 4 else ("hi" if L.top and L.k <= 4 else "list")


# generator -> the route the model must predict for it (k_range_finish's outcome, or the reason the field stays open)
GENERATORS = [
    ("list", gen_list, "list"), ("hi", gen_hi, "hi"), ("hi_edge", gen_hi_edge, "hi"), ("lo", gen_lo, "lo"),
    ("lo_edge", gen_lo_edge, "lo"), ("above", gen_above, "above"), ("below", gen_below, "below"),
    ("overflow", gen_overflow, "overflow"), ("nan", gen_nan, "nan"), ("pivots", gen_pivots, "pivots"),
    ("const", gen_const, "const"), ("zero_hi", gen_zero_hi, "hi"), ("zero_lo", gen_zero_lo, "lo"),
    ("zero_below", gen_zero_below, "below"), ("zero_hi_neg", gen_zero_hi_neg, "hi"), ("specials", gen_specials, route_specials),
]

# ring shapes: capacity, rows pushed, last_n (0 = the whole ring)
RING_SHAPES = [
    dict(name="whole_1Mi", cap=1 << 20, pushed=1 << 20, last_n=0),                   # sample ring, S = 8192 (the bench's W = CAP call)
    dict(name="last_256Ki", cap=1 << 20, pushed=1 << 20, last_n=262144),             # sample ring, S = 2048
    dict(name="last_262143", cap=1 << 20, pushed=1 << 20, last_n=262143),            # strided, stride 31, partial pair in the last window
    dict(name="last_200001", cap=1 << 20, pushed=1 << 20, last_n=200001),            # strided, stride 24
    dict(name="last_65536", cap=1 << 20, pushed=1 << 20, last_n=65536),              # strided, stride 8, list_cap = n
    dict(name="wrap_odd", cap=1 << 18, pushed=(1 << 18) + 77777, last_n=150000),     # sample ring on a wrapped range, odd start
    dict(name="wrap_strided", cap=1 << 20, pushed=(1 << 20) + 33333, last_n=100000),  # strided on a wrapped range, odd start
    dict(name="cap_1e6", cap=1000000, pushed=1000000, last_n=0),                     # 7813 slots, the last one past cap: S = 7812
    dict(name="ring_128Ki", cap=1 << 17, pushed=1 << 17, last_n=0),                  # s = 4, S = 8192
]

QUANTILES = [(99, 100), (999, 1000), (1, 2), (1, 100), (0, 1), (1, 1)]
# on ring_128Ki this quantile puts rl exactly at S: lo is the sample's minimum, one rank short of the -inf override
RL_EQ_S = (29, 8192)


def shape_n(shape):
    return shape["last_n"] or min(shape["pushed"], shape["cap"])


def cases():
    """(shape, q_num, q_den) of every sampled ring the GPU file runs"""
    out = [(s, qn, qd) for s in RING_SHAPES for qn, qd in QUANTILES]
    out.append((next(s for s in RING_SHAPES if s["name"] == "ring_128Ki"), RL_EQ_S[0], RL_EQ_S[1]))
    return out


def ring_fields(shape, q_num, q_den, seed=0):
    """the fields of one sampled ring: [(generator name, expected route, chronological x[n])], every constructible generator"""
    n = shape_n(shape)
    start = range_start(shape["cap"], shape["pushed"], n)
    _, pos = sample_positions(shape["cap"], start, n)
    k = k_from_top(n, q_num, q_den)
    out = []
    for i, (name, fn, route) in enumerate(GENERATORS):
        L = Layout(n, pos, k, np.random.default_rng([seed, i, q_num, q_den, n]))
        x = fn(L)
        if x is not None:
            out.append((name, route(L) if callable(route) else route, x))
    return out


# ------------------------------------------------------------------------------------------------ short ranges (< 64 Ki)
def short_cases():
    """(name, cap, pushed, last_n, q_num, q_den, fields[F][n]) for the radix select that short ranges take for every field"""
    out = []
    rng = np.random.default_rng(77)

    def fields(n, kinds):
        xs = []
        for kind in kinds:
            if kind == "ties":                                # > 8192 copies of the answer: every digit is fixed in k_sel_pick
                x = rng.uniform(0.0, 1000.0, n)
                x[rng.random(n) < 0.6] = 60.0
            elif kind == "cluster":                           # > 8192 keys share the first digit, the second splits them
                x = rng.uniform(0.0, 1000.0, n)
                sel = rng.random(n) < 0.6
                x[sel] = 60.0 + rng.uniform(0.0, 2.0 ** -20, int(sel.sum()))
            elif kind == "signs":                             # both signs: no common leading bit (cp = 0)
                x = rng.normal(0.0, 5.0, n)
            elif kind == "zeros":
                x = rng.choice(np.array([-1.0, -0.0, 0.0, 1.0]), n, p=[0.1, 0.4, 0.4, 0.1])
            elif kind == "special":
                x = rng.normal(60.0, 3.0, n)
                x[rng.choice(n, 6, replace=False)] = [np.inf, -np.inf, POS_NAN, NEG_NAN, np.nan, -np.inf]
            else:                                             # gauge
                x = rng.normal(60.0, 3.0, n)
            xs.append(x)
        return np.stack(xs)

    kinds = ["ties", "cluster", "signs", "zeros", "special", "gauge"]
    for name, cap, pushed, last_n, q in [
            ("short_ties_40001", 65536, 65536, 40001, (1, 2)),              # 3 blocks per field: the last slice odd, 128-bit loads
            ("short_p99_50000", 65536, 65536, 50000, (99, 100)),
            ("short_wrap_odd", 50000, 50000 + 12345, 30000, (1, 2)),        # odd start, the range wraps: 64-bit path
            ("short_wrap_p99", 50000, 50000 + 40000, 45555, (99, 100)),     # odd start and n, wraps inside a block's slice
            ("short_8192", 20000, 20000, 8192, (1, 2)),                     # no histogram pass: collect + final only
            ("short_777_min", 4000, 4000 + 1001, 777, (0, 1)),              # n odd, the minimum
            ("short_65535_max", 65536, 65536, 65535, (1, 1))]:              # one sample short of the sampled pass
        n = last_n
        out.append((name, cap, pushed, last_n, q[0], q[1], fields(n, kinds)))
    return out
