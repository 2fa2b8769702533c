"""Data and perturbations for the mean / EMA route tests (test_gpu_mean_ema_routes.py on the device, test_mean_ema_ref_model.py on the
CPU).  A gauge near 1 (so mean / (m +- 1) shows) with distinct marks on both sides of every join a route crosses and large opposite
values on the last two samples of every window, range and set, so that a sample dropped or repeated at a join, a decay exponent off
by one, a seed taken one sample late or the last two samples swapped each move the mean or the EMA by many budgets of
mean_ema_ref.py.  A small alpha (1e-6 unless a case needs the carry's guarded variant) keeps the whole range in the EMA's reach."""
import numpy as np

import mean_ema_ref as R

LD = np.longdouble
ALPHA = 1e-6
TILE = 1024                                    # GPUD_MAX_WINDOW: the long routes' tiles


def series(n, marks, seed, ends=()):
    """n samples of 1 + 0.5 N(0, 1).  Both samples at every join in `marks` (j - 1 and j) take distinct values 1 +- (10 .. 26), far
    from the mean, so that dropping or repeating one moves the mean; the last two samples before every position in `ends` take +3e4
    and -3e4, so that swapping them moves the EMA even at alpha = 1e-6"""
    rng = np.random.default_rng(seed)
    x = 1.0 + 0.5 * rng.standard_normal(n)
    pos = np.array(sorted({int(p) for j in marks for p in (j - 1, j) if 0 <= p < n}), dtype=np.int64)
    i = np.arange(pos.size)
    x[pos] = 1.0 + (1 - 2 * (i % 2)) * (10.0 + i % 13 + 0.37 * (i % 7))
    for e in ends:
        if 2 <= e <= n:
            x[e - 2:e] = (3e4, -3e4)
    return x


def ema_ld(c, alpha, seed=None, extra_decay_at=None):
    """the long-double EMA at the last sample of c (seed c[0] unless given); extra_decay_at = s multiplies the carry entering sample s
    by one more beta (a decay exponent one too large for the piece or tile that starts at s)"""
    a, b = LD(alpha), LD(1.0 - alpha)
    e = LD(c[0] if seed is None else seed)
    X = c.astype(LD)
    if extra_decay_at is None:
        return R.sg.lfilter([a], [LD(1), -b], X, zi=[b * e])[0][-1]
    s = extra_decay_at
    head = R.sg.lfilter([a], [LD(1), -b], X[:s], zi=[b * e])[0][-1] if s else e
    return R.sg.lfilter([a], [LD(1), -b], X[s:], zi=[b * b * head])[0][-1]


def perturbations(c, alpha, joins, decay_starts=()):
    """{name: (which output, perturbed value)} for one set's samples c: a sample dropped and one repeated at every join, the mean over
    m - 1 and m + 1, the seed one sample late, one more decay for the piece or tile starting at each of decay_starts, the last two
    samples swapped"""
    m = c.size
    S = np.sum(c.astype(LD))
    out = {"mean/(m-1)": ("mean", S / (m - 1)) if m > 1 else None, "mean/(m+1)": ("mean", S / (m + 1)),
           "seed late": ("ema", ema_ld(c, alpha, seed=c[1])) if m > 1 else None}
    for j in joins:
        for p in (j - 1, j):
            if 0 < p < m:                                   # the first sample is also the seed: dropping it is "seed late"
                d = np.delete(c, p)
                u = np.insert(c, p, c[p])
                out["drop %d" % p] = ("both", (np.sum(d.astype(LD)) / (m - 1), ema_ld(d, alpha)))
                out["dup %d" % p] = ("both", (np.sum(u.astype(LD)) / (m + 1), ema_ld(u, alpha)))
    for s in decay_starts:
        out["decay+1 at %d" % s] = ("ema", ema_ld(c, alpha, extra_decay_at=s))
    if m >= 2:
        sw = c.copy()
        sw[[-2, -1]] = sw[[-1, -2]]
        out["swap last two"] = ("ema", ema_ld(sw, alpha))
    return {k: v for k, v in out.items() if v is not None}


def budgets_moved(c, alpha, joins, decay_starts=(), outputs=("mean", "ema"), seed=True):
    """{perturbation: how many budgets it moves the output it touches} (for drop / dup, the larger of mean and EMA), over the
    perturbations that touch one of `outputs`; seed = False leaves out "seed late" (an EMA whose seed has decayed away)"""
    want = R.windows_fields(c[None, :], c.size, np.zeros(1), alpha)
    me, mb = LD(want["mean"][0, 0]), LD(want["mean_err"][0, 0])
    ee, eb = LD(want["ema"][0, 0]), LD(want["ema_err"][0, 0])
    moved = {}
    for k, (which, v) in perturbations(c, alpha, joins, decay_starts).items():
        if (which != "both" and which not in outputs) or (k == "seed late" and not seed):
            continue
        if which == "both":
            v = (v[0] if "mean" in outputs else me, v[1] if "ema" in outputs else ee)
        if which == "mean":
            moved[k] = float(abs(v - me) / mb)
        elif which == "ema":
            moved[k] = float(abs(v - ee) / eb)
        else:
            moved[k] = float(max(abs(v[0] - me) / mb, abs(v[1] - ee) / eb))
    return moved


def tile_starts(m, at_least=5000):
    """the long routes' tile starts (0, 1024, ...) of a range of m samples whose tile ends at least `at_least` samples before the end,
    and the last tile's start (d_last)"""
    starts = [s for s in range(TILE, m, TILE) if m - (s + TILE) >= at_least][-3:]
    last = ((m - 1) // TILE) * TILE
    return starts + ([last] if last > 0 else [])


# ------------------------------------------------------------------------------------------------ the layouts of the route tests
# Each returns the pushed streams' lengths, what the call reads, the join positions the data marks and the ends of what the call
# reduces (push-order sample numbers).
def window_layout():
    """W = 1000 over a ring of 64500 whose oldest sample sits at column 20250 (a filler of 20250 pushed first): the window across
    the physical end is window 44, the last window is partial (500)"""
    W, cap, start = 1000, 64500, 20250
    return W, cap, start, list(range(0, cap, W)) + [cap - start], list(range(W, cap, W)) + [cap]


def range_layout(last_n):
    """a wrapped ring of 2^20, the newest n = last_n (CAP for 0) samples"""
    cap = 1 << 20
    total = cap + cap // 3
    n = cap if last_n == 0 else last_n
    joins = [total - n + k * TILE for k in range(n // TILE + 1)] + [cap * (total // cap)]
    return cap, total, n, joins, [total]


def ranges_layout():
    """short ranges, tiled long ranges (some across the physical end) and one of 2.2 M samples, in a wrapped ring of 2^22"""
    cap = 1 << 22
    total = cap + 777777
    lo, end = total - cap, cap
    ranges = [(end - 500, 1000), (end - 1, 3), (total - 1023, 1023), (lo + 5, 64), (end - 150000, 300001), (lo, 1025),
              (total - 2200000, 2200000)]
    joins = [end] + [f + k * TILE for f, n in ranges for k in range(n // TILE + 1)] + [f + n for f, n in ranges]
    return cap, total, ranges, joins, [f + n for f, n in ranges]


SET_PIECES = [1, 1022, 1, 1, 50000, 1, 250000]                    # set joins at 1, 1023, 1024, 1025, 51025, 51026


def sets_layout():
    """a long set of SET_PIECES at increasing positions, and a short set of four pieces, one across the physical end"""
    cap = 1 << 20
    total = cap + 4321
    lo = total - cap
    rng = np.random.default_rng(4)
    starts = np.sort(rng.choice(np.arange(lo, total - 300000), len(SET_PIECES), replace=False))
    long_set = [(int(s), n) for s, n in zip(starts, SET_PIECES)]
    short_set = [(cap - 700, 1), (cap - 1, 1022), (lo + 3, 1), (total - 1, 1)]
    both = long_set + short_set
    joins = [a for a, _ in both] + [a + n for a, n in both] + [cap]
    return cap, total, [long_set, short_set], joins, [sum(s[-1]) for s in (long_set, short_set)]


def box_layout(n_rings, seed):
    """rings of 2^18 with different totals; three sets with one piece per ring in a random order (one short, two long) and one of
    1023 + 1025 + 1 samples over the first and last ring.  Returns (cap, totals, sets of (ring, first, n), per-ring joins, per-ring
    ends)"""
    cap = 1 << 18
    totals = [cap + 1000 * k + 17 if k % 2 else cap - 999 * (k + 1) for k in range(n_rings)]
    olds = [max(0, t - cap) for t in totals]
    rng = np.random.default_rng(seed)
    sets = []
    for s in range(3):
        pieces = []
        for k in rng.permutation(n_rings):
            n = int(rng.integers(20000, 60000)) if s else int(rng.integers(1, 300))
            pieces.append((int(k), int(rng.integers(olds[k], totals[k] - n + 1)), n))
        sets.append(pieces)
    sets.append([(0, olds[0], 1023), (n_rings - 1, olds[n_rings - 1] + 5, 1025), (0, totals[0] - 1, 1)])
    joins = [[a for st in sets for kk, a, n in st if kk == k] + [a + n for st in sets for kk, a, n in st if kk == k] + [cap]
             for k in range(n_rings)]
    ends = [[st[-1][1] + st[-1][2] for st in sets if st[-1][0] == k] for k in range(n_rings)]
    return cap, totals, sets, joins, ends


def stream_layout(span, hop):
    """the stream and hop handles' stream: W = 1000, CAP = 655002, 1.5 CAP samples; window k covers [k P, k P + L)"""
    W, cap = 1000, 655002
    n = 3 * cap // 2
    return W, cap, n, list(range(0, n, W)), list(range(span * W, n + 1, hop * W))


def tier_layout():
    """the configs[1] shape, 64 fields and CAP = 10^6, in a ring whose tier keeps every row: the newest 2.2 M samples (1.2 M of them
    decoded from the tier), a range across the tier/ring boundary and a long one wholly in the tier"""
    F, cap = 64, 1_000_000
    total = 2_200_000 + 333_333
    held = total - cap
    ranges = [(total - 2_200_000, 2_200_000), (held - 700, 1500), (10 * TILE + 17, 300001)]
    joins = [held] + [f + k * TILE for f, n in ranges for k in range(n // TILE + 1)] + [f + n for f, n in ranges] \
        + list(range(0, total, TILE))                               # the tier's block rows
    return F, cap, total, ranges, joins, [f + n for f, n in ranges]


def box_tier_layout():
    """two rings of 2^16 whose tiers keep every row: a long set spread over both rings with pieces in each tier, across each
    tier/ring boundary and in each ring, a short set across both boundaries, and one ring whole from its first sample.  Returns
    (cap, totals, sets of (ring, first, n), per-ring joins, per-ring ends)"""
    cap = 1 << 16
    totals = [5 * cap + 777, 3 * cap + 5]
    held = [t - cap for t in totals]
    sets = [[(0, held[0] - 3000, 6000), (1, 1000, 50000), (1, held[1] - 100, 1025), (0, 5, 20000), (1, totals[1] - 3000, 3000)],
            [(1, held[1] - 1, 2), (0, held[0] - 1, 1), (0, 7, 1)],
            [(1, 0, totals[1])]]
    joins = [[a for st in sets for kk, a, n in st if kk == k] + [a + n for st in sets for kk, a, n in st if kk == k] + [held[k]]
             for k in range(2)]
    ends = [[st[-1][1] + st[-1][2] for st in sets if st[-1][0] == k] for k in range(2)]
    return cap, totals, sets, joins, ends


def set_joins(pieces):
    """the positions inside a set's concatenation where one piece ends and the next begins"""
    return np.cumsum([n for n in pieces])[:-1].tolist()
