"""Window generators aimed at the branches of k_window_reduce's order-statistic cascade (gpud_b200/csrc/ring.cu), and the ring
shapes that send windows through each compiled copy of its loop.  Shared by test_window_paths_model.py (numpy model of the cascade)
and test_gpu_window_paths.py (the kernel against the oracle).

The kernel parks a window as 32 rows of 32 entries: sample t goes to row (t & 63) >> 1, entry 2 (t >> 6) + (t & 1), so lane l
holds the samples t = 2l, 2l+1 (mod 64).  Where a value sits in the window decides which lane maxima it raises, and with them the
branch.  Every generator returns one chronological window of m float64 samples; `k` is the rank (k-th largest) it aims at."""
import functools

import numpy as np

DBL_MAX = np.finfo(np.float64).max
POS_NAN = np.array([0x7FFFFFFFFFFFFFFF], dtype=np.uint64).view(np.float64)[0]    # the largest totalOrder key
NEG_NAN = np.array([0xFFFFFFFFFFFFFFFF], dtype=np.uint64).view(np.float64)[0]    # the smallest key, bit-identical to the kernel's padding
SUBNORMAL = 5e-324


def lane_positions(lane, m):
    """chronological indices t < m held by `lane` (t = 2 lane, 2 lane + 1 mod 64), in order"""
    t = np.arange(m)
    return t[((t & 63) >> 1) == lane]


def _gauge(rng, m):
    """a noisy non-integer gauge: non-zero low words, high words spread over thousands of values"""
    return 60.0 + rng.normal(0.0, 3.0, m)


def _tied(rng, m, base=45.3):
    """values that share one high word and differ in the low word (45.3 + j ulp)"""
    return np.nextafter(base, np.inf) + rng.integers(0, 1 << 20, m) * np.spacing(base)


def _lanes(rng, n):
    return rng.permutation(32)[:n]


def spike_rows(rng, m, k, n_lanes):
    """row-stacked spikes: every sample of one or two lanes (a spike repeating every 32 or 64 samples) lies above the rest, so
    the top keys fill one or two rows and both gathers overflow for k <= 32"""
    x = _gauge(rng, m)
    for lane in _lanes(rng, n_lanes):
        t = lane_positions(lane, m)
        x[t] = 1000.0 + rng.random(t.size)
    return x


def top_over_lanes(rng, m, k, extra, tied):
    """the k (+ extra) largest keys one per lane, over exactly min(32, k + extra) lanes; tied: every value shares a high word"""
    x = _tied(rng, m, 45.3) if tied else _gauge(rng, m)
    n = min(32, k + extra)
    for lane in _lanes(rng, n):
        t = lane_positions(lane, m)
        if t.size:
            x[rng.choice(t)] = (np.nextafter(45.3, np.inf) + (1 << 21) * np.spacing(45.3) + rng.integers(0, 1 << 20) * np.spacing(45.3)) if tied \
                else 500.0 + rng.random()
    return x


def _lo_zero_values(flavour, v):
    """map increasing integers v (0 <= v < 2048) to increasing doubles whose raw low word is zero"""
    v = np.asarray(v, dtype=np.float64)
    if flavour == "int":
        return v
    if flavour == "quarter":
        return v * 2.0 ** -20            # multiples of 2^-20: halves, quarters, ... all with a zero low word
    if flavour == "neg":
        return v - 2048.0                # every value negative: the key's low word is the inverse of the raw one
    return v - 150.0                     # mixed signs


def lo_zero(rng, m, k, flavour, n_big):
    """every raw low word zero.  A flat base value and n_big larger values stacked into the fewest lanes: the k-th largest lane
    maximum Lh is the base whenever those lanes are fewer than k, so exactly n_big keys are gathered above it"""
    x = np.full(m, 100.0)
    if n_big:
        order = np.concatenate([lane_positions(l, m) for l in _lanes(rng, 32)])
        n_big = min(n_big, m)
        x[order[:n_big]] = 101.0 + rng.permutation(n_big + 40)[:n_big]
    return _lo_zero_values(flavour, x)


def lo_zero_noisy(rng, m, k, flavour):
    """integer readings with ties at every rank (degrees, %, MHz)"""
    return _lo_zero_values(flavour, rng.integers(80, 120, m))


def signed_zeros(rng, m, k):
    return rng.choice(np.array([0.0, -0.0, 1.0, -1.0]), m)


def tied_shuffled(rng, m, k):
    """a monotone counter, shuffled: tied high words, the low words order it, and the positional check fails"""
    return rng.permutation(2.0 ** 39 + np.cumsum(rng.integers(0, 2001, m)).astype(np.float64))


def flat_plus_one(rng, m, k):
    """a flat 45.3 with one sample just above it (same high word)"""
    x = np.full(m, 45.3)
    x[rng.integers(0, m)] = np.nextafter(45.3, np.inf)
    return x


def tied_class(rng, m, k):
    """a class of equal keys at the bound: most lanes' maximum is the same non-integer value, the rest shares its high word"""
    x = _tied(rng, m, 45.3)
    top = np.nextafter(45.3, np.inf) + (1 << 21) * np.spacing(45.3)
    for lane in _lanes(rng, 24):
        t = lane_positions(lane, m)
        if t.size:
            x[rng.choice(t, min(t.size, 2), replace=False)] = top
    return x


def tied_select(rng, m, k):
    """tied high words; lane 0 holds the two largest keys and lanes 1..k-1 one each above the rest, so the exact 64-bit bound (the
    k-th largest lane maximum) has exactly k keys above it"""
    x = _tied(rng, m, 45.3)
    s = np.spacing(45.3)
    top = np.nextafter(45.3, np.inf) + (1 << 21) * s
    lanes = _lanes(rng, min(32, k))
    vals = top + np.sort(rng.permutation(1 << 16)[:lanes.size + 1])[::-1] * s
    for i, lane in enumerate(lanes):
        t = lane_positions(lane, m)
        if i == 0 and t.size >= 2:
            x[t[:2]] = vals[:2]
        elif t.size:
            x[rng.choice(t)] = vals[i + 1]
    return x


def min_placement(rng, m, k, n_lanes, negative):
    """the minimum's high word held by n_lanes lanes with different low words; negative: the minimum is negative, so its key's low
    word is the inverse of the raw one"""
    x = _gauge(rng, m) - (200.0 if negative else 0.0)
    lo = -300.3 if negative else 10.3
    for lane in _lanes(rng, n_lanes):
        t = lane_positions(lane, m)
        if t.size:
            x[rng.choice(t, min(t.size, 2), replace=False)] = lo + rng.integers(0, 1 << 20, min(t.size, 2)) * np.spacing(lo)
    return x


def positional(rng, m, k, fail):
    """an ascending counter (the positional shortcut's case); fail names the one sample that breaks the condition"""
    x = 2.0 ** 39 + np.cumsum(rng.integers(1, 2001, m)).astype(np.float64)
    tk = max(0, m - k)
    if fail == "before_T" and 0 < tk:
        x[rng.integers(0, tk)] = x[tk] + 0.5          # a sample before m - k above T
    elif fail == "last" and m >= 2:
        x[m - 1] = x[m - 2] - 1.0                     # the last sample is not the maximum
    elif fail == "first" and m >= 2:
        x[0] = x[1] + 0.25                            # the first sample is not the minimum
    elif fail == "nan":
        x[rng.integers(0, m)] = np.nan
    elif fail == "sign":
        # only the sign test rejects this one: +0.0 first, a -0.0 later (equal as doubles), ascending subnormals (low words non-zero)
        x = np.arange(m, dtype=np.float64) * SUBNORMAL
        x[0] = 0.0
        if m > 5:
            x[5] = -0.0
            x[1:5] = 0.0
    return x


def extreme(rng, m, k, which):
    """special bit patterns among ordinary readings; at most one finite sample with |x| > 1e300 per window"""
    x = _gauge(rng, m)
    pool = {"zeros_subnormals": [0.0, -0.0, SUBNORMAL, -SUBNORMAL, 2.2e-308, -1e-310],
            "inf": [np.inf, -np.inf, np.inf],
            "dbl_max": [DBL_MAX if rng.random() < 0.5 else -DBL_MAX],
            "pos_nan": [POS_NAN, np.inf],
            "neg_nan": [NEG_NAN, -np.inf],
            "all_neg_nan": None}[which]
    if pool is None:
        return np.full(m, NEG_NAN)                    # every sample bit-identical to the padding
    t = rng.permutation(m)[:len(pool)]
    x[t] = pool[:t.size]
    return x


# name -> generator(rng, m, k).  The kinds a window can take; each aims at one branch of the cascade (see branch_of).
KINDS = {
    "gauge": lambda r, m, k: _gauge(r, m),
    "spike_rows1": lambda r, m, k: spike_rows(r, m, k, 1),
    "spike_rows2": lambda r, m, k: spike_rows(r, m, k, 2),
    "top_k_lanes": lambda r, m, k: top_over_lanes(r, m, k, 0, False),
    "top_k1_lanes": lambda r, m, k: top_over_lanes(r, m, k, 1, False),
    "top_k_lanes_tied": lambda r, m, k: top_over_lanes(r, m, k, 0, True),
    "lz_none_int": lambda r, m, k: lo_zero(r, m, k, "int", 0),
    "lz_few_quarter": lambda r, m, k: lo_zero(r, m, k, "quarter", max(0, k - 1)),
    "lz_exact_neg": lambda r, m, k: lo_zero(r, m, k, "neg", k),
    "lz_exact_int": lambda r, m, k: lo_zero(r, m, k, "int", k),
    "lz_mid_mixed": lambda r, m, k: lo_zero(r, m, k, "mixed", min(32, k + 3)),
    "lz_over_int": lambda r, m, k: lo_zero(r, m, k, "int", 40),
    "lz_noisy_int": lambda r, m, k: lo_zero_noisy(r, m, k, "int"),
    "lz_noisy_neg": lambda r, m, k: lo_zero_noisy(r, m, k, "neg"),
    "signed_zeros": signed_zeros,
    "tied_shuffled": tied_shuffled,
    "flat_plus_one": flat_plus_one,
    "tied_class": tied_class,
    "tied_select": tied_select,
    "min_few": lambda r, m, k: min_placement(r, m, k, 3, False),
    "min_many": lambda r, m, k: min_placement(r, m, k, 20, False),
    "min_few_neg": lambda r, m, k: min_placement(r, m, k, 5, True),
    "min_many_neg": lambda r, m, k: min_placement(r, m, k, 12, True),
    "pos_pass": lambda r, m, k: positional(r, m, k, None),
    "pos_fail_before_T": lambda r, m, k: positional(r, m, k, "before_T"),
    "pos_fail_last": lambda r, m, k: positional(r, m, k, "last"),
    "pos_fail_first": lambda r, m, k: positional(r, m, k, "first"),
    "pos_fail_nan": lambda r, m, k: positional(r, m, k, "nan"),
    "pos_fail_sign": lambda r, m, k: positional(r, m, k, "sign"),
    "ext_zeros_subnormals": lambda r, m, k: extreme(r, m, k, "zeros_subnormals"),
    "ext_inf": lambda r, m, k: extreme(r, m, k, "inf"),
    "ext_dbl_max": lambda r, m, k: extreme(r, m, k, "dbl_max"),
    "ext_pos_nan": lambda r, m, k: extreme(r, m, k, "pos_nan"),
    "ext_neg_nan": lambda r, m, k: extreme(r, m, k, "neg_nan"),
    "ext_all_neg_nan": lambda r, m, k: extreme(r, m, k, "all_neg_nan"),
}
# kinds with samples that make the rest of a field's EMA infinite or NaN, or whose magnitude (DBL_MAX, 2^39 counters) dwarfs a
# gauge's: the rings keep them to every fourth field, so that most fields' EMA stays finite and on a gauge's scale
WIDE_KINDS = ("ext_inf", "ext_pos_nan", "ext_neg_nan", "ext_all_neg_nan", "ext_dbl_max", "tied_shuffled", "pos_pass",
              "pos_fail_before_T", "pos_fail_last", "pos_fail_first", "pos_fail_nan")
# kinds the tail windows (the wrap window and the trailing partial window) cycle through
ADVERSARIAL_KINDS = ("spike_rows1", "spike_rows2", "lz_exact_int", "lz_over_int", "tied_class", "tied_select", "min_many",
                     "min_many_neg", "pos_fail_sign", "ext_neg_nan", "ext_zeros_subnormals", "top_k1_lanes")


@functools.lru_cache(maxsize=4096)
def _window_cached(kind, m, k, seed):
    x = np.ascontiguousarray(KINDS[kind](np.random.default_rng(seed), m, max(1, min(k, m))), dtype=np.float64)
    assert x.shape == (m,)
    x.flags.writeable = False
    return x


def window(kind, m, k, seed):
    """one window of kind `kind`; seed: an int or a tuple of ints.  The same arguments give the same (read-only) array."""
    return _window_cached(kind, m, k, seed)


def k_of(m, q_num, q_den):
    """the rank the kernel selects: the k-th largest, k = m - ceil(m q) + 1 (oracle SPEC.md nearest rank)"""
    r = (m * q_num + q_den - 1) // q_den
    return m - max(1, min(m, r)) + 1


# Ring shapes.  `start` is the physical column of the oldest sample (set by pushing a filler prefix first); `count` samples are
# reduced.  Each names the copy of the window loop launch_windows must pick for its aligned windows (inst) and the windows it
# leaves to the tail loop inside the aligned kernel.
RING_SHAPES = [
    dict(name="w1000", W=1000, cap=64000, count=64000, start=0, inst="<1,15,0>", tail={}),
    # W = 960 leaves pair 15 of <1,15,0> empty; it runs the generic code (its EMA partial would otherwise decay once too often)
    dict(name="w960", W=960, cap=61440, count=61440, start=0, inst="<1,-1,0>", tail={}),
    dict(name="w960_partial", W=960, cap=62000, count=62000, start=0, inst="<1,-1,0>", tail={}),
    dict(name="w1022", W=1022, cap=65408, count=65408, start=0, inst="<1,15,0>", tail={}),
    dict(name="w1024", W=1024, cap=65536, count=65536, start=0, inst="<1,16,0>", tail={}),
    dict(name="w1000_tail", W=1000, cap=64500, count=64500, start=20250, inst="<1,15,0>", tail={44: "wrap", 64: "partial"}),
    dict(name="w1024_tail", W=1024, cap=66036, count=66036, start=20250, inst="<1,16,0>", tail={44: "wrap", 64: "partial"}),
    dict(name="odd_start", W=1000, cap=64000, count=64000, start=333, inst="<0,-1,0>", tail={}),
    dict(name="w999", W=999, cap=63938, count=63938, start=0, inst="<0,-1,0>", tail={}),
    dict(name="w500", W=500, cap=32250, count=32250, start=0, inst="<1,-1,0>", tail={}),
    dict(name="w62", W=62, cap=6230, count=6230, start=0, inst="<1,-1,0>", tail={}),
    dict(name="w999_single", W=999, cap=1000, count=999, start=0, inst="<1,-1,0>", tail={}),
    dict(name="short63", W=63, cap=64, count=63, start=0, inst="<1,-1,0>", tail={}),
    dict(name="short34", W=32, cap=64, count=34, start=0, inst="<1,-1,0>", tail={}),
]


def window_kind(shape, f, w):
    """the kind of window w of field f: the kinds cycle along each field (so a run of consecutive windows changes branch at every
    step), wide kinds only in every fourth field, adversarial kinds in the tail windows"""
    if w in shape["tail"]:
        names = [n for n in ADVERSARIAL_KINDS if f % 4 == 3 or n not in WIDE_KINDS]
        return names[(f + w) % len(names)]
    names = [n for n in KINDS if f % 4 == 3 or n not in WIDE_KINDS]
    return names[(f * 7 + w) % len(names)]


def field_content(shape, f, q_num=99, q_den=100, seed=0, variants=5):
    """the chronological samples of field f of a ring shape: one generated window per window slot (`variants` different windows
    of each kind and length, so that a ring of thousands of windows costs a few hundred generator calls)"""
    W, count = shape["W"], shape["count"]
    out = np.empty(count, dtype=np.float64)
    for w in range((count + W - 1) // W):
        a, b = w * W, min(count, (w + 1) * W)
        out[a:b] = window(window_kind(shape, f, w), b - a, k_of(b - a, q_num, q_den), (seed, (f + 3 * w) % variants))
    return out
