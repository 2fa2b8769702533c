"""The reference for every mean and EMA the library reports, and the rounding budget each answer must fall within.

`windows_fields` has the signature and output layout of `oracle.coracle.windows_fields`.  min / max / p99 / n_over are the C
oracle's, unchanged (they are compared bit for bit).  mean and EMA are recomputed in extended precision (x87 long double, 64-bit
significand), and four arrays are added, each [F][nw]:

* `mean_err`, `ema_err`: how far an f64 implementation of oracle/SPEC.md's definitions may be from the extended reference;
* `mean_exempt`, `ema_exempt`: the outputs that keep the former rule against the C oracle's f64 answer, see "Exemptions".

`check_mean_ema(got, want)` compares a device answer with it and returns the worst |got - ref| / err.

Reference.  mean = (sum x) / m in long double; summed in any order its own error is about n 2^-64 of sum |x| / m, 2^-11 of the
budget below.  EMA: alpha and beta = 1 - alpha are the f64 values the library uses (alpha = min(2 / (W + 1), 0.9999) when the
configured alpha is not positive); e_t = alpha x_t + beta e_(t-1) from e_(-1) = x[0] runs in long double (scipy.signal.lfilter),
which matches 300-bit arithmetic to ~1e-19 relative.  A non-finite reference (+inf, -inf, NaN) is matched by class: the recurrence
itself keeps an infinite EMA infinite and turns +inf then -inf into NaN, as SPEC.md requires.

Budget, u = 2^-53, gamma_k = k u / (1 - k u), derived from the arithmetic the library's schemes perform (DESIGN.md), not fitted:

* mean_err = gamma_(m+3) sum |x| / m + u |mean| + 2^-1074.  Any order of m - 1 f64 additions errs by at most gamma_(m-1) sum |x|
  (Higham, Accuracy and Stability, 4.2).  The window kernel, the range tiles and the box fold store a partial mean S_t / m_t and
  multiply it back by m_t: two more roundings of |S_t| <= sum |x|; the final division by m is one rounding of the result (u |mean|,
  and one more gamma step).  The last term keeps an all-zero window's budget positive.
* ema_err = u sum_t w_t |x_t| (C0 + C1 ceil(log2(m + 1)) + 2 d_t) + (m + 1/alpha) 2^-1074 max|x|, summed over every sample from the
  seed to the output's last sample: w_t = alpha beta^(d_t), plus beta^m on the seed, the exact weights; d_t the sample's distance to
  the output's last sample; m the samples from the seed to it.
  Each rounding on a sample's way to the output errs by at most u times a partial sum, which is at most sum w |x| over the samples
  in it; so the coefficient of a sample is the number of roundings on its path, and every error of a decay weight is relative.
  - 2 d_t: the weight of a sample d_t back is a product of powers of beta whose exponents add up to d_t, each rounded: one multiply
    and one add per step in the sequential recurrence; d_t / 64 fma steps with q64 = pow(beta, 64) in the device's lane Horner; the
    squarings d^(2^i), pow(d_full, t + 1), d_last and (1 - alpha)^len, each within 2 ulp of its exact power k >= 1, in the
    carry's scan and the piece composition.  2 d_t covers all of them.
  - C0 = 16: the roundings every path has whatever the length: the lane weight pw = pow(beta, e) (2 ulp), es * pw (1), the
    5-level shuffle tree of the lane partials (5), the final * alpha (1), and up to 7 more for the carry's entry (the lane and row
    carries of the scan, d_last, the piece fold): 16.
  - C1 ceil(log2(m + 1)): the scans and folds deepen with the length: the carry's Kogge-Stone scan over a row of 128 window
    partials, the cross-warp and cross-row carries, a long range's tiles, a set's pieces and the ranks each add at most one fma per
    doubling of m.  C1 = 2 leaves a factor 2 on that count.
  - The last term covers weights that underflow: each of at most m products, and the 1/alpha tail of the geometric weights past the
    point where beta^d is subnormal, loses at most 2^-1074 of max|x| (the largest finite |x| up to the output).
  On the CPU (tests/test_mean_ema_ref_model.py) the C oracle's sequential f64 recurrence uses at most 0.6 of this budget (a
  constant window after a step, where every step rounds the same way; 0.03 on gauges) and its mean at most 0.09; numpy emulations
  of the device schemes stay below 0.5.

Exemptions (`mean_exempt`, `ema_exempt`), both limited to outputs whose reference is finite:
* the mean of a window whose positive or whose negative samples sum past DBL_MAX: an f64 sum may overflow on the way;
* SPEC.md's known limit: the EMA of a window that holds two or more samples above DBL_MAX / 8 in magnitude, and of every later
  window (the lane-local EMA partial can overflow and the carry passes it on).
There the rule is oracle/SPEC.md's former one against the C oracle's f64 answer b: the same infinity or NaN as b, or
|a - b| <= 1e-6 max(|b|, max|x| of the field).  For those outputs `mean` / `ema` hold b and `mean_err` / `ema_err` that bound."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import scipy.signal as sg

from oracle import coracle

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, \
    "the mean / EMA reference needs an extended long double (64-bit significand), got %d bits" % np.finfo(LD).nmant

U = 2.0 ** -53
TINY = 2.0 ** -1074
DBL_MAX = np.finfo(np.float64).max
C0, C1 = 16, 2
FIELDS_PER_PASS = 4


def ema_alpha(W, alpha=0.0):
    """the f64 alpha the library uses for a ring of window W and configured alpha"""
    return float(alpha) if alpha > 0 else min(2.0 / (W + 1.0), 0.9999)


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


def window_bounds(n, W):
    """first and last sample of every window"""
    starts = np.arange(0, n, W, dtype=np.int64)
    return starts, np.minimum(starts + W, n) - 1


def mean_ref(x, W):
    """[F][nw]: the exact-enough mean (f64), its budget, and the exemption mask"""
    F, n = x.shape
    starts, ends = window_bounds(n, W)
    m = (ends - starts + 1).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        mean = (np.add.reduceat(x.astype(LD), starts, axis=1) / m.astype(LD)).astype(np.float64)
        A = np.add.reduceat(np.abs(x), starts, axis=1)            # a budget: f64 is ample (inf where it overflows)
        err = gamma(m + 3) * (A / m) + U * np.abs(mean) + TINY
        exempt = np.zeros(mean.shape, dtype=bool)
        if np.any(np.abs(x[np.isfinite(x)]) > DBL_MAX / (2 * W)):    # only then can a sum of one sign pass DBL_MAX
            pos = np.add.reduceat(np.where(x > 0, x, 0.0).astype(LD), starts, axis=1)
            neg = np.add.reduceat(np.where(x < 0, x, 0.0).astype(LD), starts, axis=1)
            exempt = np.isfinite(mean) & ((pos > LD(DBL_MAX)) | (neg < -LD(DBL_MAX)))
    return mean, err, exempt


def ema_ref(x, W, alpha):
    """[F][nw]: the long-double EMA at every window's last sample (f64), its budget, and the exemption mask"""
    F, n = x.shape
    starts, ends = window_bounds(n, W)
    a, b = LD(alpha), LD(1.0 - alpha)            # beta is the f64 1 - alpha, as in the library
    fin = np.isfinite(x)
    allfin = bool(fin.all())
    xf = x if allfin else np.where(fin, x, 0.0)   # lfilter's 0 * inf would be NaN: the non-finite classes come from _classes
    X = xf.astype(LD)
    AX = np.abs(xf)
    with np.errstate(invalid="ignore", over="ignore"):
        e = sg.lfilter([a], [LD(1), -b], X, axis=1, zi=(b * X[:, :1]))[0][:, ends]
        del X
        # the budget's filters in f64: Z_t = sum_s w_s |x_s| (with the seed), D_t = sum_s w_s (t - s) |x_s| (the seed at distance
        # t + 1), D_t = b D_(t-1) + b Z_(t-1)
        bf = 1.0 - alpha
        Z = sg.lfilter([alpha], [1.0, -bf], AX, axis=1, zi=(bf * AX[:, :1]))[0]
        D = sg.lfilter([0.0, bf], [1.0, -bf], Z, axis=1, zi=(bf * AX[:, :1]))[0][:, ends]
        Z = Z[:, ends]
        mt = (ends + 1).astype(np.float64)
        c = C0 + C1 * np.ceil(np.log2(mt + 1.0))
        xmax = np.maximum.accumulate(np.maximum.reduceat(AX, starts, axis=1), axis=1)
        err = U * (Z * c + 2 * D) + (mt + 1.0 / alpha) * TINY * xmax
        ema = e.astype(np.float64)
    if not allfin:
        cls = _classes(x)[:, ends]
        ema = np.where(np.isfinite(cls), ema, cls)
    big = np.add.reduceat((np.abs(x) > DBL_MAX / 8).astype(np.int64), starts, axis=1) >= 2
    exempt = np.isfinite(ema) & (np.maximum.accumulate(big, axis=1) > 0)
    return ema, err, exempt


def _classes(x):
    """[F][n]: the EMA's class after each sample - 0.0 while finite, else +inf, -inf or NaN.  Once non-finite the EMA stays so
    (beta * inf = inf whatever the weight): the seed x[0] or the first non-finite sample sets it, a later infinity of the other sign or
    a NaN makes it NaN."""
    out = np.zeros(x.shape)
    for f, row in enumerate(x):
        bad = np.flatnonzero(~np.isfinite(row))
        state = row[0] if not np.isfinite(row[0]) else 0.0
        t0 = 0
        for t in bad:
            out[f, t0:t] = state
            v = row[t]
            state = v if state == 0.0 else (state if v == state else np.nan)
            t0 = t
            if np.isnan(state):
                break
        out[f, t0:] = state
    return out


def _legacy_tol(ref, x):
    """oracle/SPEC.md's former rule, kept for the exempt outputs: 1e-6 max(|ref|, the field's largest finite |x|) around the f64
    oracle's answer ref"""
    with np.errstate(invalid="ignore"):
        scale = np.where(np.isfinite(x), np.abs(x), 0.0).max(axis=1, keepdims=True)
        return 1e-6 * np.maximum(np.abs(ref), scale)


def windows_fields(x, W, thr, alpha=0.0, q_num=0, q_den=0, threads=0):
    """coracle.windows_fields with mean and EMA from the extended reference, plus mean_err / ema_err budgets and the
    mean_exempt / ema_exempt masks (module docstring).  x: [F][n] f64 field-major."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = coracle.windows_fields(x, W, thr, alpha, q_num, q_den, threads)
    f64 = {k: out[k] for k in ("mean", "ema")}
    a = ema_alpha(W, alpha)
    # a few fields at a time (the long-double arrays take 16 B a sample), on the host's cores (the filters release the GIL)
    with ThreadPoolExecutor(max(1, min(8, os.cpu_count() or 1))) as ex:
        parts = list(ex.map(lambda f0: mean_ref(x[f0:f0 + FIELDS_PER_PASS], W) + ema_ref(x[f0:f0 + FIELDS_PER_PASS], W, a),
                            range(0, x.shape[0], FIELDS_PER_PASS)))
    for i, k in enumerate(("mean", "mean_err", "mean_exempt", "ema", "ema_err", "ema_exempt")):
        out[k] = np.concatenate([p[i] for p in parts], axis=0)
    for k in ("mean", "ema"):
        ex = out[k + "_exempt"]
        if ex.any():                                   # the former rule, against the f64 oracle (an f64 sum may overflow as it does)
            out[k] = np.where(ex, f64[k], out[k])
            out[k + "_err"] = np.where(ex, _legacy_tol(f64[k], x), out[k + "_err"])
    return out


def select(want, idx):
    """the same outputs of every array of a reference dict, e.g. select(want, (slice(None), 0)) for the first window of each field"""
    return {k: v[idx] for k, v in want.items()}


def stack(wants, axis=1):
    """reference dicts of single outputs or columns joined along `axis` (e.g. one dict per range into [F][ranges])"""
    return {k: np.stack([w[k] for w in wants], axis=axis) for k in wants[0]}


def ratios(got, want, key):
    """|got - ref| / err where the reference is finite (0 where both are equal), NaN where it is not"""
    a = np.asarray(got, dtype=np.float64)
    b, e = np.asarray(want[key], dtype=np.float64), np.asarray(want[key + "_err"], dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        d = np.abs(a - b)
        r = np.where(d == 0, 0.0, d / e)
    return np.where(np.isfinite(b), r, np.nan)


def check_mean_ema(got, want, keys=("mean", "ema"), what=""):
    """Assert every mean / EMA of `got` (dict of arrays shaped like want's) is within its budget, and that every non-finite
    reference is matched by the same class (+inf, -inf or NaN).  Returns the worst |got - ref| / err over the finite outputs."""
    worst = 0.0
    for k in keys:
        a = np.asarray(got[k], dtype=np.float64)
        b = np.asarray(want[k], dtype=np.float64)
        assert a.shape == b.shape, (what, k, a.shape, b.shape)
        fin = np.isfinite(b)
        same_class = (a == b) | (np.isnan(a) & np.isnan(b))
        bad = np.argwhere(~fin & ~same_class)
        assert bad.size == 0, (what, k, "non-finite reference", bad[:5].tolist(), a[tuple(bad[0])], b[tuple(bad[0])])
        r = ratios(a, want, k)
        bad = np.argwhere(fin & ~(r <= 1.0))
        if bad.size:
            i = tuple(bad[0])
            raise AssertionError("%s %s: %d outputs past their budget, worst %.3g budgets; first at %s: got %r ref %r err %.3g"
                                 % (what, k, len(bad), float(np.nanmax(np.where(np.isfinite(r), r, np.inf))), bad[0].tolist(),
                                    float(a[i]), float(b[i]), float(np.asarray(want[k + "_err"])[i])))
        if fin.any():
            worst = max(worst, float(np.max(r[fin])))
    return worst


def exempt_any(want):
    return bool(np.any(want["mean_exempt"]) or np.any(want["ema_exempt"]))
