"""Model check (numpy only) of the order-statistic cascade of k_window_reduce (gpud_b200/csrc/ring.cu, window_loop after pass 1) and
of the dispatch in launch_windows.  branch_of() restates, for one window, the kernel's data-dependent choices: the positional
shortcut, the lo_zero path with its three outcomes, the high-word gather, the exact 64-bit bound, the bit search, and where the
minimum comes from.  Each branch computes its answer the way the kernel does (gather counts with the kernel's early stop, the
rank rule of select_from_candidates, the k-th largest lane maximum counting multiplicity); the tests check that every branch's
answer equals a sort of the totalOrder keys bit for bit, and that the windows of window_cases.py reach every branch.
The model is evidence of coverage; test_gpu_window_paths.py checks the kernel's values whichever branch it really takes.

`PYTHONPATH=. python tests/test_window_paths_model.py` (from the repository root) prints which branches the ring tests of test_gpu_parity.py and test_gpu_work_cursor.py
reach (their windows run through branch_of instead of the GPU)."""
import collections

import numpy as np
import pytest

from oracle import pyoracle as O
import window_cases as WC

M32 = 0xFFFFFFFF
SIGN = 0x80000000
K_PAD = 0xFFFFFFFFFFFFFFFF                      # kPadStored: raw form of key 0 (-NaN, all ones)
_ROW, _COL = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
ELEM = 64 * (_COL >> 1) + 2 * _ROW + (_COL & 1)  # elem_index(row, col): chronological t of each parked entry


def key_hi_of(h):
    return (h ^ (((M32 if h & SIGN else 0)) | SIGN)) & M32


def raw_hi_of(kh):
    return kh ^ (SIGN if kh & SIGN else M32)


def true_lo(kh, raw_lo):
    return raw_lo ^ (0 if kh & SIGN else M32)


def true_key(raw):
    kh = key_hi_of(raw >> 32)
    return (kh << 32) | true_lo(kh, raw & M32)


def _s32(u):
    return u - (1 << 32) if u & SIGN else u


def park(x):
    """the 32 x 32 raw rows of shared memory: sample t at row (t & 63) >> 1, entry 2 (t >> 6) + (t & 1); padding kPadStored"""
    m = x.size
    raw = np.full((32, 32), np.uint64(K_PAD), dtype=np.uint64)
    t = np.arange(m)
    raw[(t & 63) >> 1, 2 * (t >> 6) + (t & 1)] = x.view(np.uint64)
    return [[int(v) for v in row] for row in raw]


def kth_largest_counting(vals, k):
    """warp_kth_largest_smem: the smallest value whose rank #{v > value} is < k"""
    return min(v for v in vals if sum(1 for o in vals if o > v) < k)


def gather_rows(raw, rows, Lh, Ll, hi_only):
    """gather_rows<HI_ONLY>: the flagged rows in lane order, padded with the pad row to a multiple of four, four rows per trip;
    the walk ends after the trip in which the count passes 32.  Returns (count, the first 64 hits as raw keys)."""
    order = [r for r in range(32) if rows[r]]
    n_rows = len(order)
    order += [None] * 4
    X = 0 if Lh & SIGN else 0x7FFFFFFF
    Y = _s32(Lh ^ SIGN)
    Lp = (Lh << 32) | Ll
    cnt, cand = 0, []
    i = 0
    while i < n_rows and cnt <= 32:
        for q in range(4):
            row = order[i + q]
            for kv in (raw[row] if row is not None else [K_PAD] * 32):
                hit = _s32((kv >> 32) ^ X) >= Y if hi_only else true_key(kv) > Lp
                if hit:
                    if cnt < 64:
                        cand.append(kv)
                    cnt += 1
        i += 4
    return cnt, cand


def select_from_candidates(cand, k):
    """k-th largest of the candidates (true keys) by the kernel's rank rule, and their maximum"""
    c = [true_key(v) for v in cand]
    ans = min(v for v in c if sum(1 for o in c if o > v) < k)
    return ans, max(c)


def lane_extremes(raw, m):
    """pass 1 per lane: a_smax, b_umin, c_umax of the raw high words (padding in the partially valid pair counted as the kernel
    does: -1 / all-ones / 0, neutral in each) and the OR of the raw low words"""
    J, Jfull = (m + 63) >> 6, m >> 6
    out = []
    for lane in range(32):
        a, b, c, lor = -(1 << 31), M32, 0, 0
        for i in range(32):
            j = i >> 1
            t = ELEM[lane, i]
            if j < Jfull or (j < J and t < m):
                h, lo = raw[lane][i] >> 32, raw[lane][i] & M32
                a, b, c, lor = max(a, _s32(h)), min(b, h), max(c, h), lor | lo
            elif j < J:
                a = max(a, -1)                 # padding of the partial pair: all-ones high word
        out.append((a, b, c, lor))
    return out


def branch_of(x, m, k, W=None):
    """Restates ring.cu's cascade on one window of m samples (m == x.size) for the k-th largest.  W: the ring's window (the
    positional shortcut needs m == W; default m).  Returns (path, values): path lists the branches taken in order (a gather that
    overflows appears as '<name>_overflow' before the branch that takes over) plus the minimum's source; values holds the
    totalOrder keys the branches produce for 'min', 'max' and 'kth'."""
    W = m if W is None else W
    assert x.size == m and 1 <= k <= m
    raw = park(x)
    lanes = lane_extremes(raw, m)
    rmh, mh, nh, flags, lor_all = [], [], [], 0, 0
    for a, b, c, lor in lanes:
        r = (a & M32) if a >= 0 else b
        empty = c == 0 and b == M32
        rmh.append(r)
        mh.append(key_hi_of(r))
        nh.append(M32 if empty else key_hi_of(c if c & SIGN else b))
        flags += 1 if (((mh[-1] - nh[-1]) & M32) > 8 or (c & SIGN)) else 0
        lor_all |= lor
    tied_nonneg = flags == 0
    lo_zero = lor_all == 0
    min_hi = min(nh)
    k_full = k
    path = []

    def at(t):
        return raw[(t & 63) >> 1][2 * (t >> 6) + (t & 1)]

    def f64(kv):
        return np.array([kv], dtype=np.uint64).view(np.float64)[0]

    positional = False
    if not lo_zero and tied_nonneg and m == W and m > 960 and 1 <= k_full <= 32:
        tk = m - k_full
        e0, tv, el = f64(at(0)), f64(at(tk)), f64(at(m - 1))
        ok = True
        i_low = 30 if tk >= 960 else 0
        for lane in range(32):
            for i in range(32):
                xv = f64(raw[lane][i])
                if i < i_low:
                    ok = ok and e0 <= xv <= tv
                elif ELEM[lane, i] < m:
                    ok = ok and ((e0 <= xv <= tv) if ELEM[lane, i] < tk else (tv <= xv <= el))
        positional = ok

    # ---- minimum ----
    if positional:
        vmin, min_src = true_key(at(0)), "min_positional"
    elif lo_zero:
        vmin, min_src = (min_hi << 32) | true_lo(min_hi, 0), "min_lo_zero"
    else:
        rows = [nh[l] == min_hi for l in range(32)]
        min_src = "min_row_scan" if sum(rows) > 6 else "min_row_walk"
        raw_eh = raw_hi_of(min_hi)
        el = min(true_lo(min_hi, raw[r][i] & M32) for r in range(32) if rows[r] for i in range(32)
                 if raw[r][i] >> 32 == raw_eh and ELEM[r, i] < m)
        vmin = (min_hi << 32) | el

    # ---- k-th largest and maximum ----
    done, kth, vmax = False, None, None
    if positional:
        kth, vmax, done = true_key(at(m - k)), true_key(at(m - 1)), True
        path.append("positional")
    if not done and k <= 32:
        Lh = kth_largest_counting(mh, k)
        if lo_zero:
            rows = [v > Lh for v in mh]
            cnt, cand = gather_rows(raw, rows, (Lh + 1) & M32, 0, True) if any(rows) else (0, [])
            if cnt < k:
                kth, done = (Lh << 32) | true_lo(Lh, 0), True
                path.append("lz_bound" if any(rows) else "lz_none")
            elif cnt <= 32:
                kth, _ = select_from_candidates(cand, k)
                done = True
                path.append("lz_select")
            else:
                path.append("lz_overflow")
            if done:
                mx = max(mh)
                vmax = (mx << 32) | true_lo(mx, 0)
        else:
            cnt, cand = gather_rows(raw, [v >= Lh for v in mh], Lh, 0, True)
            if cnt <= 32:
                kth, vmax = select_from_candidates(cand, k)
                done = True
                path.append("hi_select")
            else:
                path.append("hi_overflow")
    if not done:
        ml = [max([true_lo(mh[l], kv & M32) for kv in raw[l] if kv >> 32 == rmh[l]] + [0]) for l in range(32)]
        lane_max = [(mh[l] << 32) | ml[l] for l in range(32)]
        vmax = max(lane_max)
        solved = False
        if k <= 32:
            L = sorted(lane_max, reverse=True)[k - 1]
            cnt, cand = gather_rows(raw, [v > L for v in lane_max], L >> 32, L & M32, False)
            if cnt < k:
                kth, solved = L, True
                path.append("b64_bound")
            elif cnt <= 32:
                kth, _ = select_from_candidates(cand, k)
                solved = True
                path.append("b64_select")
            else:
                path.append("b64_overflow")
        if not solved:
            keys = sorted((true_key(kv) for row in raw for kv in row), reverse=True)   # every parked entry, padding included
            kth = keys[k - 1]
            path.append("bit_search" if k > 32 else "bit_search_after_overflow")
    path.append(min_src)
    return path, {"min": vmin, "max": vmax, "kth": kth}


def dispatch(start, W, count, cap):
    """launch_windows: the instantiation <ALIGNED, JF, RANGE> its aligned windows go through, and the windows it leaves to the
    tail loop (w_skip) with their reason."""
    nw = (count + W - 1) // W
    if (start & 1) or ((W & 1) and nw > 1):
        return "<0,-1,0>", {}
    tail = {}
    c_wrap = cap - start
    if start > 0 and c_wrap < count and c_wrap % W != 0:
        tail[c_wrap // W] = "wrap"
    jf = W >> 6
    special = (jf == 16 or (jf == 15 and W % 64 != 0)) and nw > 1
    if special and count % W != 0 and (nw - 1) not in tail:
        tail[nw - 1] = "partial"
    if special and jf == 15:
        return "<1,15,0>", tail
    if special and jf == 16:
        return "<1,16,0>", tail
    return "<1,-1,0>", tail


# ------------------------------------------------------------------------------------------------ the sweep
SWEEP_M = (1, 2, 31, 33, 63, 64, 65, 500, 960, 961, 999, 1000, 1022, 1024)


def _ks(m):
    return sorted({k for k in (1, 2, 11, 31, 32, 33, 34, m // 2, m) if 1 <= k <= m})


def _sweep():
    """(kind, m, k, W) for every generated window of the sweep: full windows (W = m) and, below 1000, partial ones (W = 1000)"""
    for kind in WC.KINDS:
        for m in SWEEP_M:
            for k in _ks(m):
                yield kind, m, k, m
                if m < 1000 and k in (1, 11, 32):
                    yield kind, m, k, 1000
    for m in (961, 1000, 1022, 1024):               # positional windows at the ranks that the shortcut takes
        for k in (1, 11, 31, 32):
            for kind in ("pos_pass", "pos_fail_before_T", "pos_fail_last", "pos_fail_first", "pos_fail_nan", "pos_fail_sign"):
                yield kind, m, k, m


@pytest.fixture(scope="module")
def sweep():
    out = []
    for i, (kind, m, k, W) in enumerate(_sweep()):
        x = WC.window(kind, m, k, (i, m, k))
        path, vals = branch_of(x, m, k, W)
        out.append((kind, m, k, W, x, path, vals))
    return out


def test_every_branch_gives_the_sorted_answer(sweep):
    for kind, m, k, W, x, path, vals in sweep:
        srt = np.sort(O.total_order_key(x))
        want = {"min": int(srt[0]), "max": int(srt[-1]), "kth": int(srt[m - k])}
        assert vals == want, (kind, m, k, W, path)


BRANCHES = ("positional", "lz_none", "lz_bound", "lz_select", "lz_overflow", "hi_select", "hi_overflow", "b64_bound", "b64_select",
            "b64_overflow", "bit_search", "bit_search_after_overflow", "min_positional", "min_lo_zero", "min_row_scan", "min_row_walk")


def test_every_branch_is_reached(sweep):
    seen = collections.Counter(b for *_, path, _v in sweep for b in path)
    assert set(seen) <= set(BRANCHES), set(seen) - set(BRANCHES)
    missing = {b: seen[b] for b in BRANCHES if seen[b] < 5}
    assert not missing, missing


def test_branch_edges():
    """the windows the issue of each guard turns on: the positional shortcut rejected by the sign test alone, k = 32 / 33 on the
    two sides of the k <= 32 guards, -NaN (bit-identical to the padding) in a window shorter than 64 samples"""
    x = WC.window("pos_fail_sign", 1000, 11, 1)
    path, _ = branch_of(x, 1000, 11)
    assert "positional" not in path
    flags = [(((key_hi_of((a & M32) if a >= 0 else b) - (M32 if (c == 0 and b == M32) else key_hi_of(c if c & SIGN else b))) & M32) > 8)
             for a, b, c, _ in lane_extremes(park(x), 1000)]
    assert not any(flags)                         # the span test passes: only the sign of -0.0 keeps the window off the shortcut
    x = WC.window("spike_rows1", 1000, 32, 2)
    assert branch_of(x, 1000, 32)[0][-2] == "bit_search_after_overflow"
    assert branch_of(x, 1000, 33)[0][-2] == "bit_search"
    x = WC.window("ext_neg_nan", 31, 31, 3)
    path, vals = branch_of(x, 31, 31)
    assert vals["min"] == int(np.sort(O.total_order_key(x))[0])


def test_dispatch_covers_every_copy_of_the_loop():
    seen, tails = set(), set()
    for s in WC.RING_SHAPES:
        inst, tail = dispatch(s["start"], s["W"], s["count"], s["cap"])
        assert (inst, tail) == (s["inst"], s["tail"]), s["name"]
        seen.add(inst)
        tails |= set(tail.values())
    assert seen == {"<1,15,0>", "<1,16,0>", "<1,-1,0>", "<0,-1,0>"}
    assert tails == {"wrap", "partial"}


def test_dispatch_rules():
    assert dispatch(0, 1000, 4000, 4096) == ("<1,15,0>", {})
    assert dispatch(0, 1000, 2500, 4096) == ("<1,15,0>", {2: "partial"})
    assert dispatch(1, 1000, 4096, 4096) == ("<0,-1,0>", {})
    assert dispatch(0, 999, 1998, 2000) == ("<0,-1,0>", {})
    assert dispatch(0, 999, 999, 1000) == ("<1,-1,0>", {})           # one window: an odd W needs no odd start
    assert dispatch(0, 1024, 1024, 2048) == ("<1,-1,0>", {})          # one window is not special
    assert dispatch(48, 1000, 4096, 4096) == ("<1,15,0>", {4: "wrap"})  # the wrap window is the partial last one: skipped once
    assert dispatch(2096, 500, 4096, 4096) == ("<1,-1,0>", {})         # the wrap falls on a window boundary
    assert dispatch(2048, 500, 4096, 4096) == ("<1,-1,0>", {4: "wrap"})


def test_ring_window_kinds_cross_branches():
    """in every ring shape, consecutive windows of a field change kind, and the tail windows get adversarial kinds"""
    for s in WC.RING_SHAPES:
        nw = (s["count"] + s["W"] - 1) // s["W"]
        for f in range(8):
            kinds = [WC.window_kind(s, f, w) for w in range(nw)]
            assert all(kinds[w] != kinds[w + 1] for w in range(nw - 1) if w not in s["tail"] and w + 1 not in s["tail"]), s["name"]
            assert all(kinds[w] in WC.ADVERSARIAL_KINDS for w in s["tail"]), s["name"]


# ------------------------------------------------------------------------------------------------ helper: the existing ring tests
def existing_ring_coverage(max_windows_per_test=3000):
    """Runs the ring tests of test_gpu_parity.py and test_gpu_work_cursor.py against a stand-in for the library that records every
    window it is asked to reduce and classifies it with branch_of (answering with the oracle, so the tests run to the end).
    Returns {test: Counter(branch)}.  Not a test: it documents what the GPU suite reaches."""
    import sys
    import types
    from oracle import coracle
    import test_gpu_parity as P
    import test_gpu_work_cursor as WCUR

    class Ring:
        def __init__(self, ctx, F, cap, W, thresholds=None, ema_alpha=0.0, q_num=0, q_den=0, dev=None):
            self.F, self.cap, self.W = F, cap, W
            self.qn, self.qd = (q_num, q_den) if (q_num or q_den) else (99, 100)
            self.alpha, self.thr = ema_alpha, np.asarray(thresholds if thresholds is not None else np.full(F, np.inf), dtype=np.float64)
            self.rows = np.empty((0, F))

        def push(self, rows):
            self.rows = np.concatenate([self.rows, np.asarray(rows, dtype=np.float64)])[-self.cap:]
            self.total = getattr(self, "total", 0) + len(rows)

        push_raw = push

        def set_cta_reserve(self, n):
            pass

        def counts(self):
            c = len(self.rows)
            return self.total, c, (c + self.W - 1) // self.W

        def reduce_all(self):
            x = self.rows
            seen = counter[current[0]]
            for f in range(self.F):
                for w in range(0, len(x), self.W):
                    if sum(seen.values()) >= max_windows_per_test * 3:
                        break
                    seg = np.ascontiguousarray(x[w:w + self.W, f])
                    m = seg.size
                    seen.update(branch_of(seg, m, WC.k_of(m, self.qn, self.qd), self.W)[0])
            return coracle.windows_fields(np.ascontiguousarray(x.T), self.W, self.thr, self.alpha, self.qn, self.qd)

        def close(self):
            pass

    fake = types.SimpleNamespace(Ring=Ring, Context=lambda *a: types.SimpleNamespace(close=lambda: None))
    counter = collections.defaultdict(collections.Counter)
    current = [None]
    P.g = fake
    saved = sys.modules.get("gpud_b200")
    sys.modules["gpud_b200"] = fake
    try:
        cases = [("test_ring_windows", lambda: [P.test_ring_windows(None, *a) for a in [(8, 4000, 1000, 4096), (5, 4096, 1000, 4096),
                                                                                         (3, 2777, 1024, 4096), (4, 600, 7, 1024), (64, 10000, 1000, 10000)]]),
                 ("test_ring_wrap_and_odd_start", lambda: P.test_ring_wrap_and_odd_start(None)),
                 ("test_ring_tie_heavy_gauges", lambda: [P.test_ring_tie_heavy_gauges(None, *a) for a in [(1000, 99, 100), (1000, 50, 100), (1024, 999, 1000), (250, 90, 100), (64, 99, 100)]]),
                 ("test_ring_positional_windows", lambda: [P.test_ring_positional_windows(None, *a) for a in [(1000, 99, 100), (1000, 999, 1000), (1000, 97, 100), (1024, 99, 100), (961, 99, 100), (1000, 50, 100)]]),
                 ("test_ring_special_values", lambda: P.test_ring_special_values(None)),
                 ("test_ring_quantiles_and_alpha", lambda: [P.test_ring_quantiles_and_alpha(None, *a) for a in [(50, 100, 0.1), (0, 1, 0.5), (1, 1, 0.9), (999, 1000, 0.01), (90, 100, 0.0)]]),
                 ("test_ring_push_larger_than_capacity", lambda: P.test_ring_push_larger_than_capacity(None)),
                 ("test_ring_cursor_runs_wrap_and_partial_windows", lambda: [WCUR.test_ring_cursor_runs_wrap_and_partial_windows(W) for W in (1000, 1024)])]
        for name, run in cases:
            current[0] = name
            run()
    finally:
        P.g = None
        if saved is not None:
            sys.modules["gpud_b200"] = saved
        else:
            sys.modules.pop("gpud_b200", None)
    return counter


if __name__ == "__main__":
    total = collections.Counter()
    for name, c in existing_ring_coverage().items():
        total.update(c)
        print("%-48s %s" % (name, dict(sorted(c.items()))))
    print("never reached:", [b for b in BRANCHES if not total[b]])
