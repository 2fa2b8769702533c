"""Model check (numpy only) of the routes of the whole-range order statistic (gpud_ring_reduce_range, gpud_b200/csrc/select.cu and
the RANGE pass of k_window_reduce in ring.cu).  The model restates, per field:
  - k_range_pivots: the sample (sample ring or strided reads), the sample ranks rh / rl with their clamps and the +-inf overrides,
    and the two sample order statistics that become the pivots lo, hi;
  - the fused pass: each sample classified first by the double compares (x > hi counts above; else x >= lo flags it; NaN fails
    both), then the flagged ones exactly on their totalOrder keys (above, == hi, == lo, strictly inside), or all counted as == hi
    when lo and hi are equal and not a zero; per 1024-sample window, plus the list fill;
  - k_range_finish: the outcome (constant, hi, lo, select from the list) or the reason the field stays open;
  - the radix select the open fields (and every non-constant field of a short range) go through: the k_sel_hist / k_sel_pick
    passes that do work, whether the field finishes in pick, how many keys k_sel_collect gathers for k_sel_final's list select
    (the one k_range_finish runs on its list), and which load path for_each_key takes in each block's slice.
The tests check that the model's answer equals a sort of the keys on every case, and that the cases of test_gpu_range_paths.py
reach every route, both sample sources and every load path.  test_gpu_range_paths.py checks the device against the model."""
import collections

import numpy as np

from oracle import pyoracle as O
import range_cases as RC

WP = 1024                      # the range pass's window (kMaxWindow)
COLLECT_MAX = 8192             # kCollectMax
KEY_POS_INF = int(O.total_order_key(np.array([np.inf]))[0])
KEY_NEG_INF = int(O.total_order_key(np.array([-np.inf]))[0])
H100_SMS = 132                 # the H100 SXM5; bpf only depends on it when many fields are open


def _bits(key):
    return int(O.key_to_f64(np.array([key], dtype=np.uint64)).view(np.uint64)[0])


def _f64(key):
    return float(O.key_to_f64(np.array([key], dtype=np.uint64))[0])


def _kth_largest(keys, k):
    """the k-th largest (1-based) of a uint64 key array"""
    return int(np.partition(keys, len(keys) - k)[len(keys) - k])


def pivots(x, pos, k):
    """k_range_pivots for one field: (lo key, hi key, rh, rl, S)"""
    n, S = len(x), len(pos)
    rh, rl = RC.pivot_ranks(n, k, S)
    sk = O.total_order_key(x[pos])
    hik = _kth_largest(sk, max(1, min(S, rh)))
    lok = _kth_largest(sk, max(1, min(S, rl)))
    if rh < 1:
        hik = KEY_POS_INF
    if rl > S:
        lok = KEY_NEG_INF
    return lok, hik, rh, rl, S


def classify(x, keys, lok, hik, wp=WP):
    """the fused pass: per window of wp samples (the last one shorter) [above, == hi, == lo, inside] (uint32 counts, as w_cls)
    and the flags it raised"""
    lo, hi = _f64(lok), _f64(hik)
    with np.errstate(invalid="ignore"):
        above_d = x > hi
        flagged = ~above_d & (x >= lo)
    lok_, hik_ = np.uint64(lok), np.uint64(hik)
    all_equal = lok == hik and hi != 0.0
    if all_equal:
        a, eh, el, ins = above_d, flagged, np.zeros_like(flagged), np.zeros_like(flagged)
    else:
        a = above_d | (flagged & (keys > hik_))
        eh = flagged & (keys == hik_)
        el = flagged & (keys == lok_) & (lok != hik)
        ins = flagged & (keys > lok_) & (keys < hik_)
    starts = np.arange(0, len(x), wp)
    cls = np.stack([np.add.reduceat(v.astype(np.int64), starts) for v in (a, eh, el, ins)], axis=1)
    return cls, ins


def pick_walk(keys, k, kmin, kmax):
    """k_sel_hist / k_sel_pick from k_range_finish's state, then k_sel_collect: (working passes, finished in pick, collected, answer)"""
    n = len(keys)
    diff = kmin ^ kmax
    nbits = 64 - diff.bit_length()
    prefix = kmax >> (64 - nbits) if nbits else 0
    kk, cnt, done, ans, passes = k, n, False, None, 0
    cand = keys
    if n > COLLECT_MAX:
        for _ in range(6):
            if done or cnt <= COLLECT_MAX:
                continue
            passes += 1
            d = min(11, 64 - nbits)
            shift = 64 - nbits - d
            digit = ((cand >> np.uint64(shift)) & np.uint64((1 << d) - 1)).astype(np.int64)
            hist = np.bincount(digit, minlength=1 << d)
            above = np.cumsum(hist[::-1])                    # keys in this bin or higher, from the top bin down
            j = int(np.searchsorted(above, kk))              # first bin from the top whose running count reaches kk
            b = (1 << d) - 1 - j
            acc = int(above[j - 1]) if j else 0
            prefix = ((prefix << d) if nbits else 0) | b
            nbits += d
            kk -= acc
            cand = cand[digit == b]
            cnt = len(cand)
            if nbits >= 64:
                done, ans = True, prefix
    if done:
        return passes, True, 0, ans
    return passes, False, len(cand), _kth_largest(cand, kk)


def load_paths(cap, start, n, bpf):
    """for_each_key in each of the bpf block slices: ('128', odd tail?) for an aligned run that does not wrap, else ('64', None)"""
    per = ((n + bpf - 1) // bpf + 1) & ~1
    out = []
    for blk in range(bpf):
        b = min(n, blk * per)
        e = min(n, b + per)
        p0 = start + b
        if p0 >= cap:
            p0 -= cap
        ln = e - b
        if ln > 0 and p0 + ln <= cap and p0 % 2 == 0:
            out.append(("128", ln % 2 == 1))
        else:
            out.append(("64", None))
    return out


def model_field(x, cap, start, q_num, q_den, pos=None):
    """everything the model predicts for one field of a range; pos = the sample positions (None: a short range)"""
    n = len(x)
    keys = O.total_order_key(x)
    k = RC.k_from_top(n, q_num, q_den)
    kmin, kmax = int(keys.min()), int(keys.max())
    m = dict(k=k, kmin=kmin, kmax=kmax, answer=_kth_largest(keys, k))
    if pos is not None:                                  # the pivots and the pass run for every field, constant ones too
        lok, hik, rh, rl, S = pivots(x, pos, k)
        cls, ins = classify(x, keys, lok, hik)
        tot = cls.sum(axis=0)
        c_abv, c_eh, c_el = int(tot[0]), int(tot[1]), int(tot[2])
        fill = int(tot[3])
        list_cap = min(RC.LIST_CAP, n)
        m.update(lo=_bits(lok), hi=_bits(hik), rh=rh, rl=rl, S=S, cls=cls, fill=fill)
    if kmin == kmax:
        m.update(route="const", open=False)
        return m
    if pos is None:
        m.update(route="short", open=True)
    else:
        route = None
        if kmax > KEY_POS_INF:
            route = "nan"
        elif not lok <= hik:
            route = "pivots"
        elif k <= c_abv:
            route = "above"
        elif k <= c_abv + c_eh:
            route, m["settled"] = "hi", hik
        elif k <= c_abv + c_eh + fill:
            if fill <= list_cap:
                route, m["settled"] = "list", _kth_largest(keys[ins], k - c_abv - c_eh)
            else:
                route = "overflow"
        elif k <= c_abv + c_eh + fill + c_el:
            route, m["settled"] = "lo", lok
        else:
            route = "below"
        m.update(route=route, open=route not in ("hi", "lo", "list"))
    if m["open"]:
        passes, in_pick, collected, ans = pick_walk(keys, k, kmin, kmax)
        m.update(passes=passes, in_pick=in_pick, collected=collected, settled=ans)
    return m


def model_ring(cap, pushed, last_n, q_num, q_den, xs, sm_count=H100_SMS):
    """the model over one ring's fields xs[F][n] (chronological newest n): per-field dicts, the open count and reasons of
    range_stats (sampled ranges), and for_each_key's slices for the radix select's launch"""
    n = xs.shape[1]
    start = RC.range_start(cap, pushed, n)
    sampled = n >= RC.SAMPLED_MIN
    src, pos = RC.sample_positions(cap, start, n) if sampled else (None, None)
    fields = [model_field(x, cap, start, q_num, q_den, pos) for x in xs]
    n_sel = sum(f["open"] for f in fields) if sampled else len(fields)
    bpf = max(1, min((n + 16383) // 16384, max(1, 8 * sm_count // max(1, n_sel) + 1)))
    reasons = collections.Counter(f["route"] for f in fields if f["open"]) if sampled else None
    paths = load_paths(cap, start, n, bpf) if n_sel else []
    return dict(n=n, start=start, source=src, S=len(pos) if sampled else None, fields=fields, n_open=n_sel if sampled else None,
                reasons=reasons, paths=paths, nw=(n + WP - 1) // WP)


# ------------------------------------------------------------------------------------------------ tests
_MODELS = {}


def sampled_models():
    """every sampled case of the GPU file through the model (cached: the GPU file reuses them)"""
    if "sampled" not in _MODELS:
        out = []
        for shape, qn, qd in RC.cases():
            flds = RC.ring_fields(shape, qn, qd)
            xs = np.stack([x for _, _, x in flds])
            out.append((shape, qn, qd, flds, model_ring(shape["cap"], shape["pushed"], RC.shape_n(shape), qn, qd, xs)))
        _MODELS["sampled"] = out
    return _MODELS["sampled"]


def short_models():
    if "short" not in _MODELS:
        _MODELS["short"] = [(c, model_ring(c[1], c[2], c[3], c[4], c[5], c[6])) for c in RC.short_cases()]
    return _MODELS["short"]


def test_sample_positions_follow_the_kernel():
    """the sample ring: column c with c mod 2^s = 2^(s-1), c < cap, inside the range; strided: S = min(8192, n / 8)"""
    assert RC.smp_shift(1 << 20) == 7 and RC.smp_shift(1 << 17) == 4 and RC.smp_shift(1000000) == 7
    src, pos = RC.sample_positions(1000000, 0, 1000000)
    assert src == "ring" and len(pos) == 7812                     # slot 7812 mirrors column 1 000 000: past cap
    src, pos = RC.sample_positions(1 << 20, (1 << 20) - 262144, 262144)
    assert src == "ring" and len(pos) == 2048 and np.all(pos % 128 == 64)
    assert RC.sample_positions(1 << 20, 0, 262143)[0] == "strided"
    src, pos = RC.sample_positions(1 << 20, 0, 65536)
    assert src == "strided" and len(pos) == 8192 and pos[0] == 4 and pos[-1] == 65532
    cap, start, n = 1 << 18, 189921, 150000                       # a wrapped range: columns below start map to c - start + cap
    src, pos = RC.sample_positions(cap, start, n)
    cols = (start + pos) % cap
    assert src == "ring" and np.all(cols % 32 == 16) and np.any(cols < start) and np.all(pos < n)
    assert len(pos) == sum(1 for c in range(16, cap, 32) if (c - start) % cap < n)


def test_model_answer_equals_a_sort():
    """whatever the route, the model's answer is the k-th largest key of a full sort, and settled fields agree with it"""
    for shape, qn, qd, flds, mr in sampled_models():
        for (name, _, x), f in zip(flds, mr["fields"]):
            want = int(np.sort(O.total_order_key(x))[len(x) - f["k"]])
            assert f["answer"] == want, (shape["name"], qn, qd, name)
            if "settled" in f:
                assert f["settled"] == want, (shape["name"], qn, qd, name, f["route"])
    for c, mr in short_models():
        for x, f in zip(c[6], mr["fields"]):
            assert f.get("settled", f["answer"]) == int(np.sort(O.total_order_key(x))[len(x) - f["k"]]), c[0]


def test_each_generator_takes_its_route():
    for shape, qn, qd, flds, mr in sampled_models():
        for (name, route, _), f in zip(flds, mr["fields"]):
            assert f["route"] == route, (shape["name"], qn, qd, name, f["route"])


def test_every_route_and_source_is_reached():
    routes = collections.Counter()
    sources = collections.Counter()
    corners = collections.Counter()
    for shape, qn, qd, flds, mr in sampled_models():
        sources[mr["source"]] += 1
        for f in mr["fields"]:
            routes[f["route"]] += 1
            corners["rh<1"] += f["rh"] < 1
            corners["rl>S"] += f["rl"] > f["S"]
            corners["rl==S"] += f["rl"] == f["S"]
            hi = np.array([f["hi"]], dtype=np.uint64).view(np.float64)[0]
            lo = np.array([f["lo"]], dtype=np.uint64).view(np.float64)[0]
            corners["hi=+0"] += f["hi"] == 0
            corners["hi=-0"] += f["hi"] == 1 << 63
            corners["lo=hi=+0"] += f["hi"] == 0 and f["lo"] == 0
            corners["all_equal"] += f["lo"] == f["hi"] and hi != 0.0
            corners["hi=+inf"] += hi == np.inf
            corners["lo=-inf"] += lo == -np.inf
    for r in ("list", "hi", "lo", "above", "below", "overflow", "nan", "pivots", "const"):
        assert routes[r] >= 3, (r, routes)
    assert sources["ring"] >= 3 and sources["strided"] >= 3, sources
    for c in ("rh<1", "rl>S", "rl==S", "hi=+0", "hi=-0", "lo=hi=+0", "all_equal", "hi=+inf", "lo=-inf"):
        assert corners[c] >= 1, (c, corners)


def test_pivots_reason_needs_negative_nan():
    """PIVOTS (lo above hi) happens only when rl > S forces lo = -inf over an upper pivot that is a -NaN: the sample's order
    statistics themselves are always ordered.  Only the -NaN generator gets there."""
    for shape, qn, qd, flds, mr in sampled_models():
        for (name, _, x), f in zip(flds, mr["fields"]):
            if f["route"] == "pivots":
                assert name == "pivots" and f["rl"] > f["S"] and f["rh"] >= 1
                assert np.isnan(np.array([f["hi"]], dtype=np.uint64).view(np.float64)[0]) and f["hi"] >> 63 == 1
                assert f["lo"] == 0xFFF0000000000000


def test_radix_select_paths_are_reached():
    """both load paths of for_each_key (and an odd tail on the 128-bit one), 0 / 1 / >= 2 working histogram passes, a field
    finished in k_sel_pick, and fields whose rank lies in a collected list"""
    paths, passes, in_pick, collected = set(), collections.Counter(), 0, 0
    for mr in [m for *_, m in sampled_models()] + [m for _, m in short_models()]:
        paths.update(mr["paths"])
        for f in mr["fields"]:
            if f["open"]:
                passes[min(2, f["passes"])] += 1
                in_pick += f["in_pick"]
                collected += not f["in_pick"]
    assert ("128", False) in paths and ("128", True) in paths and ("64", None) in paths, paths
    assert passes[0] >= 1 and passes[1] >= 1 and passes[2] >= 1, passes
    assert in_pick >= 1 and collected >= 1


def test_short_ranges_cover_their_shapes():
    for c, mr in short_models():
        assert mr["n"] < RC.SAMPLED_MIN and mr["source"] is None
    starts = [mr["start"] for _, mr in short_models()]
    ns = [mr["n"] for _, mr in short_models()]
    assert any(s % 2 for s in starts) and any(n % 2 for n in ns) and any(n <= COLLECT_MAX for n in ns)
    assert any(mr["start"] + mr["n"] > c[1] for c, mr in short_models())            # a range that wraps
    assert any(f["kmin"] >> 63 == 0 and f["kmax"] >> 63 == 1 for _, mr in short_models() for f in mr["fields"])   # cp = 0


if __name__ == "__main__":
    for shape, qn, qd, flds, mr in sampled_models():
        print(shape["name"], "%d/%d" % (qn, qd), mr["source"], mr["S"], "open", mr["n_open"], dict(mr["reasons"]),
              [f["route"] for f in mr["fields"]])
