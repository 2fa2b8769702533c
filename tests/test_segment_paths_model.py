"""Model check (no GPU) of the segment select of gpud_ring_reduce_ranges' long route and of span / hop handles with L > 1024
(gpud_ring_segments), and of the short route's order-statistic branches (k_ranges_short).  The model restates, per segment:
  - its pivot sample: the ring's sample ring when len >> smp_shift >= 2048 (range_cases.sample_positions), else
    S = clamp(len / 32, 64, 8192) strided reads at j stride + stride / 2; the list capacity seg_list_cap(len, S, k) with S = len >>
    smp_shift for the sample ring (the estimate ranges_plan and gpud_ring_segments size the list with, not the slots that fall in);
  - the pivots and the classification of test_range_paths_model.py on the segment's rows: 1024-sample tiles from the range's first
    sample (the last one shorter) for ranges, sub-windows of Wp for handles; the finish's route with the segment's own list capacity;
  - the long route's host plan: start columns, the flat tile list and the 1 GiB batches;
  - the short route: lane l holds t = 64 j + 2 l + {0, 1} whatever the load path, an empty lane's maximum is key 0; k > 32 takes the
    bit search, else L = the k-th largest lane maximum and cnt = the keys above it decide: cnt < k the bound, cnt <= 32 the
    candidate select, else the bit search.
The tests check that the model's answers equal a sort, that the data the GPU file builds takes the route it is built for in every
geometry that file uses, and that every route and branch is reached.  test_gpu_segment_paths.py checks the device against it."""
import collections
import ctypes as C

import numpy as np
import pytest

import range_cases as RC
import window_cases as WC
from oracle import pyoracle as O
from test_range_paths_model import KEY_POS_INF, _bits, _kth_largest, classify, pivots
from test_ring_windows_model import gen_overflow, seg_list_cap, windows_sub

TILE = 1024                                   # GPUD_MAX_WINDOW: the long route's tiles
OPEN = ("nan", "pivots", "above", "below", "overflow")
BATCH_BYTES = 1 << 30                         # kRangesBatchBytes
SEL_STATE_BYTES = 40                          # sizeof(SelState)
GENS = {name: (fn, route) for name, fn, route in RC.GENERATORS}
NAMES = [name for name, _, _ in RC.GENERATORS]


# ------------------------------------------------------------------------------------------------ one segment
def seg_geometry(cap, start, n, q):
    """a segment of n samples from physical column start under quantile q: its rank, sample source and positions, list capacity"""
    k = RC.k_from_top(n, q[0], q[1])
    if (n >> RC.smp_shift(cap)) >= 2048:
        src, pos = RC.sample_positions(cap, start, n)
        s_est = n >> RC.smp_shift(cap)
    else:
        S = min(RC.SAMPLE_MAX, max(64, n // 32))
        stride = n // S
        src, pos, s_est = "strided", np.arange(S, dtype=np.int64) * stride + stride // 2, S
    assert src == ("ring" if (n >> RC.smp_shift(cap)) >= 2048 else "strided")
    return dict(n=n, start=start, k=k, src=src, pos=pos, lcap=seg_list_cap(n, s_est, k))


def model_segment(x, geo, wp=TILE):
    """k_range_pivots, the pass's class counts per row of wp samples and k_range_finish on one segment"""
    keys = O.total_order_key(x)
    k = geo["k"]
    lok, hik, _, _, _ = pivots(x, geo["pos"], k)
    cls, ins = classify(x, keys, lok, hik, wp)
    a, eh, el, fill = (int(v) for v in cls.sum(axis=0))
    m = dict(lo=_bits(lok), hi=_bits(hik), fill=fill, cls=cls, answer=_kth_largest(keys, k))
    if keys.min() == keys.max():
        route = "const"
    elif int(keys.max()) > KEY_POS_INF:
        route = "nan"
    elif not lok <= hik:
        route = "pivots"
    elif k <= a:
        route = "above"
    elif k <= a + eh:
        route, m["settled"] = "hi", hik
    elif k <= a + eh + fill:
        if fill <= geo["lcap"]:
            route, m["settled"] = "list", _kth_largest(keys[ins], k - a - eh)
        else:
            route = "overflow"
    elif k <= a + eh + fill + el:
        route, m["settled"] = "lo", lok
    else:
        route = "below"
    m["route"] = route
    return m


def gauge(n, seed):
    return np.random.default_rng(seed).normal(60.0, 3.0, n)


def build(name, geo, seed):
    """generator `name` of range_cases.GENERATORS built against the segment's sample and list capacity: (x, the route it is built
    for), or (a gauge, None) where it cannot be built in this geometry"""
    L = RC.Layout(geo["n"], geo["pos"], geo["k"], np.random.default_rng(seed))
    fn, route = GENS[name]
    x = gen_overflow(L, geo["lcap"]) if name == "overflow" else fn(L)
    if x is None:
        return gauge(geo["n"], seed), None
    return x, (route(L) if callable(route) else route)


def reasons_of(models):
    return dict(collections.Counter(m["route"] for m in models if m["route"] in OPEN))


# ------------------------------------------------------------------------------------------------ the long route's host plan
def ranges_plan(cap, F, q, firsts, lens):
    """ranges_plan: start columns, route (0 short, 1 + batch), the flat tile list (range, column, samples) and each long range's
    (batch, first tile of the call's flat list)"""
    start = [int(f) % cap for f in firsts]
    route, tiles, tile_of = [], [], {}
    batch, nbytes, in_batch = 0, 0, 0
    for i, n in enumerate(lens):
        n = int(n)
        if n <= TILE:
            route.append(0)
            continue
        geo = seg_geometry(cap, start[i], n, q)
        nt = -(-n // TILE)
        b = F * (nt * 52 + geo["lcap"] * 8 + 16 + 4 + 40 + 4 + SEL_STATE_BYTES + 4 + 8)
        if in_batch and nbytes + b > BATCH_BYTES:
            batch, nbytes, in_batch = batch + 1, 0, 0
        nbytes += b
        in_batch += 1
        route.append(batch + 1)
        tile_of[i] = len(tiles)
        tiles += [(i, (start[i] + t * TILE) % cap, min(TILE, n - t * TILE)) for t in range(nt)]
    return dict(start=start, route=route, tiles=tiles, tile_of=tile_of)


def plan_hook(total, cap, F, q, firsts, lens):
    """gpudh_ring_ranges_plan"""
    import gpud_b200 as g
    fn = g.lib().gpudh_ring_ranges_plan
    fn.restype = C.c_int32
    fn.argtypes = [C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                   C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
    first = np.ascontiguousarray(firsts, dtype=np.int64)
    ln = np.ascontiguousarray(lens, dtype=np.int64)
    n = len(first)
    start = np.empty(n, np.int64)
    route = np.empty(n, np.int32)
    nt = C.c_int64()
    cap_t = int(sum(-(-int(v) // TILE) for v in ln if v > TILE))
    tiles = np.empty((max(1, cap_t), 3), np.int64)
    assert fn(total, cap, F, q[0], q[1], first.ctypes.data, ln.ctypes.data, n, start.ctypes.data, route.ctypes.data, tiles.ctypes.data,
              cap_t, C.byref(nt)) == 0
    return start, route, tiles[:nt.value]


# ------------------------------------------------------------------------------------------------ the GPU file's geometries
QUANTILES = RC.QUANTILES

# test_range_segment_routes: one ring of CAP = 1 Mi; long ranges at even and odd columns, one across the physical end
RANGE_CAP = 1 << 20
RANGE_LENS = [1025, 1100, 2047, 4097, 65535, 65537, 300001, 200001, 262144]   # 262144 >> 7 = 2048: the sample ring; 300001 too
RANGE_PARITY = [0, 1, 0, 1, 1, 0, 1, 0, 0]
RANGE_CROSS = 6                                                                # the range across the physical end


def range_layout():
    """(cap, samples pushed, first sample of each range): disjoint, in the held samples, the wanted column parities"""
    cap = RANGE_CAP
    before = sum(RANGE_LENS[:RANGE_CROSS]) + 2 * RANGE_CROSS
    oldest = cap - before - 150000
    firsts, cur = [], oldest + 4
    for n, par in zip(RANGE_LENS, RANGE_PARITY):
        if cur % 2 != par:
            cur += 1
        firsts.append(cur)
        cur += n + 1
    total = cap + oldest
    assert cur <= total and firsts[RANGE_CROSS] < cap < firsts[RANGE_CROSS] + RANGE_LENS[RANGE_CROSS]
    return cap, total, firsts


def range_fields(q, seed=0):
    """the fields of test_range_segment_routes: x[F][held samples] (sample total - cap first) and per (field, range) (generator,
    the route it is built for, geometry); field f of range j holds generator (f + j) % G"""
    cap, total, firsts = range_layout()
    F, oldest = len(NAMES), total - cap
    x = np.stack([gauge(cap, [seed, 99, f]) for f in range(F)])
    segs = {}
    for j, (first, n) in enumerate(zip(firsts, RANGE_LENS)):
        geo = seg_geometry(cap, first % cap, n, q)
        for f in range(F):
            name = NAMES[(f + j) % F]
            xf, route = build(name, geo, [seed, f, j, q[0], q[1]])
            x[f, first - oldest:first - oldest + n] = xf
            segs[f, j] = (name, route, geo)
    return x, segs


# test_handle_segment_routes: (name, W, span, hop, cap, pushes); every window of the last reduce built against its own sample (a hop
# handle: the windows of its last phase, which are tumbling)
HANDLE_SHAPES = [
    ("W1000_s10", 1000, 10, 10, 200000, (80000, 120000)),            # strided, S = 312, Wp = 1000
    ("W7_s600", 7, 600, 600, 50400, (16800, 33600)),                 # strided, S = 131, Wp = 840 (not a multiple of 64)
    ("W1024_s256", 1024, 256, 256, 1 << 20, (1 << 19, 1 << 19)),     # L = 256 Ki: the sample ring, S = 2048
    ("W1000_s20_h5", 1000, 20, 5, 200000, (100000, 100000)),         # hopping: four phases, the last one checked
]
HANDLE_Q = (99, 100)


def handle_windows(W, span, hop, cap, pushes):
    """per reduce (one after each push): (first new window, new windows, the windows of its last phase)"""
    L, P, p = W * span, W * hop, span // hop
    out, total, nxt = [], 0, 0
    for n in pushes:
        total += n
        assert total <= cap                                            # nothing is lost: the plan is the complete windows
        complete = 0 if total < L else (total - L) // P + 1
        n_new = complete - nxt
        r = min(p, n_new) - 1
        out.append((nxt, n_new, list(range(nxt + r, complete, p))))
        nxt = complete
    return out


def handle_fields(shape, seed=0):
    """x[F][samples pushed] for a handle shape and per (field, window) of every built window (generator, route, geometry)"""
    _, W, span, hop, cap, pushes = shape
    L, P = W * span, W * hop
    F = len(NAMES)
    total = sum(pushes)
    x = np.stack([gauge(total, [seed, 98, f]) for f in range(F)])
    plan = handle_windows(W, span, hop, cap, pushes)
    built = [k for a, n, _ in plan for k in range(a, a + n)] if hop == span else plan[-1][2]   # hopping windows overlap
    segs = {}
    for k in built:
        geo = seg_geometry(cap, k * P % cap, L, HANDLE_Q)
        for f in range(F):
            name = NAMES[(f + k) % F]
            xf, route = build(name, geo, [seed, f, k])
            x[f, k * P:k * P + L] = xf
            segs[f, k] = (name, route, geo)
    return x, segs


# test_radix_chunks: more open segments than one radix-select chunk (kSelChunk = 4096)
CHUNK = 4096
CHUNK_F, CHUNK_N = 8, 2048
CHUNK_CYCLE = ["nan", "above", "nan", "below", "nan", "overflow", "nan", "nan"]
CHUNK_CASES = [(600, (99, 100)), (600, (3, 5)), (512, (99, 100)), (513, (3, 5))]   # 4800, 4800, 4096, 4097 open segments


def chunk_fields(n_ranges, q, seed=0):
    """F = 8 fields of n_ranges disjoint 2048-sample ranges, one sample apart: (cap, firsts, x[F][cap], segs).  Every segment is forced
    open - mostly by a +NaN the sample does not read, above / below / overflow between them - except, with 513 ranges, fields 1..7 of
    the last range, which hold gauges (4104 - 7 = 4097 open)"""
    cap = n_ranges * (CHUNK_N + 1) + 2
    cap += cap % 2                                                     # a ring's capacity is even
    firsts = [1 + j * (CHUNK_N + 1) for j in range(n_ranges)]
    x = np.stack([gauge(cap, [seed, 97, f]) for f in range(CHUNK_F)])
    segs = {}
    for j, first in enumerate(firsts):
        geo = seg_geometry(cap, first, CHUNK_N, q)
        for f in range(CHUNK_F):
            name = CHUNK_CYCLE[(f * 3 + j) % len(CHUNK_CYCLE)]
            if n_ranges % 2 and j == n_ranges - 1 and f:
                name = "list"
            xf, route = build(name, geo, [seed, f, j])
            if route is None:
                xf, route = build("nan", geo, [seed, f, j])
            x[f, first:first + CHUNK_N] = xf
            segs[f, j] = (name, route, geo)
    return cap, firsts, x, segs


def span_chunk_fields(seed=0):
    """a span handle's catch-up: F = 8, W = 1000, span 2 (L = 2000), 600 windows in one reduce, every segment forced open"""
    W, span, n_win = 1000, 2, 600
    L = W * span
    cap = n_win * L
    x = np.stack([gauge(cap, [seed, 96, f]) for f in range(CHUNK_F)])
    segs = {}
    for k in range(n_win):
        geo = seg_geometry(cap, k * L, L, HANDLE_Q)
        for f in range(CHUNK_F):
            name = CHUNK_CYCLE[(f * 3 + k) % len(CHUNK_CYCLE)]
            xf, route = build(name, geo, [seed, f, k])
            if route is None:
                xf, route = build("nan", geo, [seed, f, k])
            x[f, k * L:(k + 1) * L] = xf
            segs[f, k] = (name, route, geo)
    return W, span, cap, x, segs


# test_long_route_batches: F = 16, CAP = 1 Mi, whole-ring ranges repeated, short ranges and one forced sub-range per batch
BATCH_F, BATCH_CAP = 16, 1 << 20
BATCH_Q = (99, 100)
BATCH_REPEAT = 600
BATCH_SUBS = [(0, 70001, "nan", 0), (270, 150001, "overflow", 1), (540, 100000, "nan", 0)]   # (call index, length, generator, field)


def batch_call(seed=0):
    """(total, x[F][cap] held samples, firsts, lens, {distinct (first, len): segs or None}); the ring has wrapped (total > cap)"""
    cap, F = BATCH_CAP, BATCH_F
    total = cap + 333333
    oldest = total - cap
    x = np.stack([gauge(cap, [seed, 95, f]) for f in range(F)])
    rng = np.random.default_rng([seed, 95])
    firsts, lens = [], []
    subs = {}
    sub_at = {c: (n, name, f) for c, n, name, f in BATCH_SUBS}
    used = []
    for i in range(BATCH_REPEAT):
        if i in sub_at:
            n, name, f = sub_at[i]
            first = oldest + 1000 + len(used) * 200001 + (i % 2)
            used.append(first)
            geo = seg_geometry(cap, first % cap, n, BATCH_Q)
            xf, route = build(name, geo, [seed, 94, i])
            assert route == name
            x[f, first - oldest:first - oldest + n] = xf
            firsts.append(first)
            lens.append(n)
            subs[first, n] = (f, name, route, geo)
        firsts.append(oldest)
        lens.append(cap)
        if i % 10 == 5:
            n = int(rng.choice([1, 2, 33, 700, 1024]))
            firsts.append(int(rng.integers(oldest, total - n + 1)))
            lens.append(n)
    return total, x, firsts, lens, subs


# test_short_route_branches: one field per window kind, ranges of every length at four placements
SHORT_MS = [1024, 1000, 961, 513, 65, 64, 63, 33, 32, 2, 1]
SHORT_QS = [(1, 1), (990, 1000), (969, 1000), (968, 1000), (1, 2), (0, 1), (3, 5)]   # at m = 1000: k = 1, 11, 32, 33, 500, 1000, 401
SHORT_CAP = 16384
KINDS = list(WC.KINDS)


def lane_of(t):
    return (np.asarray(t) & 63) >> 1


def short_branch(x, k):
    """(branch, answer key) of k_ranges_short on one range"""
    keys = O.total_order_key(np.asarray(x, dtype=np.float64))
    ans = _kth_largest(keys, k)
    if k > 32:
        return "bits_rank", ans
    lane_max = np.zeros(32, dtype=np.uint64)
    np.maximum.at(lane_max, lane_of(np.arange(len(keys))), keys)
    L = np.sort(lane_max)[::-1][k - 1]
    cnt = int((keys > L).sum())
    if cnt < k:
        return "bound", int(L)
    return ("select" if cnt <= 32 else "bits_overflow"), ans


def short_reachable(m, k):
    """the branches some data reaches at (m, k): keys above L lie only in the at most k - 1 lanes whose maximum exceeds it, so cnt is
    at most the samples of the k - 1 fullest lanes; the bound is always possible (all equal, or all -NaN)"""
    if k > 32:
        return {"bits_rank"}
    c = np.sort(np.bincount(lane_of(np.arange(m)), minlength=32))[::-1]
    top = int(c[:k - 1].sum())
    out = {"bound"}
    if top >= k:
        out.add("select")
    if top >= 33:
        out.add("bits_overflow")
    return out


def short_calls(q, seed=0):
    """the calls of test_short_route_branches at quantile q.  The ring (cap 16 Ki) first gets 1.5 laps, so the physical end is at
    sample 16 Ki with half a lap on either side; each later call gets one more lap.  Call 0: every length at an even and an odd start
    after the physical end (no wrap) and one wrapping range; every later call one more wrapping range.  -> [(lap samples [F][n],
    [(first, m, kinds per field)])]"""
    cap, F, K = SHORT_CAP, len(KINDS), len(KINDS)
    wraps = [(m, par) for m in SHORT_MS for par in (0, 1) if m >= 3 or (m == 2 and par == 1)]
    calls, total, i = [], 0, 0
    for c, (m_w, par_w) in enumerate(wraps):
        n_push = cap + cap // 2 if c == 0 else cap
        base = total
        total += n_push
        lap = np.stack([gauge(n_push, [seed, 93, c, f]) for f in range(F)])
        end = (total // cap) * cap                                   # the sample at physical column 0
        ranges = []
        places = []
        if c == 0:
            cur = end + 2
            for m in SHORT_MS:
                for par in (0, 1):
                    if cur % 2 != par:
                        cur += 1
                    places.append((cur, m))
                    cur += m + 1
            assert cur <= total
        a = m_w // 2
        if (cap - a) % 2 != par_w:
            a = a + 1 if a + 1 <= m_w - 1 else a - 1
        assert 1 <= a <= m_w - 1 and (end - a) % 2 == par_w
        places.append((end - a, m_w))
        for first, m in places:
            k = WC.k_of(m, q[0], q[1])
            kinds = [KINDS[(f + i) % K] for f in range(F)]
            for f in range(F):
                lap[f, first - base:first - base + m] = WC.window(kinds[f], m, k, (seed, i % 3))
            ranges.append((first, m, kinds))
            i += 1
        calls.append((lap, ranges))
    return calls


# ------------------------------------------------------------------------------------------------ tests
_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def range_models(q):
    def run():
        x, segs = range_fields(q)
        cap, total, firsts = range_layout()
        oldest = total - cap
        out = {}
        for (f, j), (name, route, geo) in segs.items():
            out[f, j] = model_segment(x[f, firsts[j] - oldest:firsts[j] - oldest + RANGE_LENS[j]], geo)
        return x, segs, out
    return _cached(("range", q), run)


def test_segment_sample_rules():
    """the strided rule and the sample ring's, the list capacity from len >> smp_shift (not the slots inside the segment)"""
    g = seg_geometry(1 << 20, 0, 10000, (99, 100))
    assert g["src"] == "strided" and len(g["pos"]) == 312 and g["pos"][0] == 16 and g["pos"][-1] == 311 * 32 + 16
    g = seg_geometry(1 << 20, 0, 1025, (99, 100))
    assert len(g["pos"]) == 64 and g["pos"][1] - g["pos"][0] == 16          # S = 64 at least
    g = seg_geometry(1 << 24, 0, 400000, (99, 100))                          # 400000 >> 11 = 195 slots
    assert g["src"] == "strided" and len(g["pos"]) == 8192                # at most 8192
    g = seg_geometry(1 << 20, 12345, 262144, (99, 100))
    assert g["src"] == "ring" and len(g["pos"]) == 2048
    assert g["lcap"] == seg_list_cap(262144, 2048, g["k"])
    g = seg_geometry(1 << 20, 64 * 1001, 300001, (99, 100))                  # 2343 slots by the estimate
    assert g["src"] == "ring" and g["lcap"] == seg_list_cap(300001, 300001 >> 7, g["k"])
    assert abs(len(g["pos"]) - (300001 >> 7)) <= 1


@pytest.mark.parametrize("q", QUANTILES)
def test_range_generators_take_their_routes(q):
    """in every range of the ring: each generator that can be built takes its route, and the model's answer is a sort's"""
    x, segs, models = range_models(q)
    cap, total, firsts = range_layout()
    oldest = total - cap
    for (f, j), (name, route, geo) in segs.items():
        m = models[f, j]
        xf = x[f, firsts[j] - oldest:firsts[j] - oldest + geo["n"]]
        assert m["answer"] == int(np.sort(O.total_order_key(xf))[geo["n"] - geo["k"]])
        if "settled" in m:
            assert m["settled"] == m["answer"], (name, m["route"])
        if route is not None:
            assert m["route"] == route, (q, name, geo["n"], m["route"])
        assert m["cls"].shape == (-(-geo["n"] // TILE), 4) and int(m["cls"].sum()) <= geo["n"]


def test_every_route_and_source_is_reached():
    routes, sources = collections.Counter(), collections.Counter()
    for q in QUANTILES:
        _, segs, models = range_models(q)
        for key, (_, _, geo) in segs.items():
            routes[models[key]["route"]] += 1
            sources[geo["src"]] += 1
    for r in ("const", "hi", "lo", "list", "above", "below", "overflow", "nan", "pivots"):
        assert routes[r] >= 2, (r, routes)
    assert sources["ring"] and sources["strided"]


def test_range_plan_agrees_with_the_library():
    """start columns, routes, the flat tile list (the last tile of each range shorter) and the batch split, model against
    gpudh_ring_ranges_plan"""
    cap, total, firsts = range_layout()
    cases = [(total, cap, len(NAMES), (99, 100), firsts, RANGE_LENS)]
    bt, _, bf, bl, _ = _cached("batch", batch_call)
    cases.append((bt, BATCH_CAP, BATCH_F, BATCH_Q, bf, bl))
    for nr, q in CHUNK_CASES[:1]:
        c_cap, c_firsts, _, _ = _cached(("chunk", nr, q), lambda: chunk_fields(nr, q))
        cases.append((c_cap, c_cap, CHUNK_F, q, c_firsts, [CHUNK_N] * nr))
    for tot, cp, F, q, fs, ls in cases:
        pl = ranges_plan(cp, F, q, fs, ls)
        start, route, tiles = plan_hook(tot, cp, F, q, fs, ls)
        assert list(start) == pl["start"]
        assert list(route) == pl["route"]
        assert [tuple(int(v) for v in t) for t in tiles] == pl["tiles"]
    pl = ranges_plan(BATCH_CAP, BATCH_F, BATCH_Q, bf, bl)
    assert max(pl["route"]) >= 3                                       # the batch call splits into three batches or more


def test_batch_call_forces_one_range_per_batch():
    total, x, firsts, lens, subs = _cached("batch", batch_call)
    pl = ranges_plan(BATCH_CAP, BATCH_F, BATCH_Q, firsts, lens)
    batches = collections.Counter(pl["route"][i] for i, (f, n) in enumerate(zip(firsts, lens)) if (f, n) in subs)
    assert sorted(batches) == list(range(1, max(pl["route"]) + 1)) and set(batches.values()) == {1}
    oldest = total - BATCH_CAP
    for (first, n), (f, name, route, geo) in subs.items():
        m = model_segment(x[f, first - oldest:first - oldest + n], geo)
        assert m["route"] == route == name


@pytest.mark.parametrize("shape", HANDLE_SHAPES, ids=[s[0] for s in HANDLE_SHAPES])
def test_handle_generators_take_their_routes(shape):
    name, W, span, hop, cap, pushes = shape
    L = W * span
    Wp = windows_sub(W, span)
    x, segs = _cached(("handle", name), lambda: handle_fields(shape))
    reached = set()
    for (f, k), (gen, route, geo) in segs.items():
        m = model_segment(x[f, k * W * hop:k * W * hop + L], geo, Wp)
        assert m["cls"].shape == (L // Wp, 4)
        if route is not None:
            assert m["route"] == route, (name, gen, m["route"])
        reached.add(m["route"])
    assert {"list", "nan", "const", "below", "overflow"} <= reached, reached
    if name == "W1024_s256":
        assert next(iter(segs.values()))[2]["src"] == "ring"
    plan = handle_windows(W, span, hop, cap, pushes)
    assert all(len(last) >= 2 for _, _, last in plan)


@pytest.mark.parametrize("case", CHUNK_CASES, ids=["%d-q%d_%d" % (n, q[0], q[1]) for n, q in CHUNK_CASES])
def test_chunk_cases_open_every_segment(case):
    n_ranges, q = case
    cap, firsts, x, segs = _cached(("chunk", n_ranges, q), lambda: chunk_fields(n_ranges, q))
    models = [model_segment(x[f, firsts[j]:firsts[j] + CHUNK_N], geo) for (f, j), (_, _, geo) in segs.items()]
    n_open = sum(m["route"] in OPEN for m in models)
    assert n_open == {600: 4800, 512: 4096, 513: 4097}[n_ranges], n_open
    why = reasons_of(models)
    assert why["nan"] > n_open // 2 and len(why) >= 3, why
    # every chunk of 4096 open segments mixes reasons (4097: the second chunk is one segment)
    order = [m["route"] for m in models if m["route"] in OPEN]
    for c0 in range(0, len(order), CHUNK):
        assert len(set(order[c0:c0 + CHUNK])) >= min(2, len(order) - c0)


def test_span_chunk_opens_every_segment():
    W, span, cap, x, segs = _cached("span_chunk", span_chunk_fields)
    L = W * span
    models = [model_segment(x[f, k * L:(k + 1) * L], geo, W) for (f, k), (_, _, geo) in segs.items()]
    assert all(m["route"] in OPEN for m in models) and len(models) == 4800
    assert len(reasons_of(models)) >= 3


def test_short_branch_model_answers_a_sort():
    rng = np.random.default_rng(1)
    for m in SHORT_MS:
        for k in sorted({1, min(m, 2), min(m, 11), min(m, 32), min(m, 33), max(1, m // 2), m}):
            for _ in range(3):
                x = rng.normal(0.0, 1.0, m)
                x[rng.random(m) < 0.3] = 0.5
                br, ans = short_branch(x, k)
                assert ans == int(np.sort(O.total_order_key(x))[m - k]), (m, k, br)
                assert br in short_reachable(m, k), (m, k, br)


def test_short_cases_reach_every_branch():
    """at m = 1024, 1000, 961, 513 and 65 every branch; at the shorter lengths every branch the model says is reachable"""
    reached = collections.defaultdict(set)
    reachable = collections.defaultdict(set)
    for q in SHORT_QS:
        for m in SHORT_MS:
            reachable[m] |= short_reachable(m, WC.k_of(m, q[0], q[1]))
        for _, ranges in short_calls(q):
            for first, m, kinds in ranges:
                k = WC.k_of(m, q[0], q[1])
                for kind in set(kinds):
                    br, ans = short_branch(WC.window(kind, m, k, (0, 0)), k)
                    reached[m].add(br)
    every = {"bound", "select", "bits_overflow", "bits_rank"}
    for m in (1024, 1000, 961, 513, 65):
        assert reached[m] == every, (m, reached[m])
    for m in SHORT_MS:
        assert reached[m] == reachable[m], (m, reached[m], reachable[m])
    assert reachable[1] == {"bound"} and reachable[2] == {"bound", "select"} and "bits_overflow" not in reachable[32]


def test_short_calls_place_every_length_four_ways():
    """even and odd starts without a wrap (the 128-bit and 64-bit loads) and across the physical end, each in the held samples"""
    seen = collections.defaultdict(set)
    total = 0
    for c, (lap, ranges) in enumerate(short_calls(SHORT_QS[0])):
        total += lap.shape[1]
        for first, m, _ in ranges:
            assert total - SHORT_CAP <= first and first + m <= total
            col = first % SHORT_CAP
            wrap = col + m > SHORT_CAP
            seen[m].add((col % 2, wrap))
        assert sum(r[0] % SHORT_CAP + r[1] > SHORT_CAP for r in ranges) == 1     # one wrapping range per call
    for m in SHORT_MS:
        want = {(0, False), (1, False)} | ({(0, True)} if m >= 3 else set()) | ({(1, True)} if m >= 2 else set())
        assert seen[m] == want, (m, seen[m])
