"""Model check (no GPU) of the layouts test_gpu_tier_paths.py runs on a tiered ring.  A range call that reaches into the tier reduces on
a virtual ring (ranges.cu reduce_sets_tier): the block rows its tier sets cover, merged and ascending, decoded to columns [1024 j,
1024 (j + 1)), the newest (partial) row copied from the ring, with capacity vcap = rows x 1024, its own sample ring (smp_shift(vcap))
and its fields in groups of G = max(1, min(F, 2^30 // (8 (vcap + ceil(vcap / 2^s))))).  The model restates, per call:
  - the split (tests/ring_tier.py split) against gpudh_ring_tier_split, for every call the GPU file makes;
  - each long range's segment geometry on that virtual ring (test_segment_paths_model.seg_geometry(vcap, vfirst, n, q)), or on the
    ring itself for a range wholly in the ring, and the field data built against it: every generator takes its route, both sample
    sources, every open reason at each quantile used, and a ring-sourced segment whose sample slots lie in the partial newest row;
  - the tier's placement (tests/ring_tier.py Tier) against gpudh_ring_tier_plan at capacities that are not a multiple of 1024, on
    random schedules and on the GPU file's own;
  - the natural group size, which splits the configs[1]-shaped call (F = 64, CAP = 1 000 000, 2.2 M samples) into 60 + 4 fields."""
import collections

import numpy as np
import pytest

import range_cases as RC
import ring_tier as T
import test_segment_paths_model as M
from oracle import pyoracle as O
from test_range_paths_model import _kth_largest
from test_gpu_ring_tier import _nvml
from test_ring_tier_model import _model, _plan, _split
from test_ring_windows_model import seg_list_cap

ROW = T.ROW
GROUP_BYTES = 1 << 30                       # kTierGroupBytes (ranges.cu)


def group_size(F, vcap):
    """fields per decoded group of a virtual ring of vcap samples"""
    s = RC.smp_shift(vcap)
    slots = -(-vcap // (1 << s))
    return max(1, min(F, GROUP_BYTES // (8 * (vcap + slots))))


def virtual(total, cap, t_first, first, length, set_off=None):
    """(route, rows, vfirst, vtotal, vcap) of one call, by the host model"""
    route, rows, vfirst, vtotal = T.split(total, cap, t_first, total // ROW, first, length, set_off)
    return route, rows, vfirst, vtotal, len(rows) * ROW


# ------------------------------------------------------------------------------------------------ routes on the decoded ring
# One ring of CAP = 32 Ki with F = 16 fields (one per generator), its tier opened empty and never evicting.  Call 0 at 190001 samples:
# two ring-sourced ranges wholly in the tier (vcap 151552, shift 5), strided ranges of 1025 and 5001 at odd starts, one across the
# tier/ring boundary and one long range wholly in the ring (its own sample ring, shift 2).  Call 1, after 44171 more samples, at
# 234172 (700 samples into the newest row): a strided range in the tier and a ring-sourced range of 40000 ending at `total` through
# the partial row (vcap 45056, shift 3) - the virtual sample ring call 0 left behind is stale for it.
ROUTE_CAP = 1 << 15
ROUTE_F = len(M.NAMES)
ROUTE_TOTALS = (190001, 234172)
ROUTE_CALLS = (
    ((5, 70001), (70011, 1025), (71041, 68001), (139047, 5001), (190001 - ROUTE_CAP - 3000, 6000), (190001 - ROUTE_CAP + 4001, 20000)),
    ((190007, 3001), (234172 - 40000, 40000)),
)
ROUTE_Q = [(99, 100), (1, 100), (1, 2)]          # pivots (lo = -inf over an upper pivot of -NaN) builds only at (1, 100)


def route_calls():
    """per call: (total, ranges, route, vfirst, vcap) with ranges [(first, n)]"""
    out = []
    for total, ranges in zip(ROUTE_TOTALS, ROUTE_CALLS):
        route, _, vfirst, _, vcap = virtual(total, ROUTE_CAP, 0, [f for f, _ in ranges], [n for _, n in ranges])
        out.append((total, ranges, route, vfirst, vcap))
    return out


def route_fields(q, seed=0):
    """x[F][234172] and per (call, range) of every long range: (geometry, [(generator, the route it is built for)] per field).
    Field f of range j of call c holds generator (f + j + 7 c) % F, built against the range's geometry: the virtual ring's for a
    range that reaches into the tier, the ring's own for one wholly in the ring."""
    F = ROUTE_F
    x = np.stack([M.gauge(ROUTE_TOTALS[-1], [seed, 92, f]) for f in range(F)])
    segs = {}
    for c, (total, ranges, route, vfirst, vcap) in enumerate(route_calls()):
        for j, (first, n) in enumerate(ranges):
            if n <= M.TILE:
                continue
            geo = M.seg_geometry(vcap, vfirst[j], n, q) if route[j] else M.seg_geometry(ROUTE_CAP, first % ROUTE_CAP, n, q)
            built = []
            for f in range(F):
                name = M.NAMES[(f + j + 7 * c) % F]
                xf, r = M.build(name, geo, [seed, c, j, f, q[0], q[1]])
                x[f, first:first + n] = xf
                built.append((name, r))
            segs[c, j] = (geo, built)
    return x, segs


def route_models(x, segs, c):
    """{range j: [model per field]} of call c's long ranges on the data"""
    _, ranges, _, _, _ = route_calls()[c]
    return {j: [M.model_segment(x[f, ranges[j][0]:ranges[j][0] + ranges[j][1]], segs[c, j][0]) for f in range(x.shape[0])]
            for j in range(len(ranges)) if (c, j) in segs}


def scratch_models(models, ranges, route, f0, F):
    """what gpudh_ring_segment_scratch holds after a tier call whose last segment select ran the tier sets' long ranges of fields
    [f0, F): ({(segment, first row): model}, segments, rows); segment (f - f0) n_long + j, its rows from (f - f0) n_tiles + tile0"""
    long = [j for j in range(len(ranges)) if route[j] and ranges[j][1] > M.TILE]
    nt = [-(-ranges[j][1] // M.TILE) for j in long]
    n_tiles = sum(nt)
    out = {}
    for f in range(f0, F):
        t0 = 0
        for i, j in enumerate(long):
            out[(f - f0) * len(long) + i, (f - f0) * n_tiles + t0] = models[j][f]
            t0 += nt[i]
    return out, (F - f0) * len(long), (F - f0) * n_tiles


def _route_cache(q):
    return M._cached(("tier_routes", q), lambda: route_fields(q))


# ------------------------------------------------------------------------------------------------ a set of pieces in the tier
# test_gpu_ring_range_sets.test_radix_reasons on a tiered ring: one set of six pieces in reverse push order (the newest two in the
# partial row, one across the tier/ring boundary, the rest in the tier), given twice, on a ring of CAP = 16 Ki.
SETS_CAP, SETS_N, SETS_Q = 1 << 14, 100001, (99, 100)
SETS_TOTAL = 118 * ROW + 500
SETS_CUTS = (0, 1, 1057, SETS_N // 3, SETS_N // 3 + 1024, SETS_N - 31, SETS_N)


def sets_layout(seed=0):
    """(pieces [(first, len)], pos, k, built [(route, x of the concatenation)]): the data built against the set's strided sample"""
    n, q = SETS_N, SETS_Q
    S = min(RC.SAMPLE_MAX, max(64, n // 32))
    stride = n // S
    pos = np.arange(S, dtype=np.int64) * stride + stride // 2
    k = RC.k_from_top(n, *q)
    built = []
    for i, (name, fn, route) in enumerate(RC.GENERATORS):
        Lay = RC.Layout(n, pos, k, np.random.default_rng([seed, i, n, 91]))
        xf = fn(Lay)
        if xf is not None:
            built.append((route(Lay) if callable(route) else route, xf))
    pieces, cur = [], SETS_TOTAL
    for a, b in zip(SETS_CUTS[:-1], SETS_CUTS[1:]):
        cur -= b - a
        pieces.append((cur, b - a))
    return pieces, pos, k, built


def sets_geo(pos, k):
    return dict(n=SETS_N, start=0, k=k, src="strided", pos=pos, lcap=seg_list_cap(SETS_N, len(pos), k))


# ------------------------------------------------------------------------------------------------ configs[1]: natural groups
# F = 64, CAP = 1 000 000, NVML-like uint32 pushed in 10 000-row chunks and odd sizes, a tier that never evicts (max_row_bytes per
# row).  Call A at 2 000 300: the newest row [1999872, 2000300) crosses the physical end at sample 2e6.  Call B at 2 213 457: the
# range [0, total) covers 2162 rows, vcap 2 213 888, shift 9: groups of 60 + 4.
C1_F, C1_CAP = 64, 1000000
C1_TOTALS = (2000300, 2213457)
C1_CHUNKS = (10000, 10000, 10000, 7777, 10000, 1, 10000, 10000, 3001, 1023)


def c1_schedule():
    """the pushes up to each call total, in order: [pushes before call A, pushes between A and B]"""
    out, total = [], 0
    for end in C1_TOTALS:
        pushes, i = [], 0
        while total < end:
            n = min(C1_CHUNKS[i % len(C1_CHUNKS)], end - total)
            pushes.append(n)
            total += n
            i += 1
        out.append(pushes)
    return out


def c1_tier_bytes():
    return T.max_row_bytes(C1_F) * (C1_TOTALS[-1] // ROW + 2)


def c1_calls():
    """per call: (total, [(first, n)]); every range starts in [lo, total) with lo = 0 (nothing evicted)"""
    cap = C1_CAP
    a, b = C1_TOTALS
    call_a = [(a - cap - 5, cap + 5),                     # from the tier through the newest row, copied across the physical end
              (0, a), (cap - 300, 600), (a - 1, 1)]
    call_b = [(0, b),                                      # every row: 60 + 4 fields per group
              (0, 1), (0, 1025), (1, 70001),               # at lo
              (b - cap, 5000), (b - cap - 1, 2), (b - cap - 777, 3000),   # at the ring's unaligned first sample and across it
              (cap - 300, 600), (cap - 5000, 12345),       # in the tier across the old physical end: rows coded across it
              (2 * cap - 777, 1500),                       # in the ring across its physical end
              (b - 1500, 1500), (b - cap - 10, cap + 10)]  # through the newest row
    return [(a, call_a), (b, call_b)]


# ------------------------------------------------------------------------------------------------ small unaligned capacities
SMALL_CAPS = (2050, 5000)
SMALL_F = 3


def small_schedule(cap):
    """(samples pushed before the tier opens, pushes after it, tier bytes): pushes of cap - 1023 and cap, one that loses rows"""
    pushes = [cap - 1023, 700, cap, 1, cap - 1023, 1024, 3 * cap + 77, 333, cap, cap - 1023, 5, cap - 1023, 2 * cap + 1]
    return cap + 300, pushes, 5 * T.max_row_bytes(SMALL_F)


def small_rows(cap, seed=0):
    """NVML-like uint32 rows [n][F] with a stretch of wide values"""
    pre, pushes, _ = small_schedule(cap)
    total = pre + sum(pushes)
    rng = np.random.default_rng([seed, cap])
    rows = _nvml(SMALL_F, total, rng)
    rows[total // 3:total // 2, 1] = rng.integers(0, 1 << 31, total // 2 - total // 3)
    return rows


def row_sizes(rows):
    bits = rows.T.astype(np.float64).view(np.uint64)
    return [T.row_bytes(bits[:, k * ROW:(k + 1) * ROW]) for k in range(rows.shape[0] // ROW)]


def edge_ranges(total, cap, lo):
    """ranges at lo, at the ring's first sample and across it, across every physical end in [lo, total) and through the newest row"""
    ring0 = total - min(total, cap)
    out = [(lo, 1), (lo, total - lo), (lo + 1, min(1500, total - lo - 1)), (ring0, min(total, cap)), (ring0 - 3, 7), (ring0 - 1100, 2300),
           (total - 1, 1), (total - 1030, 1030), (max(lo, total - cap - 700), min(total - lo, cap + 700))]
    out += [(e - 4, 9) for e in range(cap, total, cap)]
    out += [(e - 1500, 3000) for e in range(cap, total, cap)]
    return [(f, n) for f, n in out if f >= lo and n >= 1 and f + n <= total]


# ------------------------------------------------------------------------------------------------ wide rows
WIDE_FS = (301, 512)
WIDE_CAP = 4096
WIDE_PUSHES = (1500, 1024, 2000, 3073, 1, 4096, 777, 2500, 1023, 1025, 4096, 3000, 4095)


def wide_rows(F, seed=0):
    """uint16 rows [n][F]: field f holds values of 1 + (3 f + 5) % 16 bits (fields 255 and 256: 3 and 6 bits), so every block is
    INT coded and the word offsets before and after field 256 all differ"""
    n = sum(WIDE_PUSHES)
    rng = np.random.default_rng([seed, F])
    w = 1 + (3 * np.arange(F) + 5) % 16
    vals = rng.integers(0, 1 << 16, (n, F)) & ((1 << w) - 1)
    return np.ascontiguousarray(vals.astype(np.uint16))


def wide_tier_bytes(F):
    return T.max_row_bytes(F)                  # the smallest tier: about 7 rows of these, so it wraps


# ------------------------------------------------------------------------------------------------ tests
def test_group_size_rule():
    """G < F with a smaller last group on the configs[1]-shaped call B; one group on every other call of the GPU file"""
    vcap = 2162 * ROW
    assert RC.smp_shift(vcap) == 9 and group_size(C1_F, vcap) == 60
    total, ranges = c1_calls()[1]
    _, rows, _, _, vc = virtual(total, C1_CAP, 0, [f for f, _ in ranges], [n for _, n in ranges])
    assert vc == vcap and rows == list(range(2162))
    G = group_size(C1_F, vc)
    assert G < C1_F and C1_F % G == 4
    total, ranges = c1_calls()[0]
    assert group_size(C1_F, virtual(total, C1_CAP, 0, [f for f, _ in ranges], [n for _, n in ranges])[4]) == C1_F
    for _, _, _, _, vcap in route_calls():
        assert group_size(ROUTE_F, vcap) == ROUTE_F
    # the rule's edges: a field of more than 1 GiB still decodes, one field at a time
    assert group_size(8, 1 << 27) == 1 and group_size(3, ROW) == 3


def test_route_layout():
    """call 0: ring-sourced in the tier at shift 5, strided at odd starts, one range across the boundary, one wholly in the ring;
    call 1: a different shift, a range ending at `total` through the partial newest row"""
    (t0, r0, route0, vf0, vcap0), (t1, r1, route1, vf1, vcap1) = route_calls()
    assert route0 == [1, 1, 1, 1, 1, 0] and route1 == [1, 1]
    assert (vcap0, RC.smp_shift(vcap0)) == (151552, 5) and (vcap1, RC.smp_shift(vcap1)) == (45056, 3)
    assert [RC.sample_source(vcap0, n) for _, n in r0[:4]] == ["ring", "strided", "ring", "strided"]
    assert r0[1][0] % 2 and r0[3][0] % 2 and r1[0][0] % 2
    f, n = r0[4]
    assert f < t0 - ROUTE_CAP < f + n
    f, n = r0[5]
    assert t0 - ROUTE_CAP <= f and f + n <= t0 and RC.sample_source(ROUTE_CAP, n) == "ring"
    f, n = r1[1]
    assert f + n == t1 and t1 % ROW == 700 and RC.sample_source(vcap1, n) == "ring"
    # the ranges are disjoint, and call 1's lie after call 0's newest sample: every range's data is its own
    spans = sorted(r for call in ROUTE_CALLS for r in call)
    assert all(a[0] + a[1] < b[0] for a, b in zip(spans, spans[1:]))
    assert min(f for f, _ in r1) >= t0


@pytest.mark.parametrize("q", ROUTE_Q, ids=["q%d_%d" % q for q in ROUTE_Q])
def test_route_generators_take_their_routes(q):
    """every generator built for a geometry takes its route there, and the model's answer is a sort's"""
    x, segs = _route_cache(q)
    n_built = 0
    for c in range(2):
        _, ranges, _, _, _ = route_calls()[c]
        models = route_models(x, segs, c)
        for j, ms in models.items():
            geo, built = segs[c, j]
            first, n = ranges[j]
            for f, m in enumerate(ms):
                keys = O.total_order_key(x[f, first:first + n])
                assert m["answer"] == _kth_largest(keys, geo["k"])
                if "settled" in m:
                    assert m["settled"] == m["answer"]
                if built[f][1] is not None:
                    n_built += 1
                    assert m["route"] == built[f][1], (c, j, built[f][0], m["route"])
    assert n_built >= 4 * ROUTE_F


@pytest.mark.parametrize("q", ROUTE_Q, ids=["q%d_%d" % q for q in ROUTE_Q])
def test_every_source_and_reason_is_reached(q):
    """both sample sources on the virtual ring; every open reason at this quantile; the sample slots of a ring-sourced segment in the
    partial newest row"""
    x, segs = _route_cache(q)
    why = collections.Counter()
    sources = collections.Counter()
    for c in range(2):
        total, ranges, route, _, _ = route_calls()[c]
        for j, ms in route_models(x, segs, c).items():
            geo = segs[c, j][0]
            if route[j]:
                sources[geo["src"]] += 1
            why.update(m["route"] for m in ms if m["route"] in M.OPEN)
    assert sources["ring"] >= 3 and sources["strided"] >= 3, sources
    pivots = any(name == "pivots" and r is not None for _, built in segs.values() for name, r in built)
    assert set(why) == set(M.OPEN) - (set() if pivots else {"pivots"}), (q, why)
    assert pivots == (q == (1, 100))
    # call 1's last range: some of its sample slots hold samples of the partial row, which k_tier_tail writes
    total, ranges, _, _, _ = route_calls()[1]
    geo = segs[1, 1][0]
    in_tail = ranges[1][0] + geo["pos"] >= (total // ROW) * ROW
    assert geo["src"] == "ring" and 50 <= in_tail.sum() < len(in_tail)


def test_sets_layout():
    pieces, pos, k, built = sets_layout()
    total, cap = SETS_TOTAL, SETS_CAP
    assert pieces[0] == (total - 1, 1) and all(b[0] + b[1] == a[0] for a, b in zip(pieces, pieces[1:]))   # reverse push order
    assert pieces[1][0] < (total // ROW) * ROW < pieces[1][0] + pieces[1][1]                           # into the partial row
    assert pieces[2][0] < total - cap < pieces[2][0] + pieces[2][1]                                    # across the boundary
    first = [f for f, _ in pieces] * 2
    length = [n for _, n in pieces] * 2
    route, rows, _, _, _ = virtual(total, cap, 0, first, length, [0, 6, 12])
    assert route == [1, 1] and rows[-1] == total // ROW
    geo = sets_geo(pos, k)
    reached = set()
    for r, xf in built:
        m = M.model_segment(xf, geo)
        assert r is None or m["route"] == r
        reached.add(m["route"])
    assert set(M.OPEN) - {"pivots"} <= reached


def _every_call():
    """(total, cap, tier first, firsts, lens, set_off) of every call test_gpu_tier_paths.py makes"""
    out = []
    for total, ranges, _, _, _ in route_calls():
        out.append((total, ROUTE_CAP, 0, [f for f, _ in ranges], [n for _, n in ranges], None))
    pieces = sets_layout()[0]
    out.append((SETS_TOTAL, SETS_CAP, 0, [f for f, _ in pieces] * 2, [n for _, n in pieces] * 2, [0, 6, 12]))
    for total, ranges in c1_calls():
        out.append((total, C1_CAP, 0, [f for f, _ in ranges], [n for _, n in ranges], None))
    for cap in SMALL_CAPS:
        pre, pushes, tb = small_schedule(cap)
        m = T.Tier(cap, SMALL_F, tb, pre)
        sizes = row_sizes(small_rows(cap))
        m.settle(sizes)
        for n in pushes:
            m.push(n, sizes)
            lo = min(m.total - cap, m.first * ROW)
            ranges = edge_ranges(m.total, cap, lo)
            out.append((m.total, cap, m.first, [f for f, _ in ranges], [n for _, n in ranges], None))
    return out


def test_split_agrees_with_the_library(L):
    """route, rows, vfirst and vtotal of every call of the GPU file: the host model against gpudh_ring_tier_split"""
    calls = _every_call()
    n_tail = 0
    for total, cap, t_first, first, length, so in calls:
        rc, got = _split(L, total, cap, t_first, total // ROW, first, length, so)
        assert rc == 0
        want = T.split(total, cap, t_first, total // ROW, first, length, so)
        assert got == want, (total, cap)
        n_tail += bool(want[1]) and want[1][-1] == total // ROW and total % ROW > 0
    assert n_tail >= 10


@pytest.fixture(scope="module")
def L():
    import gpud_b200 as g
    return g.lib()


@pytest.mark.parametrize("cap", [2050, 5000, 10002, 1000000])
@pytest.mark.parametrize("seed", range(3))
def test_plan_at_unaligned_capacities(L, cap, seed):
    """random schedules with row sizes between a record and a row of 64-bit blocks: placement, eviction and loss"""
    rng = np.random.default_rng([seed, cap])
    F = int(rng.integers(1, 5))
    rec, top = T.rec_bytes(F), T.max_row_bytes(F)
    end = 12 * cap if cap < 100000 else 3 * cap
    n_rows = (end + 2 * cap + 3) // ROW + 2
    sizes = [int(s) for s in rec + 8 * rng.integers(F, (top - rec) // 8 + 1, n_rows)]
    tier_bytes = int(rng.integers(top, 40 * top))
    total0 = int(rng.integers(0, 2 * cap))
    pushes, t = [], total0
    while t < end:
        n = int(rng.choice([1, 1023, 1024, 1025, cap - 1023, cap - 1022, cap, cap + 1, 2 * cap + 3, int(rng.integers(1, cap))]))
        n = min(n, end - t)
        pushes.append(n)
        t += n
    pushes.append(2 * cap + 3)                                  # at least one loss
    rc, state, off = _plan(L, cap, F, tier_bytes, total0, pushes, sizes)
    assert rc == 0
    want_state, want_off = _model(cap, F, tier_bytes, total0, pushes, sizes)
    np.testing.assert_array_equal(state, want_state)
    np.testing.assert_array_equal(off, want_off)
    assert state[-1][3] > 0                                    # rows were lost


def test_plan_of_the_gpu_schedules(L):
    """the small-capacity schedules with their rows' real sizes (rows lost, the tier restarting at the first whole row of an
    unaligned ring), the wide-row schedules, and configs[1]'s, whose tier holds every row at its largest: nothing is evicted"""
    for cap in SMALL_CAPS:
        pre, pushes, tb = small_schedule(cap)
        sizes = row_sizes(small_rows(cap))
        rc, state, off = _plan(L, cap, SMALL_F, tb, pre, pushes, sizes)
        assert rc == 0
        want_state, want_off = _model(cap, SMALL_F, tb, pre, pushes, sizes)
        np.testing.assert_array_equal(state, want_state)
        np.testing.assert_array_equal(off, want_off)
        assert state[0][0] == 1                                          # opened at row 1: sample 300 is the ring's oldest
        totals = pre + np.cumsum(pushes)
        lost = [i for i in range(len(pushes)) if state[i + 1][3] > state[i][3]]
        assert lost and all(state[i + 1][0] == -(-(totals[i] - cap) // ROW) for i in lost)   # the restart at the first whole row
        assert all((totals[i] - cap) % ROW for i in lost)                                   # ... of a ring not on a row boundary
    for F in WIDE_FS:
        sizes = row_sizes(wide_rows(F))
        rc, state, off = _plan(L, WIDE_CAP, F, wide_tier_bytes(F), 0, list(WIDE_PUSHES), sizes)
        assert rc == 0
        want_state, want_off = _model(WIDE_CAP, F, wide_tier_bytes(F), 0, list(WIDE_PUSHES), sizes)
        np.testing.assert_array_equal(state, want_state)
        np.testing.assert_array_equal(off, want_off)
        assert state[-1][0] > 0 and sum(o == 0 for o in off) >= 2        # rows evicted, a row placed at offset 0 after a wrap
    pushes = [n for part in c1_schedule() for n in part]
    sizes = [T.max_row_bytes(C1_F)] * (C1_TOTALS[-1] // ROW + 1)
    rc, state, off = _plan(L, C1_CAP, C1_F, c1_tier_bytes(), 0, pushes, sizes)
    assert rc == 0
    want_state, _ = _model(C1_CAP, C1_F, c1_tier_bytes(), 0, pushes, sizes)
    np.testing.assert_array_equal(state, want_state)
    assert (state[:, 0] == 0).all() and (state[:, 3] == 0).all() and state[-1][1] == C1_TOTALS[-1] // ROW
    assert sum(c1_schedule()[0]) == C1_TOTALS[0] and sum(pushes) == C1_TOTALS[1] and len(set(pushes)) >= 5
