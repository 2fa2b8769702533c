"""The tier's range path route by route (DESIGN.md §2 "Tier"), on the layouts of test_tier_paths_model.py.  Every call is checked
against an untiered twin that holds every sample (all six outputs bit for bit) and the C oracle (min / max / p99 / n_over bit for bit,
mean and EMA within oracle/SPEC.md's tolerance).  Routes: the open count and reasons of ranges_stats() - summed over the ring's own
sets and every field group - and every pivot, list fill and class count the last segment select left (gpudh_ring_segment_scratch),
exactly as the model predicts on the virtual ring's geometry: a wrong pivot from a stale or unwritten virtual sample ring costs only
time, so only these checks see it.  Covered: each generator of range_cases.py in ranges that reach into the tier (ring-sourced and
strided, across the tier/ring boundary, through the partial newest row) and one wholly in the ring, a second call with another sample
shift on the same buffers, a set of pieces in reverse push order, forced field groups of 1, 5 and F - 1; rows of 301 and 512 fields
(block offsets past field 256) in a tier that wraps; the configs[1] shape (F = 64, CAP = 1 000 000, 2.2 M samples) in natural groups of
60 + 4; capacities of 2050 and 5000 with rows coded across the physical end, the newest row copied across it and a restart at an
unaligned first whole row.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import ring_tier as T
import test_segment_paths_model as M
import test_tier_paths_model as TM
from test_gpu_ring_range_sets import _sets
from test_gpu_ring_range_sets import _want as _want_sets
from test_gpu_ring_ranges import _alpha, _want
from test_gpu_ring_tier import _bitwise, _nvml
from test_gpu_segment_paths import _check_scratch, _scratch, _thr
from test_gpu_window_paths import _check

pytestmark = pytest.mark.gpu
ROW = T.ROW
P99 = (99, 100)


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    L = g.lib()
    L.gpudh_ring_segment_scratch.restype = C.c_int32
    L.gpudh_ring_segment_scratch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64)]
    yield g, ctx, L
    ctx.close()


def _split_args(ranges):
    return [f for f, _ in ranges], [n for _, n in ranges]


def _against_twin_and_oracle(r, twin, ranges, x, thr, alpha, q):
    """one call: all six outputs of the tiered ring equal the twin's, and the oracle on each range; -> (outputs, open count, reasons)"""
    first, length = _split_args(ranges)
    got = r.reduce_ranges(first, length)
    _, n_open, why = r.ranges_stats()
    assert _bitwise(got, twin.reduce_ranges(first, length))
    _check(got, _want(x, 0, first, length, thr, alpha, q))
    return got, n_open, why


def _push_f64(rings, x, a, b, chunk=8192):
    """samples [a, b) of x[F][n], in pushes short enough that the tier codes every row before the ring overwrites it"""
    for s in range(a, b, chunk):
        part = np.ascontiguousarray(x[:, s:min(b, s + chunk)].T)
        for r in rings:
            r.push(part)


def _push_raw(rings, rows):
    for r in rings:
        r.push_raw(rows)


@pytest.mark.parametrize("q", TM.ROUTE_Q, ids=["q%d_%d" % q for q in TM.ROUTE_Q])
def test_routes_on_the_decoded_ring(env, q):
    """call 0: ranges wholly in the tier (ring-sourced and strided), one across the boundary, one wholly in the ring, then the same call
    in forced groups of 1, 5 and F - 1 fields; call 1 after more pushes: a smaller virtual ring with another sample shift, one range
    ending at `total` whose sample slots in the partial row only k_tier_tail writes"""
    g, ctx, L = env
    x, segs = TM._route_cache(q)
    F = TM.ROUTE_F
    thr = _thr(x)
    alpha = _alpha(1000, 0.0)
    r = g.Ring(ctx, F, TM.ROUTE_CAP, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    twin = g.Ring(ctx, F, 1 << 18, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    try:
        r.tier_open(T.max_row_bytes(F) * (TM.ROUTE_TOTALS[-1] // ROW + 2))
        pos = 0
        for c, (total, ranges, route, _, _) in enumerate(TM.route_calls()):
            _push_f64((r, twin), x, pos, total)
            pos = total
            assert r.tier_counts()[:2] == (0, (total // ROW) * ROW)
            got, n_open, why = _against_twin_and_oracle(r, twin, ranges, x, thr, alpha, q)
            models = TM.route_models(x, segs, c)
            reasons = M.reasons_of([m for ms in models.values() for m in ms])
            assert why == reasons and n_open == sum(reasons.values()), (c, why, reasons)
            want, n_segs, n_rows = TM.scratch_models(models, ranges, route, 0, F)
            _check_scratch(_scratch(L, r), want, n_segs, n_rows)
            if c:
                continue
            first, length = _split_args(ranges)
            for G in (1, 5, F - 1):
                r.tier_group(G)
                try:
                    got_g = r.reduce_ranges(first, length)
                    _, n_open_g, why_g = r.ranges_stats()
                    scr = _scratch(L, r)
                finally:
                    r.tier_group(0)
                assert _bitwise(got_g, got), G
                assert (n_open_g, why_g) == (n_open, why), G
                want, n_segs, n_rows = TM.scratch_models(models, ranges, route, (F - 1) // G * G, F)   # the last group's fields
                _check_scratch(scr, want, n_segs, n_rows)
    finally:
        r.close()
        twin.close()


def test_sets_of_pieces_in_the_tier(env):
    """one set of six pieces in reverse push order - two in the partial newest row, one across the tier/ring boundary - given twice,
    its data built against the set's strided sample: every reason, pivot, list fill and class count the model's"""
    g, ctx, L = env
    pieces, pos, k, built = TM.sets_layout()
    F, cap, total, q = len(built), TM.SETS_CAP, TM.SETS_TOTAL, TM.SETS_Q
    x = np.random.default_rng(5).normal(60.0, 3.0, (F, total))
    for f, (_, xf) in enumerate(built):
        for (p, ln), a in zip(pieces, TM.SETS_CUTS[:-1]):
            x[f, p:p + ln] = xf[a:a + ln]
    thr = _thr(x)
    alpha = _alpha(1000, 0.0)
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    twin = g.Ring(ctx, F, 1 << 17, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    try:
        r.tier_open(T.max_row_bytes(F) * (total // ROW + 2))
        _push_f64((r, twin), x, 0, total)
        assert r.tier_counts()[0] == 0
        first, length, set_off = _sets([pieces, pieces])
        got = r.reduce_range_sets(first, length, set_off)
        _, n_open, why = r.ranges_stats()
        scr = _scratch(L, r)
        assert _bitwise(got, twin.reduce_range_sets(first, length, set_off))
    finally:
        r.close()
        twin.close()
    _check(got, _want_sets(x, 0, first, length, set_off, thr, alpha, q))
    expect = {}
    for route, _ in built:
        if route in M.OPEN:
            expect[route] = expect.get(route, 0) + 2
    assert why == expect and n_open == sum(expect.values()), (why, expect)
    geo = TM.sets_geo(pos, k)
    nt = -(-TM.SETS_N // M.TILE)
    models = {}
    for f, (_, xf) in enumerate(built):
        m = M.model_segment(xf, geo)
        for j in range(2):
            models[f * 2 + j, f * 2 * nt + j * nt] = m
    _check_scratch(scr, models, 2 * F, 2 * F * nt)


def _rows_against_model(r, m, bits):
    """tier_counts and every held row's bytes against the host model; -> the rows checked at offset 0 after the tier wrapped"""
    assert r.tier_counts() == (m.first * ROW, m.next * ROW, m.used, m.lost)
    wrapped = []
    for row, off, _ in m.rows:
        assert r.tier_row(row) == T.row_image(bits[:, row * ROW:(row + 1) * ROW], row, off), row
        if off == 0 and row > m.rows[0][0]:
            wrapped.append(row)
    return wrapped


@pytest.mark.parametrize("F", TM.WIDE_FS)
def test_wide_rows(env, F):
    """rows of more than 256 fields, whose block word offsets k_tier_place computes 256 fields at a time, in the smallest tier"""
    g, ctx, _ = env
    cap = TM.WIDE_CAP
    rows = TM.wide_rows(F)
    x = rows.T.astype(np.float64)
    bits = x.view(np.uint64)
    sizes = TM.row_sizes(rows)
    tb = TM.wide_tier_bytes(F)
    thr = 2.0 ** (np.arange(F) % 16)
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, ema_alpha=0.01, q_num=99, q_den=100)
    twin = g.Ring(ctx, F, 1 << 15, 1000, thresholds=thr, ema_alpha=0.01, q_num=99, q_den=100)
    try:
        r.tier_open(tb)
        m = T.Tier(cap, F, tb, 0)
        m.settle(sizes)
        a, wrapped = 0, []
        for n in TM.WIDE_PUSHES:
            _push_raw((r, twin), rows[a:a + n])
            a += n
            m.push(n, sizes)
            wrapped += _rows_against_model(r, m, bits)
            if a >= 3 * cap:
                lo = min(a - cap, m.first * ROW)
                _against_twin_and_oracle(r, twin, TM.edge_ranges(a, cap, lo), x, thr, 0.01, P99)
        assert wrapped and m.first > 0
    finally:
        r.close()
        twin.close()


def test_configs1_natural_groups(env):
    """F = 64, CAP = 1 000 000: a call whose newest row is copied across the physical end, then one whose range over every row decodes
    in groups of 60 + 4 fields with a threshold of its own per field; the oracle on the first and last field of each group"""
    g, ctx, L = env
    F, cap = TM.C1_F, TM.C1_CAP
    total_b = TM.C1_TOTALS[-1]
    rows = _nvml(F, total_b, np.random.default_rng(64))
    thr = np.array([np.quantile(rows[::97, f].astype(np.float64), 0.2 + 0.6 * f / F) + f / 128 for f in range(F)])
    assert len(set(thr.tolist())) == F
    alpha = 0.01
    sub = [0, 59, 60, 63]                                          # the first and last field of each group
    xs = np.ascontiguousarray(rows[:, sub].T.astype(np.float64))
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, ema_alpha=alpha, q_num=99, q_den=100)
    twin = g.Ring(ctx, F, 1 << 22, 1000, thresholds=thr, ema_alpha=alpha, q_num=99, q_den=100)
    try:
        r.tier_open(TM.c1_tier_bytes())
        a = 0
        for pushes, (total, ranges) in zip(TM.c1_schedule(), TM.c1_calls()):
            for n in pushes:
                _push_raw((r, twin), rows[a:a + n])
                a += n
            assert a == total and r.tier_counts()[:2] == (0, (total // ROW) * ROW) and r.tier_counts()[3] == 0
            first, length = _split_args(ranges)
            got = r.reduce_ranges(first, length)
            assert _bitwise(got, twin.reduce_ranges(first, length))
            _check({k: v[sub] for k, v in got.items()}, _want(xs, 0, first, length, thr[sub], alpha, P99))
            route, rows_v, _, _, vcap = TM.virtual(total, cap, 0, first, length)
            G = TM.group_size(F, vcap)
            if total == total_b:
                assert (G, F - F // G * G) == (60, 4)
                piv, fill, cls = _scratch(L, r)                    # the last group: 4 fields of every long tier range
                long = [n for n, rt in zip(length, route) if rt and n > M.TILE]
                assert len(fill) == 4 * len(long) and len(cls) == 4 * sum(-(-n // M.TILE) for n in long)
    finally:
        r.close()
        twin.close()


@pytest.mark.parametrize("cap", TM.SMALL_CAPS)
def test_small_unaligned_capacities(env, cap):
    """the tier opened on a wrapped ring (its first whole row 1), pushes of cap - 1023 and cap and ones that lose rows: counts and every
    row's bytes after each push, and ranges at lo, at and across the ring's first sample, across every physical end and through the
    newest row against the twin and the oracle"""
    g, ctx, _ = env
    F = TM.SMALL_F
    pre, pushes, tb = TM.small_schedule(cap)
    rows = TM.small_rows(cap)
    x = rows.T.astype(np.float64)
    bits = x.view(np.uint64)
    sizes = TM.row_sizes(rows)
    thr = np.array([np.median(x[f]) for f in range(F)])
    r = g.Ring(ctx, F, cap, 100, thresholds=thr, ema_alpha=0.01, q_num=99, q_den=100)
    twin = g.Ring(ctx, F, 1 << 16, 100, thresholds=thr, ema_alpha=0.01, q_num=99, q_den=100)
    try:
        _push_raw((r, twin), rows[:pre])
        r.tier_open(tb)
        m = T.Tier(cap, F, tb, pre)
        m.settle(sizes)
        a = pre
        for n in [0] + pushes:
            if n:
                _push_raw((r, twin), rows[a:a + n])
                a += n
                m.push(n, sizes)
            _rows_against_model(r, m, bits)
            lo = min(a - cap, m.first * ROW)
            _against_twin_and_oracle(r, twin, TM.edge_ranges(a, cap, lo), x, thr, 0.01, P99)
        assert m.lost > 0
    finally:
        r.close()
        twin.close()
