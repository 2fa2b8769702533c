"""The segment select of gpud_ring_reduce_ranges' long route and of span / hop handles with L > 1024, and the short route
(k_ranges_short), against the C oracle and the model of test_segment_paths_model.py.  Values: min / max / the order statistic / n_over
bit for bit, mean and EMA within oracle/SPEC.md's tolerance (the oracle on each range's or window's own samples).  Routes: every
segment's pivots, list fill and per-row class counts as the last segment select left them (gpudh_ring_segment_scratch), and the open
count and reasons of ranges_stats() / stats(), exactly as the model predicts - a wrong pivot, a lost list key or a wrong class count
usually costs only time, because the radix select still returns the right value, so only these checks see it.  Covered: each
generator of range_cases.py in ranges of 1025 .. 300001 samples at even and odd columns and across the physical end; span and hop
handles (strided samples, Wp = 840, the sample ring); more than 4096 open segments in one radix select (its chunk loop); a call the
long route splits into three batches; the short route's four branches on window_cases.py's windows at every length and load path,
and its EMA at alpha = 0.9999 from an infinite first sample.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import test_segment_paths_model as M
import mean_ema_ref as R
from test_gpu_ring_hop import HRun
from test_gpu_ring_ranges import _alpha, _want
from test_gpu_window_paths import _check
from test_ring_windows_model import windows_sub

pytestmark = pytest.mark.gpu

OPS = ("min", "max", "mean", "ema", "p99", "n_over")
E_STATE = -6                    # GPUD_E_STATE


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


def _scratch(L, ring, h=None):
    """(pivots [n_segs][2] as raw bits, fill [n_segs], class counts [n_rows][4]) of the last segment select, or the hook's error"""
    ns, nr = C.c_int64(), C.c_int64()
    hh = h._h if h is not None else None
    rc = L.gpudh_ring_segment_scratch(ring._h, hh, None, None, None, C.byref(ns), C.byref(nr))
    if rc:
        return rc
    piv = np.empty((ns.value, 2), dtype=np.float64)
    fill = np.empty(ns.value, dtype=np.uint32)
    cls = np.empty((nr.value, 4), dtype=np.uint32)
    assert L.gpudh_ring_segment_scratch(ring._h, hh, piv.ctypes.data, fill.ctypes.data, cls.ctypes.data, C.byref(ns), C.byref(nr)) == 0
    return piv.view(np.uint64), fill, cls


def _check_scratch(scr, models, n_segs, n_rows):
    """models: {(segment, first row): model}; the hook reports exactly n_segs segments and n_rows rows"""
    assert not isinstance(scr, int), scr
    piv, fill, cls = scr
    assert (len(fill), len(cls)) == (n_segs, n_rows)
    for (s, row0), m in models.items():
        assert (int(piv[s, 0]), int(piv[s, 1])) == (m["lo"], m["hi"]), (s, m["route"], hex(piv[s, 0]), hex(m["lo"]), hex(piv[s, 1]), hex(m["hi"]))
        assert int(fill[s]) == m["fill"], (s, m["route"], int(fill[s]), m["fill"])
        got = cls[row0:row0 + len(m["cls"])].astype(np.int64)
        bad = np.argwhere(got != m["cls"])
        assert bad.size == 0, (s, m["route"], bad[:4].tolist(), got[bad[0][0]].tolist(), m["cls"][bad[0][0]].tolist())


def _thr(x):
    return np.array([(np.inf, 60.0, x[f, x.shape[1] // 3], -np.inf, np.nan)[f % 5] for f in range(x.shape[0])])


def _push(r, x, zeros=0, chunk=1 << 18):
    """zeros rows of filler first, then x[F][n] in chunks"""
    F = x.shape[0]
    for a in range(0, zeros, chunk):
        r.push(np.zeros((min(chunk, zeros - a), F)))
    for a in range(0, x.shape[1], chunk):
        r.push(np.ascontiguousarray(x[:, a:a + chunk].T))


def _range_models(x, oldest, firsts, lens, segs, cap, q):
    """(models keyed for _check_scratch, reasons) of one batch of long ranges given in call order"""
    F = x.shape[0]
    n_long = len(firsts)
    n_tiles = sum(-(-n // M.TILE) for n in lens)
    out, every = {}, []
    tile0 = 0
    for j, (first, n) in enumerate(zip(firsts, lens)):
        for f in range(F):
            geo = segs[f, j][2] if segs else M.seg_geometry(cap, first % cap, n, q)
            m = M.model_segment(x[f, first - oldest:first - oldest + n], geo)
            out[f * n_long + j, f * n_tiles + tile0] = m
            every.append(m)
        tile0 += -(-n // M.TILE)
    return out, M.reasons_of(every), F * n_long, F * n_tiles


@pytest.mark.parametrize("q", M.QUANTILES, ids=["q%d_%d" % q for q in M.QUANTILES])
def test_range_segment_routes(env, q):
    g, ctx, L = env
    x, segs, _ = M.range_models(q)
    cap, total, firsts = M.range_layout()
    oldest = total - cap
    F = x.shape[0]
    thr = _thr(x)
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    try:
        _push(r, x, zeros=oldest)
        got = r.reduce_ranges(firsts, M.RANGE_LENS)
        _, n_radix, why = r.ranges_stats()
        scr = _scratch(L, r)
    finally:
        r.close()
    _check(got, _want(x, oldest, firsts, M.RANGE_LENS, thr, _alpha(1000, 0.0), q))
    models, reasons, n_segs, n_rows = _range_models(x, oldest, firsts, M.RANGE_LENS, segs, cap, q)
    assert why == reasons and n_radix == sum(reasons.values()), (why, reasons)
    _check_scratch(scr, models, n_segs, n_rows)


def _handle_models(run, shape, first, n_new):
    """models of the last reduce: its reasons over all its windows, and the scratch of its last phase"""
    _, W, span, hop, cap, pushes = shape
    Lw, P, p = W * span, W * hop, span // hop
    Wp = windows_sub(W, span)
    F = run.x.shape[0]
    models = {}
    for k in range(first, first + n_new):
        geo = M.seg_geometry(cap, k * P % cap, Lw, M.HANDLE_Q)
        for f in range(F):
            models[f, k] = M.model_segment(run.x[f, k * P:k * P + Lw], geo, Wp)
    last = list(range(first + min(p, n_new) - 1, first + n_new, p))
    n, sub = len(last), Lw // Wp
    scratch = {(f * n + i, f * n * sub + i * sub): models[f, k] for f in range(F) for i, k in enumerate(last)}
    return M.reasons_of(models.values()), scratch, F * n, F * n * sub


@pytest.mark.parametrize("shape", M.HANDLE_SHAPES, ids=[s[0] for s in M.HANDLE_SHAPES])
def test_handle_segment_routes(env, shape):
    """span and hop handles: the whole history against the oracle after each reduce, the last segment select against the model"""
    g, ctx, L = env
    name, W, span, hop, cap, pushes = shape
    x, _ = M._cached(("handle", name), lambda: M.handle_fields(shape))
    run = HRun(g, ctx, x, W, cap, _thr(x), span, hop, q=M.HANDLE_Q)
    try:
        assert _scratch(L, run.r, run.h) == E_STATE                  # no reduce yet
        for n in pushes:
            first0 = run.h.counts()[1]
            run.push(n)
            n_new, n_lost = run.reduce()
            assert n_lost == 0
        _, n_open, why = run.h.stats()
        scr = _scratch(L, run.r, run.h)
    finally:
        run.close()
    reasons, models, n_segs, n_rows = _handle_models(run, shape, first0, n_new)
    assert why == reasons and n_open == sum(reasons.values()), (why, reasons)
    _check_scratch(scr, models, n_segs, n_rows)


CHUNK_IDS = ["%d-q%d_%d" % (n, q[0], q[1]) for n, q in M.CHUNK_CASES] + ["span2_catch_up"]


@pytest.mark.parametrize("case", M.CHUNK_CASES + [None], ids=CHUNK_IDS)
def test_radix_chunks(env, case):
    """more than 4096 segments left open in one select (4800; exactly 4096 and 4097), so the radix select runs its chunk loop: the
    ranges of one call, and a span-2 handle's catch-up over 600 windows"""
    g, ctx, L = env
    if case is None:
        W, span, cap, x, _ = M._cached("span_chunk", M.span_chunk_fields)
        run = HRun(g, ctx, x, W, cap, _thr(x), span, span, q=M.HANDLE_Q)
        try:
            run.push(cap)
            first0 = 0
            n_new, _ = run.reduce()
            assert n_new == 600
            _, n_open, why = run.h.stats()
            scr = _scratch(L, run.r, run.h)
        finally:
            run.close()
        shape = ("span2", W, span, span, cap, (cap,))
        reasons, models, n_segs, n_rows = _handle_models(run, shape, first0, n_new)
        assert n_open == 4800 and why == reasons, (n_open, why, reasons)
        _check_scratch(scr, models, n_segs, n_rows)
        return
    n_ranges, q = case
    cap, firsts, x, segs = M._cached(("chunk", n_ranges, q), lambda: M.chunk_fields(n_ranges, q))
    lens = [M.CHUNK_N] * n_ranges
    thr = _thr(x)
    r = g.Ring(ctx, M.CHUNK_F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    try:
        _push(r, x)
        got = r.reduce_ranges(firsts, lens)
        _, n_radix, why = r.ranges_stats()
        scr = _scratch(L, r)
    finally:
        r.close()
    _check(got, _want(x, 0, firsts, lens, thr, _alpha(1000, 0.0), q))
    models, reasons, n_segs, n_rows = _range_models(x, 0, firsts, lens, segs, cap, q)
    assert n_radix == {600: 4800, 512: 4096, 513: 4097}[n_ranges] and why == reasons, (n_radix, why, reasons)
    _check_scratch(scr, models, n_segs, n_rows)


def test_long_route_batches(env):
    """one call of 600 whole-ring ranges, short ranges between them and a forced sub-range in every batch, over three batches"""
    g, ctx, L = env
    total, x, firsts, lens, subs = M._cached("batch", M.batch_call)
    cap, F, q = M.BATCH_CAP, M.BATCH_F, M.BATCH_Q
    oldest = total - cap
    pl = M.ranges_plan(cap, F, q, firsts, lens)
    n_batches = max(pl["route"])
    assert n_batches >= 3
    thr = _thr(x)
    alpha = _alpha(1000, 0.0)
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    try:
        _push(r, x, zeros=oldest)
        got = r.reduce_ranges(firsts, lens)
        _, n_radix, why = r.ranges_stats()
        scr = _scratch(L, r)
    finally:
        r.close()
    # values: the oracle once per distinct range
    distinct = {}
    for key in zip(firsts, lens):
        if key not in distinct:
            a = key[0] - oldest
            distinct[key] = R.windows_fields(x[:, a:a + key[1]], int(key[1]), thr, alpha, q[0], q[1])
    want = R.stack([R.select(distinct[key], (slice(None), 0)) for key in zip(firsts, lens)])
    _check(got, want)
    whole = [i for i, (f, n) in enumerate(zip(firsts, lens)) if n == cap]
    for k in OPS:
        col = got[k][:, whole].view(np.uint64 if k != "n_over" else np.uint32)
        assert (col == col[:, :1]).all(), k                          # bit-identical across batches
    # routes: the model's reasons over every segment of every batch
    models = {}
    for key in distinct:
        if key[1] > M.TILE:
            geo = M.seg_geometry(cap, key[0] % cap, key[1], q)
            models[key] = [M.model_segment(x[f, key[0] - oldest:key[0] - oldest + key[1]], geo) for f in range(F)]
    every = [m for key in zip(firsts, lens) if key[1] > M.TILE for m in models[key]]
    reasons = M.reasons_of(every)
    assert why == reasons and n_radix == sum(reasons.values()), (why, reasons)
    for (first, n), (f, name, _, _) in subs.items():
        assert models[first, n][f]["route"] == name
    # the hook: the last batch's segments
    last = [i for i, b in enumerate(pl["route"]) if b == n_batches]
    lf, ll = [firsts[i] for i in last], [lens[i] for i in last]
    seg_models, _, n_segs, n_rows = _range_models(x, oldest, lf, ll, None, cap, q)
    _check_scratch(scr, seg_models, n_segs, n_rows)


@pytest.mark.parametrize("q", M.SHORT_QS, ids=["q%d_%d" % q for q in M.SHORT_QS])
def test_short_route_branches(env, q):
    """one field per window kind; every length at an even and an odd start and across the physical end at both parities (a call of
    its own per wrapping range, a lap pushed between calls)"""
    g, ctx, L = env
    calls = M.short_calls(q)
    F = len(M.KINDS)
    thr = _thr(calls[0][0])
    alpha = _alpha(1000, 0.0)
    r = g.Ring(ctx, F, M.SHORT_CAP, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
    try:
        for lap, ranges in calls:
            r.push(np.ascontiguousarray(lap.T))
            total = r.counts()[0]
            base = total - lap.shape[1]
            firsts = [a for a, _, _ in ranges]
            ms = [m for _, m, _ in ranges]
            got = r.reduce_ranges(firsts, ms)
            assert _scratch(L, r) == E_STATE                          # no long range in the call
            for i, (first, m, kinds) in enumerate(ranges):
                xr = lap[:, first - base:first - base + m]
                want = R.windows_fields(xr, m, thr, alpha, q[0], q[1])
                _check({k: got[k][:, i:i + 1] for k in OPS}, want)
    finally:
        r.close()


def test_short_route_ema(env):
    """alpha = 0.9999 ((1 - alpha)^64 squared underflows): the EMA started at an infinite first sample stays infinite, +inf then
    -inf is NaN, at every length and load path"""
    g, ctx, L = env
    cap, F, alpha = M.SHORT_CAP, 4, 0.9999
    total = cap + cap // 2
    x = np.stack([M.gauge(total, [7, f]) for f in range(F)])
    ranges, cur = [], cap + 202                                      # after the wrapping range below
    for m in M.SHORT_MS:
        for par in (0, 1):
            if cur % 2 != par:
                cur += 1
            ranges.append((cur, m))
            cur += m + 1
    ranges.append((cap - 201, 400))                                   # across the physical end, odd column
    for first, m in ranges:
        x[0, first] = np.inf
        x[1, first] = -np.inf
        x[3, first] = np.inf
        x[3, first + m // 2] = -np.inf if m > 1 else np.inf
    thr = np.full(F, 60.0)
    r = g.Ring(ctx, F, cap, 1000, thresholds=thr, ema_alpha=alpha)
    try:
        r.push(np.ascontiguousarray(x.T))
        got = r.reduce_ranges([a for a, _ in ranges], [m for _, m in ranges])
    finally:
        r.close()
    for i, (first, m) in enumerate(ranges):
        xr = x[:, first:first + m]
        want = R.windows_fields(xr, m, thr, alpha, 0, 0)
        _check({k: got[k][:, i:i + 1] for k in OPS}, want)
        assert np.isposinf(got["ema"][0, i]) and np.isneginf(got["ema"][1, i])
        assert np.isnan(got["ema"][3, i]) or m == 1


def test_scratch_hook_states(env):
    """GPUD_E_STATE: a handle of L <= 1024, a handle before its first reduce, a ring whose last reduce_ranges had no long range (after
    one that had)"""
    g, ctx, L = env
    r = g.Ring(ctx, 2, 8192, 100)
    try:
        small, big = r.windows(10), r.windows(20)
        assert _scratch(L, r) == E_STATE and _scratch(L, r, big) == E_STATE
        r.push(np.random.default_rng(1).normal(60.0, 3.0, (8192, 2)))
        small.reduce()
        big.reduce()
        assert _scratch(L, r, small) == E_STATE
        piv, fill, cls = _scratch(L, r, big)
        assert len(fill) == 2 * 4 and len(cls) == 2 * 4 * 2              # 4 windows of 2000 per field, sub-windows of 1000
        r.reduce_ranges([0, 10], [3000, 50])
        piv, fill, cls = _scratch(L, r)
        assert len(fill) == 2 and len(cls) == 2 * 3
        r.reduce_ranges([0], [50])
        assert _scratch(L, r) == E_STATE
    finally:
        r.close()
