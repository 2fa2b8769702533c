"""Windows handles over chosen fields (gpud_ring_windows_open_fields, DESIGN.md §2 "Field selection").  Column g of a field handle's
history is row fields[g] of an all-field twin handle with the same span, hop and history, opened at the same moment on the same ring
and reduced after the same pushes: all six outputs bit for bit, after every reduce, through loss, restart and re-seed.  Every field
handle is also checked against the C oracle on its fields' own samples (tests/test_gpu_ring_hop.py's HRun, which checks the twin).
Covered: field lists of one field (first, last), contiguous, spread, reversed, with repeats, all F in order and a permutation of all F;
L <= 1024 on the JF = 15, JF = 16, generic and 64-bit-load paths and the wrap window; L > 1024 with strided and sample-ring pivots;
hops; every radix-select reason forced on a named field with the segment select's pivots, fill and class counts equal to the twin's
rows; an unnamed +NaN field; a large alpha through infinities; reduce results, range stats and other handles untouched; full and delta
checkpoints of mixed handle kinds, their restore, re-checkpoint and corruption; every refusal.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import ring_delta as RD
import test_ring_windows_fields_model as FM
import test_segment_paths_model as M
from test_gpu_ring_hop import HRun
from test_gpu_ring_stream import _stream, _thresholds
from test_gpu_segment_paths import _scratch, _thr
from test_gpu_window_paths import _check
from test_ring_windows_model import windows_sub

pytestmark = pytest.mark.gpu

OPS = ("min", "max", "mean", "ema", "p99", "n_over")
E_INVALID, E_CAPACITY = -1, -4


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


def field_lists(F):
    """one field (first, last), contiguous, spread, reversed, repeats, all F in order, a permutation of all F"""
    perm = list(np.random.default_rng(F).permutation(F))
    return [[0], [F - 1], [1, 2, 3], [F - 1, 0, F // 2], list(range(F - 1, -1, -1)), [2, 2, 0, 2, F - 1, 0], list(range(F)), perm]


def _read(h, first, n):
    return {k: h.read(k, first, n) for k in OPS}


def _bitwise(got, want):
    for k in OPS:
        a, b = got[k], want[k]
        assert a.shape == b.shape, k
        assert np.array_equal(a.view(np.uint64) if a.dtype == np.float64 else a, b.view(np.uint64) if b.dtype == np.float64 else b), k


def _sub(want, fields):
    """the oracle's rows of the named fields (every array of want is field-major)"""
    idx = np.asarray(fields)
    return {k: (v[idx] if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == want["min"].shape[0] else v) for k, v in want.items()}


class Twins:
    """an HRun (a ring and its all-field handle, checked against the oracle) and handles over each list, opened at the same moment"""

    def __init__(self, g, ctx, x, W, cap, thr, span, hop, lists, alpha=0.0, history=0, q=(0, 0)):
        self.run = HRun(g, ctx, x, W, cap, thr, span, hop, alpha=alpha, history=history, q=q)
        self.lists = lists
        self.hs = [self.run.r.windows(span, history, hop=hop, fields=fl) for fl in lists]

    def step(self, n, oracle=True):
        self.run.push(n)
        n_new, n_lost = self.run.reduce(check=oracle)
        first, nxt, lost = self.run.h.counts()
        twin = _read(self.run.h, first, nxt - first)
        want = self.run.want(first, nxt)[0] if oracle and nxt > first else None
        for fl, h in zip(self.lists, self.hs):
            assert h.reduce() == (n_new, n_lost) and h.counts() == (first, nxt, lost)
            got = _read(h, first, nxt - first)
            _bitwise(got, {k: v[np.asarray(fl)] for k, v in twin.items()})
            if want is not None:
                _check(got, _sub(want, fl))
        return n_new, n_lost

    def close(self):
        for h in self.hs:
            h.close()
        self.run.close()


# (W, CAP, span, hop, history, what): W = 1000 is the JF = 15 path, 1024 JF = 16, 500 the generic aligned path, 999 the 64-bit loads;
# CAP a multiple of no window puts the wrap window in the generic tail; L > 1024 with strided pivots (L = 5000) and the sample ring
# (L = 10000 of a 20500 ring); hops of s / h = 5 and 2
SHAPES = [(1000, 20500, 1, 1, 0, "jf15_wrap"), (1024, 20500, 1, 1, 0, "jf16_wrap"), (500, 20500, 1, 1, 0, "generic"),
          (999, 20500, 1, 1, 0, "loads64"), (1000, 20500, 5, 1, 0, "strided_hop5"), (1000, 20500, 10, 5, 2, "smp_hop2"),
          (100, 4102, 10, 1, 7, "L1000_hop10"), (7, 3002, 100, 25, 4, "W7_hop4")]


@pytest.mark.parametrize("W,cap,span,hop,history,what", SHAPES, ids=[s[-1] for s in SHAPES])
def test_lists_and_routes(env, W, cap, span, hop, history, what):
    """every kind of field list on one ring, push sizes through loss (a push of more than CAP), restart and re-seed"""
    g, ctx, _ = env
    F = 8
    L, P = W * span, W * hop
    sizes = [1, max(1, P - 1), P, L, L + 1, 2 * P + 3, cap, cap + P + 1, max(1, P - 1), L, 3 * P]
    x = _stream(F, W, -(-(sum(sizes) + L) // W), seed=W + span)
    t = Twins(g, ctx, x, W, cap, _thresholds(x, np.random.default_rng(W)), span, hop, field_lists(F), history=history)
    try:
        lost = 0
        for n in sizes:
            lost += t.step(n)[1]
        assert lost > 0                          # the CAP + P + 1 push lost windows: restart and re-seed were taken
        for fl, h in zip(t.lists, t.hs):
            assert list(h.fields()) == fl and h.n_fields == len(fl)
    finally:
        t.close()


@pytest.mark.parametrize("shape", M.HANDLE_SHAPES, ids=[s[0] for s in M.HANDLE_SHAPES])
def test_radix_reasons_on_named_fields(env, shape):
    """the segment-path fields of tests/test_segment_paths_model.py force every GPUD_RANGE_OPEN_* reason; a handle over a reversed
    subset with a repeat reports the reasons of its own segments, and its select's pivots, fill and class counts are the twin's rows"""
    g, ctx, L = env
    name, W, span, hop, cap, pushes = shape
    x, _ = M._cached(("handle", name), lambda: M.handle_fields(shape))
    F = x.shape[0]
    fl = [F - 1, F // 2, 1, F // 2, 0]
    run = HRun(g, ctx, x, W, cap, _thr(x), span, hop, q=M.HANDLE_Q)
    h = run.r.windows(span, 0, hop=hop, fields=fl)
    try:
        for n in pushes:
            first0 = run.h.counts()[1]
            run.push(n)
            n_new, _ = run.reduce()
            assert h.reduce()[0] == n_new
            first, nxt, _ = run.h.counts()
            twin = _read(run.h, first, nxt - first)
            _bitwise(_read(h, first, nxt - first), {k: v[np.asarray(fl)] for k, v in twin.items()})
            tw, fw = _scratch(L, run.r, run.h), _scratch(L, run.r, h)
            piv, fill, cls = tw
            n_long, rows = len(fill) // F, len(cls) // F
            idx = np.concatenate([np.arange(f * n_long, (f + 1) * n_long) for f in fl])
            ridx = np.concatenate([np.arange(f * rows, (f + 1) * rows) for f in fl])
            assert np.array_equal(fw[0], piv[idx]) and np.array_equal(fw[1], fill[idx]) and np.array_equal(fw[2], cls[ridx])
        # the reasons of the last reduce: the model's, over the named fields' segments of its windows
        Lw, P = W * span, W * hop
        models = []
        for k in range(first0, first0 + n_new):
            geo = M.seg_geometry(cap, k * P % cap, Lw, M.HANDLE_Q)
            models += [M.model_segment(x[f, k * P:k * P + Lw], geo, windows_sub(W, span)) for f in fl]
        _, n_open, why = h.stats()
        assert why == M.reasons_of(models) and n_open == sum(why.values())
    finally:
        h.close()
        run.close()


def test_unnamed_nan_field_is_never_read(env):
    """field 0 a gauge full of +NaN: the twin's segments of field 0 report NAN, a handle without field 0 none"""
    g, ctx, _ = env
    F, W, cap, span = 4, 1000, 200000, 100
    x = np.random.default_rng(3).normal(60.0, 3.0, (F, cap))
    x[0, ::97] = np.nan
    r = g.Ring(ctx, F, cap, W, thresholds=np.full(F, 61.0))
    twin, h = r.windows(span), r.windows(span, fields=[3, 1])
    try:
        r.push(np.ascontiguousarray(x.T))
        assert twin.reduce()[0] == h.reduce()[0] > 0
        assert twin.stats()[2].get("nan", 0) > 0 and "nan" not in h.stats()[2]
        first, nxt, _ = twin.counts()
        _bitwise(_read(h, first, nxt - first), {k: v[[3, 1]] for k, v in _read(twin, first, nxt - first).items()})
    finally:
        h.close()
        twin.close()
        r.close()


@pytest.mark.parametrize("span,hop", [(1, 1), (10, 2), (5, 5)])
def test_large_alpha_keeps_an_infinite_ema(env, span, hop):
    """alpha = 0.9999 with +inf and -inf runs: the guarded carry keeps an infinite EMA infinite, in the field handle as in the twin"""
    g, ctx, _ = env
    F, W, cap = 4, 100, 10000
    x = np.random.default_rng(span).normal(60.0, 3.0, (F, 4 * cap))
    x[1, 5000:5400] = np.inf
    x[2, 12000:12100] = -np.inf
    t = Twins(g, ctx, x, W, cap, np.full(F, 61.0), span, hop, [[2, 1], [1]], alpha=0.9999)
    try:
        infinite = 0
        for n in (3000, 4000, 5000, 7000):
            t.step(n)
            first, nxt, _ = t.hs[1].counts()
            infinite += int(np.isinf(t.hs[1].read("ema", first, nxt - first)).sum())
        assert infinite > 0
    finally:
        t.close()


def test_other_results_untouched(env):
    """a field handle's reduces leave gpud_ring_reduce, reduce_range and its stats, and every other handle's history bit-identical"""
    g, ctx, _ = env
    F, W, cap = 6, 1000, 300000
    x = np.random.default_rng(8).normal(60.0, 3.0, (F, 2 * cap))
    rings = [g.Ring(ctx, F, cap, W, thresholds=np.full(F, 63.0)) for _ in range(2)]
    hs = [[r.windows(1), r.windows(200, hop=20)] for r in rings]
    for r in rings:
        r.stream_open()
    fh = rings[0].windows(200, hop=20, fields=[4, 0])
    fh2 = rings[0].windows(1, fields=[5])
    try:
        pos = 0
        for n in (150000, 200000, 250000):
            outs = []
            for i, r in enumerate(rings):
                r.push(np.ascontiguousarray(x[:, pos:pos + n].T))
                if i == 0:
                    fh.reduce()
                    fh2.reduce()
                for h in hs[i]:
                    h.reduce()
                r.stream_reduce()
                if i == 0:
                    fh.reduce()
                red = r.reduce_all()
                rng_ = r.reduce_range(100000)
                stats = r.range_stats()[2], dict(r.range_open_reasons)
                hist = [_read(h, *h.counts()[:1], h.counts()[1] - h.counts()[0]) for h in hs[i]]
                first, nxt, _ = r.stream_counts()
                outs.append((red, rng_, stats, hist, r.stream_read("p99", first, nxt - first)))
            pos += n
            a, b = outs
            _bitwise(a[0], b[0])
            _bitwise(a[1], b[1])
            assert a[2] == b[2]
            for ha, hb in zip(a[3], b[3]):
                _bitwise(ha, hb)
            assert np.array_equal(a[4].view(np.uint64), b[4].view(np.uint64))
    finally:
        fh.close()
        fh2.close()
        for r in rings:
            r.close()


def _history(h):
    first, nxt, lost = h.counts()
    return (first, nxt, lost), _read(h, first, nxt - first)


def _same_handles(a, b):
    assert len(a) == len(b)
    for ha, hb in zip(a, b):
        assert list(ha.fields()) == list(hb.fields()) and ha.n_fields == hb.n_fields
        ca, ra = _history(ha)
        cb, rb = _history(hb)
        assert ca == cb
        _bitwise(ra, rb)


def _mixed(g, ctx, F, W, cap):
    r = g.Ring(ctx, F, cap, W, thresholds=np.linspace(55.0, 65.0, F))
    r.stream_open()
    hs = [r.windows(20, fields=[3, 0, 3]), r.windows(5, hop=1), r.windows(200, hop=20, fields=[F - 1]),
          r.windows(4, fields=list(range(F)))]
    return r, hs


def _reduce_all(r, hs):
    r.stream_reduce()
    for h in hs:
        h.reduce()


def test_checkpoint_chain(env):
    """full and delta checkpoints of a ring with the stream handle, all-field handles and field handles: the model reads their kind-2
    records and links, a restore gives the same histories and lists, the next reduces after it equal the original's, and
    re-checkpointing the restored ring gives the same bytes"""
    g, ctx, _ = env
    F, W, cap = 5, 100, 400000
    x = np.random.default_rng(11).normal(60.0, 3.0, (F, 3 * cap))
    r, hs = _mixed(g, ctx, F, W, cap)
    pos = 0

    def push(ring, n):
        ring.push(np.ascontiguousarray(x[:, pos:pos + n].T))

    try:
        push(r, 250000)
        pos = 250000
        _reduce_all(r, hs)
        base = r.checkpoint()
        recs, lk = FM.full_handles(base)
        assert [q["kind"] for q in recs] == [0, 2, 1, 2, 2] and [q["fields"] for q in recs][1] == [3, 0, 3]
        for q, h in zip(recs[1:], hs):
            first, nxt, _ = h.counts()
            assert np.array_equal(q["hist"][4], h.read("p99", first, nxt - first))
        deltas = []
        for n in (30000, 170000):
            push(r, n)
            pos += n
            _reduce_all(r, hs)
            d = r.checkpoint_delta()
            assert RD.header(d)["prev_link"] == lk
            lk = FM.delta_handles(d, [dict(kind=q["kind"], fields=q["fields"]) for q in recs])[1]
            deltas.append(d)
        # restore the chain into a fresh ring
        r2 = g.Ring(ctx, F, cap, W, thresholds=np.linspace(55.0, 65.0, F))
        hs2 = r2.restore(base)
        for d in deltas:
            r2.restore_delta(d)
        _same_handles(hs, hs2)
        assert r2.checkpoint() == r.checkpoint()
        # the next reduces after the restore equal the original's
        for n in (1, 99, 40000, cap + 123):
            for ring in (r, r2):
                ring.push(np.ascontiguousarray(x[:, pos:pos + n].T))
            pos += n
            _reduce_all(r, hs)
            _reduce_all(r2, hs2)
            _same_handles(hs, hs2)
        r2.close()
    finally:
        r.close()


def test_corrupt_kind2_records_are_refused(env):
    """n_fields 0 or past the blob, an id outside [0, F), non-zero padding, a list changed in a delta: refused, the ring left as
    created (the good blob restores into it afterwards)"""
    g, ctx, _ = env
    F, W, cap = 5, 100, 50000
    x = np.random.default_rng(12).normal(60.0, 3.0, (F, cap))
    r, hs = _mixed(g, ctx, F, W, cap)
    try:
        r.push(np.ascontiguousarray(x[:, :30000].T))
        _reduce_all(r, hs)
        base = r.checkpoint()
        o = _list_off(base, 1, False, F)
        bad = [FM._patched(base, o, "<q", 0), FM._patched(base, o, "<q", 1 << 40), FM._patched(base, o + 8, "<i", F),
               FM._patched(base, o + 12, "<i", -1), FM._patched(base, o + 20, "<i", 9), base[:o + 6]]
        fresh = g.Ring(ctx, F, cap, W, thresholds=np.linspace(55.0, 65.0, F))
        for b in bad:
            with pytest.raises(g.GpudError):
                fresh.restore(b)
            assert fresh.counts()[0] == 0
        hs2 = fresh.restore(base)
        _same_handles(hs, hs2)
        r.push(np.ascontiguousarray(x[:, 30000:31000].T))
        _reduce_all(r, hs)
        d = r.checkpoint_delta()
        od = _list_off(d, 1, True, F)
        with pytest.raises(g.GpudError):
            fresh.restore_delta(FM._patched(d, od + 8, "<i", 4))
        fresh.restore_delta(d)
        _same_handles(hs, hs2)
        fresh.close()
    finally:
        r.close()


def _list_off(blob, rec, is_delta, F):
    saved = FM.CFG["F"]
    FM.CFG["F"] = F
    try:
        return FM._list_off(blob, rec, is_delta)
    finally:
        FM.CFG["F"] = saved


def _last_error(L, ctx):
    buf = C.create_string_buffer(512)
    L.gpud_last_error(ctx._h, buf, 512)
    return buf.value.decode()


def test_refusals(env):
    """every refusal of gpud_ring_windows_open_fields comes before any allocation, names the argument, and leaves the ring's handle
    set as it was; gpud_ring_windows_fields reports its capacity"""
    g, ctx, L = env
    F, W, cap = 4, 100, 10000
    r = g.Ring(ctx, F, cap, W)
    L.gpud_ring_windows_open_fields.restype = C.c_int32
    try:
        h = C.c_void_p()
        ok = (C.c_int32 * 2)(1, 3)

        def call(span, hop, H, fields, n):
            return L.gpud_ring_windows_open_fields(r._h, C.c_int64(span), C.c_int64(hop), C.c_int64(H), fields, C.c_int32(n), C.byref(h))

        for args, word in [((1, 1, 0, None, 2), "NULL"), ((1, 1, 0, ok, 0), "n_fields"), ((1, 1, 0, ok, -1), "n_fields"),
                           ((1, 1, 0, (C.c_int32 * 1)(F), 1), "fields[0]"), ((1, 1, 0, (C.c_int32 * 2)(0, -1), 2), "fields[1]"),
                           ((cap // W + 1, 1, 0, ok, 2), "span"), ((4, 3, 0, ok, 2), "hop"), ((1, 1, (1 << 40) // 2 + 1, ok, 2), "history")]:
            assert call(*args) == E_INVALID, args
            assert word in _last_error(L, ctx), (args, _last_error(L, ctx))
        assert L.gpud_ring_windows_open_fields(None, 1, 1, 0, ok, 2, C.byref(h)) == E_INVALID
        assert L.gpud_ring_windows_open_fields(r._h, 1, 1, 0, ok, 2, None) == E_INVALID
        # the history limit counts the list: H = 2^40 / 2 is refused for F = 4 but allowed (in the check) for two fields
        assert L.gpud_ring_windows_open_hop(r._h, 1, 1, (1 << 40) // 2, C.byref(h)) == E_INVALID
        w = r.windows(2, fields=[3, 3, 0])
        n = C.c_int32()
        buf = (C.c_int32 * 3)()
        assert L.gpud_ring_windows_fields(w._h, buf, 2, C.byref(n)) == E_CAPACITY and n.value == 3
        assert L.gpud_ring_windows_fields(w._h, buf, 3, C.byref(n)) == 0 and list(buf) == [3, 3, 0]
        assert L.gpud_ring_windows_fields(None, buf, 3, C.byref(n)) == E_INVALID
        assert list(r.windows(1).fields()) == list(range(F))
        w.close()
    finally:
        r.close()
