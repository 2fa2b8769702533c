"""gpud_box_query_create_fields (DESIGN.md §2 "Box sets across processes", "Field selection"): the box query over chosen fields of
each rank's ring.  Simulated ranks as in test_gpu_ring_box_dist.py: 2 to 8 rings of one config on device 0 (some wrapped), each driven
by its own query in lockstep, with thresholds that differ per field.  For [f] at the first, a middle and the last field, a list out of
order with a repeat and all F in order:
  - every round's size is equal on all ranks and is the plan hook's (gpudh_box_query_plan_fields), and every rank's result is the same;
  - column g equals row fields[g] of the all-field query over the same rings, bit for bit in all six outputs, over local, short spread
    (one of odd length first) and long spread sets; it equals rings_reduce_range_sets(fields=) in one process (min / max / p99 /
    n_over everywhere, mean and EMA except for long spread sets) and the C oracle;
  - stats()["bytes_sent"] is the sum of the rounds, and the samples(0) and summaries(0) rounds are the all-field query's scaled by G / F.
Further: every radix-select reason on named fields with reasons and pivots equal to the all-field query's rows; an unnamed NaN field
that changes nothing; three long-route batches; the refusals, each on every rank at the same step; rings that report the same
afterwards; 2 and 3 gloo processes through dist.box_range_sets(fields=), and 2 NCCL processes on two GPUs (skipped with fewer).
Run on an H100: pytest -m gpu."""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if __name__ == "__main__":                                            # a worker process of test_gloo_processes
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np
import pytest

import range_cases as RC
import test_segment_paths_model as M
from test_gpu_ring_box_dist import _box_sets, _drive, _rings, _worker_call
from test_gpu_ring_box_sets import _n_gpus, _sets, _want
from test_gpu_ring_range_sets import _bits, _push
from test_gpu_ring_ranges import OPS, _alpha, _fields
from test_gpu_window_paths import _check
import mean_ema_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


def _lockstep(g, rings, args, fields=None):
    """every rank's query over the same arguments, driven to the end: (queries, result bits, round sizes)"""
    qs = [g.BoxQuery(r, k, len(rings), *args, fields=fields) for k, r in enumerate(rings)]
    sizes, outcome = _drive(qs)
    assert outcome == [None] * len(rings)
    res = [_bits(q.result()) for q in qs]
    for k in range(1, len(rings)):
        for op in OPS:
            assert np.array_equal(res[k][op], res[0][op]), (k, op)
    return qs, res[0], sizes


def _rows(d, fields):
    return {op: d[op][list(fields)] for op in OPS}


def _long_spread(args):
    ring_of, _, length, set_off = args
    return np.array([len(set(ring_of[a:b].tolist())) > 1 and length[a:b].sum() > 1024 for a, b in zip(set_off[:-1], set_off[1:])])


@pytest.mark.parametrize("n_rings,W,q,alpha", [(2, 1000, (0, 0), 0.0), (5, 999, (999, 1000), 0.9999), (8, 1, (1, 2), 0.0)])
def test_field_lists_against_all_field_query(env, n_rings, W, q, alpha):
    g, ctx = env
    F, cap = 8, 1 << 17
    rings, totals, olds, xs, thr, rng = _rings(g, ctx, n_rings, W, q, alpha, F=F, cap=cap, seed=4)
    assert len({thr[5], thr[2], thr[0]}) == 3                          # per-field thresholds: n_over through the wrong one would show
    before_reduce, before_stats = [], []
    for k, r in enumerate(rings):                                      # what the rings report must read the same afterwards
        r.reduce_all()
        before_reduce.append({op: r.read(op).copy() for op in OPS})
        r.reduce_range_sets([olds[k], olds[k] + 7], [5000, 70000], [0, 1, 2])
        before_stats.append(r.ranges_stats())
    sets = _box_sets(rng, n_rings, totals, olds, cap)
    args = _sets(sets)
    long_spread = _long_spread(args)
    assert long_spread.any() and (~long_spread).any()
    qa, full, sizes_all = _lockstep(g, rings, args)
    sent_all = qa[0].stats()["bytes_sent"]
    want = _want(xs, olds, *args, thr, _alpha(W, alpha), q)
    for fields in ([0], [F // 2], [F - 1], [5, 2, 2, 0], list(range(F))):
        G = len(fields)
        qs, got, sizes = _lockstep(g, rings, args, fields)
        rc, msg, _, _, sb, _, _, _ = g.capi.box_query_plan(totals, cap, *args, F=F, q=q if q[1] else (99, 100), fields=fields)
        assert rc == 0, msg
        assert sizes[:3] == sb.tolist(), (fields, sizes[:3], sb.tolist())
        for i in (1, 2):                                               # samples(0) and summaries(0): per column
            assert (sizes[i] - 16) * F == (sizes_all[i] - 16) * G, (fields, i)
        rows = _rows(full, fields)
        for op in OPS:
            assert np.array_equal(got[op], rows[op]), (fields, op)
        one = _bits(g.rings_reduce_range_sets(rings, *args, fields=fields))
        for op in OPS:
            cols = slice(None) if op in ("min", "max", "p99", "n_over") else ~long_spread
            bad = np.argwhere(got[op][:, cols] != one[op][:, cols])
            assert bad.size == 0, (fields, op, bad[:5].tolist())
        _check(qs[0].result(), R.select(want, (list(fields), slice(None))))
        for qq in qs:
            st = qq.stats()
            assert st["rounds"] == len(sizes) and st["bytes_sent"] == sum(sizes)
            assert st["segments_by_radix"] == int(st["reasons"].sum())
            assert st["bytes_sent"] < sent_all if G < F else st["bytes_sent"] == sent_all
            qq.close()
    for qq in qa:
        qq.close()
    for k, r in enumerate(rings):
        for op in OPS:
            assert np.array_equal(r.read(op).view(np.uint8), before_reduce[k][op].view(np.uint8)), (k, op)
        if k:                                                          # rings[0] ran the one-process calls above
            assert r.ranges_stats() == before_stats[k]
        r.close()


def test_radix_reasons_on_named_fields(env):
    """one field per generator of tests/range_cases.py in two sets spread over three ranks (one batch): a field query over the fields in
    reverse order with a repeat reports the reasons of its named fields and their pivots, equal to the all-field query's rows"""
    g, ctx = env
    n_rings, cap, n, q = 3, 1 << 20, 1 << 20, (99, 100)
    S = min(RC.SAMPLE_MAX, max(64, n // 32))
    pos = np.arange(S, dtype=np.int64) * (n // S) + (n // S) // 2
    k = RC.k_from_top(n, *q)
    built = []
    for i, (name, fn, route) in enumerate(RC.GENERATORS):
        lay = RC.Layout(n, pos, k, np.random.default_rng([i, n, 9]))
        xf = fn(lay)
        if xf is not None:
            built.append((route(lay) if callable(route) else route, xf))
    F = len(built)
    totals = [cap + cap // 2 + 1, cap - 5, cap + 17]
    olds = [max(0, t - cap) for t in totals]
    cuts = [0, 1, 1057, n // 5, n // 3, n // 3 + 1024, n // 2 + 3, n - 31, n]
    pieces, cur = [], list(totals)
    for j, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        kr = j % n_rings
        cur[kr] -= b - a
        pieces.append((kr, cur[kr], b - a))
    assert all(c >= o for c, o in zip(cur, olds))
    xs = [np.random.default_rng(5 + kr).normal(60.0, 3.0, (F, t)) for kr, t in enumerate(totals)]
    for f, (_, xf) in enumerate(built):
        for (kr, p, ln), a in zip(pieces, cuts[:-1]):
            xs[kr][f, p:p + ln] = xf[a:a + ln]
    thr = np.linspace(55.0, 65.0, F)
    rings = []
    for kr in range(n_rings):
        r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
        _push(r, xs[kr], 1 << 18)
        rings.append(r)
    args = _sets([pieces, pieces])
    qa, full, _ = _lockstep(g, rings, args)
    piv_all = qa[0].pivots()
    fields = list(range(F - 1, -1, -1)) + [F // 2]
    qs, got, _ = _lockstep(g, rings, args, fields)
    rows = _rows(full, fields)
    for op in OPS:
        assert np.array_equal(got[op], rows[op]), op
    expect = {}
    for f in fields:
        if built[f][0] in M.OPEN:
            expect[built[f][0]] = expect.get(built[f][0], 0) + 2
    assert expect
    for qq in qs:
        st = qq.stats()
        assert {g.capi.RANGE_OPEN_REASONS[i]: int(c) for i, c in enumerate(st["reasons"]) if i and c} == expect
        assert st["segments_by_radix"] == sum(expect.values())
        assert np.array_equal(qq.pivots().view(np.uint64), piv_all[fields].view(np.uint64))
        qq.close()
    held = [x[:, o:] for x, o in zip(xs, olds)]
    _check({op: v.view(np.float64) if op != "n_over" else v for op, v in got.items()},
           R.select(_want(held, olds, *args, thr, _alpha(1000, 0.0), q), (fields, slice(None))))
    for qq in qa:
        qq.close()
    for r in rings:
        r.close()


def test_unnamed_field_is_never_read(env):
    """rings whose field 3 is +NaN throughout, or garbage, answer a query that does not name it exactly as rings whose field 3 is a
    gauge, and report no NaN reason"""
    g, ctx = env
    F, cap, W = 8, 1 << 17, 1000
    rings, totals, olds, xs, thr, rng = _rings(g, ctx, 3, W, (99, 100), 0.0, F=F, cap=cap, seed=6)
    sets = _box_sets(rng, 3, totals, olds, cap)
    args = _sets(sets)
    fields = [7, 0, 4, 4, 1]
    qw, want, want_sizes = _lockstep(g, rings, args, fields)
    for fill in ("nan", "garbage"):
        others = []
        for k, t in enumerate(totals):
            x = xs[k].copy() if olds[k] == 0 else np.concatenate([np.zeros((F, olds[k])), xs[k]], axis=1)
            x[3] = np.random.default_rng(k).normal(0.0, 1e300, x.shape[1]) if fill == "garbage" else np.nan
            r = g.Ring(ctx, F, cap, W, thresholds=thr, q_num=99, q_den=100)
            _push(r, x)
            others.append(r)
        qs, got, sizes = _lockstep(g, others, args, fields)
        assert sizes == want_sizes
        for op in OPS:
            assert np.array_equal(got[op], want[op]), (fill, op)
        for qq in qs:
            assert qq.stats()["reasons"][g.capi.RANGE_OPEN_REASONS.index("nan")] == 0
            qq.close()
        for r in others:
            r.close()
    for qq in qw:
        qq.close()
    for r in rings:
        r.close()


def test_three_batches_with_a_field_list(env):
    """64 fields x 140 sets of 1 Mi samples cut into four pieces alternating between two ranks, asked for 64 columns named out of order
    with repeats: three batches of the long route, column g equal to row fields[g] of the all-field query, and min / max / p99 /
    n_over equal to the uncut range of one ring"""
    g, ctx = env
    F, cap = 64, 1 << 20
    rng = np.random.default_rng(3)
    total = cap + 12345
    thr = np.linspace(55.0, 65.0, F)
    rings = [g.Ring(ctx, F, cap, 1000, thresholds=thr) for _ in range(2)]
    for a in range(0, total, 1 << 18):
        rows = rng.normal(60.0, 3.0, (min(1 << 18, total - a), F)).astype(np.float32)
        for r in rings:
            r.push(rows)
    lo = total - cap
    sets, whole = [], []
    for i in range(140):
        a = int(rng.integers(lo, total - cap + 1)) if rng.random() < 0.2 else lo
        b = np.concatenate([[0], np.sort(rng.choice(np.arange(1, cap), 3, replace=False)), [cap]])
        sets.append([((i + j) % 2, a + int(b[j]), int(b[j + 1] - b[j])) for j in range(4)])
        whole.append((a, cap))
    args = _sets(sets)
    fields = rng.integers(0, F, F).tolist()
    assert len(set(fields)) < F and fields != sorted(fields)
    qs, got, sizes = _lockstep(g, rings, args, fields)
    assert len(sizes) >= 1 + 3 * 3                                    # the header, then samples / summaries / lists of three batches
    qa, full, _ = _lockstep(g, rings, args)
    rows = _rows(full, fields)
    for op in OPS:
        assert np.array_equal(got[op], rows[op]), op
    want = _bits(rings[0].reduce_ranges([w[0] for w in whole], [w[1] for w in whole], fields=fields))
    for op in ("min", "max", "p99", "n_over"):
        assert np.array_equal(got[op], want[op]), op
    for qq in qs + qa:
        qq.close()
    for r in rings:
        r.close()


def test_collective_refusals(env):
    g, ctx = env
    cap = 1 << 16
    rings, totals, olds, xs, thr, rng = _rings(g, ctx, 4, 100, (99, 100), 0.0, cap=cap, seed=2)
    n = len(rings)
    good = _sets([[(0, olds[0], 10), (1, olds[1], 10)], [(2, olds[2], 500)], [(0, olds[0], 6000), (3, olds[3], 6000)]])

    def run(fields_of, push_between=None):
        qs = [g.BoxQuery(r, k, n, *good, fields=fields_of(k)) for k, r in enumerate(rings)]
        sizes, outcome = _drive(qs, push_between)
        for q in qs:
            with pytest.raises(g.GpudError):
                q.result()
            q.close()
        return sizes, outcome

    def same(outcome, code, text, step):
        assert all(o is not None for o in outcome), outcome
        assert {(o[0], o[1], o[2]) for o in outcome} == {(code, outcome[0][1], step)}, outcome
        assert text in outcome[0][1], outcome[0][1]

    _, out = run(lambda k: [1, 5] if k == 2 else [1, 6])
    same(out, -1, "rank 2: its call arguments differ from rank 0's", 1)
    _, out = run(lambda k: None if k == 1 else [0, 1, 2, 3, 4, 5, 6, 7])
    same(out, -1, "rank 1: its call arguments differ from rank 0's", 1)
    _, out = run(lambda k: [3, rings[0].F])
    same(out, -1, "fields[1] is 8, not a field of the ring's 8", 1)
    _, out = run(lambda k: [-1])
    same(out, -1, "fields[0] is -1, not a field of the ring's 8", 1)
    sizes, out = run(lambda k: [6, 1], push_between=lambda: rings[1].push(np.full((3, rings[1].F), 50.0)))
    same(out, -6, "rank 1: its ring was pushed into", 2)
    assert len(sizes) == 2
    with pytest.raises(g.GpudError, match="n_fields is 0, not at least 1"):
        g.BoxQuery(rings[0], 0, n, *good, fields=[])
    for r in rings:
        r.close()


_FIELDS = [5, 2, 2, 0]


def _worker(rank, world, init, backend="gloo"):
    import torch
    import torch.distributed as dist
    import gpud_b200 as g
    from gpud_b200.dist import box_range_sets
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, init_method="file://" + init, rank=rank, world_size=world)
    F, cap, W = 8, 1 << 17, 1000
    totals = [cap + 12345 * (k + 1) if k % 2 else cap - 999 * (k + 1) for k in range(world)]
    ctx = g.Context([dev])
    thr = np.linspace(50.0, 70.0, F)
    ring = g.Ring(ctx, F, cap, W, thresholds=thr)
    _push(ring, _fields(F, totals[rank], np.random.default_rng([rank, 5])))
    args = _worker_call(world, cap, totals)
    got = _bits(box_range_sets(ring, *args, fields=_FIELDS))
    full = _bits(box_range_sets(ring, *args))
    ok = True
    for op in OPS:
        if not np.array_equal(got[op], full[op][_FIELDS]):
            print("rank %d:" % rank, op, "differs from the all-field query's rows", file=sys.stderr)
            ok = False
    if rank == 0:                                                     # rebuild every rank's ring from its seed
        rings = [ring] + [g.Ring(ctx, F, cap, W, thresholds=thr, dev=dev) for _ in range(1, world)]
        for k in range(1, world):
            _push(rings[k], _fields(F, totals[k], np.random.default_rng([k, 5])))
        want = _bits(g.rings_reduce_range_sets(rings, *args, fields=_FIELDS))
        long_spread = _long_spread(args)
        for op in OPS:                                                # mean and EMA of long spread sets fold in another order
            cols = slice(None) if op in ("min", "max", "p99", "n_over") else ~long_spread
            if not np.array_equal(got[op][:, cols], want[op][:, cols]):
                print("rank 0:", op, "differs from the one-process call", file=sys.stderr)
                ok = False
        for r in rings[1:]:
            r.close()
    dist.barrier()
    dist.destroy_process_group()
    ring.close()
    ctx.close()
    return 0 if ok else 3


def _processes(world, backend):
    with tempfile.TemporaryDirectory() as d:
        init = os.path.join(d, "init")
        procs = [subprocess.Popen([sys.executable, "-s", os.path.abspath(__file__), "--worker", str(r), str(world), init, backend]) for r in range(world)]
        try:
            codes = [p.wait(timeout=600) for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
    assert codes == [0] * world


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_processes(world):
    _processes(world, "gloo")


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_nccl_processes_on_two_devices():
    _processes(2, "nccl")


if __name__ == "__main__" and len(sys.argv) == 6 and sys.argv[1] == "--worker":
    sys.exit(_worker(int(sys.argv[2]), int(sys.argv[3]), sys.argv[4], sys.argv[5]))
