"""gpud_box_query (DESIGN.md §2 "Box sets across processes"): range sets over rings that each belong to one rank of a group.
Simulated ranks: 2 to 8 rings of one config on device 0, with different totals (some wrapped), each driven by its own query; a lockstep
driver steps every rank and "all-gathers" with device-to-device copies into one receive buffer.  Checked:
  - every round's send size is equal on all ranks, and every rank's result is the same bit for bit;
  - the result equals gpud_rings_reduce_range_sets over the same rings in one process: min / max / p99 / n_over bit for bit for every
    set, all six outputs for sets local to one rank and spread sets of up to 1024 samples (one of odd length first, so the dense
    columns after it start odd); mean and EMA of long spread sets, on both sides, within the rounding budget of mean_ema_ref.py's
    reference on each concatenation, and everything against the reference;
  - every radix-select reason forced in sets spread over ranks (tests/range_cases.py), with the reasons and every pivot equal to the
    one-process call's; a call of three long-route batches;
  - every refusal reaches every rank at the same step with the same code and message: differing arguments, a range invalid on one
    rank, and a ring pushed into between two steps (GPUD_E_STATE), with nothing to read afterwards;
  - nothing the rings report changes: their reduce results, gpud_ring_ranges_stats and range-call results read the same.
Real processes: 2 and 3 processes on the one GPU over gloo through dist.box_range_sets, and 2 over NCCL on two GPUs (skipped with
fewer), rank 0 checking against the one-process call.
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
from test_gpu_ring_box_sets import _n_gpus, _sets, _want
from test_gpu_segment_paths import _scratch
from test_gpu_ring_range_sets import _bits, _push
from test_gpu_ring_ranges import OPS, _alpha, _fields, _thr
from test_gpu_window_paths import _check
import mean_ema_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx
    ctx.close()


def _drive(queries, push_between=None):
    """step every rank in lockstep until done; returns (round sizes, per-rank outcome: None or (code, message, step))"""
    import torch
    from gpud_b200.dist import _DevBytes
    sizes, outcome, recv = [], [None] * len(queries), 0
    for step in range(256):
        outs = []
        for r, q in enumerate(queries):
            try:
                outs.append(q.step(recv))
            except Exception as e:                                   # GpudError: its code, and its message
                outcome[r] = (e.code, str(e), step)
                outs.append((0, 0))
        nbs = {nb for _, nb in outs}
        assert len(nbs) == 1, ("send sizes differ", step, [nb for _, nb in outs])
        nb = nbs.pop()
        if nb == 0:
            return sizes, outcome
        sizes.append(nb)
        buf = torch.empty(len(queries) * nb, dtype=torch.uint8, device="cuda:0")
        for r, (ptr, _) in enumerate(outs):
            buf[r * nb:(r + 1) * nb].copy_(torch.as_tensor(_DevBytes(ptr, nb), device="cuda:0"))
        torch.cuda.synchronize()
        if push_between is not None and step == 0:
            push_between()
        recv = buf.data_ptr()                                        # buf stays alive until the next round replaces it
    raise AssertionError("the query did not finish in 256 steps")


def _rings(g, ctx, n_rings, W, q, alpha, F=8, cap=1 << 17, seed=0):
    rng = np.random.default_rng([n_rings, W, q[0], seed])
    totals = [(3 * cap + 54321, cap - 12345, cap, 2 * cap + 1)[k % 4] + 1000 * (k // 4) for k in range(n_rings)]
    xs_all = [_fields(F, t, rng) for t in totals]
    thr = _thr(xs_all[0])
    rings = []
    for k in range(n_rings):
        r = g.Ring(ctx, F, cap, W, thresholds=thr, ema_alpha=alpha, q_num=q[0], q_den=q[1], dev=0)
        _push(r, xs_all[k])
        rings.append(r)
    olds = [max(0, t - cap) for t in totals]
    return rings, totals, olds, [x[:, o:] for x, o in zip(xs_all, olds)], thr, rng


def _box_sets(rng, n_rings, totals, olds, cap):
    def pick(k, n):
        return int(rng.integers(olds[k], totals[k] - n + 1))

    def anyring(n):
        k = int(rng.integers(0, n_rings))
        return (k, pick(k, n), n)
    sets = [[(0, pick(0, 7), 7), (n_rings - 1, pick(n_rings - 1, 8), 8)]]   # spread, odd length: it comes first
    for k in range(n_rings):                                          # local sets: short, one tile, the sample ring, the whole ring
        for n in (1, 33, 1025, 70000):
            sets.append([(k, pick(k, n), n)])
        sets.append([(k, pick(k, 3000), 3000), (k, pick(k, 50), 50)])
    sets.append([(k, olds[k], totals[k] - olds[k]) for k in [1]])
    sets.append([anyring(1) for _ in range(700)])                     # spread: many 1-sample ranges
    for cut in (1, 31, 32, 33, 500, 1000):                            # spread: a join at lane 0 / 31 / mid-row
        a, b = (0, 1) if cut % 2 else (n_rings - 1, 0)
        sets.append([(a, pick(a, cut), cut), (b, pick(b, 1024 - cut), 1024 - cut)])
    for k in range(n_rings):                                          # spread: pieces across each wrapped ring's physical end
        end = (totals[k] // cap) * cap
        if totals[k] > cap and end - 300 >= olds[k] and end + 300 <= totals[k]:
            sets.append([(k, end - 300, 600), ((k + 1) % n_rings, pick((k + 1) % n_rings, 400), 400)])
    sets.append([anyring(10), anyring(20), anyring(30)])
    sets.append([(k, olds[k], totals[k] - olds[k]) for k in range(n_rings)])   # long spread: every ring whole, the box
    sets.append([anyring(1) for _ in range(3000)])                    # ... a join at every sample
    for cut in (1, 1023, 1024, 1025):                                 # ... joins at a tile edge +-1
        sets.append([(0, pick(0, cut), cut), (n_rings - 1, pick(n_rings - 1, 3000), 3000), anyring(700)])
    sets.append([anyring(400), anyring(400), anyring(400)])
    order = np.concatenate([[0], 1 + rng.permutation(len(sets) - 1)])
    return [sets[i] for i in order]


def _query(g, rings, sets):
    ring_of, first, length, set_off = _sets(sets)
    qs = [g.BoxQuery(r, k, len(rings), ring_of, first, length, set_off) for k, r in enumerate(rings)]
    return qs, (ring_of, first, length, set_off)


@pytest.mark.parametrize("n_rings,W,q,alpha", [(2, 1000, (0, 0), 0.0), (5, 999, (999, 1000), 0.9999), (8, 1, (1, 2), 0.0)])
def test_simulated_ranks_against_one_process_and_oracle(env, n_rings, W, q, alpha):
    g, ctx = env
    cap = 1 << 17
    rings, totals, olds, xs, thr, rng = _rings(g, ctx, n_rings, W, q, alpha, cap=cap)
    before_reduce = []
    for r in rings:                                                    # what the rings report must read the same afterwards
        r.reduce_all()
        before_reduce.append({k: r.read(k).copy() for k in OPS})
    before_stats = []
    for k, r in enumerate(rings):
        r.reduce_range_sets([olds[k], olds[k] + 7], [5000, 70000], [0, 1, 2])
        before_stats.append(r.ranges_stats())
    sets = _box_sets(rng, n_rings, totals, olds, cap)
    qs, (ring_of, first, length, set_off) = _query(g, rings, sets)
    sizes, outcome = _drive(qs)
    assert outcome == [None] * n_rings and sizes[0] == 128
    res = [_bits(qq.result()) for qq in qs]
    for k in range(1, n_rings):
        for op in OPS:
            assert np.array_equal(res[k][op], res[0][op]), (k, op)
    one = _bits(g.rings_reduce_range_sets(rings, ring_of, first, length, set_off))
    long_spread = np.array([len({k for k, _, _ in st}) > 1 and sum(n for _, _, n in st) > 1024 for st in sets])
    assert long_spread.any() and (~long_spread).any()
    for op in OPS:
        cols = slice(None) if op in ("min", "max", "p99", "n_over") else ~long_spread
        bad = np.argwhere(res[0][op][:, cols] != one[op][:, cols])
        assert bad.size == 0, (op, bad[:5].tolist())
    _check(qs[0].result(), _want(xs, olds, ring_of, first, length, set_off, thr, _alpha(W, alpha), q))
    for k, qq in enumerate(qs):
        st = qq.stats()
        assert st["rounds"] == len(sizes) and st["bytes_sent"] == sum(sizes)
        assert st["segments_by_radix"] == int(st["reasons"].sum())
        qq.close()
    for k, r in enumerate(rings):
        for op in OPS:
            assert np.array_equal(r.read(op).view(np.uint8), before_reduce[k][op].view(np.uint8)), (k, op)
        if k:                                                          # rings[0] ran the one-process call above
            assert r.ranges_stats() == before_stats[k]
    for r in rings:
        r.close()


def test_query_owns_its_scratch(env):
    """the home ring's range-set results and stats read the same after a query"""
    g, ctx = env
    cap = 1 << 17
    rings, totals, olds, xs, thr, rng = _rings(g, ctx, 3, 100, (99, 100), 0.0, cap=cap, seed=1)
    want = [_bits(r.reduce_range_sets([olds[k], olds[k] + 3], [4000, 40000], [0, 1, 2])) for k, r in enumerate(rings)]
    stats = [r.ranges_stats() for r in rings]
    sets = _box_sets(rng, 3, totals, olds, cap)
    qs, _ = _query(g, rings, sets)
    assert _drive(qs)[1] == [None] * 3
    for k, r in enumerate(rings):
        assert r.ranges_stats() == stats[k]
        got = _bits(r.reduce_range_sets([olds[k], olds[k] + 3], [4000, 40000], [0, 1, 2]))
        assert all(np.array_equal(got[op], want[k][op]) for op in OPS), k
    for q in qs:
        q.close()
    for r in rings:
        r.close()


def test_collective_refusals(env):
    g, ctx = env
    cap = 1 << 16
    rings, totals, olds, xs, thr, rng = _rings(g, ctx, 4, 100, (99, 100), 0.0, cap=cap, seed=2)
    n = len(rings)

    def run(sets, per_rank=None, push_between=None):
        ring_of, first, length, set_off = _sets(sets)
        qs = []
        for k, r in enumerate(rings):
            a = (ring_of, first, length, set_off) if per_rank is None else per_rank(k, ring_of, first, length, set_off)
            qs.append(g.BoxQuery(r, k, n, *a))
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

    good = [[(0, olds[0], 10), (1, olds[1], 10)], [(2, olds[2], 500)], [(0, olds[0], 6000), (3, olds[3], 6000)]]

    def differ(k, ring_of, first, length, set_off):
        length = length.copy()
        if k == 2:
            length[0] += 1
        return ring_of, first, length, set_off
    _, out = run(good, per_rank=differ)
    same(out, -1, "its call arguments differ from rank 0's", 1)
    _, out = run(good + [[(3, totals[3] - 5, 10)]])                                    # past what rank 3's ring holds
    same(out, -1, "range 5", 1)
    sizes, out = run(good, push_between=lambda: rings[1].push(np.full((3, rings[1].F), 50.0)))
    same(out, -6, "rank 1: its ring was pushed into", 2)
    assert len(sizes) == 2
    for r in rings:
        r.close()


def _lockstep(g, rings, ring_of, first, length, set_off):
    qs = [g.BoxQuery(r, k, len(rings), ring_of, first, length, set_off) for k, r in enumerate(rings)]
    sizes, outcome = _drive(qs)
    assert outcome == [None] * len(rings)
    res = [_bits(q.result()) for q in qs]
    for k in range(1, len(rings)):
        for op in OPS:
            assert np.array_equal(res[k][op], res[0][op]), (k, op)
    return qs, res[0], sizes


@pytest.mark.parametrize("n_rings", [2, 4])
def test_radix_reasons_spread_over_ranks(env, n_rings):
    """one set per generator of tests/range_cases.py, its data built against the set's strided pivot sample over the concatenation and
    its pieces spread over the ranks: exact whatever the route; the reasons, the pivots and the results equal the one-process call's"""
    g, ctx = env
    cap, n, q = 1 << 20, 1 << 20, (99, 100)
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
    totals = [cap + cap // 2 + 1, cap - 5, cap + 17, cap][:n_rings]
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
    thr = np.full(F, 60.0)
    rings = []
    for kr in range(n_rings):
        r = g.Ring(ctx, F, cap, 1000, thresholds=thr, q_num=q[0], q_den=q[1])
        _push(r, xs[kr], 1 << 18)
        rings.append(r)
    ring_of, first, length, set_off = _sets([pieces, pieces])
    qs, got, sizes = _lockstep(g, rings, ring_of, first, length, set_off)
    one = _bits(g.rings_reduce_range_sets(rings, ring_of, first, length, set_off))
    for op in ("min", "max", "p99", "n_over"):
        assert np.array_equal(got[op], one[op]), op
    _, n_radix, why = rings[0].ranges_stats()
    piv_one = _scratch(g.lib(), rings[0])[0]
    expect = {}
    for route, _ in built:
        if route in M.OPEN:
            expect[route] = expect.get(route, 0) + 2
    assert why == expect and n_radix == sum(expect.values()), (why, expect)
    for qq in qs:
        st = qq.stats()
        assert st["segments_by_radix"] == n_radix
        assert {g.capi.RANGE_OPEN_REASONS[i]: int(c) for i, c in enumerate(st["reasons"]) if i and c} == why
        assert np.array_equal(qq.pivots().reshape(-1, 2).view(np.uint64), piv_one)
        qq.close()
    held = [x[:, o:] for x, o in zip(xs, olds)]
    _check({k: v.view(np.float64) if k != "n_over" else v for k, v in got.items()},
           _want(held, olds, ring_of, first, length, set_off, thr, _alpha(1000, 0.0), q))
    for r in rings:
        r.close()


def test_three_batches(env):
    """64 fields x 140 sets of 1 Mi samples cut into four pieces alternating between two ranks whose rings hold the same pushed data take
    three batches of the long route; every set reads like the uncut range of one ring"""
    g, ctx = env
    F, cap = 64, 1 << 20
    rng = np.random.default_rng(3)
    total = cap + 12345
    rings = [g.Ring(ctx, F, cap, 1000, thresholds=np.full(F, 60.0)) for _ in range(2)]
    hist = np.empty((F, total))                                       # the pushed samples, for the reference
    for a in range(0, total, 1 << 18):
        rows = rng.normal(60.0, 3.0, (min(1 << 18, total - a), F)).astype(np.float32)
        hist[:, a:a + rows.shape[0]] = rows.T
        for r in rings:
            r.push(rows)
    lo = total - cap
    hist = hist[:, lo:]
    sets, whole = [], []
    for i in range(140):
        a = int(rng.integers(lo, total - cap + 1)) if rng.random() < 0.2 else lo
        b = np.concatenate([[0], np.sort(rng.choice(np.arange(1, cap), 3, replace=False)), [cap]])
        sets.append([((i + j) % 2, a + int(b[j]), int(b[j + 1] - b[j])) for j in range(4)])
        whole.append((a, cap))
    ring_of, first, length, set_off = _sets(sets)
    qs, got, sizes = _lockstep(g, rings, ring_of, first, length, set_off)
    rc, _, route, _, _, _, _, _ = g.capi.box_query_plan([total, total], cap, ring_of, first, length, set_off, F=F)
    assert rc == 0 and np.all(route == 2)
    want = _bits(rings[0].reduce_ranges([w[0] for w in whole], [w[1] for w in whole]))
    for op in ("min", "max", "p99", "n_over"):
        assert np.array_equal(got[op], want[op]), op
    # mean and EMA fold in another order than the uncut range's: both against the reference on every field
    ref = {}
    for a in sorted({w[0] for w in whole}):
        ref[a] = R.select(R.windows_fields(hist[:, a - lo:a - lo + cap], cap, np.full(F, 60.0), _alpha(1000, 0.0)), (slice(None), 0))
    want_ref = R.stack([ref[w[0]] for w in whole])
    for side, d in (("box", got), ("one ring", want)):
        R.check_mean_ema({op: d[op].view(np.float64) for op in ("mean", "ema")}, want_ref, what=side)
    assert len(sizes) >= 1 + 3 * 3                                    # the header, then samples / summaries / lists of three batches
    for q in qs:
        q.close()
    for r in rings:
        r.close()


_WORKER_SETS = 24


def _worker_call(world, cap, totals):
    rng = np.random.default_rng([world, 77])
    olds = [max(0, t - cap) for t in totals]
    sets = []
    for s in range(_WORKER_SETS):
        if s % 3 == 0:
            k = s % world
            n = int(rng.integers(1, 90000))
            sets.append([(k, int(rng.integers(olds[k], totals[k] - n + 1)), n)])
        elif s % 4 == 1:                                              # long and spread
            sets.append([(k, int(rng.integers(olds[k], totals[k] - 30000 + 1)), 30000) for k in range(world)])
        else:
            parts = []
            for _ in range(int(rng.integers(2, 6))):
                k, n = int(rng.integers(0, world)), int(rng.integers(1, 200))
                parts.append((k, int(rng.integers(olds[k], totals[k] - n + 1)), n))
            sets.append(parts)
    return _sets(sets)


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
    thr = np.full(F, 60.0)
    ring = g.Ring(ctx, F, cap, W, thresholds=thr)
    _push(ring, _fields(F, totals[rank], np.random.default_rng([rank, 5])))
    args = _worker_call(world, cap, totals)
    got = _bits(box_range_sets(ring, *args))
    ok = True
    if rank == 0:                                                     # rebuild every rank's ring from its seed
        rings = [ring] + [g.Ring(ctx, F, cap, W, thresholds=thr, dev=dev) for _ in range(1, world)]
        for k in range(1, world):
            _push(rings[k], _fields(F, totals[k], np.random.default_rng([k, 5])))
        want = _bits(g.rings_reduce_range_sets(rings, *args))
        ring_of, _, length, set_off = args
        long_spread = np.array([len(set(ring_of[a:b].tolist())) > 1 and length[a:b].sum() > 1024 for a, b in zip(set_off[:-1], set_off[1:])])
        for op in OPS:                                                # mean and EMA of long spread sets fold in another order
            cols = slice(None) if op in ("min", "max", "p99", "n_over") else ~long_spread
            if not np.array_equal(got[op][:, cols], want[op][:, cols]):
                print("rank 0:", op, "differs from the one-process call", file=sys.stderr)
                ok = False
        ref = R.select(_want([_fields(F, t, np.random.default_rng([k, 5])) for k, t in enumerate(totals)], [0] * world, *args, thr,
                             _alpha(W, 0.0), (0, 0)), (slice(None), long_spread))
        for side, d in (("box", got), ("one process", want)):
            try:
                R.check_mean_ema({op: d[op].view(np.float64)[:, long_spread] for op in ("mean", "ema")}, ref, what=side)
            except AssertionError as e:
                print("rank 0: mean / EMA of long spread sets:", e, file=sys.stderr)
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
