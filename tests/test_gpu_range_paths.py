"""The whole-range order statistic (gpud_ring_reduce_range) against the oracle and against the numpy model of its routes
(test_range_paths_model.py), on the fields of range_cases.py: one field per route in every ring, so the fields the radix select
redoes sit at non-contiguous indices.  Values: min / max / the order statistic / n_over bit for bit, mean and EMA within
the rounding budget of mean_ema_ref.py (its extended-precision reference over one window of the whole range).  Routes, for
sampled ranges: range_stats' count of fields redone and their reasons, and the pivots, list fill and per-window class counts the
pass left in the ring's scratch (gpudh_ring_range_scratch), all exactly as the model predicts.  A fault there usually costs only
time, since the radix select still finds the right value; these checks see it.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle as O
import mean_ema_ref as R
import range_cases as RC
from test_range_paths_model import model_ring

pytestmark = pytest.mark.gpu

W = 1000                        # the ring's own window: only the EMA's alpha depends on it here
E_STATE = -6                    # GPUD_E_STATE


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    L = g.lib()
    L.gpudh_ring_range_scratch.restype = C.c_int32
    L.gpudh_ring_range_scratch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
    yield g, ctx, L
    ctx.close()


def _scratch(L, ring, F):
    """(pivots [F][2] as raw bits, fill [F], class counts [F][nw][4]) of the last reduce_range, or the hook's error code"""
    piv = np.empty((F, 2), dtype=np.float64)
    fill = np.empty(F, dtype=np.uint32)
    nw = C.c_int64()
    rc = L.gpudh_ring_range_scratch(ring._h, piv.ctypes.data, fill.ctypes.data, None, C.byref(nw))
    if rc:
        return rc
    cls = np.empty((F, nw.value, 4), dtype=np.uint32)
    assert L.gpudh_ring_range_scratch(ring._h, piv.ctypes.data, fill.ctypes.data, cls.ctypes.data, C.byref(nw)) == 0
    return piv.view(np.uint64), fill, cls


def _f64bits(key):
    return int(O.key_to_f64(np.array([key], dtype=np.uint64)).view(np.uint64)[0])


def _run(env, cap, pushed, last_n, q_num, q_den, xs):
    """push xs[F][n] as the newest n of `pushed` rows into a ring of capacity cap, reduce the range, check values against the
    oracle; returns what the routes checks need"""
    g, ctx, L = env
    F, n = xs.shape
    thr = xs[:, n // 3].copy()                                # a sample's own value: the compare is a strict >
    r = g.Ring(ctx, F, cap, W, thresholds=thr, q_num=q_num, q_den=q_den)
    try:
        rows = np.zeros((pushed, F))
        rows[pushed - n:] = xs.T
        r.push(rows)
        del rows
        got = r.reduce_range(last_n)
        stats, reasons = None, None
        try:
            stats = r.range_stats()
            reasons = dict(r.range_open_reasons)
        except g.GpudError as e:
            stats = e.code
        scratch = _scratch(L, r, F)
    finally:
        r.close()
    want = R.windows_fields(xs, n, thr, min(2.0 / (W + 1.0), 0.9999), q_num, q_den)
    for k in ("min", "max", "p99"):
        bad = np.flatnonzero(got[k].view(np.uint64) != want[k][:, 0].view(np.uint64))
        assert bad.size == 0, (k, bad.tolist(), got[k][bad[0]], want[k][bad[0], 0])
    assert np.array_equal(got["n_over"], want["n_over"][:, 0])
    R.check_mean_ema(got, R.select(want, (slice(None), 0)))
    return got, stats, reasons, scratch


@pytest.mark.parametrize("case", RC.cases(), ids=["%s-q%d_%d" % (s["name"], qn, qd) for s, qn, qd in RC.cases()])
def test_sampled_range_routes(env, case):
    shape, q_num, q_den = case
    flds = RC.ring_fields(shape, q_num, q_den)
    names = [name for name, _, _ in flds]
    xs = np.stack([x for _, _, x in flds])
    mr = model_ring(shape["cap"], shape["pushed"], RC.shape_n(shape), q_num, q_den, xs)
    got, stats, reasons, scratch = _run(env, shape["cap"], shape["pushed"], shape["last_n"], q_num, q_den, xs)
    for f, name in enumerate(names):
        assert got["p99"][f:f + 1].view(np.uint64)[0] == np.uint64(_f64bits(mr["fields"][f]["answer"])), name
    assert isinstance(stats, tuple), stats
    assert stats[2] == mr["n_open"], (stats[2], mr["n_open"], [(n, f["route"]) for n, f in zip(names, mr["fields"])])
    assert reasons == dict(mr["reasons"]), (reasons, dict(mr["reasons"]))
    piv, fill, cls = scratch
    assert cls.shape[1] == mr["nw"]
    for f, (name, m) in enumerate(zip(names, mr["fields"])):
        assert (int(piv[f, 0]), int(piv[f, 1])) == (m["lo"], m["hi"]), (name, hex(piv[f, 0]), hex(m["lo"]), hex(piv[f, 1]), hex(m["hi"]))
        assert int(fill[f]) == m["fill"], (name, int(fill[f]), m["fill"])
        bad = np.argwhere(cls[f].astype(np.int64) != m["cls"])
        assert bad.size == 0, (name, bad[:4].tolist(), cls[f][bad[0][0]].tolist(), m["cls"][bad[0][0]].tolist())


@pytest.mark.parametrize("case", RC.short_cases(), ids=[c[0] for c in RC.short_cases()])
def test_short_range_radix_select(env, case):
    """ranges below 64 Ki: every non-constant field through k_sel_hist / k_sel_pick / k_sel_collect and the list select of
    k_sel_final; no sampled pass, so range_stats and the scratch hook report GPUD_E_STATE"""
    name, cap, pushed, last_n, q_num, q_den, xs = case
    got, stats, reasons, scratch = _run(env, cap, pushed, last_n, q_num, q_den, xs)
    assert stats == E_STATE and scratch == E_STATE, (stats, scratch)
