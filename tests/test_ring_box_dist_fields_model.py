"""Model check (no GPU) of the plan and verdict of a box query over chosen fields (gpud_box_query_create_fields, DESIGN.md §2 "Box sets
across processes", "Field selection") through gpudh_box_query_plan_fields:
  - routes and owners are the all-field plan's, and the samples(0) and summaries(0) sizes are the model's formula with G = n_fields
    columns in place of F;
  - an all-field query's headers are gpudh_box_query_plan's byte for byte, and a field query's differ only in the argument hash;
  - refusals from the headers: lists that differ between ranks, a list on one rank and none on another, a field of -1 or F named with
    its position, and the segment limit counted on n_fields x n_sets."""
import ctypes as C

import numpy as np
import pytest

from gpud_b200 import capi
from test_ring_box_dist_model import _call, _model, _random_call

E_INVALID = -1
HDR_ARGS = 11


def _plan(totals, cap, ring_of, first, length, set_off, F, fields, headers=None):
    """gpudh_box_query_plan_fields with fields None passed as NULL: (rc, message, route, owner, send_bytes [3], headers)"""
    L = capi.lib()
    totals = np.ascontiguousarray(totals, dtype=np.int64)
    ro, fi, ln, so = capi._box_args(ring_of, first, length, set_off)
    n_sets = so.shape[0] - 1
    fl = None if fields is None else np.ascontiguousarray(fields, dtype=np.int32)
    hdr = np.zeros((totals.shape[0], 16), dtype=np.int64)
    hin = None if headers is None else np.ascontiguousarray(headers, dtype=np.int64)
    route, owner, sb = np.zeros(n_sets, np.int32), np.zeros(n_sets, np.int32), np.zeros(3, np.int64)
    msg = C.create_string_buffer(512)
    rc = L.gpudh_box_query_plan_fields(totals.shape[0], C.c_void_p(totals.ctypes.data), cap, F,
                                       C.c_void_p(fl.ctypes.data) if fl is not None else None, 0 if fl is None else fl.shape[0], 99, 100,
                                       C.c_void_p(ro.ctypes.data), C.c_void_p(fi.ctypes.data), C.c_void_p(ln.ctypes.data), fi.shape[0],
                                       C.c_void_p(so.ctypes.data), n_sets, C.c_void_p(hdr.ctypes.data),
                                       C.c_void_p(hin.ctypes.data) if hin is not None else None, C.c_void_p(route.ctypes.data),
                                       C.c_void_p(owner.ctypes.data), C.c_void_p(sb.ctypes.data), None, None, msg, 512)
    return rc, msg.value.decode(), route, owner, sb, hdr


def _lists(rng, F):
    """[f] for the first, a middle and the last field, a non-identity list with repeats, a random one, and all F in order"""
    return [[0], [F // 2], [F - 1], [5 % F, 2 % F, 2 % F, 0], rng.integers(0, F, int(rng.integers(1, 2 * F))).tolist(), list(range(F))]


@pytest.mark.parametrize("n_ranks", [2, 3, 8])
@pytest.mark.parametrize("seed", range(3))
def test_routes_and_sizes_against_model(n_ranks, seed):
    cap, F = 1 << 12, 8
    rng = np.random.default_rng([n_ranks, seed, 11])
    totals, ring_of, first, length, set_off = _random_call(rng, n_ranks, cap, 40, F)
    rc0, msg0, route0, owner0, sb0, hdr0 = _plan(totals, cap, ring_of, first, length, set_off, F, None)
    assert rc0 == 0, msg0
    old = capi.box_query_plan(totals, cap, ring_of, first, length, set_off, F=F)
    assert np.array_equal(hdr0, old[5]) and np.array_equal(sb0, old[4])       # the all-field query's headers are untouched
    for fields in _lists(rng, F):
        G = len(fields)
        rc, msg, route, owner, sb, hdr = _plan(totals, cap, ring_of, first, length, set_off, F, fields)
        assert rc == 0, msg
        assert np.array_equal(route, route0) and np.array_equal(owner, owner0)
        want = _model(totals, cap, ring_of, first, length, set_off, G)
        assert np.array_equal(route, want[0]) and np.array_equal(owner, want[1]) and np.array_equal(sb[:2], want[2]) and sb[2] == 0
        differ = np.argwhere(hdr != hdr0)
        assert set(differ[:, 1].tolist()) == {HDR_ARGS} and len(differ) == n_ranks, (fields, differ.tolist())


@pytest.mark.parametrize("n_ranks", [2, 3, 8])
@pytest.mark.parametrize("seed", range(3))
def test_long_spread_sizes_scale_with_the_fields(n_ranks, seed):
    """every word of samples(0) and summaries(0) after the status words is per column: one batch, G columns in place of F"""
    cap, F = 1 << 14, 8
    rng = np.random.default_rng([n_ranks, seed, 12])
    totals, ring_of, first, length, set_off = _random_call(rng, n_ranks, cap, 30, F, long_spread=True)
    rc0, msg0, route0, owner0, sb0, _ = _plan(totals, cap, ring_of, first, length, set_off, F, None)
    assert rc0 == 0, msg0
    assert (route0 == 2).any() and sb0[2] > 0
    for fields in _lists(rng, F):
        G = len(fields)
        rc, msg, route, owner, sb, _ = _plan(totals, cap, ring_of, first, length, set_off, F, fields)
        assert rc == 0, msg
        assert np.array_equal(route, route0) and np.array_equal(owner, owner0)
        assert sb[0] == 128
        for i in (1, 2):
            assert (sb0[i] - 16) % F == 0 and sb[i] - 16 == (sb0[i] - 16) // F * G, (fields, i, sb[i], sb0[i])


def test_refusals_from_headers():
    totals, ring_of, first, length, set_off = _call()
    F = 3

    def plan(fields, headers=None):
        return _plan(totals, 4096, ring_of, first, length, set_off, F, fields, headers)[:2]

    assert plan([2, 0, 0])[0] == 0
    a, b, none = [_plan(totals, 4096, ring_of, first, length, set_off, F, f)[5] for f in ([2, 0, 0], [2, 0, 1], None)]
    for mine, theirs in (([2, 0, 0], b), ([2, 0, 0], none), (None, a)):            # differing lists; a list against none; none against a list
        h = (none if mine is None else a).copy()
        h[1, HDR_ARGS] = theirs[1, HDR_ARGS]
        assert plan(mine, h) == (E_INVALID, "rank 1: its call arguments differ from rank 0's")
    assert plan([0, 1, -1]) == (E_INVALID, "fields[2] is -1, not a field of the ring's 3")
    assert plan([3]) == (E_INVALID, "fields[0] is 3, not a field of the ring's 3")
    assert plan([0, 1, 2]) == (0, "") and plan([2, 2, 2, 2, 2, 2, 2]) == (0, "")


def test_segment_limit_counts_the_fields():
    """4 fields x (2^24 / 8 + 1) sets are within GPUD_RANGES_MAX_SEGMENTS; 8 named fields over the same sets are not"""
    n_sets = (1 << 24) // 8 + 1
    so = np.arange(n_sets + 1, dtype=np.int64)
    args = ([10, 10], 16, np.zeros(n_sets, np.int32), np.zeros(n_sets, np.int64), np.ones(n_sets, np.int64), so, 4)
    rc, msg = _plan(*args, [0] * 8)[:2]
    assert rc == E_INVALID and msg == "8 fields x %d sets exceed GPUD_RANGES_MAX_SEGMENTS" % n_sets
    rc, msg = _plan(*args, [3, 1])[:2]
    assert rc == 0, msg
