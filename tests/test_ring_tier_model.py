"""The tier's host plan (gpudh_ring_tier_plan, gpudh_ring_tier_split) against the host model tests/ring_tier.py: after every push of
random sequences the rows held, bytes in use, rows lost, head and tail, and where each row was placed, with row sizes from the
checkpoint model on NVML-like and noise rows; a row that ends exactly at the buffer end, a budget of exactly one row, a push of
CAP - 1023 rows (no loss) and of one more (a row lost); and how range calls split into ring and tier work, with every refusal."""
import ctypes as C

import numpy as np
import pytest

import ring_tier as T

I64 = np.int64


@pytest.fixture(scope="module")
def L():
    import gpud_b200 as g
    return g.lib()


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None and a.size else None


def _plan(L, cap, F, tier_bytes, total0, pushes, sizes):
    pushes = np.asarray(pushes, dtype=I64)
    sizes = np.asarray(sizes, dtype=I64)
    state = np.zeros(6 * (len(pushes) + 1), dtype=I64)
    row_off = np.zeros(len(sizes), dtype=I64)
    rc = L.gpudh_ring_tier_plan(cap, F, tier_bytes, total0, _ptr(pushes), len(pushes), _ptr(sizes), len(sizes), _ptr(state), _ptr(row_off))
    return rc, state.reshape(-1, 6), row_off


def _model(cap, F, tier_bytes, total0, pushes, sizes):
    m = T.Tier(cap, F, tier_bytes, total0)
    m.settle(sizes)
    states = [m.state()]
    for n in pushes:
        m.push(n, sizes)
        states.append(m.state())
    off = np.full(len(sizes), -1, dtype=I64)
    for k, o in m.row_off.items():
        off[k] = o
    return np.array(states, dtype=I64), off


def _sizes(F, n_rows, seed):
    """row bytes from the checkpoint model: NVML-like uint32 gauges (INT blocks of varying width) and f64 noise (RAW blocks)"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_rows):
        if k % 3 == 2:
            bits = rng.normal(0.0, 1.0, (F, T.ROW)).view(np.uint64)
        else:
            step = int(rng.integers(0, 1 << int(rng.integers(0, 20))))
            bits = (1000 + np.cumsum(rng.integers(-step, step + 1, (F, T.ROW)), axis=1)).astype(np.float64).view(np.uint64)
        out.append(T.row_bytes(bits))
    return out


@pytest.mark.parametrize("seed", range(6))
def test_random_pushes(L, seed):
    rng = np.random.default_rng(seed)
    F = int(rng.integers(1, 4))
    cap = int(rng.choice([2048, 4096, 6144]))
    sizes = _sizes(F, 200, seed)
    tier_bytes = int(rng.integers(T.max_row_bytes(F), 6 * T.max_row_bytes(F)))
    total0 = int(rng.integers(0, 3 * cap))
    pushes, t = [], total0
    while t < 150 * T.ROW:
        n = int(rng.choice([1, 7, 1023, 1024, 1025, cap - 1023, cap - 1022, cap, 3 * cap, int(rng.integers(1, cap))]))
        n = min(n, 150 * T.ROW - t + 1)
        pushes.append(n)
        t += n
    rc, state, off = _plan(L, cap, F, tier_bytes, total0, pushes, sizes)
    assert rc == 0
    want_state, want_off = _model(cap, F, tier_bytes, total0, pushes, sizes)
    np.testing.assert_array_equal(state, want_state)
    np.testing.assert_array_equal(off, want_off)


def test_wrap_exactly_at_the_end(L):
    F, cap = 2, 4096
    sizes = _sizes(F, 40, 7)
    tier_bytes = sum(sizes[:5])                    # rows 0..4 fill the buffer to its last byte
    rc, state, off = _plan(L, cap, F, tier_bytes, 0, [T.ROW] * 12, sizes)
    assert rc == 0
    want_state, want_off = _model(cap, F, tier_bytes, 0, [T.ROW] * 12, sizes)
    np.testing.assert_array_equal(state, want_state)
    np.testing.assert_array_equal(off, want_off)
    assert state[5][5] == tier_bytes and state[5][0] == 0 and state[5][2] == tier_bytes   # after row 4: tail at the end, nothing evicted
    assert off[5] == 0 and state[6][0] >= 1                                               # row 5 wraps and evicts the oldest


def test_budget_of_one_row(L):
    F, cap = 3, 2048
    sizes = _sizes(F, 30, 8)
    tier_bytes = T.max_row_bytes(F)
    rc, state, off = _plan(L, cap, F, tier_bytes, 0, [T.ROW] * 20, sizes)
    assert rc == 0
    want_state, want_off = _model(cap, F, tier_bytes, 0, [T.ROW] * 20, sizes)
    np.testing.assert_array_equal(state, want_state)
    np.testing.assert_array_equal(off, want_off)
    assert (state[1:, 1] - state[1:, 0] >= 1).all() and (state[:, 2] <= tier_bytes).all() and state[-1][0] > 10   # small rows pair up
    # one byte less does not hold a row coded at 64 bits
    assert _plan(L, cap, F, tier_bytes - 1, 0, [T.ROW], sizes)[0] == -1


@pytest.mark.parametrize("extra,lost", [(0, 0), (1, 1)])
def test_push_of_cap_minus_1023(L, extra, lost):
    F, cap = 1, 8192
    sizes = _sizes(F, 64, 9)
    total0 = 5 * T.ROW + 1023                      # the newest row is one sample short of complete
    pushes = [cap - 1023 + extra]
    rc, state, off = _plan(L, cap, F, 8 * T.max_row_bytes(F), total0, pushes, sizes)
    assert rc == 0
    want_state, _ = _model(cap, F, 8 * T.max_row_bytes(F), total0, pushes, sizes)
    np.testing.assert_array_equal(state, want_state)
    assert state[1][3] == lost
    if lost:
        assert state[1][0] == 6 and off[5] == -1   # row 5 was overwritten before it was complete: the tier restarts at row 6
    else:
        assert state[1][0] == 0 and off[5] >= 0


def _split(L, total, cap, t_first, t_next, first, length, set_off=None):
    first, length = np.asarray(first, dtype=I64), np.asarray(length, dtype=I64)
    so = None if set_off is None else np.asarray(set_off, dtype=I64)
    n_sets = len(first) if so is None else len(so) - 1
    route = np.zeros(n_sets, dtype=np.int32)
    vfirst = np.zeros(len(first), dtype=I64)
    rows = np.zeros(1 << 16, dtype=I64)
    n_rows, vtotal = C.c_int64(), C.c_int64()
    rc = L.gpudh_ring_tier_split(total, cap, 4, t_first, t_next, _ptr(first), _ptr(length), len(first), _ptr(so), n_sets, _ptr(route),
                                 _ptr(vfirst), _ptr(rows), len(rows), C.byref(n_rows), C.byref(vtotal))
    if rc:
        return rc, None
    return rc, (route.tolist(), rows[:n_rows.value].tolist(), vfirst.tolist(), vtotal.value)


@pytest.mark.parametrize("seed", range(8))
def test_split(L, seed):
    rng = np.random.default_rng(100 + seed)
    cap = int(rng.choice([2048, 8192, 65536]))
    total = int(rng.integers(cap, 40 * cap))
    t_next = total // T.ROW
    t_first = int(rng.integers(0, (total - cap) // T.ROW + 1))
    lo = min(total - cap, t_first * T.ROW)
    n = int(rng.integers(1, 30))
    length = [int(rng.choice([1, 1024, 1025, int(rng.integers(1, 3 * cap))])) for _ in range(n)]
    length = [min(x, total - lo) for x in length]
    first = [int(rng.integers(lo, total - x + 1)) for x in length]
    cuts = sorted(set(rng.integers(1, n, 3).tolist())) if n > 1 else []
    set_off = [0] + cuts + [n]
    for so in (None, set_off):
        rc, got = _split(L, total, cap, t_first, t_next, first, length, so)
        assert rc == 0
        assert got == T.split(total, cap, t_first, t_next, first, length, so)
    # every refusal: before the tier's first sample, past the newest, empty, and a malformed set_off
    for f, ln in ((lo - 1, 1), (total - 5, 6), (lo, 0)):
        assert _split(L, total, cap, t_first, t_next, [f], [ln])[0] == -1
        assert T.split(total, cap, t_first, t_next, [f], [ln]) is None
    assert _split(L, total, cap, t_first, t_next, first, length, [0, n + 1] if n > 1 else [1, 1])[0] == -1


def test_split_ring_only_and_tail(L):
    cap, total = 4096, 20 * 1024 + 300
    t_first, t_next = 3, 20
    # wholly in the ring: route 0, nothing to decode
    assert _split(L, total, cap, t_first, t_next, [total - cap], [cap])[1] == ([0], [], [-1], 0)
    # from the tier up to the newest sample: every row it covers, the last one partial
    rc, (route, rows, vfirst, vtotal) = _split(L, total, cap, t_first, t_next, [5 * 1024 + 7], [total - 5 * 1024 - 7])
    assert route == [1] and rows == list(range(5, 21)) and vfirst == [7] and vtotal == 15 * 1024 + 300
    # two ranges of one set far apart: two runs, laid out one after the other
    rc, (route, rows, vfirst, vtotal) = _split(L, total, cap, t_first, t_next, [3 * 1024 + 1, total - 10], [1024, 10], [0, 2])
    assert route == [1] and rows == [3, 4, 20] and vfirst == [1, 2 * 1024 + 290] and vtotal == 2 * 1024 + 300
