"""Model check (no GPU) of the plan and verdict of gpud_box_query (DESIGN.md §2 "Box sets across processes") through gpudh_box_query_plan.
The verdict is a function of the gathered headers and the call's arguments alone, so every rank that holds the same headers reaches it:
  - each set's route and owner against a Python model, and against gpudh_rings_range_sets_plan on the same arguments (the same
    calls accepted, short spread sets on its short route, long ones on its long route with the same pivot reads, each read by the rank
    whose ring the one-process plan reads it from);
  - the header and samples rounds' send_bytes against the model's formula, which depends only on what every rank holds alike;
  - every refusal from the headers: an invalid range on one rank, differing arguments, each differing config field, a duplicated,
    misplaced or unknown rank, n_ranks that differ, a rank that could not start, m_s > UINT32_MAX and F x n_sets above the limit."""
import numpy as np
import pytest

from gpud_b200 import capi
from test_ring_box_sets_model import plan as rings_plan

E_INVALID, E_STATE = -1, -6
HDR_RANK, HDR_RANKS, HDR_ARGS, HDR_STATUS = 1, 2, 11, 12
CONFIG_WORDS = {3: "n_fields", 4: "window", 5: "capacity", 6: "ema_alpha", 7: "quantile", 8: "quantile", 9: "thresholds"}


def _model(totals, cap, ring_of, first, length, set_off, F):
    """(route, owner, send_bytes of the first two rounds) of the model: a set is local when one rank holds all its ranges, else spread,
    short up to 1024 samples (the sizes are those of calls without long spread sets)"""
    n_sets, n = len(set_off) - 1, len(totals)
    route, owner, own = np.zeros(n_sets, np.int32), np.full(n_sets, -1, np.int32), np.zeros(n, np.int64)
    for s in range(n_sets):
        ks = set(ring_of[set_off[s]:set_off[s + 1]].tolist())
        if len(ks) == 1:
            owner[s] = ks.pop()
        elif length[set_off[s]:set_off[s + 1]].sum() > 1024:
            route[s] = 2
        else:
            route[s] = 1
            for i in range(set_off[s], set_off[s + 1]):
                own[ring_of[i]] += length[i]
    n_local = int((route == 0).sum())
    return route, owner, np.array([128, 8 * (2 + 6 * F * n_local + F * int(own.max()))], np.int64)


def _random_call(rng, n_ranks, cap, n_sets, F=4, long_spread=False):
    totals = [int(rng.integers(cap // 2, 3 * cap)) for _ in range(n_ranks)]
    ring_of, first, length, set_off = [], [], [], [0]
    for s in range(n_sets):
        k = int(rng.integers(1, 6))
        one = rng.random() < 0.4
        r0 = int(rng.integers(0, n_ranks))
        budget = 1024 if not (one or long_spread) else 4 * cap
        for _ in range(k):
            r = r0 if one else int(rng.integers(0, n_ranks))
            held = min(totals[r], cap)
            n = int(rng.integers(1, max(2, min(held, budget // k) + 1)))
            ring_of.append(r)
            first.append(int(rng.integers(totals[r] - held, totals[r] - n + 1)))
            length.append(n)
        set_off.append(len(first))
    return totals, np.array(ring_of, np.int32), np.array(first, np.int64), np.array(length, np.int64), np.array(set_off, np.int64)


@pytest.mark.parametrize("n_ranks", [2, 3, 8])
@pytest.mark.parametrize("seed", range(4))
def test_routes_and_sizes_against_model(n_ranks, seed):
    cap, F = 1 << 12, 4
    rng = np.random.default_rng([n_ranks, seed])
    totals, ring_of, first, length, set_off = _random_call(rng, n_ranks, cap, 40, F)
    rc, msg, route, owner, sb, _, _, _ = capi.box_query_plan(totals, cap, ring_of, first, length, set_off, F=F)
    assert rc == 0, msg
    want = _model(totals, cap, ring_of, first, length, set_off, F)
    assert np.array_equal(route, want[0]) and np.array_equal(owner, want[1]) and np.array_equal(sb[:2], want[2]) and sb[2] == 0
    rc1, rroute = rings_plan(totals, cap, ring_of, first, length, set_off, F=F, pivots=False)[:2]
    assert rc1 == 0
    assert np.all(rroute[route == 1] == 0)     # every spread set is on the short route of the one-process call


@pytest.mark.parametrize("n_ranks", [2, 3, 8])
@pytest.mark.parametrize("seed", range(3))
def test_long_spread_sets_and_pivot_owners(n_ranks, seed):
    """long spread sets: the one-process plan's long route, its pivot reads, each owned by the rank whose ring it reads"""
    cap, F = 1 << 14, 4
    rng = np.random.default_rng([n_ranks, seed, 7])
    totals, ring_of, first, length, set_off = _random_call(rng, n_ranks, cap, 30, F, long_spread=True)
    rc, msg, route, owner, sb, _, piv_n, piv_owner = capi.box_query_plan(totals, cap, ring_of, first, length, set_off, F=F)
    assert rc == 0, msg
    assert np.array_equal(route, _model(totals, cap, ring_of, first, length, set_off, F)[0])
    assert (route == 2).any() and sb[2] > 0
    rc1, rroute, _, _, _, rpiv_n, (rpiv_rings, _) = rings_plan(totals, cap, ring_of, first, length, set_off, F=F)
    assert rc1 == 0
    assert np.all(rroute[route == 2] > 0) and np.all(rroute[route == 1] == 0)
    for s in np.flatnonzero(route == 2):
        assert piv_n[s] == rpiv_n[s] > 0
        assert np.array_equal(piv_owner[s, :piv_n[s]], rpiv_rings[s, :piv_n[s]])


def _call():
    """ranks 0..2, cap 4096: a local set per rank, two spread sets"""
    totals = [5000, 3000, 9000]
    ring_of = np.array([0, 1, 2, 0, 1, 2, 1], np.int32)
    first = np.array([4000, 100, 8000, 4500, 2900, 5000, 2000], np.int64)
    length = np.array([900, 50, 1000, 100, 100, 200, 10], np.int64)
    set_off = np.array([0, 1, 2, 3, 5, 7], np.int64)
    return totals, ring_of, first, length, set_off


def test_spread_and_local_sets():
    totals, ring_of, first, length, set_off = _call()
    rc, msg, route, owner, sb, hdr, _, _ = capi.box_query_plan(totals, 4096, ring_of, first, length, set_off, F=3)
    assert rc == 0, msg
    assert route.tolist() == [0, 0, 0, 1, 1] and owner.tolist() == [0, 1, 2, -1, -1]
    assert sb.tolist() == [128, 8 * (2 + 6 * 3 * 3 + 3 * 200), 0]     # spread samples: rank 0 holds 100, rank 1 110, rank 2 200
    assert hdr[:, HDR_RANK].tolist() == [0, 1, 2] and np.all(hdr[:, HDR_RANKS] == 3) and hdr[:, 10].tolist() == totals


def _refusal(headers=None, totals=None, **kw):
    t, ring_of, first, length, set_off = _call()
    a = dict(ring_of=ring_of, first=first, length=length, set_off=set_off)
    a.update(kw)
    rc, msg, *_ = capi.box_query_plan(totals or t, 4096, a["ring_of"], a["first"], a["length"], a["set_off"], F=3, headers=headers)
    return rc, msg


def _headers():
    t, ring_of, first, length, set_off = _call()
    return capi.box_query_plan(t, 4096, ring_of, first, length, set_off, F=3)[5].copy()


def test_refusals_from_headers():
    rc, msg = _refusal(totals=[5000, 3000, 4000])                           # range 2 is past what rank 2 holds
    assert rc == E_INVALID and "range 2" in msg and "ring 2" in msg
    h = _headers(); h[1, HDR_ARGS] ^= 1
    assert _refusal(h) == (E_INVALID, "rank 1: its call arguments differ from rank 0's")
    for w, name in CONFIG_WORDS.items():
        h = _headers(); h[2, w] += 1
        assert _refusal(h) == (E_INVALID, "rank 2: config field %s differs from rank 0's" % name)
    h = _headers(); h[2, HDR_RANK] = 1
    assert _refusal(h) == (E_INVALID, "rank 1 is duplicated (gather slots 1 and 2)")
    h = _headers(); h[[1, 2]] = h[[2, 1]]
    assert _refusal(h) == (E_INVALID, "gather slot 1 holds rank 2: the gather must be in rank order")
    h = _headers(); h[0, HDR_RANK] = 7
    assert _refusal(h)[0] == E_INVALID and "rank 7 is not a rank" in _refusal(h)[1]
    h = _headers(); h[1, HDR_RANKS] = 4
    assert _refusal(h) == (E_INVALID, "rank 1: n_ranks is 4, the gather holds 3")
    h = _headers(); h[1, 0] = 0
    assert _refusal(h) == (E_INVALID, "gather slot 1: not a box query header")
    h = _headers(); h[2, HDR_STATUS] = E_STATE
    assert _refusal(h) == (E_STATE, "rank 2 could not start the query: its ring changed")
    rc, msg = _refusal(ring_of=np.array([0, 1, 2, 0, 1, 2, 3], np.int32))
    assert rc == E_INVALID and msg.startswith("range 6: rank_of is 3")
    rc, msg = _refusal(length=np.array([900, 50, 1000, 100, 100, 1100, 10], np.int64))   # set 4: 1110 samples over ranks 2 and 1
    assert rc == 0, msg                                                     # a long spread set is answered, not refused


def test_set_and_size_refusals():
    cap = 1 << 20
    n = 4097                                                                  # 4097 x 1 Mi > UINT32_MAX samples in one set
    ring_of, first, length = np.zeros(n, np.int32), np.zeros(n, np.int64), np.full(n, cap, np.int64)
    rc, msg, *_ = capi.box_query_plan([cap, cap], cap, ring_of, first, length, [0, n], F=1)
    assert rc == E_INVALID and "set 0: more than UINT32_MAX samples" in msg
    n_sets = (1 << 24) // 4 + 1
    so = np.arange(n_sets + 1, dtype=np.int64)
    rc, msg, *_ = capi.box_query_plan([10, 10], 16, np.zeros(n_sets, np.int32), np.zeros(n_sets, np.int64), np.ones(n_sets, np.int64), so, F=4)
    assert rc == E_INVALID and "exceed GPUD_RANGES_MAX_SEGMENTS" in msg
    rc, msg, *_ = capi.box_query_plan([10, 10], 16, [0], [0], [1], [0, 0, 1], F=4)
    assert rc == E_INVALID and "set 0 is empty" in msg
