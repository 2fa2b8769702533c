"""The split of range calls over several rings that reach into their tiers (gpudh_rings_tier_split) against the host model
tests/ring_box_tier.py: rings of different totals, some untiered; tiers shorter than their ring, after eviction and after a restart that
lost rows; partial newest rows; sets that mix ring and tier ranges across rings; every ring's reach at lo_k - 1 (refused) and lo_k
(taken), and ranges ending at total_k (taken) and total_k + 1 (refused).  With one ring the hook gives gpudh_ring_tier_split's answers
on test_ring_tier_model.py's cases and on every call of test_gpu_tier_paths.py."""
import ctypes as C

import numpy as np
import pytest

import ring_box_tier as B
import test_tier_paths_model as TM
from test_ring_tier_model import _split as _split_one

I64 = np.int64
ROW = B.ROW


@pytest.fixture(scope="module")
def L():
    import gpud_b200 as g
    return g.lib()


def _ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None and a.size else None


def _split(L, totals, cap, tiers, ring_of, first, length, set_off=None):
    """the hook's answer in the model's shape, or (rc, None)"""
    nr = len(totals)
    totals = np.asarray(totals, dtype=I64)
    tf = np.array([-1 if t is None else t[0] for t in tiers], dtype=I64)
    tn = np.array([0 if t is None else t[1] for t in tiers], dtype=I64)
    ro = None if ring_of is None else np.asarray(ring_of, dtype=np.int32)
    first, length = np.asarray(first, dtype=I64), np.asarray(length, dtype=I64)
    so = None if set_off is None else np.asarray(set_off, dtype=I64)
    n = len(first)
    n_sets = n if so is None else len(so) - 1
    route = np.zeros(max(n_sets, 1), dtype=np.int32)
    vslot = np.zeros(max(n, 1), dtype=np.int32)
    vfirst = np.zeros(max(n, 1), dtype=I64)
    slot_ring = np.zeros(nr, dtype=np.int32)
    vtotal = np.zeros(nr, dtype=I64)
    slot_rows = np.zeros(nr + 1, dtype=I64)
    rows = np.zeros(1 << 16, dtype=I64)
    dec = np.zeros(1 << 16, dtype=np.uint8)
    n_slots, vcap = C.c_int32(), C.c_int64()
    rc = L.gpudh_rings_tier_split(_ptr(totals), nr, cap, _ptr(tf), _ptr(tn), _ptr(ro), _ptr(first), _ptr(length), n, _ptr(so), n_sets, _ptr(route),
                                  _ptr(vslot), _ptr(vfirst), C.byref(n_slots), _ptr(slot_ring), _ptr(vtotal), _ptr(slot_rows), _ptr(rows), _ptr(dec),
                                  len(rows), C.byref(vcap))
    if rc:
        return rc, None
    slots = [(int(slot_ring[v]), rows[slot_rows[v]:slot_rows[v + 1]].tolist(), dec[slot_rows[v]:slot_rows[v + 1]].astype(int).tolist(), int(vtotal[v]))
             for v in range(n_slots.value)]
    return rc, (route[:n_sets].tolist(), slots, vslot[:n].tolist(), vfirst[:n].tolist(), vcap.value)


def _ring(rng, cap, kind):
    """(total, tier) of one ring: untiered, a tier reaching before the ring, one shorter than the ring (eviction), one restarted at
    the first whole row after a lost row (empty or not), or a ring not yet full"""
    total = int(rng.integers(3 * cap, 30 * cap)) + int(rng.choice([0, 1, 300, 1023]))
    held = total - cap
    whole = -(-held // ROW)
    if kind == "none":
        return total, None
    if kind == "young":
        total = int(rng.integers(1, cap))
        return total, (0, total // ROW)
    if kind == "long":
        return total, (int(rng.integers(0, held // ROW + 1)), total // ROW)
    if kind == "short":
        return total, (int(rng.integers(whole + 1, total // ROW + 1)), total // ROW)
    return total, (whole, total // ROW)                                 # "restart"


def _case(rng, nr, cap):
    kinds = ["long", "none", "short", "restart", "young"]
    rings = [_ring(rng, cap, kinds[k % len(kinds)] if k else str(rng.choice(kinds))) for k in range(nr)]
    totals = [t for t, _ in rings]
    tiers = [tr for _, tr in rings]
    los = [B.reach(t, cap, tr) for t, tr in rings]

    def pick(k, n):
        n = min(n, totals[k] - los[k])
        return (k, int(rng.integers(los[k], totals[k] - n + 1)), n)
    sets = []
    for _ in range(int(rng.integers(3, 25))):
        m = int(rng.integers(1, 5))
        sets.append([pick(int(rng.integers(0, nr)), int(rng.choice([1, 31, 1024, 1025, 3000, cap + 5]))) for _ in range(m)])
    for k in range(nr):
        sets.append([(k, los[k], totals[k] - los[k])])                 # every ring whole from its reach
        sets.append([(k, totals[k] - 1, 1), pick((k + 1) % nr, 700)])  # the partial newest row, joined to another ring
    order = rng.permutation(len(sets))
    sets = [sets[i] for i in order]
    ring_of = [k for s in sets for k, _, _ in s]
    first = [f for s in sets for _, f, _ in s]
    length = [n for s in sets for _, _, n in s]
    set_off = np.cumsum([0] + [len(s) for s in sets]).tolist()
    return totals, tiers, los, ring_of, first, length, set_off


@pytest.mark.parametrize("seed", range(12))
def test_split_against_model(L, seed):
    rng = np.random.default_rng(400 + seed)
    nr = int(rng.choice([2, 3, 5, 8]))
    cap = int(rng.choice([2048, 5000, 8192, 65536]))
    totals, tiers, los, ring_of, first, length, set_off = _case(rng, nr, cap)
    want = B.split(totals, cap, tiers, ring_of, first, length, set_off)
    assert want is not None
    rc, got = _split(L, totals, cap, tiers, ring_of, first, length, set_off)
    assert rc == 0 and got == want
    # every range as its own set too (set_off NULL)
    rc, got = _split(L, totals, cap, tiers, ring_of, first, length)
    assert rc == 0 and got == B.split(totals, cap, tiers, ring_of, first, length)


def test_split_covers_every_source(L):
    """over the random cases: decoded and copied rows, copies below a short tier, from untiered rings and of partial newest rows, and
    slots of different sizes under one vcap"""
    seen = set()
    for seed in range(12):
        rng = np.random.default_rng(400 + seed)
        nr = int(rng.choice([2, 3, 5, 8]))
        cap = int(rng.choice([2048, 5000, 8192, 65536]))
        totals, tiers, _, ring_of, first, length, set_off = _case(rng, nr, cap)
        route, slots, _, _, vcap = B.split(totals, cap, tiers, ring_of, first, length, set_off)
        seen.update({"ring set" if r == 0 else "box set" for r in route})
        for k, rows, dec, vtotal in slots:
            if any(dec):
                seen.add("decoded")
            if tiers[k] is None:
                seen.add("untiered")
            elif any(not d and r < tiers[k][0] for r, d in zip(rows, dec)):
                seen.add("below a short tier")
            if rows[-1] * ROW + ROW > totals[k]:
                seen.add("partial newest")
            if len(rows) * ROW < vcap:
                seen.add("smaller than vcap")
    assert seen == {"ring set", "box set", "decoded", "untiered", "below a short tier", "partial newest", "smaller than vcap"}, seen


@pytest.mark.parametrize("seed", range(4))
def test_reach_edges(L, seed):
    """each ring's reach: lo_k - 1 refused, lo_k taken; a range ending at total_k taken, at total_k + 1 refused - alone and beside a
    valid range of every other ring"""
    rng = np.random.default_rng(500 + seed)
    nr, cap = 5, 8192
    totals, tiers, los, *_ = _case(rng, nr, cap)
    others = [(k, totals[k] - 10, 10) for k in range(nr)]
    for k in range(nr):
        for f, n, ok in ((los[k] - 1, 5, False), (los[k], 5, True), (totals[k] - 7, 7, True), (totals[k] - 7, 8, False)):
            sets = [[(k, f, n)] + [o for o in others if o[0] != k]]
            ring_of = [a for s in sets for a, _, _ in s]
            first = [b for s in sets for _, b, _ in s]
            length = [c for s in sets for _, _, c in s]
            so = [0, len(first)]
            want = B.split(totals, cap, tiers, ring_of, first, length, so)
            rc, got = _split(L, totals, cap, tiers, ring_of, first, length, so)
            if ok:
                assert want is not None and rc == 0 and got == want, (k, f, n)
            else:
                assert want is None and rc == -1, (k, f, n)
    # ring_of outside the call, an empty range, a malformed set_off
    assert _split(L, totals, cap, tiers, [nr], [los[0]], [1], [0, 1])[0] == -1
    assert _split(L, totals, cap, tiers, [0], [los[0]], [0], [0, 1])[0] == -1
    assert _split(L, totals, cap, tiers, [0, 1], [los[0], los[1]], [1, 1], [0, 3])[0] == -1


def test_shapes(L):
    """two rings, one untiered and one whose tier reaches 20 rows before its ring: a box set over both, a ring set over both"""
    cap = 4096
    totals = [30 * ROW + 300, 12 * ROW + 5]
    tiers = [(6, 30), None]
    ring_of = [0, 1, 0, 1]
    first = [7 * ROW + 3, 12 * ROW + 5 - 100, totals[0] - 50, totals[1] - 4096]
    length = [2000, 100, 50, 4096]
    rc, got = _split(L, totals, cap, tiers, ring_of, first, length, [0, 2, 4])
    route, slots, vslot, vfirst, vcap = got
    assert route == [1, 0]                             # the second set lies in its rings
    assert slots == [(0, [7, 8], [1, 1], 2 * ROW), (1, [11, 12], [0, 0], ROW + 5)]
    assert vslot == [0, 1, -1, -1] and vfirst == [3, ROW + 5 - 100, -1, -1] and vcap == 2 * ROW   # row 11 is the slot's row 0
    assert got == B.split(totals, cap, tiers, ring_of, first, length, [0, 2, 4])


def _one_ring_cases():
    """(total, cap, t_first, t_next, first, length, set_off) of test_ring_tier_model.py's split tests and test_gpu_tier_paths.py's calls"""
    out = []
    for seed in range(8):
        rng = np.random.default_rng(100 + seed)
        cap = int(rng.choice([2048, 8192, 65536]))
        total = int(rng.integers(cap, 40 * cap))
        t_next = total // ROW
        t_first = int(rng.integers(0, (total - cap) // ROW + 1))
        lo = min(total - cap, t_first * ROW)
        n = int(rng.integers(1, 30))
        length = [int(rng.choice([1, 1024, 1025, int(rng.integers(1, 3 * cap))])) for _ in range(n)]
        length = [min(x, total - lo) for x in length]
        first = [int(rng.integers(lo, total - x + 1)) for x in length]
        cuts = sorted(set(rng.integers(1, n, 3).tolist())) if n > 1 else []
        for so in (None, [0] + cuts + [n]):
            out.append((total, cap, t_first, t_next, first, length, so))
        for f, ln in ((lo - 1, 1), (total - 5, 6), (lo, 0)):
            out.append((total, cap, t_first, t_next, [f], [ln], None))
    cap, total = 4096, 20 * 1024 + 300
    out += [(total, cap, 3, 20, [total - cap], [cap], None), (total, cap, 3, 20, [5 * 1024 + 7], [total - 5 * 1024 - 7], None),
            (total, cap, 3, 20, [3 * 1024 + 1, total - 10], [1024, 10], [0, 2])]
    for total, cap, t_first, first, length, so in TM._every_call():
        out.append((total, cap, t_first, total // ROW, first, length, so))
    return out


def test_one_ring_agrees_with_the_ring_split(L):
    for total, cap, t_first, t_next, first, length, so in _one_ring_cases():
        rc1, one = _split_one(L, total, cap, t_first, t_next, first, length, so)
        rc, got = _split(L, [total], cap, [(t_first, t_next)], None, first, length, so)
        assert rc == rc1, (total, cap, first, length)
        if rc:
            continue
        route, rows, vfirst, vtotal = one
        want_slots = [(0, rows, [int(r < t_next) for r in rows], vtotal)] if rows else []
        assert got == (route, want_slots, [0 if v >= 0 else -1 for v in vfirst], vfirst, len(rows) * ROW), (total, cap)
