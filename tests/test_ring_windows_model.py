"""Model check (no GPU) of the stream windows of any span (gpud_ring_windows_*, DESIGN.md §2):
  - the sub-window the range pass runs on for L = span x W > 1024 (gpudh_ring_windows_sub) and the sub-window -> segment map of
    the pass: every window of a reduce is covered exactly once by whole sub-windows, windows that wrap the physical end too;
  - the plan with L in place of W through gpudh_ring_stream_plan;
  - a numpy model of one segment of the select: its strided pivot sample (S = L / 32), the classification, the finish with the
    segment's own list capacity, on segments built with tests/range_cases.py's generators: the model's answer is the sorted one
    and every route is reached.  test_gpu_ring_windows.py checks the device against the same routes."""
import ctypes as C
import math

import numpy as np
import pytest

import gpud_b200 as g
import range_cases as RC
from oracle import pyoracle as O
from test_range_paths_model import KEY_POS_INF, _kth_largest, classify, pivots


def windows_sub(W, span):
    """W g, g the largest divisor of span with W g <= 1024 (L <= 1024: L itself)"""
    if W * span <= 1024:
        return W * span
    return W * max(d for d in range(1, span + 1) if span % d == 0 and d * W <= 1024)


def seg_sample(L):
    """the strided pivot sample of a segment of L samples: S = L / 32 in [64, 8192] reads at j stride + stride / 2"""
    S = max(64, min(RC.SAMPLE_MAX, L // 32))
    stride = L // S
    return np.arange(S, dtype=np.int64) * stride + stride // 2


def seg_list_cap(n, S, k):
    """the list capacity of select.cu seg_sample: twice the keys the pivots are expected to leave between them, in [256, min(n, 64 Ki)]"""
    pr = k / n
    r0 = pr * S
    d = 5.0 * math.sqrt(S * pr * (1.0 - pr)) + 2.0
    ranks = min(float(S), math.ceil(r0 + d)) - max(0.0, math.floor(r0 - d)) + 1.0
    return int(min(min(n, RC.LIST_CAP), max(256.0, math.ceil(2.0 * ranks * n / S))))


def seg_route(x, pos, k, list_cap):
    """k_range_finish on one segment: (route, answer key); an open route's answer comes from the radix select (the sorted key)"""
    keys = O.total_order_key(x)
    ans = _kth_largest(keys, k)
    if keys.min() == keys.max():
        return "const", ans
    lok, hik, _, _, _ = pivots(x, pos, k)
    cls, ins = classify(x, keys, lok, hik)
    a, eh, el, fill = (int(v) for v in cls.sum(axis=0))
    if int(keys.max()) > KEY_POS_INF:
        return "nan", ans
    if not lok <= hik:
        return "pivots", ans
    if k <= a:
        return "above", ans
    if k <= a + eh:
        return "hi", hik
    if k <= a + eh + fill:
        return ("list", _kth_largest(keys[ins], k - a - eh)) if fill <= list_cap else ("overflow", ans)
    if k <= a + eh + fill + el:
        return "lo", lok
    return "below", ans


def gen_overflow(L, list_cap):
    """range_cases.gen_overflow against the segment's own list capacity: every key but the sample lies between the pivots"""
    if L.U <= list_cap or L.k > L.U + L.rlc - 1:
        return None
    mid = (L.rhc + L.rlc) // 2
    return L.build([((1e6, 2e6), mid, 0), ((-1.0, 1.0), 0, L.U), ((-2e6, -1e6), L.S - mid, 0)])


# generator -> the route it is built for (route_specials decides for the specials)
GENERATORS = [(name, gen, route) for name, gen, route in RC.GENERATORS if name != "overflow"] + [("overflow", None, "overflow")]


def build_segment(name, gen, L, k, rng):
    pos = seg_sample(L)
    lay = RC.Layout(L, pos, k, rng)
    return gen_overflow(lay, seg_list_cap(L, len(pos), k)) if gen is None else gen(lay)


def _hook(name, *types):
    fn = getattr(g.lib(), name)
    fn.restype = C.c_int32
    fn.argtypes = list(types)
    return fn


def test_sub_window_choice():
    sub = _hook("gpudh_ring_windows_sub", C.c_int32, C.c_int64)
    for W in (1, 2, 7, 10, 100, 333, 512, 513, 960, 999, 1000, 1024):
        for span in list(range(1, 40)) + [64, 97, 600, 1048, 1200, 2000, 4096]:
            wp = sub(W, span)
            assert wp == windows_sub(W, span), (W, span)
            L = W * span
            assert wp <= 1024 and L % wp == 0 and wp % W == 0 and (L <= 1024) == (wp == L)
    assert sub(0, 1) == -1 and sub(1025, 1) == -1 and sub(1000, 0) == -1
    assert windows_sub(1000, 10) == 1000 and windows_sub(7, 600) == 7 * 120 and windows_sub(1, 2000) == 1000


def _plan(fn, total, cap, L, H, first, nxt):
    out = (C.c_int64 * 8)()
    assert fn(total, cap, L, H, first, nxt, out) == 0
    return dict(zip(("n_new", "n_lost", "first", "next", "start", "write_from", "restart", "reducible_from"), list(out)))


@pytest.mark.parametrize("W,span,cap", [(1000, 10, 25500), (7, 600, 9000), (999, 3, 20500), (1000, 10, 10000), (1, 2000, 9000),
                                        (1024, 10, 20600)])
def test_plan_and_segments_cover_every_window_once(W, span, cap):
    """random pushes and reduces: the plan with L (the ring's columns kept explicitly), and the pass's sub-windows: segment
    f n_new + v / (L / Wp) of sub-window v covers exactly the columns of its window, each once, none straddling two windows"""
    fn = _hook("gpudh_ring_stream_plan", C.c_int64, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_int64))
    L = W * span
    Wp = windows_sub(W, span)
    sub = L // Wp
    H = max(1, cap // L)
    rng = np.random.default_rng(L + cap)
    cols = np.full(cap, -1, dtype=np.int64)             # sample number held by each physical column
    total, first, nxt = 0, 0, 0
    wrapped = 0
    for _ in range(60):
        n = int(rng.choice([1, L - 1, L, L + 1, 3 * L + 5, cap, cap + L + 3, int(rng.integers(1, 2 * L))]))
        s = np.arange(total + n - min(n, cap), total + n)
        cols[s % cap] = s
        total += n
        p = _plan(fn, total, cap, L, H, first, nxt)
        oldest = max(0, total - cap)
        reducible = -(-oldest // L)
        assert p["reducible_from"] == reducible and p["next"] == total // L
        assert p["n_lost"] == max(0, reducible - nxt) and p["restart"] == (p["n_lost"] > 0)
        frm = reducible if p["restart"] else nxt
        assert p["n_new"] == total // L - frm and p["start"] == frm * L % cap
        assert p["first"] == max(frm if p["restart"] else first, total // L - H)
        for f in (0, 2):                                 # two fields of a 3-field ring: segments f n_new + j
            seen = {}
            for v in range(p["n_new"] * sub):
                c = (p["start"] + v * Wp + np.arange(Wp)) % cap
                wrapped += int(c[-1] < c[0])
                seg = f * p["n_new"] + v // sub
                samples = cols[c]
                assert (samples // L == frm + v // sub).all(), (v, seg)      # no sub-window straddles two windows
                seen.setdefault(seg, []).append(samples)
            for j in range(p["n_new"]):
                got = np.sort(np.concatenate(seen[f * p["n_new"] + j]))
                assert np.array_equal(got, np.arange((frm + j) * L, (frm + j + 1) * L))
        first, nxt = p["first"], p["next"]
    assert wrapped > 0 or cap % Wp == 0                 # a sub-window wrapped the physical end where the shapes allow it


@pytest.mark.parametrize("L", [2000, 10000, 20000, 600000])
@pytest.mark.parametrize("q", [(99, 100), (1, 100), (1, 2), (999, 1000)])
def test_segment_model_routes(L, q):
    """segments built for each route: the model's answer is the sorted key, and the route is the one built for (600 000 samples:
    strided reads only if the ring's sample ring is too sparse - at CAP = 1 Mi it is not, so that length only checks the list size)"""
    k = RC.k_from_top(L, q[0], q[1])
    pos = seg_sample(L)
    cap_list = seg_list_cap(L, len(pos), k)
    assert 256 <= cap_list <= min(L, RC.LIST_CAP)
    rng = np.random.default_rng(L * 7 + q[0])
    reached = set()
    for name, gen, route in GENERATORS:
        x = build_segment(name, gen, L, k, rng)
        if x is None:
            continue
        want_route = route(RC.Layout(L, pos, k, rng)) if callable(route) else route
        got_route, ans = seg_route(x, pos, k, cap_list)
        assert ans == _kth_largest(O.total_order_key(x), k), name
        assert got_route == want_route, (name, got_route, want_route)
        reached.add(got_route)
    assert {"list", "const", "nan"} <= reached
    if L == 20000 and q == (99, 100):
        assert {"hi", "lo", "below", "overflow"} <= reached
    if L == 20000 and q == (1, 2):
        assert "above" in reached


def test_list_memory_scales_with_the_window():
    """a 512 x 1 Mi catch-up at L = 10 000: 53 248 segments, each with a list sized for its own expected fill, not kListCap"""
    L, k = 10000, RC.k_from_top(10000, 99, 100)
    cap_list = seg_list_cap(L, len(seg_sample(L)), k)
    segs = 512 * ((1 << 20) // L)
    assert segs == 53248 and segs * cap_list * 8 < 1 << 30
    # the continuous gauge the pivots are built for fills well under half of it
    rng = np.random.default_rng(3)
    x = rng.normal(60.0, 3.0, L)
    pos = seg_sample(L)
    lok, hik, _, _, _ = pivots(x, pos, k)
    _, ins = classify(x, O.total_order_key(x), lok, hik)
    assert 0 < int(ins.sum()) <= cap_list // 2 + 64
