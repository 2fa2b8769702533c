"""The ring's ingest bit for bit: k_ring_append and the staging pipeline of gpud_ring_push_raw that feeds it, against the host
model of ring_ingest.py.  After each push the physical ring [F][CAP] and the sample ring (gpudh_ring_snapshot) must equal the
model as uint64 bit patterns, so NaN payloads and -0 count.  Covered: every entry point (push, push_raw of all nine sample
types from pageable memory, from pinned memory and from pinned memory at a row offset, push_device) on one ring in turn; pushes
that cross staging pieces of every type, start or end one row short of a piece and wrap the physical end inside one; the
transpose tile's edges (F = 1, 31, 33, 512, 4097); heads at 0 and CAP - 1 with n = 1, CAP, CAP + 1 and several CAP; sample
shifts 0, 1, 3, 5 and 7 (with a sample slot past the ring); the widening edges of every type; a source overwritten as soon as
the push returns, on a caller stream that is still busy; the bench's e2e transport; and the argument errors.
Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import mean_ema_ref as R
import ring_ingest as RI
from test_range_paths_model import model_ring

pytestmark = pytest.mark.gpu

E_INVALID = -1                  # GPUD_E_INVALID
DT = {name: i for i, name in enumerate(RI.DTYPES)}


@pytest.fixture(scope="module")
def env():
    import torch
    import gpud_b200 as g
    ctx = g.Context([0])
    L = g.lib()
    L.gpudh_ring_snapshot.restype = C.c_int32
    L.gpudh_ring_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
    L.gpudh_ring_range_scratch.restype = C.c_int32
    L.gpudh_ring_range_scratch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
    yield g, ctx, L, torch
    ctx.close()


# ------------------------------------------------------------------------------------------------ helpers
def snapshot(L, ring):
    """(ring [F][CAP], sample [F][slots]) as uint64 bits, and the ring's sample shift"""
    s, slots = C.c_int32(), C.c_int64()
    assert L.gpudh_ring_snapshot(ring._h, None, None, C.byref(s), C.byref(slots)) == 0
    rb = np.empty((ring.F, ring.cap), dtype=np.uint64)
    sb = np.empty((ring.F, slots.value), dtype=np.uint64)
    assert L.gpudh_ring_snapshot(ring._h, C.c_void_p(rb.ctypes.data), C.c_void_p(sb.ctypes.data), C.byref(s), C.byref(slots)) == 0
    return rb, sb, s.value


def _first_diff(got, want):
    eq = got == want
    n_bad = eq.size - int(np.count_nonzero(eq))
    if n_bad == 0:
        return None
    i = np.unravel_index(int(np.argmin(eq)), eq.shape)
    return n_bad, tuple(int(v) for v in i), hex(int(got[i])), hex(int(want[i]))


def check(env, ring, model, what=""):
    """the snapshot equals the model bit for bit: the ring, every sample slot, the shift and total"""
    g, ctx, L, torch = env
    rb, sb, s = snapshot(L, ring)
    assert ring.counts()[0] == model.total, what
    assert s == model.s and sb.shape[1] == model.slots, (what, s, model.s)
    d = _first_diff(rb, model.ring)
    assert d is None, (what, "ring: n_bad, [field, column], got, want", d)
    d = _first_diff(sb, model.sample())
    assert d is None, (what, "sample ring: n_bad, [field, slot], got, want", d)


def rand_rows(rng, dt, n, F):
    """random samples of one type over its whole range; the float types include random bit patterns (NaNs, subnormals)"""
    if dt in ("float32", "float64"):
        x = (rng.standard_normal((n, F)) * 1e3).astype(dt)
        ut = np.uint32 if dt == "float32" else np.uint64
        bits = rng.integers(0, np.iinfo(ut).max, (n, F), dtype=ut, endpoint=True).view(dt)
        return np.where(rng.random((n, F)) < 0.25, bits, x)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, (n, F), dtype=dt, endpoint=True)


def push(env, ring, model, mode, rows):
    """one push of rows [n][F] through an entry point; the caller's source is overwritten as soon as the push returns
      push        gpud_ring_push (float64) from pageable memory
      pageable    gpud_ring_push_raw from pageable memory
      pinned      gpud_ring_push_raw from a pinned tensor
      pinned_off  the same, the rows starting 3 rows into the pinned tensor
      device      gpud_ring_push_device (float64) from a CUDA tensor"""
    g, ctx, L, torch = env
    n, F = rows.shape
    if mode in ("push", "pageable"):
        src = np.array(rows, copy=True)
        if mode == "push":
            ring.push(src)
        else:
            ring.push_raw(src)
        src.view(np.uint8)[...] = 0xA5
    elif mode in ("pinned", "pinned_off"):
        off = 3 if mode == "pinned_off" else 0
        esz = rows.dtype.itemsize
        buf = torch.full(((n + off) * F * esz,), 0x5A, dtype=torch.uint8).pin_memory()
        a = buf.numpy().view(rows.dtype).reshape(n + off, F)
        a[off:] = rows
        ring.push_raw_ptr(buf.data_ptr() + off * F * esz, n, DT[rows.dtype.name])
        buf.fill_(0xA5)
    elif mode == "device":
        assert rows.dtype == np.float64
        t = torch.from_numpy(np.ascontiguousarray(rows)).to("cuda")
        torch.cuda.synchronize()
        ring.push_device(t.data_ptr(), n)
        ring.sync()                                   # the append has read t
        del t
    else:
        raise ValueError(mode)
    model.push(rows)


def _pieces_crossed(pushes, cap, p):
    """for each push (n, head before): the number of staging pieces it takes and whether it wraps inside a piece"""
    out, total = [], 0
    for n in pushes:
        kept = min(n, cap)
        total += n - kept
        head = total % cap
        wrap_at = cap - head                           # rows of this push before the physical end
        out.append((-(-kept // p), kept > wrap_at and wrap_at % p != 0))
        total += kept
    return out


# ------------------------------------------------------------------------------------------------ entry points x memory
@pytest.mark.parametrize("dt", RI.DTYPES)
def test_entry_points_and_memory(env, dt):
    """pageable, pinned and pinned-at-an-offset pushes of one raw type, with float64 pushes (host and device) in between"""
    g, ctx, L, torch = env
    F, cap = 37, 4096
    rng = np.random.default_rng(DT[dt] + 1)
    ring = g.Ring(ctx, F, cap, 256)
    model = RI.RingModel(F, cap)
    try:
        seq = [("pageable", dt, 1000), ("pinned", dt, 1500), ("push", "float64", 7), ("pinned_off", dt, 2000), ("device", "float64", 333),
               ("pageable", dt, 1), ("pinned", dt, 4095), ("device", "float64", 4097), ("pinned_off", dt, 9000), ("push", "float64", 1)]
        for i, (mode, t, n) in enumerate(seq):
            push(env, ring, model, mode, rand_rows(rng, t, n, F))
            check(env, ring, model, (i, mode, t, n))
    finally:
        ring.close()


# ------------------------------------------------------------------------------------------------ staging pieces
@pytest.mark.parametrize("mem", ["pageable", "pinned"])
@pytest.mark.parametrize("dt", RI.DTYPES)
def test_pieces(env, dt, mem):
    """F = 4097 (not a multiple of 32): a piece is 1023 rows of float64 and 8 / itemsize times as many of a narrower type.
    Pushes of piece - 1, piece, piece + 1 and 2.5 pieces (which wraps the physical end 100 rows into a piece), then 4 pieces
    + 3 into a ring of 3 pieces + 100 (the newest CAP rows only)."""
    g, ctx, L, torch = env
    F = 4097
    p = RI.piece_rows(F, dt)
    assert p == 1023 * (8 // np.dtype(dt).itemsize)
    cap = 3 * p + 100
    cap += cap & 1
    sizes = [p - 1, p, p + 1, 5 * p // 2, 4 * p + 3]
    crossed = _pieces_crossed(sizes, cap, p)
    assert crossed[2][0] == 2 and crossed[3] == (3, True) and crossed[4][0] == 4, crossed
    rng = np.random.default_rng(100 + DT[dt])
    ring = g.Ring(ctx, F, cap, 1000)
    model = RI.RingModel(F, cap)
    try:
        for n in sizes:
            push(env, ring, model, mem, rand_rows(rng, dt, n, F))
            check(env, ring, model, (dt, mem, n))
    finally:
        ring.close()


# ------------------------------------------------------------------------------------------------ heads and tile edges
@pytest.mark.parametrize("F,cap", [(1, 1000000), (31, 16384), (33, 8192), (512, 8192), (33, 32770), (32, 1 << 18)],
                         ids=["F1-s7", "F31-s1", "F33-s0", "F512-s0", "F33-s3", "F32-s5"])
def test_heads_and_tiles(env, F, cap):
    """n = 1 at head 0, a push that leaves the head at CAP - 1, n = 1 and n = 2 there, n = CAP, n = CAP + 1 through the device
    entry point (the trim in launch_append), 3 CAP + 5 pinned at an offset (the trim in push_raw)"""
    g, ctx, L, torch = env
    rng = np.random.default_rng(F * 7 + cap)
    ring = g.Ring(ctx, F, cap, min(1000, cap))
    model = RI.RingModel(F, cap)
    assert model.s == {1000000: 7, 16384: 1, 8192: 0, 32770: 3, 1 << 18: 5}[cap]
    try:
        def to_last(total):
            return (cap - 1 - total % cap) % cap or cap

        steps = [("push", "float64", lambda t: 1), ("pinned", "uint32", to_last), ("device", "float64", lambda t: 1),
                 ("pageable", "uint8", to_last), ("pinned_off", "int64", lambda t: 2), ("pageable", "int16", lambda t: cap),
                 ("device", "float64", lambda t: cap + 1), ("pinned_off", "float32", lambda t: 3 * cap + 5), ("push", "float64", lambda t: 5)]
        for mode, t, nf in steps:
            n = nf(model.total)
            head = model.total % cap
            push(env, ring, model, mode, rand_rows(rng, t, n, F))
            check(env, ring, model, (mode, t, n, head))
        assert model.total > 5 * cap
    finally:
        ring.close()


# ------------------------------------------------------------------------------------------------ widening edges
def _tie_values(kmax=11):
    """values exactly halfway between neighbouring doubles at every exponent from 2^53 to 2^64, and their neighbours"""
    vals = []
    for k in range(1, kmax + 1):
        base = 1 << (52 + k)
        for m in (0, 1, 2, 3, (1 << 52) - 2, (1 << 52) - 1):
            half = base + (m << k) + (1 << (k - 1))
            vals += [half - 1, half, half + 1]
    return vals


EDGES = {
    "uint64": [0, 1, (1 << 53) - 1, 1 << 53, (1 << 53) + 1, (1 << 53) + 3, 1 << 63, (1 << 64) - 1, (1 << 64) - (1 << 10),
               (1 << 64) - (1 << 11)] + [v for v in _tie_values() if v < 1 << 64],
    "int64": [-(1 << 63), (1 << 63) - 1, (1 << 53) + 1, -((1 << 53) + 1), (1 << 53) + 3, -((1 << 53) + 3), 0, -1]
             + [s * v for v in _tie_values(10) for s in (1, -1)],
    "float32": [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000,
                0x7F7FFFFF, 0xFF7FFFFF, 0x7FC00000, 0xFFC00000, 0x7FC12345, 0xFFD54321, 0x7F800001, 0xFF800001, 0x7FA5A5A5,
                0xFF812345, 0x7FFFFFFF, 0xFFFFFFFF],
    "float64": [0x0000000000000000, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001,
                0x800FFFFFFFFFFFFF, 0x7FEFFFFFFFFFFFFF, 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001,
                0xFFF4000000ABCDEF, 0x7FFFFFFFFFFFFFFF],
}


def edge_values(dt):
    if dt == "float32":
        return np.array(EDGES[dt], dtype=np.uint32).view(np.float32)
    if dt == "float64":
        return np.array(EDGES[dt], dtype=np.uint64).view(np.float64)
    if dt in EDGES:
        return np.array(EDGES[dt], dtype=dt)
    info = np.iinfo(dt)
    return np.array([info.min, info.min + 1, -1 if info.min else 2, 0, 1, info.max - 1, info.max], dtype=dt)


@pytest.mark.parametrize("mem", ["pageable", "pinned_off", "device"])
@pytest.mark.parametrize("dt", RI.DTYPES)
def test_widening_edges(env, dt, mem):
    """every edge value in every field of a 7-field ring, at a known column: rows[i][f] = edges[(i + 3 f) % E], pushed twice so
    the second copy wraps the ring"""
    if mem == "device" and dt != "float64":
        pytest.skip("push_device takes float64 rows")
    g, ctx, L, torch = env
    F = 7
    e = edge_values(dt)
    E = len(e)
    rows = np.stack([np.roll(e, -3 * f) for f in range(F)], axis=1)
    assert rows.shape == (E, F) and rows[5:6, 2].tobytes() == e[(5 + 6) % E:(5 + 6) % E + 1].tobytes()
    cap = E + (E & 1) + 2
    ring = g.Ring(ctx, F, cap, min(64, cap))
    model = RI.RingModel(F, cap)
    try:
        push(env, ring, model, mem, rows)
        check(env, ring, model, (dt, mem, "first"))
        push(env, ring, model, mem, rows[::-1])
        check(env, ring, model, (dt, mem, "wrapped"))
    finally:
        ring.close()


# ------------------------------------------------------------------------------------------------ the caller's contract
def test_busy_caller_stream_and_stream_switch(env):
    """Pushes on a caller stream that is still busy with earlier work when they are issued: the staging copies run ahead of
    the appends, so the pageable path must not refill a staging buffer whose copy has not run yet, and a source overwritten
    as soon as the push returns must not reach the ring.  reduce() in between; then back to the ring's own stream."""
    g, ctx, L, torch = env
    F = 4097
    p64 = RI.piece_rows(F, "float64")
    cap = 8 * p64
    rng = np.random.default_rng(9)
    thr = np.full(F, 100.0)
    ring = g.Ring(ctx, F, cap, 1000, thresholds=thr)
    model = RI.RingModel(F, cap)
    stream = torch.cuda.Stream()
    try:
        ring.set_stream(stream.cuda_stream)
        for dt, mem, n in (("float64", "pageable", 5 * p64 + 17), ("uint16", "pinned", 2 * RI.piece_rows(F, "uint16") + 5),
                           ("int32", "pageable", 3 * RI.piece_rows(F, "int32") + 1)):
            rows = rng.standard_normal((n, F)) * 100 if dt == "float64" else rand_rows(rng, dt, n, F)
            with torch.cuda.stream(stream):
                torch.cuda._sleep(2_000_000_000)         # ~1 s of GPU time queued ahead of the push on the caller's stream
            push(env, ring, model, mem, rows)
            ring.reduce()
        check(env, ring, model, "caller stream")
        ring.sync()                                       # the caller orders its stream before handing the ring back
        ring.set_stream(0)
        for dt, mem, n in (("float32", "pageable", 1500), ("float64", "device", 2000), ("uint32", "pinned_off", 3000)):
            rows = (rng.standard_normal((n, F)) * 100).astype(dt) if dt.startswith("float") else rand_rows(rng, dt, n, F)
            push(env, ring, model, mem, rows)
            ring.reduce()
        check(env, ring, model, "own stream")
        got = ring.reduce_all()
        sel = [0, 1, 31, 32, 2048, F - 1]
        want = R.windows_fields(model.chronological(sel), 1000, thr[sel])
        for k in ("min", "max", "p99"):
            assert np.array_equal(got[k][sel].view(np.uint64), want[k].view(np.uint64)), k
        assert np.array_equal(got["n_over"][sel], want["n_over"])
        R.check_mean_ema({k: got[k][sel] for k in ("mean", "ema")}, want)
    finally:
        ring.close()


# ------------------------------------------------------------------------------------------------ the bench's e2e transport
def test_bench_e2e_transport_quarter_ring(env):
    """bench.py's headline e2e at a quarter of its ring: F = 512, CAP = 2^18, pinned uint32 rows of 2^17 polls pushed on a caller
    stream (two staging pieces each), the pinned buffer refilled after every push.  The ring equals the model; the window
    reduce equals the oracle on a few fields; and the whole-range reduce redoes no field and takes the model's pivots, which
    it reads from the sample ring the same pushes kept."""
    g, ctx, L, torch = env
    F, cap, W, n = 512, 1 << 18, 1000, 1 << 17
    assert RI.piece_rows(F, "uint32") == 1 << 14 and RI.smp_shift(cap) == 5
    thr = np.full(F, 60000.0)
    ring = g.Ring(ctx, F, cap, W, thresholds=thr)
    model = RI.RingModel(F, cap)
    stream = torch.cuda.Stream()
    host = torch.empty((n, F), dtype=torch.int32).pin_memory()
    try:
        ring.set_stream(stream.cuda_stream)
        for step in range(3):
            torch.manual_seed(step)
            host.copy_(torch.randint(30000, 90000, (n, F), dtype=torch.int32))
            ring.push_raw_ptr(host.data_ptr(), n, DT["uint32"])
            model.push(host.numpy().view(np.uint32))
        check(env, ring, model, "e2e")
        got = ring.reduce_all()
        sel = [0, 1, 255, 256, 511]
        x = model.chronological(sel)
        want = R.windows_fields(x, W, thr[sel])
        for k in ("min", "max", "p99"):
            assert np.array_equal(got[k][sel].view(np.uint64), want[k].view(np.uint64)), k
        assert np.array_equal(got["n_over"][sel], want["n_over"])
        R.check_mean_ema({k: got[k][sel] for k in ("mean", "ema")}, want)
        ring.reduce_range(0)
        assert ring.range_stats()[2] == 0, ring.range_open_reasons
        piv = np.empty((F, 2), dtype=np.float64)
        fill = np.empty(F, dtype=np.uint32)
        nw = C.c_int64()
        assert L.gpudh_ring_range_scratch(ring._h, C.c_void_p(piv.ctypes.data), C.c_void_p(fill.ctypes.data), None, C.byref(nw)) == 0
        mr = model_ring(cap, model.total, cap, 99, 100, x)
        assert mr["source"] == "ring"
        for i, f in enumerate(sel):
            m = mr["fields"][i]
            assert (int(piv.view(np.uint64)[f, 0]), int(piv.view(np.uint64)[f, 1])) == (m["lo"], m["hi"]), f
            assert int(fill[f]) == m["fill"], f
    finally:
        ring.close()


# ------------------------------------------------------------------------------------------------ errors
def test_argument_errors_leave_the_ring_alone(env):
    """unknown dtype, n < 0, NULL with n > 0 and device memory given to push_raw / push: GPUD_E_INVALID, total unchanged, ring
    unchanged.  n = 0 is a no-op on every entry point, NULL source included."""
    g, ctx, L, torch = env
    F, cap = 4, 64
    ring = g.Ring(ctx, F, cap, 16)
    model = RI.RingModel(F, cap)
    try:
        rows = np.arange(5 * F, dtype=np.float64).reshape(5, F)
        push(env, ring, model, "push", rows)
        ptr = C.c_void_p(rows.ctypes.data)
        dev = torch.arange(64 * F, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        dptr = C.c_void_p(dev.data_ptr())
        h = ring._h
        bad = [("push_raw dtype 9", L.gpud_ring_push_raw(h, ptr, 1, 9)), ("push_raw dtype -1", L.gpud_ring_push_raw(h, ptr, 1, -1)),
               ("push_raw n -1", L.gpud_ring_push_raw(h, ptr, -1, 0)), ("push_raw NULL", L.gpud_ring_push_raw(h, None, 1, 1)),
               ("push n -1", L.gpud_ring_push(h, ptr, -1)), ("push NULL", L.gpud_ring_push(h, None, 3)),
               ("push_device n -1", L.gpud_ring_push_device(h, dptr, -1)), ("push_device NULL", L.gpud_ring_push_device(h, None, 2)),
               ("push_raw device f64", L.gpud_ring_push_raw(h, dptr, 3, 0)), ("push_raw device u32", L.gpud_ring_push_raw(h, dptr, 3, 1)),
               ("push device", L.gpud_ring_push(h, dptr, 3)), ("push_raw device n > CAP", L.gpud_ring_push_raw(h, dptr, 100, 1))]
        for what, rc in bad:
            assert rc == E_INVALID, (what, rc)
            assert ring.counts()[0] == model.total, what
        noop = [L.gpud_ring_push(h, ptr, 0), L.gpud_ring_push(h, None, 0), L.gpud_ring_push_raw(h, ptr, 0, 3), L.gpud_ring_push_raw(h, None, 0, 8),
                L.gpud_ring_push_device(h, dptr, 0), L.gpud_ring_push_device(h, None, 0)]
        assert noop == [0] * len(noop)
        check(env, ring, model, "after the errors")
        push(env, ring, model, "pageable", rows[:2].astype(np.uint16))    # the ring still takes rows
        check(env, ring, model, "after a good push")
        del dev
    finally:
        ring.close()
