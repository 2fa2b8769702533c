"""Ring checkpoints on the GPU (gpud_ring_checkpoint / gpud_ring_restore): the bytes equal the host model's encoding
(ring_checkpoint.py) of the ring's chronological samples, byte for byte; a restore rebuilds the physical ring and the sample ring
exactly (gpudh_ring_snapshot), and every reduce, range and windows handle of the restored ring answers bit for bit what the original
answers, before and after the same further pushes.  Refusals come before any launch and leave the ring as created.
Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import ring_checkpoint as RC

pytestmark = pytest.mark.gpu

E_INVALID, E_CAPACITY, E_STATE = -1, -4, -6
OPS = ("min", "max", "mean", "ema", "p99", "n_over")


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    L = g.lib()
    L.gpudh_ring_snapshot.restype = C.c_int32
    L.gpudh_ring_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
    yield g, ctx, L
    ctx.close()


# ------------------------------------------------------------------------------------------------ helpers
def snapshot(L, ring):
    s, slots = C.c_int32(), C.c_int64()
    assert L.gpudh_ring_snapshot(ring._h, None, None, C.byref(s), C.byref(slots)) == 0
    rb = np.empty((ring.F, ring.cap), dtype=np.uint64)
    sb = np.empty((ring.F, slots.value), dtype=np.uint64)
    assert L.gpudh_ring_snapshot(ring._h, C.c_void_p(rb.ctypes.data), C.c_void_p(sb.ctypes.data), C.byref(s), C.byref(slots)) == 0
    return rb, sb


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def same(a, b, what=""):
    a, b = bits(a), bits(b)
    assert a.shape == b.shape and np.array_equal(a, b), (what, int(np.count_nonzero(a != b)) if a.shape == b.shape else (a.shape, b.shape))


class Cfg:
    def __init__(self, F, cap, W, alpha=0.0, q=(0, 0), thr=None):
        self.F, self.cap, self.W, self.alpha, self.q = F, cap, W, alpha, q
        self.thr = thr

    def ring(self, g, ctx):
        return g.Ring(ctx, self.F, self.cap, self.W, thresholds=self.thr, ema_alpha=self.alpha, q_num=self.q[0], q_den=self.q[1])

    def model(self):
        alpha = self.alpha if self.alpha > 0 else min(2.0 / (self.W + 1.0), 0.9999)
        q = self.q if self.q != (0, 0) else (99, 100)
        thr = np.full(self.F, np.inf) if self.thr is None else self.thr
        return {"F": self.F, "W": self.W, "cap": self.cap, "alpha": alpha, "q_num": q[0], "q_den": q[1], "thr": thr}


def all_reads(ring) -> dict:
    """gpud_ring_reduce + the six reads, reduce_range(0) and of a last_n, and a batch of short and long ranges"""
    total, count, _ = ring.counts()
    out = {}
    ring.reduce()
    for k in OPS:
        out["w_" + k] = ring.read(k)
    for last in (0, max(1, count // 3)):
        for k, v in ring.reduce_range(last).items():
            out["r%d_%s" % (last, k)] = v
    o = total - count
    first = [o, o + count // 2, total - min(count, 1500), total - 1, o + count // 5]
    length = [min(count, 2000), max(1, count // 4), min(count, 1500), 1, max(1, min(count - count // 5, 1024))]
    for k, v in ring.reduce_ranges(first, length).items():
        out["rs_" + k] = v
    return out


def same_reads(a: dict, b: dict):
    assert a.keys() == b.keys()
    for k in a:
        same(a[k], b[k], k)


def feed_rows(kind: str, F: int, n: int, seed: int):
    """n poll rows [n][F] of one feed: NVML-like uint32 gauges, the survey stream, or the special-value classes"""
    rng = np.random.default_rng(seed)
    if kind == "u32":
        temp = 40 + np.cumsum(rng.integers(-1, 2, (n, F)), axis=0) % 30
        power = 300000 + np.cumsum(rng.integers(-500, 501, (n, F)), axis=0)
        clock = np.full((n, F), 1980)
        col = np.arange(F) % 3
        return np.where(col == 0, temp, np.where(col == 1, power, clock)).astype(np.uint32)
    if kind == "survey":
        import synth_device as SD
        return np.concatenate([t[:rows].cpu().numpy() for t, rows in SD.chunks("survey", F, n, 1 << 14, seed, "cuda")])[:n]
    # special: random bit patterns and IEEE classes, integers around +-2^53, constants, integer gauges with a -0.0 now and then
    x = np.empty((n, F))
    cls = np.arange(F) % 4
    specials = np.array([0.0, -0.0, 5e-324, -5e-324, np.inf, -np.inf, np.nan, 1.5]).view(np.uint64)
    specials = np.concatenate([specials, np.array([0x7FF0000000000001, 0xFFF8DEADBEEF0001, 0x7FF800000000ABCD], dtype=np.uint64)])
    raw = np.where(rng.random((n, F)) < 0.5, rng.integers(0, 2 ** 64, (n, F), dtype=np.uint64, endpoint=False),
                   specials[rng.integers(0, len(specials), (n, F))]).view(np.float64)
    big = 2.0 ** 53 - 2000 + np.cumsum(rng.integers(0, 3, (n, F)), axis=0).astype(np.float64)
    big *= np.where(np.arange(F) % 8 < 4, 1.0, -1.0)
    gauge = rng.integers(30, 90, (n, F)).astype(np.float64)
    gauge[rng.random((n, F)) < 0.001] = -0.0
    x[:] = np.where(cls == 0, raw, np.where(cls == 1, big, np.where(cls == 2, 75.0, gauge)))
    return x


def push(ring, kind, rows):
    if kind == "u32":
        ring.push_raw(rows)
    else:
        ring.push(rows)


def checkpoint_checked(ring, cfg, L) -> bytes:
    """the checkpoint, checked against the model's encoding of the ring's chronological samples and against the bound"""
    blob = ring.checkpoint()
    assert ring.checkpoint_bound() >= len(blob)
    total, count, _ = ring.counts()
    rb, _ = snapshot(L, ring)
    want = RC.encode(RC.chronological(rb, total, ring.cap), total, cfg.model())
    hs = RC.decode(blob)["handles"] if RC.header(blob)["n_handles"] else []
    if hs:
        want = RC.encode(RC.chronological(rb, total, ring.cap), total, cfg.model(), hs)
    assert blob == want, "checkpoint bytes differ from the model's encoding"
    d = RC.decode(blob)
    _, _, blocks = ring.checkpoint_stats()
    assert blocks == {"raw": int((d["dir"] >> 7 == 0).sum()), "int": int((d["dir"] >> 7 == 1).sum())}
    return blob


def restored(g, ctx, cfg, blob):
    r = cfg.ring(g, ctx)
    hs = r.restore(blob)
    return r, hs


# ------------------------------------------------------------------------------------------------ 1. round trips
SHAPES = [Cfg(1, 3000, 10, alpha=0.25), Cfg(3, 5000, 100, q=(95, 100)), Cfg(64, 10002, 1000), Cfg(512, 4098, 64, alpha=0.9999)]


@pytest.mark.parametrize("kind", ["u32", "survey", "special"])
@pytest.mark.parametrize("si", range(len(SHAPES)))
def test_roundtrip(env, kind, si):
    g, ctx, L = env
    cfg = SHAPES[si]
    F, cap = cfg.F, cfg.cap
    if cfg.thr is None and kind != "special":
        cfg = Cfg(F, cap, cfg.W, cfg.alpha, cfg.q, thr=np.linspace(50, 400000, F))
    ring = cfg.ring(g, ctx)
    rows = feed_rows(kind, F, 3 * cap + 3000, 7 + si)
    pos = 0
    # total = 0, < CAP, = CAP, > CAP and not a multiple, after one push of more than CAP rows
    for step in (0, cap // 3, cap - cap // 3, 777, cap + 1234):
        if step:
            push(ring, kind, rows[pos:pos + step])
            pos += step
        blob = checkpoint_checked(ring, cfg, L)
        r2, hs = restored(g, ctx, cfg, blob)
        assert hs == []
        assert r2.counts() == ring.counts()
        a, b = snapshot(L, ring), snapshot(L, r2)
        same(a[0], b[0], "ring")
        same(a[1], b[1], "sample ring")
        enc, dec, blocks = r2.checkpoint_stats()
        assert dec >= 0 and sum(blocks.values()) == F * -(-min(pos, cap) // 1024)
        if pos:
            with pytest.raises(g.GpudError):
                r2.read("min")                               # no reduce yet, as on a new ring
            same_reads(all_reads(ring), all_reads(r2))
            # the restored ring goes on like the original
            more = rows[pos:pos + 1000]
            push(ring, kind, more)
            push(r2, kind, more)
            same_reads(all_reads(ring), all_reads(r2))
            assert r2.checkpoint() == ring.checkpoint()
            # take the pushed rows back out of the original: a fresh restore of the same blob for the next step
            ring.close()
            ring, _ = restored(g, ctx, cfg, blob)
        r2.close()
    ring.close()


def test_large_ring_pageable_and_pinned(env):
    """a survey ring of 512 x 64 Ki samples: the payload crosses the staging pair in several pieces; pinned buffers both ways"""
    g, ctx, L = env
    import synth_device as SD
    F, cap, W = 512, 1 << 16, 1000
    cfg = Cfg(F, cap, W, thr=SD.thresholds("survey", F, cap, 3))
    ring = cfg.ring(g, ctx)
    SD.fill_ring(ring, "survey", F, cap, 3, "cuda")
    ring.push(feed_rows("special", F, 4321, 5))
    blob = ring.checkpoint()
    assert len(blob) > 32 << 20                       # more than one piece of the 32 MiB staging buffers
    d = RC.decode(blob)
    rb, sb = snapshot(L, ring)
    total = ring.counts()[0]
    same(d["samples"], RC.chronological(rb, total, cap), "model decode")
    size = len(blob)
    p = C.c_void_p()
    assert L.gpud_host_alloc(size, C.byref(p)) == 0
    try:
        pinned = np.frombuffer((C.c_char * size).from_address(p.value), dtype=np.uint8)
        assert ring.checkpoint(out=pinned) == size
        assert pinned.tobytes() == blob
        for src in (blob, pinned):
            r2, _ = restored(g, ctx, cfg, src)
            a = snapshot(L, r2)
            same(a[0], rb, "ring")
            same(a[1], sb, "sample ring")
            r2.close()
    finally:
        L.gpud_host_free(p)
    ring.close()


# ------------------------------------------------------------------------------------------------ 2. handles
def handle_state(ring, hs):
    """counts and every history read of the stream handle and each windows handle"""
    out = []
    first, nxt, lost = ring.stream_counts()
    out.append((first, nxt, lost, {k: ring.stream_read(k, first, nxt - first) for k in OPS}))
    for h in hs:
        first, nxt, lost = h.counts()
        out.append((first, nxt, lost, {k: h.read(k, first, nxt - first) for k in OPS}))
    return out


def same_handles(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x[:3] == y[:3], (i, x[:3], y[:3])
        for k in OPS:
            same(x[3][k], y[3][k], (i, k))


def test_handles_roundtrip(env):
    g, ctx, L = env
    F, cap, W = 3, 8192, 8
    cfg = Cfg(F, cap, W, alpha=0.05, thr=np.array([60.0, 300500.0, 1980.0]))
    rows = feed_rows("u32", F, 40000, 11).astype(np.float64)
    rows[:, 0] += np.random.default_rng(1).standard_normal(len(rows))        # one non-integer field: RAW blocks too
    ring = cfg.ring(g, ctx)
    ring.push(rows[:2000])
    ring.stream_open(50)
    hs = [ring.windows(10), ring.windows(6, 20, hop=2), ring.windows(200, 0, hop=100), ring.windows(2)]
    ring.stream_reduce()
    for h in hs:
        h.reduce()
    ring.push(rows[2000:2700])
    ring.stream_reduce()
    hs[0].reduce(); hs[1].reduce(); hs[2].reduce()
    ring.push(rows[2700:11000])                       # hs[3] is not reduced through this: its oldest windows are lost
    hs.append(ring.windows(5, 7))                     # opened and never reduced: its first commit re-seeds
    ring.stream_reduce()
    hs[0].reduce(); hs[2].reduce()
    n_new, n_lost = hs[3].reduce()
    assert n_lost > 0
    ring.push(rows[11000:11333])
    ring.stream_reduce()
    hs[0].reduce()
    blob = checkpoint_checked(ring, cfg, L)
    d = RC.decode(blob)
    assert [h["kind"] for h in d["handles"]] == [0, 1, 1, 1, 1, 1]
    assert [(h["span"], h["hop"]) for h in d["handles"][1:]] == [(10, 10), (6, 2), (200, 100), (2, 2), (5, 5)]
    assert d["handles"][5]["reseed"] == 1 and d["handles"][1]["reseed"] == 0 and d["handles"][4]["lost"] > 0
    r2, hs2 = restored(g, ctx, cfg, blob)
    assert [(h.span, h.hop) for h in hs2] == [(h.span, h.hop) for h in hs]
    same_handles(handle_state(ring, hs), handle_state(r2, hs2))
    assert r2.checkpoint() == blob
    # the same further pushes into both, including one of more than CAP rows that makes windows lost
    pos = 11333
    lost = 0
    for step in (5, 999, 1600, cap + 2222, 37):
        for r in (ring, r2):
            r.push(rows[pos:pos + step])
        pos += step
        got = [r2.stream_reduce()] + [h.reduce() for h in hs2]
        want = [ring.stream_reduce()] + [h.reduce() for h in hs]
        assert got == want, step
        lost += sum(nl for _, nl in want)
        same_handles(handle_state(ring, hs), handle_state(r2, hs2))
    assert lost > 0
    same_reads(all_reads(ring), all_reads(r2))
    ms, _, _ = hs2[2].stats()
    assert ms > 0
    r2.close()
    ring.close()


def test_empty_ring_with_open_stream(env):
    g, ctx, L = env
    cfg = Cfg(4, 2048, 16)
    ring = cfg.ring(g, ctx)
    ring.stream_open(0)
    w = ring.windows(3)
    blob = checkpoint_checked(ring, cfg, L)
    r2, hs = restored(g, ctx, cfg, blob)
    assert len(hs) == 1 and r2.counts() == (0, 0, 0) and r2.stream_counts() == ring.stream_counts()
    rows = feed_rows("special", 4, 3000, 2)
    for r, h in ((ring, w), (r2, hs[0])):
        r.push(rows)
    assert ring.stream_reduce() == r2.stream_reduce() and w.reduce() == hs[0].reduce()
    same_handles(handle_state(ring, [w]), handle_state(r2, hs))
    r2.close()
    ring.close()


# ------------------------------------------------------------------------------------------------ 3. refusals
def raw_restore(L, ring, blob, cap_handles=8):
    buf = (C.c_char * max(1, len(blob))).from_buffer_copy(bytes(blob) or b"\0")
    hs = (C.c_void_p * max(1, cap_handles))()
    n = C.c_int32(-1)
    rc = L.gpud_ring_restore(ring._h, C.cast(buf, C.c_void_p), len(blob), hs, cap_handles, C.byref(n))
    return rc, n.value


def last_error(g, ctx):
    buf = C.create_string_buffer(512)
    g.lib().gpud_last_error(ctx._h, buf, 512)
    return buf.value.decode()


def untouched(L, ring):
    assert ring.counts() == (0, 0, 0)
    rb, sb = snapshot(L, ring)
    assert not rb.any() and not sb.any()


def test_refusals(env):
    g, ctx, L = env
    F, cap, W = 3, 6000, 10
    thr = np.array([50.0, 60.0, 70.0])
    cfg = Cfg(F, cap, W, alpha=0.3, q=(9, 10), thr=thr)
    src = cfg.ring(g, ctx)
    rows = feed_rows("u32", F, 9000, 3).astype(np.float64)
    src.push(rows[:7777])
    src.stream_open(0)
    src.windows(4)
    src.stream_reduce()
    blob = src.checkpoint()
    hd = RC.header(blob)
    lay = RC.layout(F, hd["count"], hd["payload_bytes"] // 8, hd["handle_bytes"])

    # every config field, each with the whole message
    for bad, msg in ((Cfg(F + 1, cap, W, 0.3, (9, 10), np.append(thr, 1.0)), "restore: n_fields 3, the ring has 4"),
                     (Cfg(F, cap, W + 1, 0.3, (9, 10), thr), "restore: window 10, the ring has 11"),
                     (Cfg(F, cap + 2, W, 0.3, (9, 10), thr), "restore: capacity 6000, the ring has 6002"),
                     (Cfg(F, cap, W, 0.3000000001, (9, 10), thr), "restore: ema_alpha %.17g, the ring has %.17g" % (0.3, 0.3000000001)),
                     (Cfg(F, cap, W, 0.3, (8, 10), thr), "restore: q_num 9, the ring has 8"),
                     (Cfg(F, cap, W, 0.3, (9, 11), thr), "restore: q_den 10, the ring has 11"),
                     (Cfg(F, cap, W, 0.3, (9, 10), np.array([50.0, -0.0 + 60.000000000001, 70.0])),
                      "restore: thresholds[1] %.17g, the ring has %.17g" % (60.0, 60.000000000001)),
                     (Cfg(F, cap, W, 0.3, (9, 10), np.array([50.0, 60.0, -70.0])), "restore: thresholds[2] 70, the ring has -70")):
        r = bad.ring(g, ctx)
        assert raw_restore(L, r, blob)[0] == E_INVALID, msg
        assert last_error(g, ctx) == msg
        untouched(L, r)
        r.close()

    # a target that is not as created
    r = cfg.ring(g, ctx)
    r.push(rows[:1])
    assert raw_restore(L, r, blob)[0] == E_STATE
    assert last_error(g, ctx) == "restore: the ring has been pushed into"
    assert r.counts()[0] == 1
    r.close()
    for opener in (lambda r: r.stream_open(0), lambda r: r.windows(2)):
        r = cfg.ring(g, ctx)
        opener(r)
        assert raw_restore(L, r, blob)[0] == E_STATE
        assert last_error(g, ctx) == "restore: the ring has a stream or windows handle open"
        untouched(L, r)
        r.close()

    # cap_handles too small
    r = cfg.ring(g, ctx)
    assert raw_restore(L, r, blob, cap_handles=0) == (E_CAPACITY, 1)
    assert last_error(g, ctx) == "restore: 1 windows handles, room for 0"
    untouched(L, r)

    # malformed bytes
    def edit(off, fmt, value, b=blob):
        b = bytearray(b)
        import struct
        struct.pack_into(fmt, b, off, value)
        return bytes(b)
    hs = RC.decode(blob)["handles"]

    def bad_handle(i, **edits):
        h = dict(hs[i], **edits)
        return "restore: handle %d (kind %d, span %d, hop %d, history %d, windows [%d, %d)) is not one this ring can hold" % (
            i, h["kind"], h["span"], h["hop"], h["H"], h["first"], h["next"])
    n, pay = len(blob), hd["payload_bytes"]
    malformed = {
        "truncated by 8": (blob[:-8], "restore: section lengths do not add up to the %d bytes given" % (n - 8)),
        "header only": (blob[:128], "restore: truncated thresholds section"),
        "short header": (blob[:100], "restore: not a ring checkpoint"), "empty": (b"", "restore: not a ring checkpoint"),
        "magic": (b"GPUDRCK0" + blob[8:], "restore: not a ring checkpoint"),
        "version": (edit(8, "<I", 2), "restore: checkpoint version 2, this library reads 1"),
        "header padding": (edit(120, "<Q", 1), "restore: header byte 120 is not zero"),
        "width 65": (edit(lay["dir"] + 1, "<B", 65), "restore: block 1 has width 65"),
        "width 127 INT": (edit(lay["dir"], "<B", 0xFF), "restore: block 0 has width 127"),
        "directory padding": (edit(lay["dir"] + F * lay["nb"], "<B", 1), "restore: directory padding is not zero"),
        "payload length": (edit(80, "<q", pay + 8)[:lay["payload"]] + bytes(8) + blob[lay["payload"]:],
                           "restore: the directory codes %d payload bytes, the section has %d" % (pay, pay + 8)),
        "count": (edit(56, "<q", hd["count"] - 1), "restore: total %d and count %d disagree" % (hd["total"], hd["count"] - 1)),
        "total": (edit(48, "<q", -1), "restore: total -1 and count %d disagree" % hd["count"]),
        "n_handles": (edit(20, "<I", 3), "restore: truncated handle 2"),
        "handle span": (edit(lay["handles"] + 8, "<q", cap), bad_handle(0, span=cap)),
        "handle history": (edit(lay["handles"] + 24, "<q", 0), bad_handle(0, H=0)),
        "handle next": (edit(lay["handles"] + 40, "<q", 10 ** 6), bad_handle(0, next=10 ** 6)),
        "handle first > next": (edit(lay["handles"] + 32, "<q", 10 ** 6), bad_handle(0, first=10 ** 6)),
        "two stream handles": (edit(lay["handles"] + 64 + RC.handle_body_bytes(F, hs[0]["next"] - hs[0]["first"]), "<q", 0), bad_handle(1, kind=0)),
        "handle reseed 2": (edit(lay["handles"] + 56, "<q", 2), bad_handle(0)),
        "trailing byte": (blob + b"\0", "restore: section lengths do not add up to the %d bytes given" % (n + 1)),
    }
    for what, (b, msg) in malformed.items():
        assert raw_restore(L, r, b)[0] == E_INVALID, what
        assert last_error(g, ctx) == msg, what
        untouched(L, r)

    # a flipped payload bit: the checksum catches it after the decode, and the ring is as created again
    b = bytearray(blob)
    b[lay["payload"] + 40] ^= 0x04
    assert raw_restore(L, r, bytes(b))[0] == E_INVALID
    assert last_error(g, ctx) == "restore: checksum mismatch in field 0: the checkpoint is corrupt"
    untouched(L, r)
    fresh = cfg.ring(g, ctx)
    for x in (r, fresh):
        x.push(rows[:2500])
    same_reads(all_reads(r), all_reads(fresh))
    r.close()
    fresh.close()

    # the real thing still restores
    r, hs = restored(g, ctx, cfg, blob)
    assert len(hs) == 1 and r.counts() == src.counts()
    r.close()

    # checkpoint into a buffer one byte short: the exact size, nothing written
    n = C.c_int64()
    buf = (C.c_char * len(blob))()
    assert L.gpud_ring_checkpoint(src._h, C.cast(buf, C.c_void_p), len(blob) - 1, C.byref(n)) == E_CAPACITY
    assert n.value == len(blob) and bytes(buf) == bytes(len(blob))
    assert L.gpud_ring_checkpoint(src._h, None, 0, C.byref(n)) == E_CAPACITY and n.value == len(blob)
    assert L.gpud_ring_checkpoint(src._h, C.cast(buf, C.c_void_p), len(blob), C.byref(n)) == 0 and bytes(buf) == blob
    src.close()


def test_stats_before_any_checkpoint(env):
    g, ctx, L = env
    r = Cfg(2, 100, 10).ring(g, ctx)
    with pytest.raises(g.GpudError) as e:
        r.checkpoint_stats()
    assert e.value.code == E_STATE
    r.checkpoint()
    enc, dec, blocks = r.checkpoint_stats()
    assert blocks == {"raw": 0, "int": 0}
    r.close()
