"""Ring delta checkpoints on the GPU (gpud_ring_checkpoint_delta / gpud_ring_restore_delta): the delta bytes equal the host model's
(ring_delta.py) byte for byte; a base restored into a fresh ring with its deltas applied in order equals the original ring at the
moment the last delta was written (physical ring and sample ring, full checkpoint bytes, reduces, ranges and handle reads), and the
chain goes on from there to the same next delta.  Every refusal comes before any launch and leaves the ring and its marker as they
were.  Run on an H100: pytest -m gpu."""
import ctypes as C
import struct

import numpy as np
import pytest

import ring_checkpoint as RC
import ring_delta as RD
from test_gpu_ring_checkpoint import Cfg, all_reads, feed_rows, handle_state, last_error, push, same, same_handles, same_reads, snapshot

pytestmark = pytest.mark.gpu

E_INVALID, E_CAPACITY, E_STATE = -1, -4, -6


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    L = g.lib()
    L.gpudh_ring_snapshot.restype = C.c_int32
    L.gpudh_ring_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
    yield g, ctx, L
    ctx.close()


def raw_apply(L, ring, blob):
    buf = (C.c_char * max(1, len(blob))).from_buffer_copy(bytes(blob) or b"\0")
    return L.gpud_ring_restore_delta(ring._h, C.cast(buf, C.c_void_p), len(blob))


def raw_delta(L, ring, cap):
    buf = (C.c_char * max(1, cap))()
    n = C.c_int64(-1)
    rc = L.gpud_ring_checkpoint_delta(ring._h, C.cast(buf, C.c_void_p), cap, C.byref(n))
    return rc, n.value, bytes(buf)[:max(0, min(cap, n.value))]


def model_delta(L, ring, base_total, base_link):
    """the model's delta of a ring without handles whose marker is a full checkpoint at base_total with link base_link"""
    rb, _ = snapshot(L, ring)
    st = RD.new_ring(ring.F, ring.W, ring.cap)
    st["ring"], st["total"] = rb, ring.counts()[0]
    st["marker"] = {"total": base_total, "link": base_link, "next": []}
    return RD.encode(st)


def same_ring(L, a, b):
    assert a.counts() == b.counts()
    x, y = snapshot(L, a), snapshot(L, b)
    same(x[0], y[0], "ring")
    same(x[1], y[1], "sample ring")


# ------------------------------------------------------------------------------------------------ 1. bytes = the model's
RUNS = [0, 1, 1023, 1024, 1025, "cap-1", "cap", "cap+1", "3cap"]


@pytest.mark.parametrize("kind", ["u32", "survey", "special"])
def test_delta_bytes_equal_the_model(env, kind):
    g, ctx, L = env
    cfg = Cfg(3, 5000, 100, alpha=0.25, thr=np.array([60.0, 300500.0, 1980.0]))
    cap = cfg.cap
    rows = feed_rows(kind, 3, 5 * cap, 21)
    for m in (0, cap + 700):                                 # a base before any wrap, and one whose delta wraps at the physical end
        for run in RUNS:
            n = {"cap-1": cap - 1, "cap": cap, "cap+1": cap + 1, "3cap": 3 * cap}.get(run, run)
            ring = cfg.ring(g, ctx)
            if m:
                push(ring, kind, rows[:m])
            base = ring.checkpoint()
            if n:
                push(ring, kind, rows[m:m + n])
            assert ring.checkpoint_delta_bound() >= 0
            bound = ring.checkpoint_delta_bound()
            delta = ring.checkpoint_delta()
            assert len(delta) <= bound
            assert delta == model_delta(L, ring, m, RD.full_link(base)), (m, run)
            d = RD.decode(delta)
            _, _, blocks = ring.checkpoint_stats()
            assert blocks == {"raw": int((d["dir"] >> 7 == 0).sum()), "int": int((d["dir"] >> 7 == 1).sum())}
            r2 = cfg.ring(g, ctx)
            r2.restore(base)
            r2.restore_delta(delta)
            same_ring(L, ring, r2)
            _, dec, blocks2 = r2.checkpoint_stats()
            assert blocks2 == blocks and dec >= 0
            if n:
                with pytest.raises(g.GpudError):
                    r2.read("min")                           # no reduce since the apply
                same_reads(all_reads(ring), all_reads(r2))
            assert r2.checkpoint() == ring.checkpoint()
            r2.close()
            ring.close()


# ------------------------------------------------------------------------------------------------ 2. the chain contract
class Twin:
    """two rings fed and reduced identically: `a` writes the chain, `b` answers full checkpoints and reads without moving a's marker"""

    def __init__(self, g, ctx, cfg):
        self.r = [cfg.ring(g, ctx), cfg.ring(g, ctx)]
        self.hs = [[], []]

    def push(self, rows):
        for r in self.r:
            r.push(rows)

    def open(self):
        for r, hs in zip(self.r, self.hs):
            r.stream_open(50)
            hs += [r.windows(10), r.windows(200, 0), r.windows(6, 20, hop=2), r.windows(2), r.windows(5, 7)]

    def reduce(self, which):
        out = []
        for r, hs in zip(self.r, self.hs):
            out.append([r.stream_reduce() if w == "s" else hs[w].reduce() for w in which])
        assert out[0] == out[1]
        return out[0]

    def close(self):
        for r in self.r:
            r.close()


def test_chain_contract(env):
    g, ctx, L = env
    F, cap, W = 3, 8192, 8
    cfg = Cfg(F, cap, W, alpha=0.05, thr=np.array([60.0, 300500.0, 1980.0]))
    rows = feed_rows("u32", F, 60000, 11).astype(np.float64)
    rows[:, 0] += np.random.default_rng(1).standard_normal(len(rows))        # one non-integer field: RAW blocks too
    t = Twin(g, ctx, cfg)
    a, b = t.r
    t.push(rows[:2000])
    t.open()                                          # stream, span L = 80, span L = 1600 > 1024, hop, span 2, and one never reduced
    t.reduce(["s", 0, 1, 2, 3])
    base = a.checkpoint()
    pos = 2000
    # (rows pushed, then the handles reduced) before each delta; 2: empty; 3: > CAP rows, handle 3 left behind; 4: its loss and re-seed
    script = [(700, ["s", 0, 1, 2]), (0, []), (cap + 108, ["s", 0, 2]), (333, [3, "s"]), (5000, [1, 3, 4]), (1, []), (2500, ["s", 0, 1, 2, 3, 4])]
    deltas, lost = [], 0
    for k, (n, which) in enumerate(script):
        t.push(rows[pos:pos + n])
        pos += n
        lost += sum(nl for _, nl in t.reduce(which))
        deltas.append(a.checkpoint_delta())
        d = RD.decode(deltas[-1])
        prev = RD.decode(deltas[-2]) if k else {"total": 2000, "link": RD.full_link(base)}
        assert (d["prev_total"], d["prev_link"], d["total"]) == (prev["total"], prev["link"], pos)
        if n == 0 and not which:
            assert d["payload_bytes"] == 0 and all(h["next"] == h["from"] for h in d["handles"])
        # the records hold the history a's handles read for windows [from, next)
        for h, rec in zip([None] + t.hs[0], d["handles"]):
            cnt = rec["next"] - rec["from"]
            got = a.stream_read("min", rec["from"], cnt) if h is None else h.read("min", rec["from"], cnt)
            same(got, rec["hist"][0], ("hist", k))
        # a fresh ring: the base, then d1 .. dk
        r2 = cfg.ring(g, ctx)
        hs2 = r2.restore(base)
        for x in deltas:
            r2.restore_delta(x)
        same_ring(L, a, r2)
        same_handles(handle_state(a, t.hs[0]), handle_state(r2, hs2))
        assert r2.checkpoint() == b.checkpoint(), k
        same_reads(all_reads(b), all_reads(r2))
        r2.close()
    assert lost > 0
    # the handle opened before the base and first reduced in step 5 re-seeds its EMA then
    assert [RD.decode(x)["handles"][5]["reseed"] for x in deltas] == [1, 1, 1, 1, 0, 0, 0]
    # the chain goes on across the restart: the same further pushes and reduces give the same next delta, byte for byte
    r2 = cfg.ring(g, ctx)
    hs2 = r2.restore(base)
    for x in deltas:
        r2.restore_delta(x)
    more = rows[pos:pos + 3000]
    for r, hs in ((a, t.hs[0]), (r2, hs2)):
        r.push(more)
        r.stream_reduce()
        for h in hs:
            h.reduce()
    nxt = a.checkpoint_delta()
    assert r2.checkpoint_delta() == nxt
    assert r2.checkpoint() == a.checkpoint()
    r2.close()
    t.close()


# ------------------------------------------------------------------------------------------------ 3. refusals
def test_write_refusals(env):
    g, ctx, L = env
    cfg = Cfg(2, 4000, 10)
    rows = feed_rows("special", 2, 9000, 4)
    r = cfg.ring(g, ctx)
    r.push(rows[:1000])
    assert raw_delta(L, r, 1 << 20)[0] == E_STATE            # no marker yet
    assert last_error(g, ctx) == "checkpoint_delta: no checkpoint written or restored on this ring yet"
    r.checkpoint()
    for change in (lambda r: r.stream_open(0), lambda r: r.windows(3), lambda r: r.windows(3).close()):
        x = cfg.ring(g, ctx)
        x.push(rows[:1000])
        x.checkpoint()
        change(x)
        assert raw_delta(L, x, 1 << 20)[0] == E_STATE
        assert last_error(g, ctx) == "checkpoint_delta: a handle was opened or closed since the last checkpoint: write a full one"
        x.checkpoint()                                       # a full checkpoint starts a new chain
        assert RD.decode(x.checkpoint_delta())["total"] == 1000
        x.close()
    # cap too small: the exact size, nothing written, the marker where it was: the retry equals a twin's fresh call
    twin = cfg.ring(g, ctx)
    twin.push(rows[:1000])
    twin.checkpoint()
    for x in (r, twin):
        x.push(rows[1000:3333])
    want = twin.checkpoint_delta()
    rc, n, got = raw_delta(L, r, len(want) - 1)
    assert rc == E_CAPACITY and n == len(want) and got == bytes(len(want) - 1)
    assert last_error(g, ctx) == "checkpoint_delta needs %d bytes" % len(want)
    assert raw_delta(L, r, 0)[:2] == (E_CAPACITY, len(want))
    assert last_error(g, ctx) == "checkpoint_delta needs %d bytes" % len(want)
    assert r.checkpoint_delta() == want
    r.close()
    twin.close()


def test_apply_refusals(env):
    g, ctx, L = env
    F, cap, W = 3, 6000, 10
    cfg = Cfg(F, cap, W, alpha=0.3, thr=np.array([50.0, 60.0, 70.0]))
    rows = feed_rows("u32", F, 20000, 3).astype(np.float64)
    src = cfg.ring(g, ctx)
    src.push(rows[:7777])
    src.stream_open(0)
    w = src.windows(4)
    src.stream_reduce()
    base = src.checkpoint()
    src.push(rows[7777:9000])
    src.stream_reduce()
    w.reduce()
    d1 = src.checkpoint_delta()
    src.push(rows[9000:9500])
    d2 = src.checkpoint_delta()
    other = cfg.ring(g, ctx)                                 # another chain of the same config
    other.push(rows[:7777])
    other.stream_open(0)
    other.windows(4)
    other.checkpoint()
    other.push(rows[:100])
    d_other = other.checkpoint_delta()
    other.close()

    def target():
        r = cfg.ring(g, ctx)
        hs = r.restore(base)
        return r, hs, snapshot(L, r)

    def unchanged(r, snap, code, blob, what, msg):
        assert raw_apply(L, r, blob) == code, (what, last_error(g, ctx))
        assert last_error(g, ctx) == msg, what
        x = snapshot(L, r)
        same(x[0], snap[0], what)
        same(x[1], snap[1], what)
        assert r.checkpoint() == base, what                  # also re-marks the target at the base's own link
        r.restore_delta(d1)                                  # and the right delta still applies
        r.close()

    def bad_link(blob, ring_link):
        return ("restore_delta: the delta follows link %016x, the ring is at %016x (out of order, applied twice, or another chain)" %
                (RD.header(blob)["prev_link"], ring_link))

    # the chain
    for what, blob in (("out of order", d2), ("another chain", d_other)):
        r, _, snap = target()
        unchanged(r, snap, E_INVALID, blob, what, bad_link(blob, RD.full_link(base)))
    r, _, _ = target()
    r.restore_delta(d1)
    snap = snapshot(L, r)
    assert raw_apply(L, r, d1) == E_INVALID                  # applied twice
    assert last_error(g, ctx) == bad_link(d1, RD.decode(d1)["link"])
    same(snapshot(L, r)[0], snap[0], "twice")
    r.restore_delta(d2)
    r.close()
    # the target moved on since its marker
    r, _, snap = target()
    r.push(rows[:1])
    assert raw_apply(L, r, d1) == E_STATE and r.counts()[0] == 7778
    assert last_error(g, ctx) == "restore_delta: the ring has been pushed into since its last checkpoint"
    r.close()
    for change in (lambda r, hs: hs[0].close(), lambda r, hs: r.windows(2)):
        r, hs, snap = target()
        change(r, hs)
        assert raw_apply(L, r, d1) == E_STATE
        assert last_error(g, ctx) == "restore_delta: a handle was opened or closed since the ring's last checkpoint"
        same(snapshot(L, r)[0], snap[0], "handles changed")
        r.close()
    # a handle that committed windows since the marker, with nothing pushed: the base's windows handle had never been reduced
    r, hs, snap = target()
    n_new, _ = hs[0].reduce()
    assert n_new > 0 and raw_apply(L, r, d1) == E_STATE
    assert last_error(g, ctx) == "restore_delta: a handle has committed windows since the ring's last checkpoint"
    r.close()
    r = cfg.ring(g, ctx)
    assert raw_apply(L, r, d1) == E_STATE                    # no marker
    assert last_error(g, ctx) == "restore_delta: no checkpoint written or restored on this ring yet"
    r.close()

    # malformed bytes
    hd = RD.header(d1)
    lay = RD.layout(F, hd["total"] - hd["first_d"], hd["payload_bytes"] // 8, hd["handle_bytes"])

    def edit(off, fmt, value, b=d1):
        b = bytearray(b)
        struct.pack_into(fmt, b, off, value)
        return bytes(b)
    hs = RD.decode(d1)["handles"]
    h0 = lay["handles"]
    h1 = h0 + 80 + RC.handle_body_bytes(F, hs[0]["next"] - hs[0]["from"])

    def bad_handle(i, **edits):
        h = dict(hs[i], **edits)
        return ("restore_delta: handle %d (kind %d, span %d, hop %d, history %d, windows [%d, %d) from %d) is not this ring's handle's successor" %
                (i, h["kind"], h["span"], h["hop"], h["H"], h["first"], h["next"], h["from"]))
    n, pay = len(d1), hd["payload_bytes"]
    sections = "restore_delta: section lengths do not add up to the %d bytes given"
    totals = "restore_delta: totals %d -> %d and first sample %d disagree"
    malformed = {
        "empty": (b"", "restore_delta: not a ring delta checkpoint"), "short header": (d1[:100], "restore_delta: not a ring delta checkpoint"),
        "header only": (d1[:128], sections % 128), "truncated by 8": (d1[:-8], sections % (n - 8)), "trailing byte": (d1 + b"\0", sections % (n + 1)),
        "magic": (b"GPUDRCK1" + d1[8:], "restore_delta: not a ring delta checkpoint"),
        "version": (edit(8, "<I", 2), "restore_delta: delta version 2, this library reads 1"),
        "header padding": (edit(120, "<Q", 1), "restore_delta: header byte 120 is not zero"),
        "F": (edit(12, "<I", F + 1), "restore_delta: n_fields 4, the ring has 3"), "W": (edit(16, "<I", W + 1), "restore_delta: window 11, the ring has 10"),
        "CAP": (edit(24, "<q", cap + 1), "restore_delta: capacity 6001, the ring has 6000"),
        "prev_total": (edit(32, "<q", 7776), totals % (7776, 9000, 7777)),
        # a consistent total one sample on: field 1's last block (width 10) codes one payload word more than the section holds
        "total": (edit(40, "<q", 9001), "restore_delta: the directory codes %d payload bytes, the section has %d" % (pay + 8, pay)),
        "first_d": (edit(48, "<q", 7778), totals % (7777, 9000, 7778)),
        "width 65": (edit(lay["dir"], "<B", 65), "restore_delta: block 0 has width 65"),
        "directory padding": (edit(lay["dir"] + F * lay["nb"], "<B", 1), "restore_delta: directory padding is not zero"),
        "payload length": (edit(72, "<q", pay + 8)[:lay["payload"]] + bytes(8) + d1[lay["payload"]:],
                           "restore_delta: the directory codes %d payload bytes, the section has %d" % (pay, pay + 8)),
        "n_handles": (edit(20, "<I", 1), "restore_delta: 1 handle records, the ring has 2 handles"),
        "kind": (edit(h0, "<q", 1), bad_handle(0, kind=1)), "span": (edit(h1 + 8, "<q", 5), bad_handle(1, span=5)),
        "hop": (edit(h1 + 16, "<q", 2), bad_handle(1, hop=2)), "H": (edit(h1 + 24, "<q", 99), bad_handle(1, H=99)),
        "first > from": (edit(h0 + 32, "<q", 10 ** 6), bad_handle(0, first=10 ** 6)), "next": (edit(h0 + 40, "<q", 10 ** 6), bad_handle(0, next=10 ** 6)),
        "prev_next": (edit(h0 + 64, "<q", 1), bad_handle(0)), "from": (edit(h0 + 72, "<q", 0), bad_handle(0, **{"from": 0})),
        "reseed 2": (edit(h0 + 56, "<q", 2), bad_handle(0)),
    }
    for what, (blob, msg) in malformed.items():
        r, _, snap = target()
        unchanged(r, snap, E_INVALID, blob, what, msg)
    for bad, msg in ((Cfg(F + 1, cap, W, 0.3, thr=np.array([50.0, 60.0, 70.0, 1.0])), "restore_delta: n_fields 3, the ring has 4"),
                     (Cfg(F, cap, W + 1, 0.3, thr=np.array([50.0, 60.0, 70.0])), "restore_delta: window 10, the ring has 11")):
        r = bad.ring(g, ctx)
        assert raw_apply(L, r, d1) == E_INVALID
        assert last_error(g, ctx) == msg
        r.close()

    # a flipped payload bit: the check pass catches it and nothing is written; the right delta applies afterwards
    b = bytearray(d1)
    b[lay["payload"] + 40] ^= 0x04
    r, _, snap = target()
    assert raw_apply(L, r, bytes(b)) == E_INVALID
    assert last_error(g, ctx) == "restore_delta: checksum mismatch in field 0: the delta is corrupt; nothing was written"
    x = snapshot(L, r)
    same(x[0], snap[0], "flip")
    same(x[1], snap[1], "flip")
    r.restore_delta(d1)
    r.restore_delta(d2)
    same_ring(L, src, r)
    assert r.checkpoint() == src.checkpoint()
    r.close()
    src.close()


# ------------------------------------------------------------------------------------------------ 4. buffers and shapes
def test_pinned_pageable_one_field_no_handles(env):
    g, ctx, L = env
    cfg = Cfg(1, 70000, 100)
    rows = feed_rows("special", 1, 200000, 8)
    a = cfg.ring(g, ctx)
    a.push(rows[:50000])
    base = a.checkpoint()
    a.push(rows[50000:125000])                               # more than CAP since the base
    size = a.checkpoint_delta_bound()
    p = C.c_void_p()
    assert L.gpud_host_alloc(size, C.byref(p)) == 0
    try:
        pinned = np.frombuffer((C.c_char * size).from_address(p.value), dtype=np.uint8)
        n = a.checkpoint_delta(out=pinned)
        d1 = pinned[:n].tobytes()
        assert d1 == model_delta(L, a, 50000, RD.full_link(base))
        a.push(rows[125000:126000])
        page = np.zeros(a.checkpoint_delta_bound(), dtype=np.uint8)
        n2 = a.checkpoint_delta(out=page)
        d2 = page[:n2].tobytes()
        assert RD.decode(d2)["prev_link"] == RD.decode(d1)["link"]
        r2 = cfg.ring(g, ctx)
        r2.restore(base)
        r2.restore_delta(pinned[:n])                         # from pinned memory
        r2.restore_delta(page[:n2])                          # from pageable memory
        same_ring(L, a, r2)
        assert r2.checkpoint() == a.checkpoint()
        r2.close()
    finally:
        L.gpud_host_free(p)
    a.close()
