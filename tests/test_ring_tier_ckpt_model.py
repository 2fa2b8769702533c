"""Tier checkpoint chains on the host: gpudh_ring_tier_chain_plan (gpud_ring_tier_restore's checks and placement, with no device)
against the host model tests/ring_tier_ckpt.py.  Chains are written by the model from NVML-like and noise rows and a model tier that
evicts, loses rows and restarts, with an empty delta among them; they are restored into the original, a smaller and a larger
tier_bytes, and every refusal is built by editing a model blob.  Verdict codes, texts, the rows kept, their offsets and the tier's
state must all agree."""
import ctypes as C
import struct

import numpy as np
import pytest

import ring_checkpoint as CK
import ring_tier as T
import ring_tier_ckpt as TK

ROW = T.ROW
F, W, CAP = 3, 100, 4096


@pytest.fixture(scope="module")
def L():
    import gpud_b200 as g
    return g.lib()


def hook(L, blobs, total, tier_bytes, F=F, W=W, cap=CAP):
    bufs = [C.create_string_buffer(bytes(b), max(1, len(b))) for b in blobs]
    ptrs = (C.c_void_p * max(1, len(blobs)))(*[C.addressof(b) for b in bufs])
    sizes = (C.c_int64 * max(1, len(blobs)))(*[len(b) for b in blobs])
    row_off = np.zeros(1 << 12, dtype=np.int64)
    state = np.zeros(6, dtype=np.int64)
    n = C.c_int64()
    msg = C.create_string_buffer(512)
    rc = L.gpudh_ring_tier_chain_plan(F, W, cap, total, tier_bytes, ptrs, sizes, len(blobs), C.c_void_p(row_off.ctypes.data), len(row_off), C.byref(n),
                                      C.c_void_p(state.ctypes.data), msg, 512)
    if rc:
        return rc, msg.value.decode(), None, None
    return rc, "", row_off[:n.value].tolist(), tuple(state.tolist())


def samples(n_rows, seed):
    """[F][n_rows * 1024] bits in push order: NVML-like integer gauges (INT blocks), a stretch of wide integers, f64 noise (RAW)"""
    rng = np.random.default_rng(seed)
    n = n_rows * ROW
    x = np.stack([40 + np.cumsum(rng.integers(-1, 2, n)) % 40, 1980 - 15 * rng.integers(0, 3, n), rng.normal(0.0, 1.0, n)]).astype(np.float64)
    x[1, 20 * ROW:30 * ROW] = rng.integers(0, 1 << 40, 10 * ROW)
    return x.view(np.uint64)


def scenario(seed=0, tier_bytes=None, pushes=None):
    """a model tier fed `pushes` and the chain written along the way: a base after the third push, then a delta after every later one
    -> (bits, tier, blobs, tier_bytes)"""
    bits = samples(80, seed)
    sizes = [T.row_bytes(bits[:, k * ROW:(k + 1) * ROW]) for k in range(80)]
    tier_bytes = tier_bytes or 3 * T.max_row_bytes(F)
    pushes = pushes or [3000, 2500, 5000, 1024, 0, 6000, CAP + 1500, 2048, 0, 7000, 3 * ROW, 5 * ROW]
    m = T.Tier(CAP, F, tier_bytes, 0)
    m.settle(sizes)
    w = TK.Writer(W, CAP)
    blobs = []
    for i, n in enumerate(pushes):
        m.push(n, sizes)
        if i == 2:
            blobs.append(w.full(bits, m))
        elif i > 2:
            blobs.append(w.delta(bits, m))
    return bits, m, blobs, tier_bytes


def test_scenario_covers_eviction_loss_and_empty_deltas():
    _, m, blobs, tier_bytes = scenario()
    hs = [TK.header(b) for b in blobs]
    assert m.lost > 0 and hs[-1]["lost"] == m.lost
    assert any(h["from"] == h["next"] for h in hs[1:])                         # an empty delta
    assert any(h["first"] > h["prev_next"] for h in hs[1:])                    # rows lost or evicted past the marker
    assert any(a["first"] < b["first"] for a, b in zip(hs, hs[1:]))           # eviction
    assert m.used <= tier_bytes


@pytest.mark.parametrize("seed", range(3))
def test_chains_and_placement(L, seed):
    bits, m, blobs, tier_bytes = scenario(seed)
    total = m.total
    for k in range(1, len(blobs) + 1):                 # every prefix of the chain is a chain
        h = TK.header(blobs[k - 1])
        t_total = max(h["next"] * ROW, total if k == len(blobs) else h["next"] * ROW)
        for tb in (tier_bytes, T.max_row_bytes(F), 10 * tier_bytes):
            got = hook(L, blobs[:k], t_total, tb)
            want = TK.plan(F, W, CAP, t_total, tb, blobs[:k])
            assert got == want, (k, tb)
            assert got[0] == 0
    # into the original's size: exactly the rows it held, where it held them; larger: the same rows
    rc, _, row_off, state = hook(L, blobs, total, tier_bytes)
    assert state[:4] == (m.first, m.next, m.used, m.lost)
    rc, _, row_off, state = hook(L, blobs, total, 10 * tier_bytes)
    assert (state[0], state[1], state[3]) == (m.first, m.next, m.lost) and min(row_off) >= 0
    # smaller: the newest rows that fit
    rc, _, row_off, state = hook(L, blobs, total, T.max_row_bytes(F))
    assert state[1] == m.next and state[0] > m.first and row_off[-1] >= 0 and row_off[0] == -1


def put(blob, off, fmt, v):
    b = bytearray(blob)
    struct.pack_into(fmt, b, off, v)
    return bytes(b)


def row_at(blob, j):
    """byte offset in the blob of its j-th row"""
    h = TK.header(blob)
    off = TK.HEADER.size
    for _ in range(j):
        s0, _ = struct.unpack_from("<qq", blob, off)
        dirs = blob[off + 16:off + 16 + F]
        off += T.rec_bytes(F) + 8 * sum(CK.block_words(ROW, d & 127) for d in dirs)
    assert off < TK.HEADER.size + h["rows_len"]
    return off


def refusal_cases():
    bits, m, blobs, tier_bytes = scenario()
    total = m.total
    b0, hs = blobs[0], [TK.header(b) for b in blobs]
    r0 = TK.HEADER.size
    lossy = next(i for i in range(1, len(blobs)) if hs[i]["first"] > hs[i]["prev_next"])
    grown = lambda b: b[:r0 + TK.header(b)["rows_len"]] + bytes(8) + b[r0 + TK.header(b)["rows_len"]:]
    ch = list(blobs)
    return total, tier_bytes, [
        ("capacity", dict(cap=2046), blobs, "capacity 2046 is below 2048"),
        ("tier_bytes", dict(tier_bytes=T.max_row_bytes(F) - 8), blobs, "do not hold one row"),
        ("magic", {}, [b"GPUDRCK1" + b0[8:]] + ch[1:], "blob 0 is not a ring tier checkpoint"),
        ("short", {}, [b0[:100]] + ch[1:], "blob 0 is not a ring tier checkpoint"),
        ("version", {}, [put(b0, 8, "<I", 2)] + ch[1:], "version 2"),
        ("pad word", {}, [put(b0, 20, "<I", 1)] + ch[1:], "header byte 20 is not zero"),
        ("pad tail", {}, ch[:1] + [put(ch[1], 127, "<B", 1)] + ch[2:], "blob 1: header byte 127 is not zero"),
        ("fields", dict(F=F + 1), blobs, "n_fields 3, the ring has 4"),
        ("window", dict(W=W + 1), blobs, "window 100, the ring has 101"),
        ("cap", dict(cap=2 * CAP), blobs, "capacity 4096, the ring has 8192"),
        ("truncated", {}, [b0[:-1]] + ch[1:], "section lengths"),
        ("rows_len", {}, [put(b0, 80, "<q", hs[0]["rows_len"] - 8)] + ch[1:], "section lengths"),
        ("from", {}, [put(b0, 48, "<q", hs[0]["from"] + 1)] + ch[1:], "disagree"),
        ("lost", {}, ch[:2] + [put(ch[2], 64, "<q", -1)] + ch[3:], "blob 2: first"),
        ("delta first", {}, ch[1:], "blob 0 is a delta"),
        ("base again", {}, ch[:2] + [b0] + ch[3:], "blob 2 is a full tier checkpoint"),
        ("skipped", {}, ch[:1] + ch[2:], "blob 1 follows link"),
        ("swapped", {}, ch[:1] + [ch[2], ch[1]] + ch[3:], "blob 1 follows link"),
        ("prev_next", {}, ch[:lossy] + [put(ch[lossy], 56, "<q", hs[lossy]["prev_next"] - 1)] + ch[lossy + 1:], "blob %d follows row" % lossy),
        ("record sample", {}, [put(b0, row_at(b0, 1), "<q", 5)] + ch[1:], "record starts at sample 5"),
        ("offset word", {}, [put(b0, row_at(b0, 1) + 8, "<q", 0)] + ch[1:], "offset word is 0"),
        ("width", {}, [put(b0, row_at(b0, 0) + 16 + 1, "<B", 65)] + ch[1:], "field 1 has width 65"),
        ("dir padding", {}, [put(b0, row_at(b0, 0) + 16 + F, "<B", 1)] + ch[1:], "record padding is not zero"),
        ("woff padding", {}, [put(b0, row_at(b0, 0) + 16 + 8 + 4 * F, "<B", 1)] + ch[1:], "record padding is not zero"),
        ("word offset", {}, [put(b0, row_at(b0, 0) + 16 + 8 + 4, "<I", 3)] + ch[1:], "field 1's word offset is 3"),
        ("row truncated", {}, [put(put(b0, 80, "<q", hs[0]["rows_len"] - 8), len(b0) - 8 * F - 8, "<q", 0)[:-8]] + ch[1:], "is truncated"),
        ("extra bytes", {}, [put(grown(b0), 80, "<q", hs[0]["rows_len"] + 8)] + ch[1:], "8 bytes after its last row"),
        ("past total", dict(total=hs[-1]["next"] * ROW - 1), blobs, "the chain holds samples up to"),
        ("before ring", dict(total=(hs[-1]["next"] + 5) * ROW + CAP), blobs, "before the ring's first whole row"),
    ]


def test_refusals(L):
    total, tier_bytes, cases = refusal_cases()
    for name, kw, blobs, text in cases:
        a = dict(dict(F=F, W=W, cap=CAP, total=total, tier_bytes=tier_bytes), **kw)
        got = hook(L, blobs, a["total"], a["tier_bytes"], a["F"], a["W"], a["cap"])
        want = TK.plan(a["F"], a["W"], a["cap"], a["total"], a["tier_bytes"], blobs)
        assert got == want, name
        assert got[0] == TK.E_INVALID and text in got[1], (name, got[1])
