"""Host model of kind-2 handle records (DESIGN.md "Ring checkpoint format", "Ring delta checkpoint format"): a windows handle over
chosen fields is recorded as its kind's head words, i64 n_fields, the i32 field ids zero-padded to 8 bytes, then the body of the
other kinds with n_fields in place of F; the chain link folds the n_fields word and the padded list words after the head words.

The model extends tests/ring_checkpoint.py and tests/ring_delta.py: a model handle of kind 2 carries `fields`, and its hist / nover /
ema have n_fields rows.  `full` and `delta` write blobs, `decode_handles` reads a handle section back with every check the library
makes of a record (each refusal raises Refused), `apply_delta` applies a delta onto a model ring.  The tests below round-trip records
of every kind through it; tests/test_gpu_ring_windows_fields.py compares the library's bytes with it."""
import struct

import numpy as np
import pytest

import ring_checkpoint as RC
import ring_delta as RD

KIND_STREAM, KIND_WINDOWS, KIND_FIELDS = 0, 1, 2
HISTORY_LIMIT = 1 << 40          # H x the handle's fields


class Refused(ValueError):
    pass


def n_rows(h: dict, F: int) -> int:
    """the fields a handle's body counts: its list's for kind 2, else the ring's"""
    return len(h["fields"]) if h["kind"] == KIND_FIELDS else F


def list_bytes(fields) -> bytes:
    """i64 n_fields, then the i32 ids zero-padded to 8 bytes"""
    ids = np.ascontiguousarray(fields, dtype="<i4").tobytes()
    return struct.pack("<q", len(fields)) + ids + bytes(RC.pad8(len(ids)) - len(ids))


def list_words(fields):
    """the words the link folds after a kind-2 record's head words"""
    b = list_bytes(fields)
    return list(struct.unpack("<%dq" % (len(b) // 8), b))


def new_handle(F: int, kind: int, span: int, hop: int, H: int, fields=None) -> dict:
    h = RD.new_handle(len(fields) if kind == KIND_FIELDS else F, kind, span, hop, H)
    if kind == KIND_FIELDS:
        h["fields"] = list(fields)
    return h


def body(h: dict, lo: int, nf: int) -> bytes:
    """windows [lo, next) of h: [5][nf][n] f64, [nf][n] u32 padded to 8 bytes, [nf] f64 EMA state (zeros while a re-seed is pending)"""
    slots = np.arange(lo, h["next"]) % h["H"]
    hist = np.ascontiguousarray(h["hist"][:, :, slots], dtype="<f8")
    nover = np.ascontiguousarray(h["nover"][:, slots], dtype="<u4").tobytes()
    ema = np.zeros(nf) if h["reseed"] else np.ascontiguousarray(h["ema"], dtype="<f8")
    return hist.tobytes() + nover + bytes(RC.pad8(len(nover)) - len(nover)) + ema.tobytes()


def record(h: dict, F: int, head) -> tuple:
    """(record bytes, the words the link folds) of h with the given head words"""
    extra = list_bytes(h["fields"]) if h["kind"] == KIND_FIELDS else b""
    words = list(head) + (list_words(h["fields"]) if h["kind"] == KIND_FIELDS else [])
    lo = head[9] if len(head) == 10 else h["first"]
    return struct.pack("<%dq" % len(head), *head) + extra + body(h, lo, n_rows(h, F)), words


def with_handles(blob: bytes, hnd: bytes, n: int, hnd_len_off: int) -> bytes:
    """a blob written without handles, with handle section hnd of n records instead"""
    out = bytearray(blob)
    struct.pack_into("<I", out, 20, n)
    struct.pack_into("<q", out, hnd_len_off, len(hnd))
    return bytes(out) + hnd


def full(st: dict, cfg: dict) -> bytes:
    """the full checkpoint of model ring st (any handle kinds); its marker moves to it"""
    blob = RD.full(dict(st, handles=[]), cfg)
    recs, heads = [], []
    for h in st["handles"]:
        rec, words = record(h, st["F"], (h["kind"], h["span"], h["hop"], h["H"], h["first"], h["next"], h["lost"], int(h["reseed"])))
        recs.append(rec)
        heads += words
    out = with_handles(blob, b"".join(recs), len(recs), 96)
    d = RC.header(out)
    sums = np.frombuffer(out, "<u8", st["F"], RC.layout(st["F"], d["count"], d["payload_bytes"] // 8, 0)["sum"])
    RD.mark(st, RD.link(0, st["total"], sums, heads))
    return out


def delta(st: dict) -> bytes:
    """the delta since st's marker (any handle kinds); the marker moves to it"""
    m = st["marker"]
    bare = dict(st, handles=[], marker=dict(m, next=[]))
    blob = RD.encode(bare)
    recs, heads = [], []
    for h, prev_next in zip(st["handles"], m["next"]):
        lo = RD.from_window(h["first"], prev_next)
        rec, words = record(h, st["F"], (h["kind"], h["span"], h["hop"], h["H"], h["first"], h["next"], h["lost"], int(h["reseed"]), prev_next, lo))
        recs.append(rec)
        heads += words
    out = with_handles(blob, b"".join(recs), len(recs), 88)
    d = RD.header(out)
    count = d["total"] - d["first_d"]
    sums = np.frombuffer(out, "<u8", st["F"], RD.layout(st["F"], count, d["payload_bytes"] // 8, 0)["sum"])
    RD.mark(st, RD.link(m["link"], st["total"], sums, heads))
    return out


def decode_handles(blob: bytes, F: int, off: int, end: int, n_rec: int, is_delta: bool, prev=None) -> tuple:
    """the handle records of a blob's section [off, end): -> (records, the words the link folds).  Every check the library makes of
    a record's kind and list raises Refused: kind 2 at a windows position with 1 <= n_fields, every id in [0, F), zero padding, the
    history limit on n_fields, nothing truncated; a delta's record must have its predecessor's kind and list (prev: those handles)."""
    nh = 10 if is_delta else 8
    recs, words = [], []
    for i in range(n_rec):
        if off + 8 * nh > end:
            raise Refused("truncated handle %d" % i)
        head = struct.unpack_from("<%dq" % nh, blob, off)
        kind, span, hop, H, first, nxt = head[:6]
        words += head
        off += 8 * nh
        if not (kind == KIND_WINDOWS or kind == KIND_FIELDS or (kind == KIND_STREAM and i == 0)):
            raise Refused("handle %d of kind %d" % (i, kind))
        nf, fields = F, None
        if kind == KIND_FIELDS:
            if off + 8 > end:
                raise Refused("truncated handle %d" % i)
            nf = struct.unpack_from("<q", blob, off)[0]
            if nf < 1 or nf > (end - off - 8) // 4 or off + 8 + RC.pad8(4 * nf) > end:
                raise Refused("handle %d has a list of %d fields" % (i, nf))
            fields = list(np.frombuffer(blob, "<i4", nf, off + 8))
            if min(fields) < 0 or max(fields) >= F:
                raise Refused("handle %d names a field outside [0, %d)" % (i, F))
            if any(blob[off + 8 + 4 * nf:off + 8 + RC.pad8(4 * nf)]):
                raise Refused("handle %d: field list padding is not zero" % i)
            words += list_words(fields)
            off += 8 + RC.pad8(4 * nf)
        if H < 1 or H > HISTORY_LIMIT // nf:
            raise Refused("handle %d: history of %d windows" % (i, H))
        if prev is not None and (kind != prev[i]["kind"] or fields != prev[i].get("fields")):
            raise Refused("handle %d is not the successor of the ring's handle" % i)
        lo = head[9] if is_delta else first
        n = nxt - lo
        size = 40 * nf * n + RC.pad8(4 * nf * n) + 8 * nf
        if off + size > end:
            raise Refused("truncated handle %d" % i)
        recs.append({"head": head, "kind": kind, "fields": fields, "from": lo,
                     "hist": np.frombuffer(blob, "<f8", 5 * nf * n, off).reshape(5, nf, n),
                     "nover": np.frombuffer(blob, "<u4", nf * n, off + 40 * nf * n).reshape(nf, n),
                     "ema": np.frombuffer(blob, "<f8", nf, off + 40 * nf * n + RC.pad8(4 * nf * n))})
        off += size
    if off != end:
        raise Refused("the handle section has %d bytes after its last handle" % (end - off))
    return recs, words


def full_handles(blob: bytes):
    """the records and link of a full checkpoint"""
    d = RC.header(blob)
    F = d["F"]
    lay = RC.layout(F, d["count"], d["payload_bytes"] // 8, d["handle_bytes"])
    recs, words = decode_handles(blob, F, lay["handles"], lay["size"], d["n_handles"], False)
    sums = np.frombuffer(blob, "<u8", F, lay["sum"])
    return recs, RD.link(0, d["total"], sums, words)


def delta_handles(blob: bytes, prev_handles):
    d = RD.header(blob)
    F = d["F"]
    lay = RD.layout(F, d["total"] - d["first_d"], d["payload_bytes"] // 8, d["handle_bytes"])
    recs, words = decode_handles(blob, F, lay["handles"], lay["size"], d["n_handles"], True, prev_handles)
    sums = np.frombuffer(blob, "<u8", F, lay["sum"])
    return recs, RD.link(d["prev_link"], d["total"], sums, words)


def strip_handles(blob: bytes, hnd_len_off: int) -> bytes:
    """the blob without its handle section (its samples alone, for ring_checkpoint.decode / ring_delta.decode)"""
    n = struct.unpack_from("<q", blob, hnd_len_off)[0]
    return with_handles(blob[:len(blob) - n], b"", 0, hnd_len_off)


def apply_delta(st: dict, blob: bytes):
    """a delta onto model ring st in place: its samples through ring_delta's model, its records here"""
    recs, lk = delta_handles(blob, st["handles"])
    d = RD.decode(strip_handles(blob, 88))
    assert d["prev_link"] == st["marker"]["link"] and d["prev_total"] == st["total"]
    count = d["total"] - d["first_d"]
    st["ring"][:, (d["first_d"] + np.arange(count)) % st["cap"]] = d["samples"]
    st["total"] = d["total"]
    for h, r in zip(st["handles"], recs):
        kind, span, hop, H, first, nxt, lost, reseed, prev_next, lo = r["head"]
        assert prev_next == h["next"]
        slots = np.arange(lo, nxt) % H
        h["hist"][:, :, slots] = r["hist"]
        h["nover"][:, slots] = r["nover"]
        h.update(first=first, next=nxt, lost=lost, reseed=reseed, ema=r["ema"].copy())
    RD.mark(st, lk)


# ------------------------------------------------------------------------------------------------ tests
CFG = dict(F=6, W=16, cap=256, alpha=0.25, q_num=99, q_den=100)


def _cfg():
    return dict(CFG, thr=np.linspace(-1.0, 1.0, CFG["F"]))


def _commit(h: dict, rng, n_new: int):
    """n_new more windows into h's history, random contents"""
    nf = h["hist"].shape[1]
    for _ in range(n_new):
        k = h["next"] % h["H"]
        h["hist"][:, :, k] = rng.standard_normal((5, nf))
        h["nover"][:, k] = rng.integers(0, 100, nf)
        h["next"] += 1
        h["first"] = max(h["first"], h["next"] - h["H"])
    h["ema"] = rng.standard_normal(nf)
    h["reseed"] = 0


def _ring(rng):
    st = RD.new_ring(CFG["F"], CFG["W"], CFG["cap"])
    st["handles"] = [new_handle(CFG["F"], KIND_STREAM, 1, 1, 16), new_handle(CFG["F"], KIND_FIELDS, 2, 1, 8, [5, 0, 5]),
                     new_handle(CFG["F"], KIND_WINDOWS, 4, 2, 6), new_handle(CFG["F"], KIND_FIELDS, 1, 1, 4, [1, 2, 3, 4, 0])]
    RD.push(st, rng.standard_normal((300, CFG["F"])))
    for h in st["handles"]:
        _commit(h, rng, 5)
    return st


def test_kind2_record_layout():
    """head words, i64 n_fields, the ids zero-padded to 8 bytes, then the body with n_fields rows"""
    rng = np.random.default_rng(1)
    st = _ring(rng)
    blob = full(st, _cfg())
    recs, lk = full_handles(blob)
    assert [r["kind"] for r in recs] == [0, 2, 1, 2]
    assert recs[1]["fields"] == [5, 0, 5] and recs[3]["fields"] == [1, 2, 3, 4, 0]
    assert list_bytes([5, 0, 5]) == struct.pack("<q3i4x", 3, 5, 0, 5)
    assert list_bytes([1, 2]) == struct.pack("<q2i", 2, 1, 2)                # no padding for an even count
    for h, r in zip(st["handles"], recs):
        slots = np.arange(h["first"], h["next"]) % h["H"]
        assert np.array_equal(r["hist"], h["hist"][:, :, slots]) and np.array_equal(r["nover"], h["nover"][:, slots])
        assert np.array_equal(r["ema"], h["ema"])
    assert lk == st["marker"]["link"]
    # the samples are the ring format's own, untouched by the records
    d = RC.decode(strip_handles(blob, 96))
    assert np.array_equal(d["samples"], RD.chronological(st, st["total"] - min(st["total"], st["cap"])))


def test_no_field_handle_keeps_the_blob():
    """a ring with no kind-2 handle: the extended writer's bytes are ring_delta's, link included"""
    rng = np.random.default_rng(2)
    st = _ring(rng)
    st["handles"] = [h for h in st["handles"] if h["kind"] != KIND_FIELDS]
    a, b = RD.copy(st), RD.copy(st)
    assert full(a, _cfg()) == RD.checkpoint(b, _cfg()) and a["marker"] == b["marker"]
    RD.push(a, rng.standard_normal((40, CFG["F"])))
    b["ring"], b["total"] = a["ring"].copy(), a["total"]
    for h, g in zip(a["handles"], b["handles"]):
        _commit(h, np.random.default_rng(3), 2)
        _commit(g, np.random.default_rng(3), 2)
    assert delta(a) == RD.encode(b) and a["marker"] == b["marker"]


def test_link_folds_the_list():
    """the link changes with any word of a list: n_fields, an id, and its order"""
    rng = np.random.default_rng(4)
    links = set()
    for fields in ([5, 0, 5], [5, 0, 4], [0, 5, 5], [5, 0, 5, 1]):
        st = _ring(np.random.default_rng(4))
        st["handles"][1] = new_handle(CFG["F"], KIND_FIELDS, 2, 1, 8, fields)
        _commit(st["handles"][1], rng, 3)
        st["handles"][1]["hist"][:] = 0.0
        st["handles"][1]["nover"][:] = 0
        st["handles"][1]["ema"][:] = 0.0
        full(st, _cfg())
        links.add(st["marker"]["link"])
    assert len(links) == 4


def test_delta_chain_round_trip():
    """full, then deltas with new samples and windows: each applies onto the model restored from the chain before it, and the
    result equals the ring; restore + re-checkpoint gives the same bytes"""
    rng = np.random.default_rng(5)
    st = _ring(rng)
    base = full(st, _cfg())
    recs, lk = full_handles(base)
    mirror = RD.restore(strip_handles(base, 96))
    mirror["handles"] = []
    for h, r in zip(st["handles"], recs):
        g = new_handle(CFG["F"], r["kind"], h["span"], h["hop"], h["H"], r["fields"])
        slots = np.arange(h["first"], h["next"]) % h["H"]
        g["hist"][:, :, slots] = r["hist"]
        g["nover"][:, slots] = r["nover"]
        g.update(first=h["first"], next=h["next"], lost=h["lost"], reseed=h["reseed"], ema=r["ema"].copy())
        mirror["handles"].append(g)
    RD.mark(mirror, lk)
    assert full(RD.copy(mirror), _cfg()) == base
    for step in range(3):
        RD.push(st, rng.standard_normal((37 + 50 * step, CFG["F"])))
        for i, h in enumerate(st["handles"]):
            _commit(h, rng, (i + step) % 4)
        blob = delta(st)
        apply_delta(mirror, blob)
        assert mirror["total"] == st["total"] and np.array_equal(mirror["ring"], st["ring"])
        assert mirror["marker"]["link"] == st["marker"]["link"]
        for h, g in zip(st["handles"], mirror["handles"]):
            assert (g["first"], g["next"], g["reseed"]) == (h["first"], h["next"], h["reseed"])
            slots = np.arange(h["first"], h["next"]) % h["H"]
            assert np.array_equal(g["hist"][:, :, slots], h["hist"][:, :, slots]) and np.array_equal(g["ema"], h["ema"])
    # a delta with nothing new holds the lists again and no windows
    blob = delta(st)
    recs, _ = delta_handles(blob, st["handles"])
    assert [r["fields"] for r in recs] == [None, [5, 0, 5], None, [1, 2, 3, 4, 0]] and all(r["hist"].shape[2] == 0 for r in recs)


def _list_off(blob: bytes, rec: int, is_delta: bool) -> int:
    """byte offset of record rec's n_fields word (rec is a kind-2 record)"""
    F = CFG["F"]
    if is_delta:
        d = RD.header(blob)
        off = RD.layout(F, d["total"] - d["first_d"], d["payload_bytes"] // 8, d["handle_bytes"])["handles"]
    else:
        d = RC.header(blob)
        off = RC.layout(F, d["count"], d["payload_bytes"] // 8, d["handle_bytes"])["handles"]
    nh = 10 if is_delta else 8
    for i in range(rec):
        head = struct.unpack_from("<%dq" % nh, blob, off)
        nf = F
        off += 8 * nh
        if head[0] == KIND_FIELDS:
            nf = struct.unpack_from("<q", blob, off)[0]
            off += 8 + RC.pad8(4 * nf)
        lo = head[9] if is_delta else head[4]
        n = head[5] - lo
        off += 40 * nf * n + RC.pad8(4 * nf * n) + 8 * nf
    return off + 8 * nh


def _patched(blob: bytes, off: int, fmt: str, *v) -> bytes:
    out = bytearray(blob)
    struct.pack_into(fmt, out, off, *v)
    return bytes(out)


@pytest.mark.parametrize("is_delta", [False, True])
def test_corrupt_kind2_records_are_refused(is_delta):
    rng = np.random.default_rng(6)
    st = _ring(rng)
    blob = full(st, _cfg())
    prev = [dict(h) for h in st["handles"]]
    if is_delta:
        RD.push(st, rng.standard_normal((20, CFG["F"])))
        _commit(st["handles"][1], rng, 2)
        blob = delta(st)
    read = (lambda b: delta_handles(b, prev)) if is_delta else full_handles
    read(blob)
    o = _list_off(blob, 1, is_delta)                       # record 1: fields [5, 0, 5], one pad word
    bad = {
        "n_fields 0": _patched(blob, o, "<q", 0),
        "n_fields negative": _patched(blob, o, "<q", -3),
        "n_fields past the blob": _patched(blob, o, "<q", 1 << 40),
        "n_fields shifts the body": _patched(blob, o, "<q", 2),
        "field F": _patched(blob, o + 8, "<i", CFG["F"]),
        "field -1": _patched(blob, o + 12, "<i", -1),
        "padding": _patched(blob, o + 20, "<i", 7),
        "kind 2 as the stream position": _patched(blob, _list_off(blob, 0, is_delta) - 8 * (10 if is_delta else 8), "<q", KIND_FIELDS),
        "kind 1 with a list": _patched(blob, o - 8 * (10 if is_delta else 8), "<q", KIND_WINDOWS),
        "truncated list": blob[:o + 6],
    }
    if is_delta:
        bad["another list"] = _patched(blob, o + 8, "<i", 4)
        bad["kind 2 for a windows handle"] = _patched(blob, _list_off(blob, 2, True) - 80, "<q", KIND_FIELDS)
    for why, b in bad.items():
        with pytest.raises((Refused, struct.error)):
            read(b)
            raise AssertionError(why)


def test_history_limit_counts_the_list():
    """H x n_fields, not H x F, is held to 2^40"""
    st = RD.new_ring(CFG["F"], CFG["W"], CFG["cap"])
    st["handles"] = [new_handle(CFG["F"], KIND_FIELDS, 1, 1, 2, [3])]
    blob = full(st, _cfg())
    o = _list_off(blob, 0, False)
    ok = _patched(blob, o - 40, "<q", HISTORY_LIMIT)            # H of a one-field handle: at the limit
    full_handles(ok)
    with pytest.raises(Refused):
        full_handles(_patched(blob, o - 40, "<q", HISTORY_LIMIT + 1))
