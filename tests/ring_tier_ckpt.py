"""Host model of tier checkpoints (DESIGN.md "Ring tier checkpoint format"): the bytes of a full tier checkpoint and a tier delta
written from a ring's samples and the state of its tier (tests/ring_tier.py), the verdict gpud_ring_tier_restore's host checks reach
on a chain, in their order and with their texts, and the placement of the chain's rows in a new tier."""
import struct

import numpy as np

import ring_checkpoint as CK
import ring_tier as T

ROW = T.ROW
MAGIC = (b"GPUDRTK1", b"GPUDRTD1")                     # [delta]
VERSION = 1
HEADER = struct.Struct("<8sIIIIqqqqqqQqq32x")          # 128 bytes
FIELDS = ("magic", "version", "F", "W", "zero", "cap", "first", "next", "from", "prev_next", "lost", "prev_link", "rows_len", "sums_len")
E_INVALID, E_CAPACITY, E_STATE = -1, -4, -6
M64 = (1 << 64) - 1


def _mix(x: int) -> int:
    return int(CK.mix64(np.array([x & M64], dtype=np.uint64))[0])


def link(prev: int, nxt: int, first: int, sums) -> int:
    """h = mix(prev + golden), then mix(h + next), mix(h + first) and mix(h + c_f) for every field"""
    h = _mix(prev + int(CK.GOLDEN))
    h = _mix(h + nxt)
    h = _mix(h + first)
    for c in sums:
        h = _mix(h + int(c))
    return h


def header(blob: bytes) -> dict:
    return dict(zip(FIELDS, HEADER.unpack_from(blob, 0)))


def sums_of(blob: bytes):
    h = header(blob)
    return np.frombuffer(blob, "<u8", h["F"], HEADER.size + h["rows_len"]).astype(np.uint64)


def blob_link(blob: bytes) -> int:
    h = header(blob)
    return link(h["prev_link"], h["next"], h["first"], sums_of(blob))


def write(bits: np.ndarray, W: int, cap: int, first: int, nxt: int, frm: int, lost: int, prev_next: int = 0, prev_link: int = 0,
          delta: bool = False) -> bytes:
    """A tier blob of rows [frm, nxt) of the samples bits [F][>= 1024 nxt] (uint64, push order): each row's image as the tier codes it,
    its offset word the row's offset in the rows section, then the checksums with i = 0 at sample 1024 frm."""
    F = bits.shape[0]
    rows, off = [], 0
    for k in range(frm, nxt):
        img = T.row_image(bits[:, k * ROW:(k + 1) * ROW], k, off)
        rows.append(img)
        off += len(img)
    sec = b"".join(rows)
    sums = CK.checksum(bits[:, frm * ROW:nxt * ROW]) if nxt > frm else np.zeros(F, dtype=np.uint64)
    head = HEADER.pack(MAGIC[delta], VERSION, F, W, 0, cap, first, nxt, frm, prev_next, lost, prev_link, len(sec), 8 * F)
    return head + sec + sums.astype("<u8").tobytes()


class Writer:
    """The blobs a tiered ring writes, from its samples and its tier (a ring_tier.Tier), and its tier marker (next, link)."""

    def __init__(self, W: int, cap: int):
        self.W, self.cap = W, cap
        self.marker = None

    def full(self, bits, tier) -> bytes:
        b = write(bits, self.W, self.cap, tier.first, tier.next, tier.first, tier.lost)
        self.marker = (tier.next, blob_link(b))
        return b

    def delta(self, bits, tier) -> bytes:
        assert self.marker is not None
        pn, pl = self.marker
        b = write(bits, self.W, self.cap, tier.first, tier.next, max(tier.first, pn), tier.lost, pn, pl, delta=True)
        self.marker = (tier.next, blob_link(b))
        return b


class Refused(Exception):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.code, self.msg = code, msg


def _frame(F, W, cap, blob, i, prev):
    """one blob's checks in gpud_ring_tier_restore's order -> (header dict, row sizes, link)"""
    def no(msg):
        raise Refused(E_INVALID, "tier_restore: " + msg)
    blob = bytes(blob)
    if len(blob) < HEADER.size or blob[:8] not in MAGIC:
        no("blob %d is not a ring tier checkpoint" % i)
    delta = blob[:8] == MAGIC[1]
    h = header(blob)
    if h["version"] != VERSION:
        no("blob %d: version %d, this library reads %d" % (i, h["version"], VERSION))
    for k in list(range(20, 24)) + list(range(96, 128)):
        if blob[k]:
            no("blob %d: header byte %d is not zero" % (i, k))
    if h["F"] != F:
        no("blob %d: n_fields %d, the ring has %d" % (i, h["F"], F))
    if h["W"] != W:
        no("blob %d: window %d, the ring has %d" % (i, h["W"], W))
    if h["cap"] != cap:
        no("blob %d: capacity %d, the ring has %d" % (i, h["cap"], cap))
    rl, sl = h["rows_len"], h["sums_len"]
    if rl < 0 or rl & 7 or rl > len(blob) or sl != 8 * F or HEADER.size + rl + sl != len(blob):
        no("blob %d: section lengths do not add up to the %d bytes given" % (i, len(blob)))
    first, nxt, frm, pn, lost, pl = h["first"], h["next"], h["from"], h["prev_next"], h["lost"], h["prev_link"]
    ok = 0 <= first <= nxt <= 1 << 52 and lost >= 0 and (pn <= nxt and frm == max(first, pn) if delta else pn == 0 and pl == 0 and frm == first)
    if not ok:
        no("blob %d: first %d, next %d, from %d, prev_next %d and lost %d disagree" % (i, first, nxt, frm, pn, lost))
    if i == 0 and delta:
        no("blob 0 is a delta: a chain starts with a full tier checkpoint")
    if i > 0 and not delta:
        no("blob %d is a full tier checkpoint: only blob 0 may be" % i)
    if prev is not None:
        ph, plink = prev
        if pl != plink:
            no("blob %d follows link %016x, blob %d's is %016x (out of order, or another chain)" % (i, pl, i - 1, plink))
        if pn != ph["next"]:
            no("blob %d follows row %d, blob %d ends at row %d" % (i, pn, i - 1, ph["next"]))
        if first < ph["first"] or lost < ph["lost"]:
            no("blob %d starts at row %d with %d lost, before blob %d's row %d with %d lost" % (i, first, lost, i - 1, ph["first"], ph["lost"]))
    sec = blob[HEADER.size:HEADER.size + rl]
    rec = T.rec_bytes(F)
    sizes, off = {}, 0
    for row in range(frm, nxt):
        if off + rec > rl:
            no("blob %d: row %d is truncated" % (i, row))
        s0, o = struct.unpack_from("<qq", sec, off)
        if s0 != row * ROW:
            no("blob %d: row %d's record starts at sample %d" % (i, row, s0))
        if o != off:
            no("blob %d: row %d's offset word is %d, the row is at %d" % (i, row, o, off))
        words = 0
        dirs = sec[off + 16:off + 16 + CK.pad8(F)]
        woff = sec[off + 16 + CK.pad8(F):off + rec]
        for f in range(F):
            w = dirs[f] & 127
            if w > 64:
                no("blob %d: row %d field %d has width %d" % (i, row, f, w))
            wo = struct.unpack_from("<I", woff, 4 * f)[0]
            if wo != words:
                no("blob %d: row %d field %d's word offset is %d, its directory gives %d" % (i, row, f, wo, words))
            words += CK.block_words(ROW, w)
        if any(dirs[F:]) or any(woff[4 * F:]):
            no("blob %d: row %d's record padding is not zero" % (i, row))
        size = rec + 8 * words
        if off + size > rl:
            no("blob %d: row %d is truncated" % (i, row))
        sizes[row] = size
        off += size
    if off != rl:
        no("blob %d: the rows section has %d bytes after its last row" % (i, rl - off))
    return h, sizes, blob_link(blob)


def plan(F, W, cap, total, tier_bytes, blobs):
    """gpud_ring_tier_restore's host work (gpudh_ring_tier_chain_plan) -> (code, message, row_off of rows [last first, last next),
    state (first, next, used, lost, head, tail)); a refusal -> (code, message, None, None)"""
    try:
        if cap < 2 * ROW:
            raise Refused(E_INVALID, "tier_restore: capacity %d is below %d" % (cap, 2 * ROW))
        if tier_bytes < T.max_row_bytes(F):
            raise Refused(E_INVALID, "tier_restore: %d bytes do not hold one row coded at 64 bits (%d bytes)" % (tier_bytes, T.max_row_bytes(F)))
        frames, prev = [], None
        for i, b in enumerate(blobs):
            h, sizes, lk = _frame(F, W, cap, b, i, prev)
            frames.append((h, sizes))
            prev = (h, lk)
        last = frames[-1][0]
        whole = -(-(total - min(total, cap)) // ROW)
        if last["next"] * ROW > total:
            raise Refused(E_INVALID, "tier_restore: the chain holds samples up to %d, the ring has %d" % (last["next"] * ROW, total))
        if last["next"] < whole:
            raise Refused(E_INVALID, "tier_restore: the chain ends at row %d, before the ring's first whole row %d: the samples between are in neither"
                          % (last["next"], whole))
    except Refused as e:
        return e.code, e.msg, None, None
    m = place(F, cap, tier_bytes, last, {k: s for _, sizes in frames for k, s in sizes.items()})
    row_off = [m.row_off[k] if k >= m.first else -1 for k in range(last["first"], last["next"])]
    return 0, "", row_off, m.state()


def place(F, cap, tier_bytes, last, sizes):
    """a new tier of tier_bytes holding rows [last first, last next), placed oldest first, with the last blob's next and lost count"""
    m = T.Tier(cap, F, tier_bytes, 0)
    m.rows, m.tail, m.row_off = [], 0, {}
    m.next = last["first"]
    for k in range(last["first"], last["next"]):
        m._place(k, sizes[k])
    m.next, m.lost = last["next"], last["lost"]
    return m
