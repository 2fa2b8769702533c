"""Blocks of the checkpoint codec aimed at one route each (csrc/ring_ckpt.cu; the format is DESIGN.md "Ring checkpoint format",
its host model ring_checkpoint.py).  Shared by test_ckpt_cases_model.py (every case reaches its target in the model) and
test_gpu_ckpt_paths.py (the kernels code, pack and unpack every case byte for byte as the model does).

A block is up to 1024 chronological samples of one field (uint64 bit patterns): an anchor and the n - 1 residuals at one width w,
RAW (bits XOR the previous sample's bits) or INT (zigzag of the int64 difference, for blocks of exact integers |x| <= 2^53), the
narrower mode, INT on a tie.  Residual j of sample t = j sits at bits [(t - 1) w, t w) of the payload words after the anchor, and
sample t is lane t % 32 of step t // 32 of the warp that codes the block.

A target is a dict:
  {"kind": "plain", "mode": RAW | INT, "w", "n", "t"}: exactly one residual has bit w - 1 set, the one of sample t (the widest);
      every other residual is narrower.  t is None when w == 0 or n == 1.
  {"kind": "eligible_raw", "k", "n"}: integers 2^52 and 2^52 + 2^k alternating: INT is allowed, but RAW (w = k + 1) is narrower.
  {"kind": "tie", "k", "n"}: 2^52 + 2^(k-1) and 2^52 + 2^k alternating: both modes have w = k + 1, so the block codes INT.
  {"kind": "edge", "edge", "at", "n"}: small integers with EDGES[edge] at sample `at`: INT when that value is allowed, else RAW.
  {"kind": "const", "value", "n"}: n copies of one bit pattern: w = 0, INT when the value is an allowed integer.
`block(target)` builds the samples, `route(bits)` reads any block back into these terms, `column(blocks)` chains the blocks of one
field in chronological order."""
import zlib

import numpy as np

import ring_checkpoint as RC
import ring_delta as RD

U64 = np.uint64
BLOCK = RC.BLOCK
RAW, INT = RC.MODE_RAW, RC.MODE_INT
TWO53 = 1 << 53


def _bits(x) -> int:
    return int(np.array([x], dtype=np.float64).view(U64)[0])


# the values at the edge of INT eligibility; only +-2^53 are allowed
EDGES = {
    "+2^53": _bits(2.0 ** 53), "-2^53": _bits(-2.0 ** 53), "+(2^53+2)": _bits(2.0 ** 53 + 2), "-(2^53+2)": _bits(-2.0 ** 53 - 2),
    "-0.0": _bits(-0.0), "5e-324": _bits(5e-324), "+inf": _bits(np.inf), "-inf": _bits(-np.inf),
    "NaN": 0x7FF8000000000000, "-NaN": 0xFFF8000000000000, "sNaN payload": 0x7FF0000000000001, "-NaN payload": 0xFFF4DEADBEEF0001,
    "+2^63": _bits(2.0 ** 63), "-2^63": _bits(-2.0 ** 63),        # cvt.rzi saturates: (double)(int64)x == x, only |x| <= 2^53 refuses
}
ALLOWED_EDGES = ("+2^53", "-2^53")
STRADDLES = ("inside", "end", "one", "more")    # a residual inside one word, ending on a word boundary, into the next by 1 / > 1 bit


def straddle(t: int, w: int) -> str:
    """where the residual of sample t (>= 1) sits at width w > 0: bits [(t - 1) w, t w) against the 64-bit payload words"""
    end = ((t - 1) * w) % 64 + w
    return "end" if end == 64 else "one" if end == 65 else "more" if end > 65 else "inside"


def _rng(target: dict):
    return np.random.default_rng(zlib.crc32(repr(sorted(target.items())).encode()))


def _below(rng, k: int, size: int) -> np.ndarray:
    """size uniform uint64 values in [0, 2^k), 0 <= k <= 63"""
    return rng.integers(0, 1 << k, size=size, dtype=U64, endpoint=False) if k else np.zeros(size, dtype=U64)


def _raw_plain(tg: dict, rng) -> np.ndarray:
    w, n, t = tg["w"], tg["n"], tg["t"]
    res = _below(rng, max(w - 1, 0), n - 1)
    if w:
        res[t - 1] = U64(1 << (w - 1)) | _below(rng, w - 1, 1)[0]
    for _ in range(8):
        # a NaN anchor (bit 51 set) stays NaN under residuals below 2^51: the block is never INT-eligible
        anchor = U64(0x7FF8000000000000) | _below(rng, 51, 1)[0] if w <= 51 else rng.integers(0, 2 ** 64, dtype=U64, endpoint=False)
        bits = np.bitwise_xor.accumulate(np.concatenate([[anchor], res]).astype(U64))
        if not RC.int_allowed(bits):
            return bits
    raise AssertionError(tg)


def _int_plain(tg: dict, rng) -> np.ndarray:
    w, n, t = tg["w"], tg["n"], tg["t"]
    # every other difference is <= 0 with a zigzag narrower than w (at most 40 bits), so the path only climbs at sample t
    c = min(w - 1, 40)
    d = -rng.integers(0, 1 << (c - 1), size=n - 1, dtype=np.int64) if c >= 1 else np.zeros(n - 1, dtype=np.int64)
    if w:
        if w <= 54:
            z = (1 << (w - 1)) | int(_below(rng, w - 1, 1)[0])
        elif w == 55:
            z = (1 << 54) | (int(_below(rng, 53, 1)[0]) << 1)      # even: d in [2^53, 2^54)
        else:
            z = 1 << 55                                            # d = 2^54 exactly: from -2^53 to +2^53
        d[t - 1] = (z >> 1) ^ -(z & 1)
    path = np.concatenate([[0], np.cumsum(d)]).astype(np.int64)
    lo, hi = -TWO53 - int(path.min()), TWO53 - int(path.max())
    assert lo <= hi, tg
    # prefer a start near 0, where the RAW residuals of integers are wide; the range check below settles it
    near = (max(lo, -(1 << 40)), min(hi, 1 << 40))
    for i in range(16):
        a, b = near if near[0] <= near[1] and i < 12 else (lo, hi)
        v0 = a + int(rng.integers(0, b - a + 1, dtype=np.uint64)) if b > a else a
        bits = (path + v0).astype(np.float64).view(U64)
        if RC.block_mode(bits) == (INT, w):
            return bits
    raise AssertionError(tg)


def block(tg: dict) -> np.ndarray:
    """the uint64 samples of one block that codes to target tg"""
    rng, n, kind = _rng(tg), tg["n"], tg["kind"]
    assert 1 <= n <= BLOCK
    if kind == "plain":
        assert (tg["t"] is None) == (tg["w"] == 0 or n == 1) and (tg["t"] is None or 1 <= tg["t"] < n)
        return _raw_plain(tg, rng) if tg["mode"] == RAW else _int_plain(tg, rng)
    if kind in ("eligible_raw", "tie"):
        k = tg["k"]
        a, b = (1 << 52, (1 << 52) + (1 << k)) if kind == "eligible_raw" else ((1 << 52) + (1 << (k - 1)), (1 << 52) + (1 << k))
        return np.where(np.arange(n) % 2 == 0, a, b).astype(np.int64).astype(np.float64).view(U64)
    if kind == "const":
        return np.full(n, tg["value"], dtype=U64)
    assert kind == "edge"
    v = 1000 + np.cumsum(rng.integers(-3, 4, size=n))
    bits = v.astype(np.float64).view(U64).copy()
    bits[tg["at"]] = U64(EDGES[tg["edge"]])
    return bits


def column(blocks) -> np.ndarray:
    """one field's chronological samples from its blocks: every block but the last has 1024 samples"""
    assert all(len(b) == BLOCK for b in blocks[:-1])
    return np.concatenate([np.asarray(b, dtype=U64) for b in blocks]) if blocks else np.zeros(0, dtype=U64)


def route(bits: np.ndarray) -> dict:
    """what the codec does with one block: its mode and width, both modes' widths (w_int None when INT is not allowed), the
    position t of the one residual that sets the width's top bit (None if no such single residual) with its lane and step, where
    that residual and the last one sit against the payload words, and the positions of INT-breaking samples and of +-2^53"""
    bits = np.ascontiguousarray(bits, dtype=U64)
    n = len(bits)
    mode, w = RC.block_mode(bits)
    allowed = RC.int_allowed(bits)
    w_raw = RC.width(np.bitwise_or.reduce(RC.residuals(bits, RAW), initial=U64(0)))
    w_int = RC.width(np.bitwise_or.reduce(RC.residuals(bits, INT), initial=U64(0))) if allowed else None
    t = None
    if w and n > 1:
        top = np.flatnonzero((RC.residuals(bits, mode) >> U64(w - 1)) & U64(1)) + 1
        t = int(top[0]) if len(top) == 1 else None
    x = bits.view(np.float64)
    with np.errstate(invalid="ignore"):
        ok = (np.abs(x) <= 2.0 ** 53) & (x.astype(np.int64).astype(np.float64).view(U64) == bits)
    breaks = [int(i) for i in np.flatnonzero(~ok)]
    return {"mode": mode, "w": w, "n": n, "allowed": allowed, "w_raw": w_raw, "w_int": w_int, "t": t,
            "lane": None if t is None else t % 32, "step": None if t is None else t // 32,
            "wide": None if t is None else straddle(t, w), "last": straddle(n - 1, w) if w and n > 1 else None,
            "breaks": breaks, "extremes": [int(i) for i in np.flatnonzero(np.abs(x) == 2.0 ** 53)]}


def reaches(tg: dict, r: dict) -> bool:
    """route r is what target tg aims at"""
    if tg["kind"] == "plain":
        return (r["mode"], r["w"], r["n"], r["t"]) == (tg["mode"], tg["w"], tg["n"], tg["t"])
    if tg["kind"] == "eligible_raw":
        return r["allowed"] and (r["mode"], r["w"], r["w_int"]) == (RAW, tg["k"] + 1, tg["k"] + 2) and r["n"] == tg["n"]
    if tg["kind"] == "tie":
        return (r["mode"], r["w"], r["w_raw"], r["n"]) == (INT, tg["k"] + 1, tg["k"] + 1, tg["n"])
    if tg["kind"] == "const":
        return (r["mode"], r["w"], r["n"]) == (INT if RC.int_allowed(np.array([tg["value"]], dtype=U64)) else RAW, 0, tg["n"])
    allowed = tg["edge"] in ALLOWED_EDGES
    return (r["mode"] == (INT if allowed else RAW) and r["n"] == tg["n"] and
            (r["extremes"] == [tg["at"]] if allowed else r["breaks"] == [tg["at"]]))


# ------------------------------------------------------------------------------------------------ the families
POSITIONS = (1, 31, 32, 33, 992)                 # and n - 1: the widest residual in lane 1 / 31 / 0 / 1 of steps 0, 0, 1, 1, 31
EDGE_AT = (0, 31, 32, 992)                       # and n - 1
TAILS = (1, 2, 3, 7, 31, 32, 33, 63, 64, 65, 511, 512, 513, 1023, 1024)


def plain(mode: int, w: int, n: int = BLOCK, t=None) -> dict:
    if n == 1:
        w = 0                                    # a lone anchor
    if w == 0:
        t = None
    elif t is None:
        t = 1 + (w * 37) % (n - 1)
    return {"kind": "plain", "mode": mode, "w": w, "n": n, "t": t}


def one_bit_t(w: int, n: int = BLOCK):
    """the first sample whose residual at odd width w >= 3 reaches exactly one bit into the next word (t w = 1 mod 64)"""
    if w % 2 == 0 or w < 3:
        return None
    t = pow(w, -1, 64)
    return t if t < n else None


def width_matrix() -> list:
    """every RAW width 0..64 and INT width 0..56 (each also with its widest residual at a one-bit straddle where the width is odd
    and in lane 0 of a later step), INT-allowed blocks that code RAW, and ties"""
    out = []
    for mode, top in ((RAW, 64), (INT, 56)):
        for w in range(top + 1):
            out.append(plain(mode, w))
            if w:
                out.append(plain(mode, w, t=32 * (1 + w % 31)))
            if one_bit_t(w):
                out.append(plain(mode, w, t=one_bit_t(w)))
    out += [{"kind": "eligible_raw", "k": k, "n": BLOCK} for k in (0, 1, 7, 30, 51)]
    out += [{"kind": "tie", "k": k, "n": BLOCK} for k in (1, 2, 13, 40, 51)]
    return out


def tail_cases(n: int) -> list:
    """blocks of n samples: the widest residual at every aimed position and in each straddle class of the last residual that n
    allows, in both modes"""
    out = [plain(RAW, 0, n), plain(INT, 0, n)]
    if n == 1:
        return out
    ts = sorted({t for t in POSITIONS + (n - 1,) if 1 <= t < n})
    widths = {}
    for w in range(1, 57):
        widths.setdefault(straddle(n - 1, w), []).append(w)
    for i, t in enumerate(ts):
        for j, cls in enumerate(STRADDLES):
            ws = widths.get(cls)
            if ws:
                w = ws[(i + j) % len(ws)]
                out.append(plain((i + j) % 2, w, n, t))
    for w in (64, 63):
        out.append(plain(RAW, w, n, n - 1))
    return out


def edge_cases(n: int = BLOCK) -> list:
    return [{"kind": "edge", "edge": e, "at": at, "n": n} for e in EDGES for at in sorted(set(EDGE_AT + (n - 1,))) if at < n]


def mixed(n: int, i: int) -> dict:
    """case i of a rotation through both modes and many widths, with the widest residual anywhere: filler blocks of n samples"""
    mode = i % 2
    w = (i * 29) % (65 if mode == RAW else 57)
    return plain(mode, w, n, None if w == 0 or n == 1 else 1 + (i * 131) % (n - 1))


def fields(count: int, cases=(), seed: int = 0, at: int = 0) -> np.ndarray:
    """[F][count] uint64, F = len(cases): field f's chronological samples are blocks of a rotation (mixed), its block `at`
    replaced by cases[f] (which must have that block's samples)"""
    nb = -(-count // BLOCK)
    F = max(1, len(cases))
    cols = []
    for f in range(F):
        blocks = []
        for b in range(nb):
            n = min(BLOCK, count - b * BLOCK)
            tg = cases[f] if b == at and f < len(cases) else mixed(n, seed + 7 * f + 3 * b)
            blocks.append(block(tg))
        cols.append(column(blocks))
    return np.array(cols, dtype=U64).reshape(F, count)


# ------------------------------------------------------------------------------------------------ corruptions
def _layout(blob: bytes):
    """(header, layout, samples per field, first sample) of a full checkpoint or a delta"""
    if blob[:8] == RC.MAGIC:
        h = RC.header(blob)
        count, first = h["count"], h["total"] - h["count"]
        return h, RC.layout(h["F"], count, h["payload_bytes"] // 8, h["handle_bytes"]), count, first
    h = RD.header(blob)
    count = h["total"] - h["first_d"]
    return h, RD.layout(h["F"], count, h["payload_bytes"] // 8, h["handle_bytes"]), count, h["first_d"]


def blocks_of(blob: bytes):
    """-> [F][nb] of (directory offset, payload word offset, n, mode, w) of every block of a full checkpoint or delta"""
    h, lay, count, _ = _layout(blob)
    F, nb = h["F"], lay["nb"]
    out, off = [], 0
    for f in range(F):
        row = []
        for b in range(nb):
            u = f * nb + b
            d = blob[lay["dir"] + u]
            n = min(BLOCK, count - b * BLOCK)
            row.append((lay["dir"] + u, off, n, d >> 7, d & 127))
            off += RC.block_words(n, d & 127)
        out.append(row)
    return out


def decode_samples(blob: bytes) -> np.ndarray:
    """[F][count] samples a full checkpoint or delta decodes to, without checking its checksums: what restore would write"""
    h, lay, count, _ = _layout(blob)
    payload = np.frombuffer(blob, "<u8", h["payload_bytes"] // 8, lay["payload"]).astype(U64)
    out = np.zeros((h["F"], count), dtype=U64)
    for f, row in enumerate(blocks_of(blob)):
        for b, (doff, off, n, mode, w) in enumerate(row):
            out[f, b * BLOCK:b * BLOCK + n] = RC.decode_block(blob[doff], payload[off:off + RC.block_words(n, w)], n)
    return out


def _flip(blob: bytes, byte: int, bit: int) -> bytes:
    b = bytearray(blob)
    b[byte] ^= 1 << bit
    return bytes(b)


def bit_flips(blob: bytes, f: int, b: int) -> dict:
    """one flipped payload bit of block (f, b): in its anchor, its first residual word, the top bit of its last word (padding
    unless the residuals end on a word boundary), the top bit of its last residual, and the top bit of its first residual that
    reaches into the next word"""
    _, lay, _, _ = _layout(blob)
    doff, off, n, mode, w = blocks_of(blob)[f][b]
    base = lay["payload"] + 8 * off
    nw = RC.block_words(n, w)
    out = {"anchor": _flip(blob, base + 2, 3)}
    if nw > 1:
        out["first residual word"] = _flip(blob, base + 8 + 1, 0)
        out["last word"] = _flip(blob, base + 8 * nw - 1, 7)
        top = (n - 1) * w - 1                                     # the last residual's top bit in the residual stream
        out["last residual"] = _flip(blob, base + 8 + top // 8, top % 8)
    for t in range(1, n):
        if w and straddle(t, w) in ("one", "more"):
            top = (t * w) - 1                                     # the residual's top bit, in the word after its first
            out["straddling residual"] = _flip(blob, base + 8 + top // 8, top % 8)
            break
    return out


def swap_blocks(blob: bytes, u1: tuple, u2: tuple) -> bytes:
    """blocks (f1, b1) and (f2, b2) of equal n exchanged with their directory bytes: the payload length and every other block's
    offset stay consistent, so only the checksums can tell"""
    _, lay, _, _ = _layout(blob)
    rows = blocks_of(blob)
    (d1, o1, n1, _, w1), (d2, o2, n2, _, w2) = rows[u1[0]][u1[1]], rows[u2[0]][u2[1]]
    assert n1 == n2
    if o1 > o2:
        (d1, o1, w1), (d2, o2, w2) = (d2, o2, w2), (d1, o1, w1)
    k1, k2 = RC.block_words(n1, w1), RC.block_words(n2, w2)
    p = lay["payload"]
    a, b = blob[p + 8 * o1:p + 8 * (o1 + k1)], blob[p + 8 * o2:p + 8 * (o2 + k2)]
    out = bytearray(blob[:p + 8 * o1] + b + blob[p + 8 * (o1 + k1):p + 8 * o2] + a + blob[p + 8 * (o2 + k2):])
    out[d1], out[d2] = blob[d2], blob[d1]
    return bytes(out)


def flip_mode(blob: bytes, f: int, b: int) -> bytes:
    return _flip(blob, blocks_of(blob)[f][b][0], 7)


def swap_widths(blob: bytes, u1: tuple, u2: tuple) -> bytes:
    """the widths of two blocks of equal n exchanged in the directory, payload untouched: the total length is unchanged"""
    rows = blocks_of(blob)
    (d1, _, n1, _, w1), (d2, _, n2, _, w2) = rows[u1[0]][u1[1]], rows[u2[0]][u2[1]]
    assert n1 == n2 and w1 != w2
    out = bytearray(blob)
    out[d1], out[d2] = (blob[d1] & 0x80) | w2, (blob[d2] & 0x80) | w1
    return bytes(out)


def corruptions(blob: bytes, aimed: dict, swaps=(), mode_flips=(), width_swaps=()) -> dict:
    """name -> edited bytes: every bit flip of each aimed block {name: (f, b)}, the block swaps, mode flips and width swaps"""
    out = {}
    for name, (f, b) in aimed.items():
        for what, e in bit_flips(blob, f, b).items():
            out["%s: %s" % (name, what)] = e
    for u1, u2 in swaps:
        out["swap %s %s" % (u1, u2)] = swap_blocks(blob, u1, u2)
    for u in mode_flips:
        out["mode bit %s" % (u,)] = flip_mode(blob, *u)
    for u1, u2 in width_swaps:
        out["widths %s %s" % (u1, u2)] = swap_widths(blob, u1, u2)
    return out


def accepted(edited: bytes, samples: np.ndarray) -> bool:
    """the model decodes the edited bytes to the original samples [F][count]: a restore must then accept them"""
    return np.array_equal(decode_samples(edited), samples)


# ------------------------------------------------------------------------------------------------ the corruption rings
def corruption_fields():
    """[6][2049] samples (blocks of 1024, 1024 and 1) and where to corrupt them: block 0 of the fields is RAW w=64, RAW w=1,
    INT w=56, INT w=0, all zeros (INT w=0: its mode bit does not change what it decodes to) and RAW w=64 again; block 2 is an
    n = 1 tail.  -> (cols, aimed {name: (f, b)}, swaps, mode flips, width swaps)"""
    first = [plain(RAW, 64, t=33), plain(RAW, 1, t=992), plain(INT, 56, t=32), plain(INT, 0), {"kind": "const", "value": 0, "n": BLOCK},
             plain(RAW, 64, t=1023)]
    cols = fields(2 * BLOCK + 1, first, seed=5)
    aimed = {"RAW w=64": (0, 0), "RAW w=1": (1, 0), "INT w=56": (2, 0), "INT w=0": (3, 0), "n = 1 tail": (0, 2)}
    swaps = [((0, 0), (5, 0)), ((0, 0), (0, 1)), ((1, 2), (4, 2))]
    mode_flips = [(4, 0), (3, 0), (0, 0), (1, 2)]
    width_swaps = [((1, 0), (2, 0))]
    return cols, aimed, swaps, mode_flips, width_swaps


def wrap_fields():
    """[2][1026] samples for a ring of CAP 1026 whose physical end falls between samples 32 and 33 of block 0 (total 2019): an INT
    and a RAW block with the widest residual on sample 33, the first one after the end"""
    return fields(1026, [plain(INT, 20, t=33), plain(RAW, 40, t=33)], seed=9)


def wrap_cases(n: int, t: int) -> list:
    """blocks of n samples for a block that the ring's physical end cuts before sample t: both modes at several widths, the widest
    residual on sample t (the first after the end) or on sample t - 1 (the last before it)"""
    out = []
    for i, (mode, w) in enumerate(((RAW, 1), (RAW, 33), (RAW, 64), (INT, 3), (INT, 31), (INT, 56), (RAW, 0), (INT, 0))):
        tw = t if i % 2 == 0 or t == 1 else t - 1
        out.append(plain(mode, w, n, tw if 1 <= tw < n else None))
    return out
