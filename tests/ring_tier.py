"""Host model of the ring's tier (DESIGN.md §2 "Tier"): the bytes of each block row, their placement in the tier's byte ring, the loss
rule, and how a range call splits into ring and tier work.  Row k is samples [1024 k, 1024 (k + 1)) of every field; each field's block
is coded by the checkpoint model (tests/ring_checkpoint.py)."""
import struct

import numpy as np

import ring_checkpoint as CK

ROW = CK.BLOCK


def rec_bytes(F: int) -> int:
    """a row record: first sample, byte offset, F directory bytes and F u32 block word offsets, each part padded to 8 bytes"""
    return 16 + CK.pad8(F) + CK.pad8(4 * F)


def max_row_bytes(F: int) -> int:
    """a row whose every block is coded at 64 bits, with its record: the smallest tier"""
    return rec_bytes(F) + 8 * F * ROW


def encode_row(bits: np.ndarray):
    """-> (directory bytes [F], payload words per field) of one row: bits [F][1024] uint64"""
    dirs, words = [], []
    for f in range(bits.shape[0]):
        d, w = CK.encode_block(bits[f])
        dirs.append(d)
        words.append(w)
    return dirs, words


def row_bytes(bits: np.ndarray) -> int:
    _, words = encode_row(bits)
    return rec_bytes(bits.shape[0]) + 8 * sum(len(w) for w in words)


def row_image(bits: np.ndarray, row: int, off: int) -> bytes:
    """row `row` as it lies in the tier at byte offset off: its record, then the blocks in field order"""
    F = bits.shape[0]
    dirs, words = encode_row(bits)
    woff = np.cumsum([0] + [len(w) for w in words[:-1]]).astype("<u4")
    rec = struct.pack("<qq", row * ROW, off) + bytes(dirs) + bytes(CK.pad8(F) - F) + woff.tobytes() + bytes(CK.pad8(4 * F) - 4 * F)
    return rec + np.concatenate(words).astype("<u8").tobytes()


class Tier:
    """Placement, eviction and loss of the tier of a ring of capacity cap and F fields, opened with tier_bytes at total0 samples."""

    def __init__(self, cap: int, F: int, tier_bytes: int, total0: int = 0):
        self.cap, self.F = cap, F
        self.B = tier_bytes & ~7
        self.total = total0
        self.lost = 0
        whole = self._whole()
        self.next = whole                         # rows encoded so far
        self.rows = []                            # held rows, oldest first: [row, off, bytes]
        self.tail = 0
        self.row_off = {}

    def _whole(self):
        return (self.total - min(self.total, self.cap) + ROW - 1) // ROW

    @property
    def first(self):
        return self.rows[0][0] if self.rows else self.next

    @property
    def used(self):
        return sum(b for _, _, b in self.rows)

    @property
    def head(self):
        return self.rows[0][1] if self.rows else 0

    def _place(self, row, s):
        while True:
            off = self.tail if self.tail + s <= self.B else 0
            # a held row overlaps [off, off + s)
            if not any(o < off + s and off < o + b for _, o, b in self.rows):
                break
            self.rows.pop(0)
        self.rows.append([row, off, s])
        self.tail = off + s
        self.row_off[row] = off

    def settle(self, sizes):
        """after the open or a push: the loss rule, then every row the ring completed, sizes[k] bytes for row k"""
        whole, done = self._whole(), self.total // ROW
        if self.next < whole:
            self.lost += whole - self.next
            self.next = whole
            self.rows, self.tail = [], 0
        for k in range(self.next, done):
            self._place(k, sizes[k])
        self.next = max(self.next, done)

    def push(self, n, sizes):
        self.total += n
        self.settle(sizes)

    def state(self):
        """(first row, next row, bytes in use, rows lost, head, tail): gpudh_ring_tier_plan's state"""
        return (self.first, self.next, self.used, self.lost, self.head, self.tail)


def split(total, cap, t_first, t_next, first, length, set_off=None):
    """-> (route [n_sets], rows, vfirst [n], vtotal) of one range call on a tiered ring, or None when the call is refused"""
    first, length = list(first), list(length)
    n = len(first)
    count = min(total, cap)
    lo = min(total - count, t_first * ROW)
    if any(ln < 1 or f < lo or f + ln > total for f, ln in zip(first, length)):
        return None
    sets = [(s, s + 1) for s in range(n)] if set_off is None else list(zip(set_off[:-1], set_off[1:]))
    if set_off is not None and (set_off[0] != 0 or set_off[-1] != n or any(b <= a for a, b in sets)):
        return None
    route = [int(any(first[i] < total - count for i in range(a, b))) for a, b in sets]
    need = set()
    for (a, b), r in zip(sets, route):
        for i in range(a, b) if r else ():
            need.update(range(first[i] // ROW, -(-(first[i] + length[i]) // ROW)))
    rows = sorted(need)
    at = {k: j for j, k in enumerate(rows)}
    vfirst = [-1] * n
    for (a, b), r in zip(sets, route):
        for i in range(a, b) if r else ():
            vfirst[i] = at[first[i] // ROW] * ROW + first[i] % ROW
    vtotal = len(rows) * ROW
    if rows and rows[-1] == t_next:
        vtotal -= ROW - (total - t_next * ROW)
    return route, rows, vfirst, vtotal
