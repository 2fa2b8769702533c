"""Seeded inputs that drive the kmsg scan through each of its paths, and the expected value of every hit field.

- xid_fuzz_lines / xid_fuzz_records: mutations of the Xid / SXid vectors aimed at the R1-R6 automata (the NVLink5 extended
  format above all), as lines and as /dev/kmsg records whose text is broken by continuation lines.
- dense_lines / dense_buffer: one verified anchor per short line, so the candidate count is exact (several match rounds,
  exactly 2^20 - the largest list the family sort takes - and one more).
- raw_boundary_buffer / separator_run_buffer: RAW_KMSG separators whose next byte sits in the next word, lane, chunk, run or tile.
- large_plan: where hit lines are planted in a multi-GiB device buffer (tile boundaries, 2^31, the last bytes).
- anchor_count: the candidates the filter must verify.
- expect_xid / expect_lines / expect_records: the oracle's match of every unit, field by field, in the layout of gpud_xid_hit.
"""
import re

import numpy as np

import synth
from oracle import pyoracle as O

CHUNK = 512                  # bytes per filter warp step
RUN = 4 * CHUNK              # bytes per filter load run
TILE = 1024 * CHUNK          # chunks per separator-prefix tile
STAGE_PIECE = 8 << 20        # pageable host buffers are staged in pieces of this size
SIDE_CAP = 1 << 20           # the family sort runs on candidate lists up to this length

XID_LITS = [b"NVRM: Xid (", b"fallen off the bus", b"SXid"]
EXT_LITS = [b"segfault at", b"ERROR detected invalid context, skipping further processing", b"Detected insufficient power on the PCIe slot (",
            b"Port module event", b"mlx5_cmd_out_err", b"task ", b"soft lockup - CPU#", b"VFS: file-max limit ", b"md/raid",
            b"Remounting filesystem read-only", b"block nvme", b"nvme nvme", b"attempt to access beyond end of device",
            b"Buffer I/O error on dev ", b"I/O error while writing superblock", b"Kernel ", b"CPU: ", b"invoked oom-killer:",
            b"oom-kill:constraint=", b"Task in ", b"Killed process "]
_ANCHOR_RE = {ext: re.compile(b"|".join(b"(?=" + re.escape(l) + b")" for l in XID_LITS + (EXT_LITS if ext else []))) for ext in (False, True)}

HIT_EXTENDED, HIT_FALLEN_OFF_BUS, HIT_DEV_TRUNCATED, HIT_HAS_RULE = 1, 2, 4, 8
_VARIANT_DESC = {}
for _sc, _v in ((4, 1), (10, 2)):
    if _sc in O.DETAILS_WITH_SUBCODES.get(149, {}):
        _VARIANT_DESC[O.DETAILS_WITH_SUBCODES[149][_sc].description] = _v


def anchor_count(buf: bytes, ext: bool = False) -> int:
    """Occurrences the filter verifies: every (overlapping) "NVRM: Xid (", "fallen off the bus" and "SXid" and, with the extra
    matchers, every occurrence of their 21 anchor literals - each wholly inside the buffer."""
    return sum(1 for _ in _ANCHOR_RE[ext].finditer(buf))


# ------------------------------------------------------------------------------------------------ expected hits
def _sp(m, i):
    return (m.group(i) or b"") if m is not None else b""


def expect_xid(msg: bytes):
    """xid.Match of one message as the fields of a gpud_xid_hit (spans as the bytes they cover), or None.  `outcome` names the
    branch that decided it."""
    info = O.extract_nvrm_xid_info_extended(msg)
    if info is not None:
        d = O.detail_from_nvlink_info(info)
        if d is not None:
            m = O.R2.search(msg)
            rule, _ = O.lookup_nvlink_rule(info)
            flags = HIT_EXTENDED | (HIT_HAS_RULE if rule >= 0 else 0)
            if len(m.group(1)) + 4 > 39 or len(m.group(5)) >= 40:
                flags |= HIT_DEV_TRUNCATED
            return {"outcome": "ext_rule" if rule >= 0 else "ext_norule", "kind": 1, "code": info.xid, "flags": flags,
                    "device": ("PCI:" + info.device)[:39], "dev": m.group(1), "unit": _sp(m, 5), "pid": _sp(m, 3), "pname": _sp(m, 4),
                    "inj": _sp(m, 8), "severity_fatal": int(m.group(6) == b"Fatal"), "xc": int(m.group(7)[2:]), "link": info.link,
                    "intrinfo": info.intrinfo, "error_status": info.error_status, "extra": list(info.extra), "sub_code": info.sub_code,
                    "event_type": d.event_type, "actions": d.actions, "rule_index": rule, "variant": _VARIANT_DESC.get(d.description, 0)}
    m = O.R1.search(msg)
    code = O.go_atoi(m.group(2)) if m else None
    if code:
        d = O.get_detail(code)
        if d is None:
            return {"outcome": "r1_unknown"}
        near = b" Link" in msg and b"(0x" in msg
        return dict(_plain(code, d.event_type, d.actions), outcome="ext_fallback_r1" if near else "r1_known", device=m.group(1).decode("latin-1")[:39],
                    dev=m.group(1), flags=HIT_DEV_TRUNCATED if len(m.group(1)) > 39 else 0)
    for name, rx in (("r4", O.R4), ("r3", O.R3)):
        m = rx.search(msg)
        if m:
            d = O.get_detail(79)
            return dict(_plain(79, d.event_type, d.actions), outcome=name, device=O.normalize_pci_bdf(m.group(1).decode("latin-1")), dev=m.group(1),
                        flags=HIT_FALLEN_OFF_BUS)
    return None


def _plain(code, event_type, actions):
    return {"kind": 1, "code": code, "unit": b"", "pid": b"", "pname": b"", "inj": b"", "severity_fatal": 0, "xc": 0, "link": 0,
            "intrinfo": 0, "error_status": 0, "extra": [], "sub_code": 0, "event_type": event_type, "actions": actions,
            "rule_index": -1, "variant": 0}


def expect_sxid(msg: bytes):
    s = O.sxid_match(msg)
    if s is None:
        return None
    m = O.R6.search(msg)
    dev = m.group(1) if m else b""
    return dict(_plain(s["sxid"], s["detail"]["event_type"], s["detail"]["actions"]), outcome="sxid_dev" if m else "sxid_nodev",
                kind=2, device=dev.decode("latin-1")[:39], dev=dev, flags=HIT_DEV_TRUNCATED if len(dev) > 39 else 0)


def outcome(msg: bytes) -> str:
    """the branch of the Xid decision a message takes ("none" when neither Xid nor SXid matches)"""
    x = expect_xid(msg)
    if x is not None:
        return x["outcome"]
    s = expect_sxid(msg)
    return s["outcome"] if s is not None else "none"


def _unit_hits(msg: bytes, unit: int, offset: int, msg_off: int, kmsg=(0, 0, 0)):
    out = []
    for h in (expect_xid(msg), expect_sxid(msg)):
        if h is None or "kind" not in h:
            continue
        out.append(dict(h, line=unit, offset=offset, msg_off=msg_off, kmsg=kmsg))
    return out


def expect_lines(lines):
    """LINES: every Xid / SXid hit of the buffer b"\\n".join(lines), in (line, kind) order."""
    out, off = [], 0
    for i, l in enumerate(lines):
        out += _unit_hits(l, i, off, off)
        off += len(l) + 1
    return out


def split_records(buf: bytes):
    return re.split(rb"\n(?! )", buf)


def expect_records(buf: bytes):
    """RAW_KMSG: every Xid / SXid hit of the records of `buf` (a record continues on lines that start with ' ';
    records parseLine rejects are skipped).  Returns (hits, n_units)."""
    out, off = [], 0
    recs = split_records(buf)
    for i, rec in enumerate(recs):
        try:
            prio, seq, usec, msg = O.parse_kmsg_line(0, rec.decode("latin-1"))
        except ValueError:
            pass
        else:
            out += _unit_hits(msg.encode("latin-1"), i, off, off + rec.index(b";") + 1, (prio, seq, usec))
        off += len(rec) + 1
    return out, len(recs)


def oracle_units(buf: bytes, raw: bool, ext: bool = False):
    """O.scan_lines / O.scan_raw_kmsg of `buf`, computed once per distinct unit (the dense and boundary buffers repeat a few
    units millions of times).  Returns (hits, n_units)."""
    units = split_records(buf) if raw else buf.split(b"\n")
    cache, out, off = {}, [], 0
    for i, u in enumerate(units):
        r = cache.get(u)
        if r is None:
            r = cache[u] = O.scan_raw_kmsg(u, ext)[0] if raw else O.scan_lines(u, ext)
        for h in r:
            out.append(dict(h, line=i, offset=off))
        off += len(u) + 1
    return out, len(units)


# ------------------------------------------------------------------------------------------------ Xid fuzz
def _is_extended_base(l: str) -> bool:
    return O.R2.search(l.encode()) is not None


_EDIT_ALPHABET = list("0123456789abcdefABCDEFxX:,()./_-") + list("NVRMXIDLKPQZ") + [" ", "\t", "\f", "\r"]
_WS_RUNS = [" ", "  ", "\t", "\f", "\r", " \t", "\t\f", "\r ", " \f\r"]


def _mutate(l: str, rng) -> str:
    op = int(rng.integers(0, 10))
    n = len(l)
    if op == 0 and n:                                            # truncation at any byte
        return l[: int(rng.integers(0, n + 1))]
    if op == 1:                                                  # one-byte edit: replace, insert or delete
        p = int(rng.integers(0, n + 1))
        c = _EDIT_ALPHABET[int(rng.integers(0, len(_EDIT_ALPHABET)))]
        k = int(rng.integers(0, 3))
        return l[:p] + (c if k < 2 else "") + l[p + (k != 1):]
    if op == 2:                                                  # whitespace runs replaced by other [\t\f\r ] runs
        runs = list(re.finditer(r"[ \t\f\r]+", l))
        if runs:
            m = runs[int(rng.integers(0, len(runs)))]
            return l[:m.start()] + _WS_RUNS[int(rng.integers(0, len(_WS_RUNS)))] + l[m.end():]
    if op == 3:                                                  # numeric fields: past int64 / uint32, leading zeros, signed link
        nums = list(re.finditer(r"0x[0-9a-fA-F]+|-?\d+", l))
        if nums:
            m = nums[int(rng.integers(0, len(nums)))]
            t = m.group(0)
            k = int(rng.integers(0, 6))
            if t.startswith("0x"):
                new = ["0x100000000", "0xffffffff", "0x" + "0" * 12 + t[2:], "0x", "0xFFFFFFFFF", t.upper().replace("0X", "0x")][k]
            else:
                new = ["9223372036854775808", "9223372036854775807", "000" + t.lstrip("-"), "-" + t.lstrip("-"), "-0", "99999999999999999999999"][k]
            return l[:m.start()] + new + l[m.end():]
    if op == 4:                                                  # pid/name group dropped or added
        m = re.search(r", pid=\d+, name=[^,]+", l)
        if m:
            return l[:m.start()] + ("" if rng.random() < 0.5 else m.group(0) + m.group(0)) + l[m.end():]
        m = re.search(r"\): \d+", l)
        if m:
            return l[:m.end()] + ", pid=%d, name=%s" % (int(rng.integers(0, 99999)), ["proc", "a b", "x(y)", "NVRM"][int(rng.integers(0, 4))]) + l[m.end():]
    if op == 5:                                                  # hex words 3-6 dropped or duplicated
        m = re.search(r"\((0x[0-9a-fA-F]+(?:[ \t\f\r]+0x[0-9a-fA-F]+)*)", l)
        if m:
            words = m.group(1).split()
            k = int(rng.integers(0, 3))
            if k == 0 and len(words) > 2:
                words.pop(int(rng.integers(2, len(words))))
            elif k == 1:
                words += words[: int(rng.integers(1, 5))]
            else:
                words = words[:2]
            return l[:m.start(1)] + " ".join(words) + l[m.end(1):]
    if op == 6:                                                  # PCI: removed or doubled
        if "PCI:" in l:
            return l.replace("PCI:", "" if rng.random() < 0.5 else "PCI:PCI:", 1)
        return l.replace("(", "(PCI:", 1)
    if op == 7:                                                  # Fatal / Nonfatal case, XC2, "i" without digits
        subs = [("Nonfatal", "nonfatal"), ("Nonfatal", "NonFatal"), ("Fatal", "fatal"), ("Fatal", "FATAL"), ("Nonfatal", "Fatal"),
                ("Fatal", "Nonfatal"), ("XC0", "XC2"), ("XC1", "XC2"), ("XC0", "XC1"), (" i0 ", " i "), (" i1", " i")]
        a, b = subs[int(rng.integers(0, len(subs)))]
        if a in l:
            return l.replace(a, b, 1)
        m = re.search(r" i\d+ ", l)
        if m:
            return l[:m.start()] + " i " + l[m.end():]
    if op == 8:                                                  # the extended unit: digits, lowercase, a second slash
        m = re.search(r", ([A-Z_]+(?:/[A-Z_]+)?)[ \t\f\r]", l)
        if m:
            u = m.group(1)
            k = int(rng.integers(0, 4))
            new = [u.lower(), u + "/X", u + "2", "A" * int(rng.integers(30, 50))][k]
            return l[:m.start(1)] + new + l[m.end(1):]
    return l


def _glue(a: str, b: str, rng) -> str:
    return a + ("" if rng.random() < 0.3 else " ") + b


def xid_fuzz_lines(n: int, seed: int = synth.SEED):
    """n mutated Xid / SXid lines (no '\\n'), each at most a few hundred bytes: the reference's vectors and EDGE_LINES with
    extra weight on the NVLink5 extended lines, one to three mutations each, sometimes two lines glued together"""
    rng = np.random.default_rng(seed)
    base = [l.replace("\n", " ") for l in synth.hit_lines() + synth.EDGE_LINES]
    ext = [l for l in base if _is_extended_base(l)]
    out = []
    for _ in range(n):
        pool = ext if rng.random() < 0.5 else base
        l = pool[int(rng.integers(0, len(pool)))]
        if rng.random() < 0.08:
            l = _glue(l, base[int(rng.integers(0, len(base)))], rng)
        for _k in range(int(rng.integers(1, 4))):
            l = _mutate(l, rng)
        out.append(l.replace("\n", " ")[:320])
    return out


def xid_fuzz_records(n: int, seed: int = synth.SEED) -> bytes:
    """n /dev/kmsg records carrying the fuzz lines, with "\\n " continuation breaks inserted at token boundaries - inside R2's
    whitespace, inside R3's span, between a number and its comma - and some records a continuation line of their own"""
    rng = np.random.default_rng(seed + 1)
    lines = xid_fuzz_lines(n, seed)
    recs = []
    for i, l in enumerate(lines):
        b = l.encode()
        cuts = [m.start() for m in re.finditer(rb"(?<=[^0-9A-Za-z])|(?=[^0-9A-Za-z])", b)]
        for _ in range(int(rng.integers(0, 3)) if cuts else 0):
            p = cuts[int(rng.integers(0, len(cuts)))]
            b = b[:p] + (b"\n " if rng.random() < 0.7 else b"\n  ") + b[p:]
            cuts = [c + 2 if c > p else c for c in cuts]
        rec = b"%d,%d,%d,-;" % (int(rng.integers(0, 8)), 1000 + i, 5_000_000 + 137 * i) + b
        if i % 11 == 5:
            rec += b"\n SUBSYSTEM=pci\n DEVICE=+pci:0000:05:00.0"
        recs.append(rec)
    return b"\n".join(recs) + b"\n"


# ------------------------------------------------------------------------------------------------ dense candidates
DENSE_JUNK = [b"NVRM: Xid (junk", b"SXid seen, no code", b"NVRM: Xid (PCI:0000:05:00) no code",
              b"GPU has fallen off the bus", b"SXid (PCI:0000:05:00.0): x"]
DENSE_JUNK_EXT = DENSE_JUNK + [b"segfault at 0", b"task x", b"Kernel x", b"CPU: x", b"nvme nvme: x", b"md/raid x",
                               b"Killed process x", b"Task in x", b"oom-kill:constraint=x"]


def _dense_hit_lines(ext: bool):
    out = []
    for l in synth.hit_lines():
        b = l.encode()
        if b"\n" not in b and len(b) < 300 and O.scan_lines(b, ext) and 1 <= anchor_count(b, ext) <= 3:
            out.append(b)
    return out


def dense_lines(n_cand: int, ext: bool = False, seed: int = synth.SEED):
    """short lines holding exactly n_cand verified anchors in all: one per junk line (the filter keeps it, the automaton rejects
    it), real hit lines mixed in at about one in twenty"""
    rng = np.random.default_rng(seed)
    junk = DENSE_JUNK_EXT if ext else DENSE_JUNK
    hits = _dense_hit_lines(ext)
    hit_n = [anchor_count(h, ext) for h in hits]
    u, kh, kj = rng.random(n_cand), rng.integers(0, len(hits), n_cand).tolist(), rng.integers(0, len(junk), n_cand).tolist()
    real = (u < 0.05).tolist()
    out, left, i = [], n_cand, 0
    while left:
        if real[i] and hit_n[kh[i]] <= left:
            out.append(hits[kh[i]])
            left -= hit_n[kh[i]]
        else:
            out.append(junk[kj[i]])
            left -= 1
        i += 1
    return out


def kmsg_prefix(i: int) -> bytes:
    k = i % 7
    return b"%d,%d,%d,-;" % (k, 100 + k, 1000 * k)


def dense_buffer(n_cand: int, raw: bool, ext: bool = False, seed: int = synth.SEED) -> bytes:
    lines = dense_lines(n_cand, ext, seed)
    if raw:
        lines = [kmsg_prefix(i) + l for i, l in enumerate(lines)]
    return b"\n".join(lines)


# ------------------------------------------------------------------------------------------------ separators at load boundaries
BOUNDARIES = [16, 512, 2048, 512 << 10, 1 << 20]
HIT_REC = b"6,7,8,-;NVRM: Xid (PCI:0000:05:00): 79, pid=1, GPU has fallen off the bus."
CONT_HIT = b" cont NVRM: Xid (PCI:0000:06:00): 13, Graphics Exception"
_FILLER = b"6,1,2,-;usb 1-1: new high-speed USB device number 3 using xhci_hcd"


def _fill_to(p: int) -> bytes:
    """records of noise that end with a separator at byte p - 1 ... precisely: bytes [0, p) hold records, the last one unterminated"""
    out, size = [], 0
    while p - size > len(_FILLER) + 40:
        out.append(_FILLER)
        size += len(_FILLER) + 1
    last = p - size
    assert last >= 9
    out.append(b"6,1,2,-;" + b"x" * (last - 8))
    return b"\n".join(out)


def raw_boundary_buffer(B: int, d: int, cont: bool) -> bytes:
    """a record ends at offset p = B - 1 - d with '\\n'; the next byte is ' ' (cont: the record continues, with a hit in the
    continuation line) or the first byte of a record holding a hit.  Another hit record follows right after."""
    p = B - 1 - d
    head = _fill_to(p)
    assert len(head) == p
    nxt = CONT_HIT if cont else HIT_REC
    return head + b"\n" + nxt + b"\n" + HIT_REC + b"\n" + _FILLER


def separator_run_buffer(start: int, n: int, after: bytes, raw: bool) -> bytes:
    """n bare '\\n' from offset `start` (filler before it), then `after` (a hit unit, or ' ' + text: a continuation of the run's
    last empty unit) and one more hit unit"""
    head = _fill_to(start) if raw else b"x" * start
    hit = HIT_REC if raw else HIT_REC.split(b";", 1)[1]
    return head + b"\n" * n + after + b"\n" + hit


def boundary_cases():
    """(name, buffer, raw) of every boundary case"""
    out = []
    for B in BOUNDARIES:
        for d in range(5):
            for cont in (True, False):
                out.append(("B%d_d%d_%s" % (B, d, "cont" if cont else "sep"), raw_boundary_buffer(B, d, cont), True))
    for raw in (False, True):
        hit = HIT_REC if raw else HIT_REC.split(b";", 1)[1]
        tag = "raw" if raw else "lines"
        out.append(("chunk_run_" + tag, separator_run_buffer(CHUNK, CHUNK, hit, raw), raw))
        out.append(("tile_runs_" + tag, separator_run_buffer(TILE - 3, 3 * TILE + 5, hit, raw), raw))
        out.append(("run_then_cont_" + tag, separator_run_buffer(CHUNK, CHUNK, b" " + hit, raw), raw))
    return out


# ------------------------------------------------------------------------------------------------ large device buffer
LARGE_FILLER = b"[ 1234.567890] kernel: filler line with no anchor in it, 64 b.\n"
LARGE_HITS = [b"NVRM: Xid (PCI:0000:05:00): 79, pid=1, GPU has fallen off the bus.",
              b"nvidia-nvswitch3: SXid (PCI:0000:05:00.0): 12028, Non-fatal, Link 32 egress",
              b"NVRM: Xid (PCI:0000:04:00): 149, NETIR_LINK_EVT/NETIR_LINK_DOWN Fatal XC1 i12 Link -1 (0x00a00011 0x00000000)",
              b"NVRM: GPU 0000:29:00.0: GPU has fallen off the bus."]


def large_plan(total: int):
    """(offset, line) of the hit lines planted in a `total`-byte buffer of LARGE_FILLER: each is written as '\\n' + line + '\\n'
    (the last one without the final '\\n', ending the buffer), so the line starts at offset + 1.  Lines straddle the first and
    a few later tile boundaries, the 2^31 and 2^32 boundaries that fit, and end at the buffer's last byte."""
    spots = [TILE - 20, 2 * TILE - 1, 7 * TILE - 40, 1023 * TILE - 10, 1024 * TILE - 1, 1025 * TILE - 60]
    for edge in (1 << 31, 1 << 32):
        spots += [edge - 40, edge + TILE - 1, edge + 3 * TILE - 2]
    spots.append(total // 2 - total // 2 % TILE - 7)
    out = []
    for s in sorted(spots):
        if 0 < s and s + 300 < total and (not out or s - out[-1][0] > 300):
            out.append((s, LARGE_HITS[len(out) % len(LARGE_HITS)]))
    last = LARGE_HITS[0]
    out.append((total - len(last) - 1, last))
    return out
