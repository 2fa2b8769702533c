"""Every path of the kmsg scan against the oracle, field by field (pytest -m gpu on an H100): the Xid / SXid automata under
fuzz, several match rounds and the unsorted candidate list, unaligned device buffers and caller streams, the staged host
copies, RAW_KMSG separators at load boundaries, buffers past 2^31 (and 2^32 when the device has room) and the hit-list
overflow contract.  The inputs come from tests/scan_cases.py, whose CPU test checks that each reaches its regime."""
import ctypes as C

import numpy as np
import pytest

import scan_cases as S
import synth
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

g = None
torch = None
E_CAPACITY = -4


@pytest.fixture(scope="module")
def ctx():
    global g, torch
    import gpud_b200 as _g
    import torch as _t
    g, torch = _g, _t
    c = g.Context([0])
    yield c
    c.close()


def _mode(name):
    return {"lines": g.SCAN_LINES, "raw": g.SCAN_RAW_KMSG, "ext": g.SCAN_LINES | g.SCAN_EXT_MATCHERS}[name]


def _b(h):
    return bytes(memoryview(h))


def _cmp_full(got, want, span, raw):
    """every field of each hit against the expectation of tests/scan_cases.py; span(off, n) = those bytes of the buffer"""
    assert len(got) == len(want)
    for h, w in zip(got, want):
        d = h.as_dict()
        ctx_ = (d, {k: v for k, v in w.items()})
        assert (h.unit_index, h.unit_offset, h.kind, h.code, h.flags) == (w["line"], w["offset"], w["kind"], w["code"], w["flags"]), ctx_
        assert d["device"] == w["device"], ctx_
        spans = [span(o, n) for o, n in ((h.dev_off, h.dev_len), (h.unit_name_off, h.unit_name_len), (h.pid_off, h.pid_len),
                                        (h.pname_off, h.pname_len), (h.inj_off, h.inj_len))]
        assert spans == [w["dev"], w["unit"], w["pid"], w["pname"], w["inj"]], ctx_
        assert d["unit"] == w["unit"].decode("latin-1")[:39], ctx_
        assert (h.severity_fatal, h.xc, h.link, h.intrinfo, h.error_status, d["extra"], h.sub_code) == \
               (w["severity_fatal"], w["xc"], w["link"], w["intrinfo"], w["error_status"], w["extra"], w["sub_code"]), ctx_
        assert (h.event_type, d["actions"], d["actions_nil"], h.rule_index, h.detail_variant) == \
               (w["event_type"], list(w["actions"] or []), w["actions"] is None, w["rule_index"], w["variant"]), ctx_
        if raw:
            assert d["kmsg"] == tuple(w["kmsg"]), ctx_


def _key(h):
    return (h["line"], h["offset"], h["kind"], h["code"], h["device"][:39], h["event_type"], list(h["actions"] or []))


def _cmp_oracle(got, want, raw):
    assert [_key(h.as_dict()) for h in got] == [_key(w) for w in want]
    if raw:
        assert [h.as_dict()["kmsg"] for h in got] == [tuple(w["kmsg"]) for w in want]


# ------------------------------------------------------------------------------------------------ 1. fuzz
@pytest.mark.parametrize("seed", [1, 2])
def test_xid_fuzz_lines_every_field(ctx, seed):
    lines = [l.encode() for l in S.xid_fuzz_lines(25000, seed=seed)]
    buf = b"\n".join(lines)
    hits, n_units = ctx.kmsg_scan(buf)
    want = S.expect_lines(lines)
    assert n_units == len(lines) and len(want) > 12000
    _cmp_full(hits, want, lambda o, n: buf[o:o + n], raw=False)
    _cmp_oracle(hits, O.scan_lines(buf), raw=False)
    print("fuzz lines seed %d: %d lines, %d hits" % (seed, len(lines), len(hits)))


@pytest.mark.parametrize("seed", [3, 4])
def test_xid_fuzz_records_every_field(ctx, seed):
    buf = S.xid_fuzz_records(10000, seed=seed)
    hits, n_units = ctx.kmsg_scan(buf, mode=g.SCAN_RAW_KMSG)
    want, n = S.expect_records(buf)
    assert n_units == n and len(want) > 4000
    _cmp_full(hits, want, lambda o, k: buf[o:o + k], raw=True)
    _cmp_oracle(hits, O.scan_raw_kmsg(buf)[0], raw=True)
    print("fuzz records seed %d: %d records, %d hits" % (seed, n, len(hits)))


# ------------------------------------------------------------------------------------------------ 2. dense candidates
@pytest.mark.parametrize("mode", ["lines", "raw", "ext"])
@pytest.mark.parametrize("size", ["rounds", "side", "side_plus_1"])
def test_dense_candidates(ctx, mode, size):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = {"rounds": 2 * sms * 2048, "side": S.SIDE_CAP, "side_plus_1": S.SIDE_CAP + 1}[size]
    raw, ext = mode == "raw", mode == "ext"
    buf = S.dense_buffer(n, raw=raw, ext=ext)
    assert S.anchor_count(buf, ext) == n
    want, n_want = S.oracle_units(buf, raw, ext)
    runs = []
    for phased in (False, True):
        ctx.scan_phase_timing(phased)
        try:
            hits, n_units = ctx.kmsg_scan(buf, mode=_mode(mode), cap=1 << 17)
        finally:
            ctx.scan_phase_timing(False)
        runs.append(([_b(h) for h in hits], n_units, ctx.scan_stats()))
        assert n_units == n_want
        assert ctx.scan_stats()["candidates"] == n
        _cmp_oracle(hits, want, raw)
    assert runs[0] == runs[1]
    print("dense %s %s: %d candidates (2 x SMs x 2048 = %d, side list %d), %d hits, %d units" %
          (mode, size, runs[0][2]["candidates"], 2 * sms * 2048, S.SIDE_CAP, len(runs[0][0]), runs[0][1]))


# ------------------------------------------------------------------------------------------------ 3. unaligned device buffers
def _alignment_buffer(mode):
    lines = [b"NVRM: GPU 0000:29:00.0: GPU has fallen off the bus.", b"nvidia-nvswitch3: SXid (PCI:0000:05:00.0): 12028, Non-fatal, Link 32 egress",
             b"NVRM:   The NVIDIA GPU 0000:18:00.0 (PCI ID) has fallen off the bus and is not responding to commands.",
             b"fallen off the bus", b"SXid", b"XXid SXi called allen len 64 fall alle llen X fallen off the bu",
             b"x" * 300 + b" NVRM: Xid (PCI:0000:05:00): 79, pid=1, name=p" + b"y" * 400,
             b"N" * 270 + b"NVRM: GPU 0000:29:00.0: GPU has fallen off the bus." + b"f" * 290,
             b"SXid (PCI:0000:05:00.0): 1, x " + b"S" * 250 + b" SXid (PCI:0000:05:00.0): 12028, Non-fatal",
             b"NVRM: Xid (PCI:0000:04:00): 149, NETIR_LINK_EVT/NETIR_LINK_DOWN Fatal XC1 i12 Link -1 (0x00a00011 0x00000000)"]
    if mode == "ext":
        lines += [l.encode() for l in synth.ext_lines()[:60] + synth.PRIM_EDGE_LINES]
    units = []
    for i, line in enumerate(lines):
        for pad in (0, 1, 2, 3, 5, 13, 17, 495, 509, 511, 2045, 2047):
            units.append(b"a" * pad + b"\n" + line if i % 2 else b"a" * pad + line)
    if mode == "raw":
        return b"\n".join(S.kmsg_prefix(i) + u.replace(b"\n", b"\n ") if i % 3 == 0 else S.kmsg_prefix(i) + u.replace(b"\n", b" ")
                          for i, u in enumerate(units))
    return b"\n".join(units)


@pytest.mark.parametrize("mode", ["lines", "raw", "ext"])
def test_unaligned_device_buffers(ctx, mode):
    full = _alignment_buffer(mode)
    raw = mode == "raw"
    L0 = len(full) - len(full) % 16
    d = torch.zeros(len(full) + 64, dtype=torch.uint8, device="cuda")
    n_scans = 0
    for L in (L0, L0 - 15, L0 - 1):
        buf = full[:L]
        ref, ref_units = ctx.kmsg_scan(buf, mode=_mode(mode))
        want, n_want = S.oracle_units(buf, raw, mode == "ext")
        assert ref_units == n_want and len(want) > 50
        _cmp_oracle(ref, want, raw)
        src = torch.frombuffer(bytearray(buf), dtype=torch.uint8)
        for off in range(16):
            d.zero_()
            d[off:off + L].copy_(src)
            hits, n_units = ctx.kmsg_scan_device(d.data_ptr() + off, L, mode=_mode(mode))
            assert n_units == ref_units, (L, off)
            assert [_b(h) for h in hits] == [_b(h) for h in ref], (L, off)
            n_scans += 1
    assert n_scans == 48
    del d
    torch.cuda.empty_cache()


def test_caller_stream_unsynchronised_write(ctx):
    buf = _alignment_buffer("lines")
    ref, ref_units = ctx.kmsg_scan(buf)
    host = torch.frombuffer(bytearray(buf), dtype=torch.uint8).pin_memory()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = torch.empty(len(buf) + 3, dtype=torch.uint8, device="cuda")
        d[3:].copy_(host, non_blocking=True)                 # written on s, scanned on s, no synchronisation in between
        hits, n_units = ctx.kmsg_scan_device(d.data_ptr() + 3, len(buf), stream=s.cuda_stream)
    s.synchronize()
    assert n_units == ref_units and [_b(h) for h in hits] == [_b(h) for h in ref]


# ------------------------------------------------------------------------------------------------ 4. host staging
def test_host_staging_pageable_pinned_device(ctx):
    total = 2 * S.STAGE_PIECE + (5 << 20)
    arr = bytearray((S.LARGE_FILLER * (total // len(S.LARGE_FILLER) + 1))[:total])
    spots = [(k * S.STAGE_PIECE - 40, S.LARGE_HITS[k % 4]) for k in (1, 2)] + [(7 << 20, S.LARGE_HITS[2]), (total - 200, S.LARGE_HITS[1])]
    for o, l in spots:
        seg = b"\n" + l + b"\n"
        arr[o:o + len(seg)] = seg
    buf = bytes(arr)
    want, n_want = S.oracle_units(buf, raw=False)
    starts = {w["offset"] for w in want}
    assert len(want) == len(spots) and all(k * S.STAGE_PIECE - 39 in starts for k in (1, 2))      # lines cut by the piece boundaries
    pageable, nu = ctx.kmsg_scan(buf)
    assert nu == n_want
    _cmp_oracle(pageable, want, raw=False)
    pinned = torch.frombuffer(bytearray(buf), dtype=torch.uint8).pin_memory()
    arr_h = (g.XidHit * 64)()
    nh, nu2 = C.c_int64(), C.c_int64()
    rc = ctx._L.gpud_kmsg_scan(ctx._h, 0, C.c_void_p(pinned.data_ptr()), len(buf), g.SCAN_LINES, arr_h, 64, C.byref(nh), C.byref(nu2))
    assert rc == 0 and nu2.value == n_want
    dev = pinned.to("cuda")
    device, nu3 = ctx.kmsg_scan_device(dev.data_ptr(), len(buf))
    assert nu3 == n_want
    ref = [_b(h) for h in pageable]
    assert [_b(arr_h[i]) for i in range(nh.value)] == ref and [_b(h) for h in device] == ref
    # the staged copy must not leave the previous piece's bytes behind: scan a shorter buffer right after
    short = buf[: S.STAGE_PIECE + 100]
    h2, n2 = ctx.kmsg_scan(short)
    w2, wn2 = S.oracle_units(short, raw=False)
    assert n2 == wn2
    _cmp_oracle(h2, w2, raw=False)


# ------------------------------------------------------------------------------------------------ 5. RAW separators at boundaries
@pytest.mark.parametrize("case", range(len(S.BOUNDARIES) * 10 + 6))
def test_separators_at_load_boundaries(ctx, case):
    name, buf, raw = S.boundary_cases()[case]
    hits, n_units = ctx.kmsg_scan(buf, mode=g.SCAN_RAW_KMSG if raw else g.SCAN_LINES)
    want, n_want = S.oracle_units(buf, raw)
    assert n_units == n_want, name
    assert [h.unit_index for h in hits] == [w["line"] for w in want], name
    _cmp_oracle(hits, want, raw)


# ------------------------------------------------------------------------------------------------ 6. large device buffers
def _large_case(total):
    c = g.Context([0])
    try:
        filler = torch.frombuffer(bytearray(S.LARGE_FILLER), dtype=torch.uint8).to("cuda")
        d = filler.repeat(total // len(S.LARGE_FILLER) + 1)[:total]
        plan = S.large_plan(total)
        for k, (o, l) in enumerate(plan):
            seg = b"\n" + l + (b"\n" if k + 1 < len(plan) else b"")
            d[o:o + len(seg)] = torch.frombuffer(bytearray(seg), dtype=torch.uint8).to("cuda")
        step = 1 << 28

        def newlines(end):
            return sum(int((d[a:min(a + step, end)] == 10).sum()) for a in range(0, end, step))
        n_units_want = newlines(total) + 1
        want = []
        for o, l in plan:
            for w in S.expect_lines([l]):
                want.append(dict(w, line=newlines(o + 1), offset=o + 1))
        hits, n_units = c.kmsg_scan_device(d.data_ptr(), total)
        stats = c.scan_stats()
        assert n_units == n_units_want
        assert stats["candidates"] == sum(S.anchor_count(l) for _, l in plan)

        def span(o, n):
            return bytes(d[o:o + n].cpu().numpy()) if n else b""
        _cmp_full(hits, want, span, raw=False)
        print("large buffer: %d bytes, %d tiles, %d units, largest hit offset %d" % (total, (total + S.TILE - 1) // S.TILE, n_units,
                                                                                    max(h.unit_offset for h in hits)))
    finally:
        c.close()
        d = filler = None
        torch.cuda.empty_cache()


def test_large_device_buffer_past_2_31(ctx):
    _large_case((9 << 30) // 4)


def test_large_device_buffer_past_2_32(ctx):
    free, _ = torch.cuda.mem_get_info()
    if free < (24 << 30):
        pytest.skip("needs 24 GiB of free device memory for a 4.25 GiB buffer and its candidate list; %.1f GiB free" % (free / 2**30))
    _large_case((17 << 30) // 4)


# ------------------------------------------------------------------------------------------------ 7. hit-list overflow
def _overflow_buffers():
    hit_lines = [l.encode() for l in synth.hit_lines() + synth.EDGE_LINES if "\n" not in l and O.scan_lines(l.encode())]
    lines = (hit_lines * (5200 // len(hit_lines) + 1))[:5200]
    rng = np.random.default_rng(7)
    lines = [lines[i] for i in rng.permutation(len(lines))]
    dup = [b"Kernel panic - not syncing: Kernel Panic", b"segfault at 1 in libnccl.so segfault at 2 in libnccl.so",
           b"nvme nvme1: I/O 5 timeout, reset controller nvme nvme2: I/O 6 timeout, reset controller"]
    ext = [dup[i % 3] if i % 2 else hit_lines[i % len(hit_lines)] for i in range(6000)]
    return [("lines", b"\n".join(lines)), ("ext", b"\n".join(ext))]


@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("entry", ["host", "device"])
def test_hit_list_overflow_keeps_the_first_hits(ctx, which, entry):
    name, buf = _overflow_buffers()[which]
    mode = g.SCAN_LINES | (g.SCAN_EXT_MATCHERS if name == "ext" else 0)
    ref_ctx = g.Context([0])
    try:
        full, n_units = ref_ctx.kmsg_scan(buf, mode=mode, cap=1 << 16)
        found = ref_ctx.scan_stats()["hits"]
    finally:
        ref_ctx.close()
    total = len(full)
    assert total >= 5000
    if name == "ext":
        assert found > total                  # the device list holds (unit, kind) duplicates the host drops
    ref = [_b(h) for h in full]
    d = torch.frombuffer(bytearray(buf), dtype=torch.uint8).to("cuda") if entry == "device" else None
    c = g.Context([0])                        # fresh: its device hit list has not grown
    try:
        for cap in (0, 1, 100, 1023, 1024, total - 1, total, total + 1):
            arr = (g.XidHit * cap)() if cap else None
            nh, nu = C.c_int64(), C.c_int64()
            if entry == "host":
                rc = c._L.gpud_kmsg_scan(c._h, 0, C.cast(C.c_char_p(buf), C.c_void_p), len(buf), mode, arr, cap, C.byref(nh), C.byref(nu))
            else:
                rc = c._L.gpud_kmsg_scan_device(c._h, 0, C.c_void_p(d.data_ptr()), len(buf), mode, arr, cap, C.byref(nh), C.byref(nu), None)
            assert rc == (E_CAPACITY if cap < total else 0), (cap, rc)
            assert nh.value == total and nu.value == n_units, cap
            got = [_b(arr[i]) for i in range(min(cap, total))]
            assert got == ref[:cap], "cap %d: first differing hit %d" % (cap, next(i for i, (a, b) in enumerate(zip(got, ref)) if a != b))
    finally:
        c.close()
    print("overflow %s %s: %d hits after dedup, %d on the device" % (name, entry, total, found))
