"""CPU checks of tests/scan_cases.py: every builder reaches the regime it is meant for, and the field-by-field expectation the
GPU tests compare against agrees with the oracle's own scan."""
import collections

import pytest

import scan_cases as S
from oracle import pyoracle as O

H100_SMS = 132


@pytest.fixture(scope="module")
def fuzz_lines():
    return S.xid_fuzz_lines(50000, seed=1)


def test_fuzz_lines_reach_every_outcome(fuzz_lines):
    assert max(len(l.encode()) for l in fuzz_lines) <= 320 and not any("\n" in l for l in fuzz_lines)
    c = collections.Counter(S.outcome(l.encode()) for l in fuzz_lines)
    for k, least in (("ext_rule", 2000), ("ext_norule", 500), ("ext_fallback_r1", 2000), ("r1_known", 2000), ("r1_unknown", 100),
                     ("r3", 30), ("r4", 50), ("sxid_dev", 100), ("sxid_nodev", 50), ("none", 2000)):
        assert c[k] >= least, (k, c)


def test_fuzz_is_seeded():
    assert S.xid_fuzz_lines(300, seed=5) == S.xid_fuzz_lines(300, seed=5) != S.xid_fuzz_lines(300, seed=6)
    assert S.xid_fuzz_records(300, seed=5) == S.xid_fuzz_records(300, seed=5)


def test_expectation_agrees_with_the_oracle_scan(fuzz_lines):
    lines = [l.encode() for l in fuzz_lines[:8000]]
    got = S.expect_lines(lines)
    want = O.scan_lines(b"\n".join(lines))
    key = lambda h: (h["line"], h["offset"], h["kind"], h["code"], h["device"][:39], h["event_type"], list(h["actions"] or []))
    assert [key(h) for h in got] == [key(h) for h in want]
    for h, w in zip(got, want):
        assert bool(h["flags"] & S.HIT_EXTENDED) == w["extended"]
        if w["extended"]:
            assert (h["sub_code"], h["error_status"], h["intrinfo"], h["link"]) == (w["sub_code"], w["error_status"], w["intrinfo"], w["link"])
            assert h["unit"].decode("latin-1") == w["unit"]


def test_fuzz_records_break_lines_and_agree_with_the_oracle():
    buf = S.xid_fuzz_records(6000, seed=3)
    recs = S.split_records(buf)
    assert sum(b"\n " in r for r in recs) > 2000
    # continuation breaks inside the extended format's whitespace and inside R3's span, both matching and not
    assert sum(1 for r in recs if O.R2.search(r) and b"\n " in O.R2.search(r).group(0)) > 50
    assert sum(1 for r in recs if O.R3.search(r) and b"\n " in O.R3.search(r).group(0)) >= 1
    got, n = S.expect_records(buf)
    want, wn = O.scan_raw_kmsg(buf)
    assert n == wn
    key = lambda h: (h["line"], h["offset"], h["kind"], h["code"], h["device"][:39], h["event_type"], tuple(h["kmsg"]))
    assert [key(h) for h in got] == [key(h) for h in want]
    c = collections.Counter(h["outcome"] for h in got)
    assert c["ext_rule"] > 300 and c["ext_fallback_r1"] > 300 and c["r1_known"] > 300, c


def test_anchor_count_overlaps_and_buffer_end():
    assert S.anchor_count(b"SXidSXid NVRM: Xid (x fallen off the bus") == 4
    assert S.anchor_count(b"NVRM: Xid ") == 0 and S.anchor_count(b"fallen off the bu") == 0 and S.anchor_count(b"SXi") == 0
    assert S.anchor_count(b"nvme nvme nvme", ext=True) == 2 and S.anchor_count(b"nvme nvme nvme") == 0
    assert S.anchor_count(b"task Kernel CPU: SXid", ext=True) == 4
    assert len(S.EXT_LITS) == 21


@pytest.mark.parametrize("raw", [False, True])
@pytest.mark.parametrize("ext", [False, True])
def test_dense_counts_are_exact(raw, ext):
    for n in (2 * H100_SMS * 2048, S.SIDE_CAP, S.SIDE_CAP + 1):
        buf = S.dense_buffer(n, raw=raw, ext=ext)
        assert S.anchor_count(buf, ext) == n
        units = S.split_records(buf) if raw else buf.split(b"\n")
        assert max(len(u) for u in units) < 320
        real = sum(1 for u in units if u.split(b";", 1)[-1] not in (S.DENSE_JUNK_EXT if ext else S.DENSE_JUNK))
        assert 0.02 * len(units) < real < 0.08 * len(units)


@pytest.mark.parametrize("ext", [False, True])
def test_dense_junk_is_rejected_by_the_automata(ext):
    for l in S.DENSE_JUNK_EXT if ext else S.DENSE_JUNK:
        assert S.anchor_count(l, ext) == 1, l
        assert O.scan_lines(l, ext) == [], l
        assert O.scan_raw_kmsg(S.kmsg_prefix(3) + l, ext)[0] == [], l


def test_boundary_cases_put_the_separator_where_meant():
    cases = S.boundary_cases()
    assert len(cases) == len(S.BOUNDARIES) * 5 * 2 + 6
    for name, buf, raw in cases:
        if name.startswith("B"):
            B, d = (int(x[1:]) for x in name.split("_")[:2])
            p = B - 1 - d
            assert buf[p] == 0x0A and buf.rfind(b"\n", 0, p) < p - 8
            assert buf[p + 1:p + 2] == (b" " if name.endswith("cont") else b"6")
            hits, _ = S.expect_records(buf)
            assert len(hits) == 2 and hits[0]["line"] + 1 == hits[1]["line"]
            assert hits[0]["offset"] == (buf.rfind(b"\n", 0, p) + 1 if name.endswith("cont") else p + 1)
        else:
            start = S.CHUNK if "chunk" in name or "cont" in name else S.TILE - 3
            n = S.CHUNK if start == S.CHUNK else 3 * S.TILE + 5
            assert buf[start - 1] != 0x0A and buf[start:start + n] == b"\n" * n and buf[start + n] != 0x0A
            want, _ = S.oracle_units(buf, raw)
            assert len(want) == (1 if "cont" in name and raw else 2)


def test_oracle_units_equals_the_whole_buffer_oracle():
    for name, buf, raw in S.boundary_cases()[:12]:
        got = S.oracle_units(buf, raw)
        want = O.scan_raw_kmsg(buf) if raw else (O.scan_lines(buf), buf.count(b"\n") + 1)
        assert got == want, name


def test_large_plan_crosses_tiles_and_the_31_bit_offset():
    total = (9 << 30) // 4                      # 2.25 GiB
    plan = S.large_plan(total)
    spans = [(o + 1, o + 1 + len(l)) for o, l in plan]
    assert all(b[1] + 1 <= a[0] for a, b in zip(spans[1:], spans))          # no overlap, '\n' between
    assert spans[-1][1] == total
    assert any(s < (1 << 31) < e for s, e in spans) and any(s == (1 << 31) + S.TILE for s, _ in spans)
    assert any(s < S.TILE < e for s, e in spans) and any(s == 2 * S.TILE for s, _ in spans) and any(s == 1024 * S.TILE for s, _ in spans)
    assert total // S.TILE > 4 * 1024                                        # the last block scans several tiles per thread
    assert not S.anchor_count(S.LARGE_FILLER) and all(O.scan_lines(l) for l in S.LARGE_HITS)
    big = S.large_plan((1 << 32) + (1 << 30))
    assert any(s < (1 << 32) < e for s, e in ((o + 1, o + 1 + len(l)) for o, l in big))
