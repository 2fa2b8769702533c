"""The checkpoint codec's aimed blocks (ckpt_cases.py) against the host model of the format (ring_checkpoint.py): every case
reaches its target, together they reach every route of the codec, every case round-trips, and the model decode of each corruption
of test_gpu_ckpt_paths.py says whether a restore must accept it (the same samples) or refuse it (a checksum mismatch)."""
import numpy as np
import pytest

import ckpt_cases as K
import ring_checkpoint as RC
import ring_delta as RD

ALL = K.width_matrix() + [c for n in K.TAILS for c in K.tail_cases(n)] + K.edge_cases() + K.edge_cases(33) + K.edge_cases(1)


@pytest.fixture(scope="module")
def routes():
    return [(tg, K.block(tg)) for tg in ALL]


def test_every_case_reaches_its_target(routes):
    for tg, bits in routes:
        r = K.route(bits)
        assert K.reaches(tg, r), (tg, r)


def test_every_width_and_both_tie_directions(routes):
    rs = [K.route(b) for _, b in routes]
    assert {r["w"] for r in rs if r["mode"] == K.RAW} == set(range(65))
    assert {r["w"] for r in rs if r["mode"] == K.INT} == set(range(57))
    # INT allowed but RAW narrower (2^52, 2^52 + 1: RAW w=1 against INT w=2), and the tie that codes INT (2^52 + 1, 2^52 + 2)
    assert any(r["mode"] == K.RAW and r["allowed"] and (r["w"], r["w_int"]) == (1, 2) for r in rs)
    assert any(r["mode"] == K.INT and (r["w"], r["w_raw"]) == (2, 2) for r in rs)
    assert len({r["w"] for r in rs if r["mode"] == K.RAW and r["allowed"]}) >= 5
    assert len({r["w"] for r in rs if r["mode"] == K.INT and r["w_raw"] == r["w"]}) >= 5
    # INT w=56 only from -2^53 straight to +2^53
    b = next(b for tg, b in routes if tg.get("mode") == K.INT and tg.get("w") == 56)
    t = K.route(b)["t"]
    assert (b[t - 1], b[t]) == (K.EDGES["-2^53"], K.EDGES["+2^53"])


def test_every_eligibility_edge_at_every_position(routes):
    for n in (K.BLOCK, 33, 1):
        got = set()
        for tg, b in routes:
            if tg["kind"] == "edge" and tg["n"] == n:
                r = K.route(b)
                at = r["extremes"] if tg["edge"] in K.ALLOWED_EDGES else r["breaks"]
                assert r["mode"] == (K.INT if tg["edge"] in K.ALLOWED_EDGES else K.RAW)
                got |= {(tg["edge"], p) for p in at}
        want = {(e, p) for e in K.EDGES for p in set(K.EDGE_AT + (n - 1,)) if p < n}
        assert got == want, sorted(want - got)


def test_every_tail_straddle_and_position(routes):
    rs = [K.route(b) for _, b in routes]
    assert {r["n"] for r in rs} >= set(K.TAILS) | {1, 2, 31, 32, 33, 63, 64, 65, 511, 512, 513, 1023, 1024}
    assert {r["last"] for r in rs} == set(K.STRADDLES) | {None}
    assert {r["wide"] for r in rs} == set(K.STRADDLES) | {None}
    for n in K.TAILS:
        here = [r for r in rs if r["n"] == n]
        # the widest residual at every aimed position n allows, in both modes across the positions
        assert {r["t"] for r in here if r["t"] is not None} >= {t for t in K.POSITIONS + (n - 1,) if 1 <= t < n}, n
        # every straddle class of the last residual that n allows at some width
        possible = {K.straddle(n - 1, w) for w in range(1, 65)} if n > 1 else set()
        assert {r["last"] for r in here if r["last"]} == possible, n
    # lane 0 of a later step carries the widest residual, at every width of both modes
    for mode, top in ((K.RAW, 64), (K.INT, 56)):
        assert {r["w"] for r in rs if r["mode"] == mode and r["lane"] == 0 and r["step"]} == set(range(1, top + 1))
    # a one-bit straddle of the widest residual at every odd width >= 3 of both modes
    for mode, top in ((K.RAW, 64), (K.INT, 56)):
        assert {r["w"] for r in rs if r["mode"] == mode and r["wide"] == "one"} == set(range(3, top + 1, 2))


def test_every_case_round_trips(routes):
    for tg, bits in routes:
        d, words = RC.encode_block(bits)
        assert (d >> 7, d & 127) == RC.block_mode(bits)
        assert len(words) == RC.block_words(len(bits), d & 127)
        assert np.array_equal(RC.decode_block(d, words, len(bits)), bits), tg


def test_fields_chain_blocks():
    cols = K.fields(2 * K.BLOCK + 5, [K.plain(K.RAW, 7), K.plain(K.INT, 9)], seed=3)
    assert cols.shape == (2, 2 * K.BLOCK + 5)
    assert K.route(cols[0, :K.BLOCK])["w"] == 7 and K.route(cols[1, :K.BLOCK])["mode"] == K.INT
    assert K.route(cols[1, 2 * K.BLOCK:])["n"] == 5


# ------------------------------------------------------------------------------------------------ corruptions
CFG = {"W": 1, "alpha": 0.5, "q_num": 99, "q_den": 100}


def corruption_blobs():
    """(name, blob, samples, corruptions) of the full checkpoint and the delta of the corruption fields and of the wrap fields"""
    cols, aimed, swaps, flips, widths = K.corruption_fields()
    F, count = cols.shape
    cfg = dict(CFG, F=F, cap=4096, thr=np.full(F, np.inf))
    full = RC.encode(cols, count, cfg)
    st = RD.new_ring(F, 1, 4096)
    RD.push(st, np.zeros((3000, F), dtype=np.uint64))
    RD.checkpoint(st, cfg)
    RD.push(st, cols.T)
    delta = RD.encode(st)
    wcols = K.wrap_fields()
    wcfg = dict(CFG, F=2, cap=1026, thr=np.full(2, np.inf))
    wrap = RC.encode(wcols, 2019, wcfg)
    daimed = dict(aimed, **{"wrap block": (2, 1)})
    return [("full", full, cols, K.corruptions(full, aimed, swaps, flips, widths)),
            ("delta", delta, cols, K.corruptions(delta, daimed, swaps, flips, widths)),
            ("wrap", wrap, wcols, K.corruptions(wrap, {"wrap block INT": (0, 0), "wrap block RAW": (1, 0)}, [((0, 1), (1, 1))]))]


def test_corruption_outcomes():
    for name, blob, cols, edits in corruption_blobs():
        assert np.array_equal(K.decode_samples(blob), cols)
        outcome = {what: K.accepted(e, cols) for what, e in edits.items()}
        for what, e in edits.items():
            assert len(e) == len(blob) and e != blob, (name, what)
        # a changed anchor, residual word, last or straddling residual, block order or width always changes the samples
        for what, ok in outcome.items():
            if any(k in what for k in ("anchor", "first residual", "last residual", "straddling")) or what.startswith(("swap", "widths")):
                assert not ok, (name, what)
        # every aimed block with residuals has its last residual flipped
        for what in edits:
            if what.endswith("first residual word"):
                assert what.replace("first residual word", "last residual") in edits, (name, what)
        if name != "wrap":
            # the mode bit of an all-zero block: INT 0 and RAW +0.0 are the same samples, so restore must accept it
            assert outcome["mode bit (4, 0)"] and not outcome["mode bit (3, 0)"] and not outcome["mode bit (0, 0)"]
            # RAW w=1: 1023 residuals end 1023 bits in, so its last word's top bit is padding; RAW w=64 has none
            assert outcome["RAW w=1: last word"] and not outcome["RAW w=64: last word"]
            # ... but the top bit of every aimed block's last residual is data
            assert {w for w in edits if w.endswith("last residual")} >= {"RAW w=64: last residual", "RAW w=1: last residual",
                                                                          "INT w=56: last residual"}
            # INT w=56 has residuals across two words; RAW w=64 and w=1 never straddle
            assert "INT w=56: straddling residual" in edits and "RAW w=64: straddling residual" not in edits
        print(name, sorted(outcome.items()))


def test_corruption_sites():
    """the flips land where they aim: the straddling residual's top bit lies in the word after its first bit"""
    cols, aimed, *_ = K.corruption_fields()
    blob = RC.encode(cols, cols.shape[1], dict(CFG, F=6, cap=4096, thr=np.full(6, np.inf)))
    lay = RC.layout(6, cols.shape[1], RC.header(blob)["payload_bytes"] // 8, 0)
    doff, off, n, mode, w = K.blocks_of(blob)[2][0]
    assert (n, mode, w) == (K.BLOCK, K.INT, 56)
    e = K.bit_flips(blob, 2, 0)["straddling residual"]
    diff = [i for i in range(len(blob)) if blob[i] != e[i]]
    assert len(diff) == 1
    bit = 8 * (diff[0] - lay["payload"] - 8 * (off + 1)) + (blob[diff[0]] ^ e[diff[0]]).bit_length() - 1
    t = next(t for t in range(1, n) if K.straddle(t, w) in ("one", "more"))
    assert bit == t * w - 1 and bit // 64 == ((t - 1) * w) // 64 + 1
