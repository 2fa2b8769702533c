"""Tier checkpoints on the GPU (DESIGN.md "Ring tier checkpoint format"), on NVML-like uint32 rows pushed raw (INT blocks) and f64
fields with noise, infinities and NaN (RAW blocks): a ring and its tier checkpointed and restored into a new ring give the same tier
counts, the same row bytes but for the offset word, and ranges and sets in the tier, across its boundary and in the ring equal bit for
bit in all six outputs and checked against the C oracle; after identical further pushes the next ring delta and tier delta are
byte-equal; a base plus deltas restores the tier a full tier checkpoint restores; blobs are a function of the rows alone; a smaller
tier keeps the model's newest rows; blobs equal the host model's (tests/ring_tier_ckpt.py); every refusal with its full text, leaving
the ring without a tier and open to tier_open; tier calls never move the ring's chain marker; a capped codec grid changes nothing.
Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import ring_tier as T
import ring_tier_ckpt as TK
from test_gpu_ring_ranges import OPS, _fields, _thr
from test_gpu_ring_tier import _bitwise, _cases, _nvml, _oracle
from test_gpu_window_paths import _check
from test_ring_tier_ckpt_model import refusal_cases, scenario

pytestmark = pytest.mark.gpu
ROW = T.ROW
F, CAP, W, ALPHA = 6, 16384, 1000, 0.01


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    yield g, ctx, g.lib()
    ctx.close()


def last_error(g, ctx):
    buf = C.create_string_buffer(512)
    g.lib().gpud_last_error(ctx._h, buf, 512)
    return buf.value.decode()


def data(kind, total, seed):
    """-> (rows [total][F] as pushed, x [F][total] f64, thresholds)"""
    rng = np.random.default_rng(seed)
    if kind == "nvml":
        rows = _nvml(F, total, rng)
        x = rows.T.astype(np.float64)
        thr = np.array([np.median(x[f]) for f in range(F)])
    else:
        x = _fields(F, total, rng)
        rows = np.ascontiguousarray(x.T)
        thr = _thr(x)
    return rows, x, thr


def push(r, rows, a, b, step=5000):
    for i in range(a, b, step):
        part = rows[i:min(b, i + step)]
        r.push_raw(part) if rows.dtype != np.float64 else r.push(part)


def new_ring(g, ctx, thr):
    return g.Ring(ctx, F, CAP, W, thresholds=thr, ema_alpha=ALPHA)


def held_rows(r):
    t0, t1, _, _ = r.tier_counts()
    return {k: r.tier_row(k) for k in range(t0 // ROW, t1 // ROW)}


def no_offset(img):
    return img[:8] + img[16:]


def same_answers(a, b, x, thr, total, lo, seed):
    rng = np.random.default_rng(seed)
    cases = _cases(total, CAP, lo, rng)
    first = np.array([f for f, _ in cases], dtype=np.int64)
    length = np.array([n for _, n in cases], dtype=np.int64)
    got, want = b.reduce_ranges(first, length), a.reduce_ranges(first, length)
    assert _bitwise(got, want)
    _check(got, _oracle(x, first, length, np.arange(len(first) + 1), thr, ALPHA))
    order = rng.permutation(len(cases))
    sf, sl = first[order], length[order]
    so = np.array(sorted({0, len(sf)} | set(rng.integers(1, len(sf), 5).tolist())), dtype=np.int64)
    got, want = b.reduce_range_sets(sf, sl, so), a.reduce_range_sets(sf, sl, so)
    assert _bitwise(got, want)
    _check(got, _oracle(x, sf, sl, so, thr, ALPHA))


@pytest.mark.parametrize("kind", ["nvml", "noise"])
def test_round_trip_and_further_pushes(env, kind):
    g, ctx, _ = env
    total, more = 10 * CAP + 777, 3 * CAP + 5
    rows, x, thr = data(kind, total + more, 1)
    tb = 8 * F * (total + more) + (1 << 20)              # holds every row: both tiers evict nothing
    a = new_ring(g, ctx, thr)
    a.tier_open(tb)
    push(a, rows, 0, total)
    with pytest.raises(g.GpudError) as e:
        a.tier_checkpoint_stats()
    assert e.value.code == -6
    ring_blob, tier_blob = a.checkpoint(), a.tier_checkpoint()
    enc, _, n = a.tier_checkpoint_stats()
    assert enc > 0 and n == total // ROW - a.tier_counts()[0] // ROW
    b = new_ring(g, ctx, thr)
    b.restore(ring_blob)
    b.tier_restore(tb, [tier_blob])
    _, dec, n_b = b.tier_checkpoint_stats()
    assert dec > 0 and n_b == n
    assert b.tier_counts() == a.tier_counts()
    ra, rb = held_rows(a), held_rows(b)
    assert ra.keys() == rb.keys() and all(no_offset(ra[k]) == no_offset(rb[k]) for k in ra)
    lo = a.tier_counts()[0]
    assert lo < total - CAP
    same_answers(a, b, x[:, :total], thr, total, lo, 2)
    # identical further pushes: the same ring delta and tier delta, and the same answers.  b's first tier call after its restore is
    # this delta, so it follows the tier marker the restore set: the chain's last next row and link.
    for r in (a, b):
        push(r, rows, total, total + more)
    ring_delta = a.checkpoint_delta()
    assert ring_delta == b.checkpoint_delta()
    da, db = a.tier_checkpoint_delta(), b.tier_checkpoint_delta()
    assert da == db and TK.header(da)["from"] == total // ROW
    assert TK.header(db)["prev_next"] == total // ROW and TK.header(db)["prev_link"] == TK.blob_link(tier_blob)
    same_answers(a, b, x, thr, total + more, lo, 3)
    # a second restart: the ring's chain, then the tier's base and the delta b wrote, restore the same tier again
    c = new_ring(g, ctx, thr)
    c.restore(ring_blob)
    c.restore_delta(ring_delta)
    c.tier_restore(tb, [tier_blob, db])
    assert c.tier_counts() == a.tier_counts()
    full = a.tier_checkpoint()
    assert b.tier_checkpoint() == full and c.tier_checkpoint() == full
    same_answers(a, c, x, thr, total + more, lo, 4)
    for r in (a, b, c):
        r.close()


@pytest.mark.parametrize("kind", ["nvml", "noise"])
def test_chain_equals_full_and_blob_bytes(env, kind):
    """a small tier that evicts and wraps: a base plus deltas (one empty) restores what a full tier checkpoint restores, into a tier of
    the original's size, a larger one (every row, and the same blob bytes as the original's) and a smaller one (the model's newest rows)"""
    g, ctx, _ = env
    steps = [3 * CAP, 5000, 0, 2 * CAP + 1, 9000, CAP, 4 * CAP]
    total = sum(steps)
    rows, x, thr = data(kind, total, 4)
    tb = 12 * T.max_row_bytes(F)
    a = new_ring(g, ctx, thr)
    a.tier_open(tb)
    chain, pos = [], 0
    for i, n in enumerate(steps):
        push(a, rows, pos, pos + n)
        pos += n
        chain.append(a.tier_checkpoint() if i == 0 else a.tier_checkpoint_delta())
    assert any(TK.header(b)["from"] == TK.header(b)["next"] for b in chain[1:])                 # an empty delta
    assert TK.header(chain[-1])["first"] > TK.header(chain[0])["first"]                          # rows were evicted
    full = a.tier_checkpoint()
    ring_blob = a.checkpoint()
    used = a.tier_counts()[2]
    outs = {}
    for name, blobs, size in (("chain", chain, tb), ("full", [full], tb), ("large", chain, 4 * tb), ("small", chain, T.max_row_bytes(F) + 4096)):
        r = new_ring(g, ctx, thr)
        r.restore(ring_blob)
        r.tier_restore(size, blobs)
        outs[name] = r
    c, f, big, small = outs["chain"], outs["full"], outs["large"], outs["small"]
    assert c.tier_counts() == f.tier_counts() and held_rows(c) == held_rows(f)
    assert c.tier_counts()[:2] == a.tier_counts()[:2] and c.tier_counts()[2] == used
    # a larger tier holds every row the original held; its blob is the original's, byte for byte
    assert big.tier_counts()[:2] == a.tier_counts()[:2] and big.tier_checkpoint() == full == c.tier_checkpoint()
    # a smaller tier keeps the model's newest rows, where the model places them
    bits = np.ascontiguousarray(x).view(np.uint64)
    last = TK.header(chain[-1])
    sizes = {k: T.row_bytes(bits[:, k * ROW:(k + 1) * ROW]) for k in range(last["first"], last["next"])}
    m = TK.place(F, CAP, T.max_row_bytes(F) + 4096, last, sizes)
    assert small.tier_counts() == (m.first * ROW, m.next * ROW, m.used, m.lost)
    for k, img in held_rows(small).items():
        assert int.from_bytes(img[8:16], "little") == m.row_off[k]
    lo = a.tier_counts()[0]
    for r in (c, f, big):
        same_answers(a, r, x, thr, total, lo, 5)
    same_answers(a, small, x, thr, total, small.tier_counts()[0], 6)
    for r in (a, c, f, big, small):
        r.close()


PUSHES = [3000, 2500, 5000, 1024, 0, 6000, 4096 + 1500, 2048, 0, 7000, 3 * ROW, 5 * ROW]     # test_ring_tier_ckpt_model.scenario's


def model_ring(g, ctx):
    """the model scenario's pushes into a ring of its config, the GPU's blobs at the same points -> (ring, blobs, model blobs,
    samples [3][total], tier_bytes)"""
    bits, m, mblobs, tb = scenario(0, pushes=PUSHES)
    pushes = PUSHES
    x = bits.view(np.float64)
    r = g.Ring(ctx, 3, 4096, 100)
    r.tier_open(tb)
    blobs, pos = [], 0
    for i, n in enumerate(pushes):
        if n:
            r.push(np.ascontiguousarray(x[:, pos:pos + n].T))
        pos += n
        if i == 2:
            blobs.append(r.tier_checkpoint())
        elif i > 2:
            blobs.append(r.tier_checkpoint_delta())
    return r, blobs, mblobs, x[:, :pos], tb


def test_blobs_equal_the_model_and_refusals(env):
    g, ctx, L = env
    r, blobs, mblobs, x, tb = model_ring(g, ctx)
    assert blobs == mblobs
    total = x.shape[1]
    assert r.counts()[0] == total
    ring_blob = r.checkpoint()

    def target(cap=4096, F_=3, W_=100, n=None):
        t = g.Ring(ctx, F_, cap, W_)
        if n is None and (cap, F_, W_) == (4096, 3, 100):
            t.restore(ring_blob)
        elif n:
            t.push(np.zeros((n, F_)))
        return t

    def restore_rc(t, size, chain):
        bufs = [C.create_string_buffer(bytes(b), max(1, len(b))) for b in chain]
        ptrs = (C.c_void_p * len(chain))(*[C.addressof(b) for b in bufs])
        sizes = (C.c_int64 * len(chain))(*[len(b) for b in chain])
        return L.gpud_ring_tier_restore(t._h, size, ptrs, sizes, len(chain))

    total_m, tb_m, cases = refusal_cases()
    assert total_m == total and tb_m == tb
    b0 = blobs[0]
    flipped = bytearray(b0)
    flipped[TK.HEADER.size + T.rec_bytes(3)] ^= 1                        # the anchor of row 0's first block
    # a chain from another ring with the same pushes: its rows differ from this ring's where both hold them
    rng = np.random.default_rng(9)
    y = x.copy()
    y[0] = np.round(rng.normal(50.0, 5.0, y.shape[1]))
    o = g.Ring(ctx, 3, 4096, 100)
    o.tier_open(tb)
    pos = 0
    for i, n in enumerate(PUSHES):
        if n:
            o.push(np.ascontiguousarray(y[:, pos:pos + n].T))
        pos += n
    other_chain = [o.tier_checkpoint()]
    oh = TK.header(other_chain[0])
    whole = -(-(total - 4096) // ROW)
    table = []
    for name, kw, chain, _ in cases:
        want = TK.plan(kw.get("F", 3), kw.get("W", 100), kw.get("cap", 4096), kw.get("total", total), kw.get("tier_bytes", tb), chain)
        assert want[0] == -1, name
        table.append((name, kw, chain, want[1]))
    table += [
        ("checksum", {}, [bytes(flipped)] + blobs[1:], "tier_restore: blob 0: checksum mismatch in field 0: the blob is corrupt"),
        ("another ring", {}, other_chain, "tier_restore: rows [%d, %d) of the chain differ from the ring's samples in field 0: the chain is from another ring"
         % (max(whole, oh["first"]), oh["next"])),
    ]
    for name, kw, chain, text in table:
        n = kw.get("total")
        t = target(kw.get("cap", 4096), kw.get("F", 3), kw.get("W", 100), n)
        assert restore_rc(t, kw.get("tier_bytes", tb), chain) == -1, name
        assert last_error(g, ctx) == text, name
        with pytest.raises(g.GpudError) as e:
            t.tier_counts()
        assert e.value.code == -6, name
        if t.cap >= 2 * ROW:
            t.tier_open(tb)
        t.close()
    # a ring that already has a tier
    t = target()
    t.tier_open(tb)
    assert restore_rc(t, tb, blobs) == -6 and last_error(g, ctx) == "tier_restore: the ring already has a tier"
    t.close()
    # the chain restores, and the restored tier's blob is the original's
    t = target()
    t.tier_restore(tb, blobs)
    assert t.tier_counts() == r.tier_counts()
    assert t.tier_checkpoint() == r.tier_checkpoint()
    t.close()
    # the writers' refusals
    u = g.Ring(ctx, 3, 4096, 100)
    for call, text in ((u.tier_checkpoint, "tier_checkpoint: the ring has no tier"), (u.tier_checkpoint_delta, "tier_checkpoint_delta: the ring has no tier")):
        with pytest.raises(g.GpudError) as e:
            call()
        assert e.value.code == -6 and last_error(g, ctx) == text
    u.tier_open(tb)
    with pytest.raises(g.GpudError) as e:
        u.tier_checkpoint_delta()
    assert e.value.code == -6
    assert last_error(g, ctx) == "tier_checkpoint_delta: no tier checkpoint written or restored on this ring yet: write a full tier checkpoint"
    need = r.tier_checkpoint_bound()
    buf = (C.c_char * 64)()
    n_b = C.c_int64()
    assert L.gpud_ring_tier_checkpoint(r._h, C.cast(buf, C.c_void_p), 64, C.byref(n_b)) == -4
    assert n_b.value == need and last_error(g, ctx) == "tier_checkpoint needs %d bytes" % need
    for q in (u, r, o):
        q.close()


def test_ring_marker_and_capped_grid(env):
    """tier checkpoints and restores leave the ring's chain marker where ring checkpoints put it (the ring's deltas equal an untiered
    twin's); a codec grid of 1 or 3 CTAs writes the same tier blob and restores the same tier"""
    g, ctx, L = env
    total = 6 * CAP + 333
    rows, x, thr = data("noise", total + 5000, 7)
    tb = 6 * T.max_row_bytes(F)
    a, twin = new_ring(g, ctx, thr), new_ring(g, ctx, thr)
    a.tier_open(tb)
    for r in (a, twin):
        push(r, rows, 0, total)
    base = a.checkpoint()
    assert base == twin.checkpoint()
    chain = [a.tier_checkpoint()]
    for r in (a, twin):
        push(r, rows, total, total + 5000)
    chain.append(a.tier_checkpoint_delta())
    ring_delta = a.checkpoint_delta()
    assert ring_delta == twin.checkpoint_delta()
    empty = twin.checkpoint_delta()
    full = a.tier_checkpoint()
    outs = []
    for grid in (0, 1, 3):
        assert L.gpudh_ring_ckpt_grid(a._h, grid) == 0
        assert a.tier_checkpoint() == full
        r = new_ring(g, ctx, thr)
        assert L.gpudh_ring_ckpt_grid(r._h, grid) == 0
        r.restore(base)
        r.restore_delta(ring_delta)
        r.tier_restore(tb, chain)
        assert r.checkpoint_delta() == empty                      # the restore left the ring's marker at ring_delta
        outs.append(r)
    assert L.gpudh_ring_ckpt_grid(a._h, 0) == 0
    for r in outs:
        assert r.tier_counts() == a.tier_counts() and held_rows(r) == held_rows(outs[0])
        assert r.tier_checkpoint() == full
    same_answers(a, outs[1], x, thr, total + 5000, a.tier_counts()[0], 8)
    lo = a.tier_counts()[0]
    assert _bitwise(outs[1].reduce_ranges([lo], [total - lo]), outs[2].reduce_ranges([lo], [total - lo]))
    for r in [a, twin] + outs:
        r.close()
