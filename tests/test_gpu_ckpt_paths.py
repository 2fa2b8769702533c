"""The checkpoint codec route by route on the GPU (k_ckpt_size, k_ckpt_pack and k_ckpt_unpack of csrc/ring_ckpt.cu): every field
of a test ring carries one aimed block of ckpt_cases.py, and every case is checked four ways: the checkpoint (or delta) bytes equal
the host model's (ring_checkpoint.py / ring_delta.py) byte for byte, the restored ring equals the original bit for bit (physical
ring and sample ring), checkpoint_stats reports the model's RAW / INT block counts, and the restored ring checkpoints to the same
bytes again.  Each family runs at the default grid and with the codec grid capped at 1 and 3 CTAs (gpudh_ring_ckpt_grid), where
every warp codes, packs and unpacks many blocks of mixed modes and widths in turn.  Corruptions that keep every length consistent
are accepted exactly when the model decodes them to the same samples, and refused as a checksum mismatch otherwise, leaving the
ring (and, for a delta, its handles and chain marker) as it was.  Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import ckpt_cases as K
import ring_checkpoint as RC
import ring_delta as RD
from test_gpu_ring_checkpoint import Cfg, handle_state, last_error, same, same_handles, snapshot
from test_gpu_ring_delta import model_delta, raw_apply

pytestmark = pytest.mark.gpu

E_INVALID = -1
GRIDS = (0, 1, 3)          # the codec grid: the default, and capped at 1 and 3 CTAs


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    ctx = g.Context([0])
    L = g.lib()
    L.gpudh_ring_snapshot.restype = C.c_int32
    L.gpudh_ring_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
    yield g, ctx, L
    ctx.close()


# ------------------------------------------------------------------------------------------------ helpers
def new_ring(env, cfg, grid):
    g, ctx, L = env
    r = cfg.ring(g, ctx)
    assert L.gpudh_ring_ckpt_grid(r._h, grid) == 0
    return r


def push_cols(ring, cols, total):
    """a ring whose chronological samples are cols [F][count] after `total` pushes: filler rows first, then the columns"""
    F, count = cols.shape
    if total > count:
        ring.push(np.zeros((total - count, F)))
    ring.push(np.ascontiguousarray(cols.T).view(np.float64))


def blocks(blob, model):
    d = model.decode(blob)["dir"]
    return {"raw": int((d >> 7 == 0).sum()), "int": int((d >> 7 == 1).sum())}


def checked_full(env, cfg, grid, cols, total):
    """push the columns, checkpoint, and check the four ways; -> (ring, blob)"""
    g, ctx, L = env
    ring = new_ring(env, cfg, grid)
    push_cols(ring, cols, total)
    rb, sb = snapshot(L, ring)
    same(RC.chronological(rb, total, cfg.cap), cols, "pushed")
    blob = ring.checkpoint()
    assert blob == RC.encode(cols, total, cfg.model()), "checkpoint bytes differ from the model's"
    assert ring.checkpoint_stats()[2] == blocks(blob, RC)
    r2 = new_ring(env, cfg, grid)
    assert r2.restore(blob) == []
    x = snapshot(L, r2)
    same(x[0], rb, "ring")
    same(x[1], sb, "sample ring")
    assert r2.checkpoint_stats()[2] == blocks(blob, RC)
    assert r2.checkpoint() == blob
    r2.close()
    return ring, blob


def untouched(L, ring):
    assert ring.counts() == (0, 0, 0)
    rb, sb = snapshot(L, ring)
    assert not rb.any() and not sb.any()


# ------------------------------------------------------------------------------------------------ a. modes and widths
@pytest.mark.parametrize("grid", GRIDS)
def test_mode_width_matrix(env, grid):
    cases = K.width_matrix()
    cols = K.fields(K.BLOCK, cases)
    ring, _ = checked_full(env, Cfg(len(cases), K.BLOCK, 1), grid, cols, K.BLOCK)
    ring.close()


# ------------------------------------------------------------------------------------------------ b. tails and positions
@pytest.mark.parametrize("grid", GRIDS)
def test_tails_positions_straddles(env, grid):
    """per tail length n, one ring whose fields are a full block and then a tail case of n samples: every aimed position of the
    widest residual, every straddle class of the last one, and the eligibility edges at n = 1, 33 and 1024"""
    for n in K.TAILS:
        cases = K.tail_cases(n) + (K.edge_cases(n) if n in (1, 33, K.BLOCK) else [])
        count = K.BLOCK + n
        cap = count + count % 2
        ring, _ = checked_full(env, Cfg(len(cases), cap, 1), grid, K.fields(count, cases, seed=n, at=1), count)
        ring.close()
        # and the same cases as the only block of a ring of n samples
        ring, _ = checked_full(env, Cfg(len(cases), n + n % 2, 1), grid, K.fields(n, cases, seed=n), n)
        ring.close()


# ------------------------------------------------------------------------------------------------ c. wraps
def wraps():
    """(CAP, total, block, t): the physical end falls just before sample t of that block of the checkpoint's samples"""
    out = []
    for cap, spots in ((2, [(0, 1)]), (30, [(0, 1), (0, 29)]), (34, [(0, t) for t in (1, 31, 32, 33)]),
                       (1022, [(0, t) for t in (1, 31, 32, 33)]), (1026, [(0, t) for t in (1, 31, 32, 33, 1023)] + [(1, 1)]),
                       (8192, [(3, 33), (7, 1023)]), (16382, [(5, 1023), (15, 1)]), (16386, [(2, 32), (16, 1)]), (40002, [(9, 31)])):
        for b, t in spots:
            start = cap - (K.BLOCK * b + t)
            out.append((cap, cap + start, b, t))
    return out


@pytest.mark.parametrize("grid", GRIDS)
def test_wraps(env, grid):
    """CAP < 1024, CAP = 2 (mod 4), sample rings at smp_shift 0, 1, 2 and 3: restore writes both across the physical end"""
    g, ctx, L = env
    shifts = set()
    for cap, total, b, t in wraps():
        n = min(K.BLOCK, cap - b * K.BLOCK)
        cases = K.wrap_cases(n, t)
        ring, _ = checked_full(env, Cfg(len(cases), cap, 1), grid, K.fields(cap, cases, seed=t, at=b), total)
        s = C.c_int32()
        L.gpudh_ring_snapshot(ring._h, None, None, C.byref(s), None)
        shifts.add(s.value)
        ring.close()
    assert shifts == {0, 1, 2, 3}


# ------------------------------------------------------------------------------------------------ d. deltas
DELTAS = [  # CAP, marker total, rows pushed after it, block of the run the cases go to
    (4096, 3039, 2049, 1),        # the run crosses the physical end before sample 33 of its block 1
    (2050, 1000, 3000, 0),        # more than CAP since the marker: first_d = total - CAP, the end before sample 100 of block 0
    (1026, 500, 1025, 0),         # a run of 1024 + 1 whose end falls before sample 526
    (34, 17, 34, 0),              # a whole ring of 34 from sample 17 on
]


@pytest.mark.parametrize("grid", GRIDS)
def test_deltas(env, grid):
    """first_d cuts the blocks off the multiples of 1024 of the push order, and runs cross the physical end; a second delta in
    the chain follows the first"""
    g, ctx, L = env
    for cap, m, pushed, b in DELTAS:
        total = m + pushed
        count = total - RD.first_d(m, total, cap)
        n = min(K.BLOCK, count - b * K.BLOCK)
        t = (cap - RD.first_d(m, total, cap) % cap) % K.BLOCK
        cases = K.wrap_cases(n, min(max(t, 1), n - 1) if n > 1 else 1)
        F = len(cases)
        cfg = Cfg(F, cap, 1)
        cols = K.fields(count, cases, seed=m, at=b)
        ring = new_ring(env, cfg, grid)
        ring.push(np.random.default_rng(m).integers(-5, 5, (m, F)).astype(np.float64))
        base = ring.checkpoint()
        push_cols(ring, cols, pushed)
        d1 = ring.checkpoint_delta()
        assert d1 == model_delta(L, ring, m, RD.full_link(base)), (cap, m)
        same(RD.decode(d1)["samples"], cols, "delta samples")
        assert ring.checkpoint_stats()[2] == blocks(d1, RD)
        # a second delta: 1500 more samples from where the first left off
        more = K.fields(1500, [K.mixed(K.BLOCK, i) for i in range(F)], seed=cap)
        push_cols(ring, more, 1500)
        d2 = ring.checkpoint_delta()
        assert d2 == model_delta(L, ring, total, RD.decode(d1)["link"])
        r2 = new_ring(env, cfg, grid)
        r2.restore(base)
        r2.restore_delta(d1)
        assert r2.checkpoint_stats()[2] == blocks(d1, RD)
        r2.restore_delta(d2)
        assert r2.counts() == ring.counts()
        x, y = snapshot(L, ring), snapshot(L, r2)
        same(x[0], y[0], "ring")
        same(x[1], y[1], "sample ring")
        assert r2.checkpoint() == ring.checkpoint()
        r2.close()
        ring.close()


def delta_families():
    """the width matrix, tails with every aimed position and straddle class, and the eligibility edges, each family as block 1 of
    a run of 1024 + n samples"""
    out = [K.width_matrix()]
    for n in (1, 2, 31, 33, 65, 513, K.BLOCK):
        out.append(K.tail_cases(n) + (K.edge_cases(n) if n in (1, 33, K.BLOCK) else []))
    return out


@pytest.mark.parametrize("grid", GRIDS)
def test_families_through_deltas(env, grid):
    """every family of a-b as a delta of CAP 4096: the marker puts first_d off the multiples of 1024, and the run crosses the
    physical end just after its middle sample"""
    g, ctx, L = env
    cap = 4096
    for cases in delta_families():
        n = cases[0]["n"]
        count = K.BLOCK + n
        m = cap - count // 2 - 1
        assert m % K.BLOCK and m + count > cap
        F = len(cases)
        cfg = Cfg(F, cap, 1)
        cols = K.fields(count, cases, seed=n, at=1)
        ring = new_ring(env, cfg, grid)
        ring.push(np.random.default_rng(n).integers(-5, 5, (m, F)).astype(np.float64))
        base = ring.checkpoint()
        push_cols(ring, cols, count)
        delta = ring.checkpoint_delta()
        assert delta == model_delta(L, ring, m, RD.full_link(base)), n
        same(RD.decode(delta)["samples"], cols, "delta samples")
        assert ring.checkpoint_stats()[2] == blocks(delta, RD)
        r2 = new_ring(env, cfg, grid)
        r2.restore(base)
        r2.restore_delta(delta)
        assert r2.checkpoint_stats()[2] == blocks(delta, RD)
        x, y = snapshot(L, ring), snapshot(L, r2)
        same(x[0], y[0], "ring")
        same(x[1], y[1], "sample ring")
        assert r2.checkpoint() == ring.checkpoint()
        r2.close()
        ring.close()


# ------------------------------------------------------------------------------------------------ e. more blocks than warps
def test_more_blocks_than_warps_at_the_default_grid(env):
    """F x nb above 16 CTAs x 8 warps per SM: at the default grid every warp of all three kernels codes more than one block"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cases = K.width_matrix()[::9][:32]
    F = len(cases)
    nb = 16 * sms * 8 // F + 2
    count = (nb - 1) * K.BLOCK + 513
    assert F * nb > 16 * sms * 8
    ring, _ = checked_full(env, Cfg(F, count + 1, 1), 0, K.fields(count, cases, seed=1), count)
    ring.close()


# ------------------------------------------------------------------------------------------------ f. corruptions
def expect_outcome(env, rc, edited, cols, what):
    g, ctx, L = env
    if K.accepted(edited, cols):
        assert rc == 0, (what, last_error(g, ctx))
        return True
    assert rc == E_INVALID and "checksum" in last_error(g, ctx), (what, rc, last_error(g, ctx))
    return False


def raw_restore(L, ring, blob):
    buf = (C.c_char * len(blob)).from_buffer_copy(blob)
    hs = (C.c_void_p * 1)()
    n = C.c_int32()
    return L.gpud_ring_restore(ring._h, C.cast(buf, C.c_void_p), len(blob), hs, 1, C.byref(n))


@pytest.mark.parametrize("grid", GRIDS)
def test_corrupt_full(env, grid):
    g, ctx, L = env
    cols, aimed, swaps, flips, widths = K.corruption_fields()
    wcols = K.wrap_fields()
    for cfg, cols, total, edits in ((Cfg(6, 4096, 1), cols, cols.shape[1], lambda b: K.corruptions(b, aimed, swaps, flips, widths)),
                                    (Cfg(2, 1026, 1), wcols, 2019, lambda b: K.corruptions(b, {"wrap INT": (0, 0), "wrap RAW": (1, 0)},
                                                                                         [((0, 1), (1, 1))]))):
        ring, blob = checked_full(env, cfg, grid, cols, total)
        want = snapshot(L, ring)
        n_ok = 0
        for what, e in edits(blob).items():
            r = new_ring(env, cfg, grid)
            if expect_outcome(env, raw_restore(L, r, e), e, cols, what):
                n_ok += 1
                x = snapshot(L, r)
                same(x[0], want[0], what)
                same(x[1], want[1], what)
            else:
                untouched(L, r)
            r.close()
        assert n_ok >= (2 if cfg.F == 6 else 0)        # the zero block's mode bit and RAW w=1's padding bit
        ring.close()


@pytest.mark.parametrize("grid", GRIDS)
def test_corrupt_delta(env, grid):
    """a refused delta leaves the ring, the sample ring, every handle's reads and counts and the chain marker as they were: the
    genuine delta still applies afterwards and gives the original"""
    g, ctx, L = env
    cols, aimed, swaps, flips, widths = K.corruption_fields()
    F, count = cols.shape
    cfg = Cfg(F, 4096, 8)
    src = new_ring(env, cfg, grid)
    src.push(np.random.default_rng(3).integers(0, 100, (3000, F)).astype(np.float64))
    src.stream_open(0)
    w = src.windows(2)
    src.stream_reduce()
    w.reduce()
    base = src.checkpoint()
    push_cols(src, cols, count)
    src.stream_reduce()
    w.reduce()
    delta = src.checkpoint_delta()
    same(RD.decode(delta)["samples"], cols, "delta samples")
    want = snapshot(L, src)
    want_handles = handle_state(src, [w])
    want_blob = src.checkpoint()
    edits = K.corruptions(delta, dict(aimed, **{"wrap block": (2, 1)}), swaps, flips, widths)
    for what, e in edits.items():
        r = new_ring(env, cfg, grid)
        hs = r.restore(base)
        before, before_handles = snapshot(L, r), handle_state(r, hs)
        if not expect_outcome(env, raw_apply(L, r, e), e, cols, what):
            x = snapshot(L, r)
            same(x[0], before[0], what)
            same(x[1], before[1], what)
            same_handles(handle_state(r, hs), before_handles)
            r.restore_delta(delta)                      # the marker did not move
        x = snapshot(L, r)
        same(x[0], want[0], what)
        same(x[1], want[1], what)
        same_handles(handle_state(r, hs), want_handles)
        assert r.checkpoint() == want_blob, what
        r.close()
    src.close()


# ------------------------------------------------------------------------------------------------ g. staging pieces
STAGE_BYTES = 32 << 20     # the ring's pinned staging pieces: stage_rows x F x 8 bytes


@pytest.mark.parametrize("F,count", [(64, 65536), (64, 65537), (1, (4 << 20) - 1), (1, 4 << 20), (1, (4 << 20) + 1)])
def test_staging_boundaries(env, F, count):
    """random bit patterns: every block RAW w = 64, the payload exactly 8 F count bytes, one staging piece, a piece and 512 B, or
    a piece and 8 B either side; checkpoint, restore, delta and delta apply through pageable, pinned and odd-address pinned memory"""
    g, ctx, L = env
    assert (STAGE_BYTES // (8 * F)) * 8 * F == STAGE_BYTES
    cap = count + count % 2
    cfg = Cfg(F, cap, 1)
    bits = np.random.default_rng(count + F).integers(0, 2 ** 64, size=(F, count), dtype=np.uint64, endpoint=False)
    rows = np.ascontiguousarray(bits.T).view(np.float64)
    src = [new_ring(env, cfg, 0) for _ in range(2)]
    base = [r.checkpoint() for r in src]                # empty: the deltas hold every sample
    assert base[0] == base[1]
    for r in src:
        r.push(rows)
    want = snapshot(L, src[0])
    full = RC.encode(bits, count, cfg.model())
    hd = RC.header(full)
    assert hd["payload_bytes"] == 8 * F * count and hd["payload_bytes"] - STAGE_BYTES in (-8, 0, 8, 512)
    bufs = []
    try:
        for size, odd in ((len(full) + 16, False), (RD.bound(F, count, 0) + 16, True)):
            p = C.c_void_p()
            assert L.gpud_host_alloc(size, C.byref(p)) == 0
            bufs.append(p)
        pin_full = np.frombuffer((C.c_char * len(full)).from_address(bufs[0].value), dtype=np.uint8)
        assert src[0].checkpoint() == full                                 # pageable
        assert src[0].checkpoint_stats()[2] == blocks(full, RC) == {"raw": F * -(-count // K.BLOCK), "int": 0}
        assert src[0].checkpoint(out=pin_full) == len(full) and pin_full.tobytes() == full
        for blob in (full, pin_full):
            r = new_ring(env, cfg, 0)
            r.restore(blob)
            x = snapshot(L, r)
            same(x[0], want[0], "ring")
            same(x[1], want[1], "sample ring")
            r.close()
        # deltas: src[1] still has its marker at the empty base
        d_page = src[1].checkpoint_delta()
        assert d_page == model_delta(L, src[1], 0, RD.full_link(base[1]))
        r = new_ring(env, cfg, 0)
        r.restore(base[0])
        r.push(rows)
        room = RD.bound(F, count, 0)
        pin_odd = np.frombuffer((C.c_char * room).from_address(bufs[1].value + 1), dtype=np.uint8)
        n = r.checkpoint_delta(out=pin_odd)
        assert pin_odd[:n].tobytes() == d_page
        r.close()
        for blob in (d_page, pin_odd[:n]):
            r = new_ring(env, cfg, 0)
            r.restore(base[0])
            r.restore_delta(blob)
            x = snapshot(L, r)
            same(x[0], want[0], "ring")
            same(x[1], want[1], "sample ring")
            r.close()
    finally:
        for p in bufs:
            L.gpud_host_free(p)
        for r in src:
            r.close()
