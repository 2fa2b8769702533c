"""Every device buffer, pinned buffer, event and stream libgpud_b200 keeps belongs to one of the owner types of
gpud_b200/csrc/internal.h, which count the live ones (gpudh_cuda_objects).  On the GPU: every object a ctx, ring, handle, tier, box
query or call creates is gone once it is closed, and a call repeated at the same size keeps the scratch its first run grew.  On the
CPU: no raw CUDA allocation, free, create or destroy call is left outside those owner types, where it would escape the count."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gpud_b200", "csrc")
KINDS = ("device buffers", "pinned buffers", "events", "streams")

RAW = re.compile(r"\bcuda(Malloc\w*|Free\w*|EventCreate\w*|EventDestroy|StreamCreate\w*|StreamDestroy)\s*\(")
# where a raw call may stand: the owner types, and the two ABI functions whose memory belongs to the caller
ALLOWED = {"internal.h": [("class gpud_buf", "using gpud_pinned")] + [("class gpud_event", "};\n"), ("class gpud_stream", "};\n")],
           "api.cu": [('int32_t gpud_host_alloc(', "\n}\n"), ('int32_t gpud_host_free(', "\n}\n")]}


def raw_calls(name, text):
    """-> the raw CUDA resource calls of one source file that lie outside the spans it may hold them in, as (line, call)"""
    spans = []
    for start, end in ALLOWED.get(name, []):
        a = text.index(start)
        spans.append((a, text.index(end, a)))
    return [(text.count("\n", 0, m.start()) + 1, m.group(0)) for m in RAW.finditer(text)
            if not any(a <= m.start() < b for a, b in spans)]


def sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cpp", ".h", ".inc")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, f.read()


def test_no_raw_cuda_objects_outside_the_owner_types():
    found = {name: calls for name, text in sources() for calls in [raw_calls(name, text)] if calls}
    assert not found, found
    # the check sees a raw call in any file, the owner types' own file included
    for name, text in sources():
        if name.endswith(".cu"):
            assert raw_calls(name, text + "\nvoid f(void** p) { cudaMalloc(p, 8); }\n")
    head = dict(sources())["internal.h"]
    assert raw_calls("internal.h", head + "\ninline void f(cudaEvent_t e) { cudaEventDestroy(e); }\n")


@pytest.fixture(scope="module")
def env():
    import gpud_b200 as g
    L = g.lib()
    L.gpudh_cuda_objects.argtypes = [C.POINTER(C.c_int64)]
    L.gpudh_cuda_objects.restype = None

    def live():
        out = (C.c_int64 * 4)()
        L.gpudh_cuda_objects(out)
        return dict(zip(KINDS, out))
    ctx = g.Context([0])
    yield g, ctx, live
    ctx.close()


def fields(F, n, seed):
    rng = np.random.default_rng(seed)
    x = np.cumsum(rng.normal(size=(F, n)), axis=1) + rng.normal(size=(F, 1)) * 100
    return np.ascontiguousarray(x)


def push(r, x, a, b, step=20000):
    for i in range(a, b, step):
        r.push(np.ascontiguousarray(x[:, i:min(b, i + step)].T))


def box_query_to_end(g, ring, first, length, set_off):
    """one rank (n_ranks = 1): every round's all-gather is the rank's own send bytes"""
    import torch
    from gpud_b200.dist import _DevBytes
    q = g.BoxQuery(ring, 0, 1, np.zeros(len(first), dtype=np.int32), first, length, set_off)
    recv = None
    ptr, nb = q.step()
    while nb:
        recv = torch.as_tensor(_DevBytes(ptr, nb), device="cuda:0").clone()
        torch.cuda.synchronize()
        ptr, nb = q.step(recv.data_ptr())
    out = q.result()
    q.close()
    return out


@pytest.mark.gpu
def test_ctx_scans_release_everything(env):
    g, _, live = env
    before = live()
    ctx = g.Context([0])
    buf = "\n".join(synth.hit_lines()).encode()
    hits, _ = ctx.kmsg_scan(buf)
    assert hits
    dd = g.KmsgDedupDevice(ctx)
    dd.scan(buf, now_unix=1000)
    dd.close()
    ctx.ib_scan([[(1, True, 0), (2, False, 1)], [(1, False, 0)]], 1, 240, 3)
    assert live() != before
    ctx.close()
    assert live() == before


@pytest.mark.gpu
def test_ring_and_every_call_release_everything(env):
    g, ctx, live = env
    F, CAP, W = 8, 1 << 16, 100
    x = fields(F, 3 * CAP + 4321, 1)
    total = x.shape[1]
    before = live()
    r = g.Ring(ctx, F, CAP, W)
    push(r, x, 0, total)
    r.reduce_all()
    r.reduce_range(0)
    r.reduce_range(5000)
    first = np.array([total - 10, total - 3000, total - CAP, total - 50000], dtype=np.int64)
    length = np.array([7, 2500, CAP, 40000], dtype=np.int64)
    r.reduce_ranges(first, length)
    r.reduce_range_sets(first, length, np.array([0, 2, 4], dtype=np.int64))
    r.stream_open()
    hs = [r.windows(20), r.windows(20, hop=5)]                        # L = 2000 > 1024: the segment select's scratch
    push(r, x, 0, 5000)
    r.stream_reduce()
    for h in hs:
        h.reduce()
    blob = r.checkpoint()
    push(r, x, 5000, 9000)
    delta = r.checkpoint_delta()
    r2 = g.Ring(ctx, F, CAP, W)
    r2.restore(blob)
    r2.restore_delta(delta)
    r2.close()
    total += 9000
    got = box_query_to_end(g, r, np.array([total - 3000, total - 5, total - CAP], dtype=np.int64),
                           np.array([2000, 5, CAP], dtype=np.int64), np.array([0, 2, 3], dtype=np.int64))
    assert got["p99"].shape == (F, 2)
    hs[0].close()
    r.close()                                                         # hs[1] and the stream handle go with the ring
    assert live() == before


@pytest.mark.gpu
def test_tier_and_its_checkpoint_release_everything(env):
    g, ctx, live = env
    F, CAP, W = 4, 1 << 14, 100
    x = fields(F, 12 * CAP + 555, 2)
    total = x.shape[1]
    tb = 8 * F * total + (1 << 20)
    before = live()
    r = g.Ring(ctx, F, CAP, W)
    r.tier_open(tb)
    push(r, x, 0, total, step=5000)                                   # a push longer than the ring would lose tier rows
    first = np.array([total - 8 * CAP, total - 100], dtype=np.int64)
    length = np.array([CAP - 100, 50], dtype=np.int64)
    want = r.reduce_ranges(first, length)                             # the first range reaches back into the tier
    blob, tier_blob = r.checkpoint(), r.tier_checkpoint()
    r2 = g.Ring(ctx, F, CAP, W)
    r2.restore(blob)
    r2.tier_restore(tb, [tier_blob])
    assert all(np.array_equal(r2.reduce_ranges(first, length)[k], want[k]) for k in want)
    r2.close()
    r.close()
    assert live() == before


@pytest.mark.gpu
def test_repeated_calls_keep_their_scratch(env):
    g, ctx, live = env
    F, CAP, W = 8, 1 << 16, 100
    x = fields(F, 2 * CAP, 3)
    r = g.Ring(ctx, F, CAP, W)
    push(r, x, 0, 2 * CAP)
    h = r.windows(20)
    first = np.array([2 * CAP - 10, 2 * CAP - 50000], dtype=np.int64)
    length = np.array([7, 40000], dtype=np.int64)
    buf = "\n".join(synth.hit_lines()).encode()
    calls = [r.reduce_all, lambda: r.reduce_range(0), lambda: r.reduce_range(30000), lambda: r.reduce_ranges(first, length),
             lambda: r.reduce_range_sets(first, length, np.array([0, 2], dtype=np.int64)), lambda: ctx.kmsg_scan(buf)]
    for call in calls:
        call()
        after_first = live()
        for _ in range(3):
            call()
            assert live() == after_first, call
    push(r, x, 0, 4000)
    h.reduce()
    after_first = live()
    for _ in range(3):
        push(r, x, 0, 4000)
        h.reduce()
        assert live() == after_first
    r.close()
