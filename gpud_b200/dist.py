"""Host-side multi-GPU plumbing (one process per GPU, torch.distributed for rendezvous / collectives).

Only three things on this path cross GPUs (SURVEY.md §8e):
  * the whole-box NVLink/fabric view: one 128-byte record per GPU, all-gathered (NCCL over NVLink) and evaluated
    redundantly on every rank  — replaces the single-process loops of nvlink/component.go:164-311 and
    fabric-manager/fabric_state.go:67-113;
  * an optional split of one large kmsg buffer across ranks at unit boundaries, hits concatenated in unit order;
  * box range sets (box_range_sets): a fixed header per rank, the results of the sets one rank's ring holds, and for a set spread over
    several ranks only small objects: the samples of a short one, or for a long one its pivot sample, the per-rank class counts and
    EMA partials, the keys between the pivots and, for the rare segment the pivots miss, digit histograms and the last candidates.
Ring data is never exchanged: every GPU reduces its own counter stream.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple


def split_at_units(buf: bytes, world: int, raw_kmsg: bool = False) -> List[Tuple[int, int]]:
    """Byte ranges [b, e) for `world` ranks, cut just after a unit separator ('\\n'; in RAW_KMSG mode a '\\n' that is not
    followed by ' ', so a record and its continuation lines stay together).  Every range except the last ends with its
    separator, so the ranks' unit counts add up exactly: units(whole) = sum(units(part_i) - 1) + 1."""
    n = len(buf)
    cuts = [0]
    for r in range(1, world):
        pos = max(cuts[-1], (n * r) // world)
        while True:
            nl = buf.find(b"\n", pos)
            if nl < 0:
                pos = n
                break
            pos = nl + 1
            if not raw_kmsg or pos >= n or buf[pos:pos + 1] != b" ":
                break
        cuts.append(pos)
    cuts.append(n)
    return [(cuts[i], cuts[i + 1]) for i in range(world)]


def merge_hits(parts: Sequence[Tuple[int, int, list]]):
    """parts[i] = (byte_offset_of_part, n_units_in_part, hits) with hits as dicts carrying 'line' and 'offset' relative to
    the part.  Returns (hits with global line/offset, n_units_total)."""
    out, line0 = [], 0
    for i, (off, n_units, hits) in enumerate(parts):
        for h in hits:
            g = dict(h)
            g["line"] = h["line"] + line0
            g["offset"] = h["offset"] + off
            out.append(g)
        # a part that ends with its separator counts one trailing empty unit that really belongs to the next part
        line0 += n_units - 1 if i + 1 < len(parts) else n_units
    return out, line0


def gather_fabric(ctx, raw, at_least: int = 0, group=None, device=None):
    """pack kernel -> all_gather_into_tensor (NCCL) -> verdict kernel, one process per GPU.  Returns FabricVerdict."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    send = torch.zeros(128, dtype=torch.uint8, device=dev)
    table = torch.zeros(128 * world, dtype=torch.uint8, device=dev)
    # the library treats a NULL stream as "use my own": give it a real stream so kernels and the collective are ordered
    cur = torch.cuda.current_stream(dev)
    side = cur if cur.cuda_stream != 0 else torch.cuda.Stream(device=dev)
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        ctx.fabric_pack(raw, send.data_ptr(), dev=dev.index, stream=side.cuda_stream)   # K7 writes straight into the send buffer
        dist.all_gather_into_tensor(table, send, group=group)
        v = ctx.fabric_verdict(table.data_ptr(), world, at_least, dev=dev.index, stream=side.cuda_stream)
    cur.wait_stream(side)
    return v


class _DevBytes:
    """a zero-copy uint8 view of library-owned device memory for torch.as_tensor"""

    def __init__(self, ptr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def box_range_sets(ring, rank_of, first, length, set_off, group=None, fields=None) -> dict:
    """Range sets over the rings of every rank of the group, this process holding ring `rank` (gpud_box_query, DESIGN.md §2 "Box sets
    across processes"): every rank calls this with the same arguments and gets the same {op: [F][n_sets]} result, identical to
    capi.rings_reduce_range_sets over all the rings in one process.  With a list of fields (the same on every rank), only those are
    read and exchanged, and row g is field fields[g]: {op: [len(fields)][n_sets]}.  NCCL all-gathers device buffers; any other
    backend (gloo) stages through host memory."""
    import torch
    import torch.distributed as dist
    from .capi import BoxQuery
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    dev = torch.device("cuda", ring.dev)
    nccl = dist.get_backend(group) == "nccl"
    q = BoxQuery(ring, rank, world, rank_of, first, length, set_off, fields=fields)
    try:
        send_ptr, nb = q.step()
        while nb:
            send = torch.as_tensor(_DevBytes(send_ptr, nb), device=dev)
            if nccl:
                recv = torch.empty(world * nb, dtype=torch.uint8, device=dev)
                dist.all_gather_into_tensor(recv, send, group=group)
            else:
                host = torch.empty(world * nb, dtype=torch.uint8)
                dist.all_gather_into_tensor(host, send.cpu(), group=group)
                recv = host.to(dev)
            torch.cuda.synchronize(dev)          # the library reads recv on the ring's own stream
            send_ptr, nb = q.step(recv.data_ptr())
        return q.result()
    finally:
        q.close()
