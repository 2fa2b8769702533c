"""Host model of a range call over several rings that reaches into their tiers (DESIGN.md §2 "Tier", "Box sets"): which sets go to the
virtual box, and its layout.  Ring k of the call has pushed totals[k] samples into capacity cap and, tiered, a tier that holds block rows
[t_first, t_next) (tiers[k] = (t_first, t_next), or None for an untiered ring).  A tiered ring's ranges may start at
lo_k = min(total_k - count_k, 1024 t_first); an untiered ring's at total_k - count_k."""
ROW = 1024


def reach(total, cap, tier):
    """lo_k: the first sample a range of this ring may start at"""
    held = total - min(total, cap)
    return held if tier is None else min(held, tier[0] * ROW)


def split(totals, cap, tiers, ring_of, first, length, set_off=None):
    """-> (route [n_sets], slots [(ring, rows, dec, vtotal)], vslot [n], vfirst [n], vcap), or None when the call is refused.
    A set goes to the box (route 1) when one of its ranges starts before its ring's first sample.  Per ring its box sets touch, in
    ring order, one slot: the block rows those sets' ranges cover, merged and ascending, each decoded from the ring's tier (dec 1) when
    the tier holds it, else copied from the ring (dec 0); row j of the slot at virtual columns [1024 j, 1024 (j + 1)).  vtotal: the
    slot's samples (its newest row may be partial).  vcap: the largest slot's rows x 1024."""
    first, length = list(first), list(length)
    n = len(first)
    ring_of = [0] * n if ring_of is None else list(ring_of)
    nr = len(totals)
    for i in range(n):
        k = ring_of[i]
        if not 0 <= k < nr:
            return None
        if length[i] < 1 or first[i] < reach(totals[k], cap, tiers[k]) or first[i] + length[i] > totals[k]:
            return None
    sets = [(s, s + 1) for s in range(n)] if set_off is None else list(zip(set_off[:-1], set_off[1:]))
    if set_off is not None and (set_off[0] != 0 or set_off[-1] != n or any(b <= a for a, b in sets)):
        return None
    held = [t - min(t, cap) for t in totals]
    route = [int(any(first[i] < held[ring_of[i]] for i in range(a, b))) for a, b in sets]
    need = [set() for _ in range(nr)]
    for (a, b), r in zip(sets, route):
        for i in range(a, b) if r else ():
            need[ring_of[i]].update(range(first[i] // ROW, -(-(first[i] + length[i]) // ROW)))
    slots, slot_of = [], {}
    for k in range(nr):
        if not need[k]:
            continue
        rows = sorted(need[k])
        tier = tiers[k]
        dec = [int(tier is not None and tier[0] <= row < tier[1]) for row in rows]
        vtotal = (len(rows) - 1) * ROW + min(ROW, totals[k] - rows[-1] * ROW)
        slot_of[k] = len(slots)
        slots.append((k, rows, dec, vtotal))
    vslot, vfirst = [-1] * n, [-1] * n
    for (a, b), r in zip(sets, route):
        for i in range(a, b) if r else ():
            v = slot_of[ring_of[i]]
            vslot[i] = v
            vfirst[i] = slots[v][1].index(first[i] // ROW) * ROW + first[i] % ROW
    vcap = max((len(s[1]) for s in slots), default=0) * ROW
    return route, slots, vslot, vfirst, vcap

