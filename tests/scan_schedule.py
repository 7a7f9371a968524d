"""Exact host restatement of how the persistent scan kernels walk a shard (test infrastructure).

k_scan_pw (minivite_b200/csrc/scan_pipe.cuh) and k_scan_pq (scan_queue.cuh) give every warp the 32-vertex groups
g, g + gstride, g + 2 gstride, ... (g = its global warp index, gstride = 8 x the CTAs of the grid).  Per group the
kernels decide, from the row offsets alone, whether the prefetched edge block covers the whole group, which lanes are
left to k_scan_heavy, and how the rest is cut into sub-ranges that each fit one staging buffer (with a synchronous
bulk copy when the prefetched block does not cover one).  k_scan_pq additionally bounds every vertex's best gain,
parks the vertices that may move in a 64-slot per-warp ring and drains it 32 at a time.

This module restates those rules line by line, in the kernels' integer and fp64 arithmetic, for a CSR in the kernels'
own vertex numbering (reorder = 0 keeps the caller's), so that a test can say exactly which boundary each group of an
engineered graph lands on, and assert that it lands there.  It never runs a kernel.
"""
from collections import Counter

import numpy as np

MV_WCAP_UNIT = 512          # edges per staging buffer, unit weights (scan_pipe.cuh)
MV_WCAP_W = 320             # ... weighted (4-byte tail + 8-byte weight per edge)
MV_Q_ENT = 12               # leftover communities one ring slot holds (scan_queue.cuh)
MV_Q_SLOTS = 64             # ring slots per warp
MV_Q_DRAIN = 32             # parked vertices that trigger a pass-1 round
PW_WARPS = 8                # warps per CTA
K_ECAP = 2048               # edges per sub-range of k_scan_ws (kernels.cuh, scan_variant 3)
K_TILE_V = 128              # vertices per tile of k_scan_ws


def cap_of(unit):
    return MV_WCAP_UNIT if unit else MV_WCAP_W


def heavy_deg_of(variant, unit, force_heavy_deg=0):
    """heavy_launch (mvgpu.cu): one staging buffer minus the 16-byte alignment slack for the persistent kernels, kECap
    for k_scan_ws; force_heavy_deg > 0 can only lower it."""
    tile_cap = cap_of(unit) - 4 if variant >= 4 else K_ECAP
    return min(force_heavy_deg, tile_cap) if force_heavy_deg > 0 else tile_cap


def heavy_info(rowptr, heavy_deg):
    """(nheavy, maxdeg) as shard_info() reports them: vertices above heavy_deg, counted only when the maximum is."""
    deg = np.diff(np.asarray(rowptr, np.int64))
    maxdeg = int(deg.max()) if deg.size else 0
    return (int((deg > heavy_deg).sum()) if maxdeg > heavy_deg else 0), maxdeg


def heavy_table_size(d):
    """Hash-table entries k_scan_heavy gives a vertex of degree d (heavy_finish)."""
    t = 64
    while t < 2 * d:
        t <<= 1
    return t


def warp_groups(ngroups, ctas):
    """Groups of each warp of a grid of `ctas` CTAs, clipped to the grid launch_scan_t starts."""
    grid = min((ngroups + PW_WARPS - 1) // PW_WARPS, ctas)
    gstride = grid * PW_WARPS
    return [list(range(w, ngroups, gstride)) for w in range(gstride)]


def extent(rowptr, g, cap):
    """The prefetched edge block of group g: [lo4, lo4 + n4), widened to 16 bytes, clipped to one buffer."""
    lnv = len(rowptr) - 1
    nv = min(32, lnv - 32 * g)
    e0, e1 = int(rowptr[32 * g]), int(rowptr[32 * g + nv])
    lo4 = e0 & ~3
    n4 = min(cap, (e1 - lo4 + 3) & ~3) if e1 > lo4 else 0
    return lo4, n4


def group_plan(rowptr, g, cap, heavy_deg, has_heavy):
    """One group's schedule: nvalid, lo4 / n4, whole, heavy lanes, and every sub-range as a dict
    {start, end, a_sub, e_lo, e_end, sync, copy_n, stop} (stop: 'cap', 'heavy' or None when end == nvalid / 32)."""
    lnv = len(rowptr) - 1
    nvalid = min(32, lnv - 32 * g)
    ra = [int(rowptr[32 * g + l]) for l in range(nvalid)]
    rb = [int(rowptr[32 * g + l + 1]) for l in range(nvalid)]
    deg = [b - a for a, b in zip(ra, rb)]
    heavy = [has_heavy and d > heavy_deg for d in deg]
    lo4, n4 = extent(rowptr, g, cap)
    have_lo, have_n = lo4, n4
    g_e0, g_e1 = int(rowptr[32 * g]), int(rowptr[32 * g + nvalid])
    whole = (not has_heavy) and (g_e1 - have_lo) <= have_n
    subs, skipped = [], []
    if whole:
        subs.append({"start": 0, "end": nvalid, "a_sub": lo4, "e_lo": g_e0, "e_end": g_e1, "sync": False, "copy_n": 0,
                     "stop": None})
    else:
        start = 0
        while start < nvalid:
            if heavy[start]:
                skipped.append(start)
                start += 1
                continue
            e_lo = ra[start]
            a_sub = e_lo & ~3
            # the start vertex always fits: deg + (ra mod 4) <= CAP for every non-heavy vertex (heavy_deg <= CAP - 4)
            assert rb[start] - a_sub <= cap, ("start vertex does not fit", g, start, deg[start], ra[start] % 4, cap)
            end = start
            while end < 32 and end < nvalid and not heavy[end] and rb[end] - a_sub <= cap:
                end += 1
            assert end > start
            stop = None if end >= nvalid else ("heavy" if heavy[end] else "cap")
            e_end = rb[end - 1]
            sync = not (a_sub >= have_lo and e_end <= have_lo + have_n)
            copy_n = 0
            if sync:
                have_lo, have_n = a_sub, (e_end - a_sub + 3) & ~3
                assert have_n <= cap
                copy_n = have_n
            subs.append({"start": start, "end": end, "a_sub": a_sub, "e_lo": e_lo, "e_end": e_end, "sync": sync,
                         "copy_n": copy_n, "stop": stop})
            start = end
    return {"g": g, "nvalid": nvalid, "lo4": lo4, "n4": n4, "whole": whole, "heavy": skipped, "subs": subs,
            "deg": deg, "ra": ra, "e0": g_e0, "e1": g_e1}


def schedule(rowptr, cap, heavy_deg, ctas):
    """Per warp, the plans of its groups in the order the warp takes them."""
    rowptr = np.asarray(rowptr, np.int64)
    lnv = len(rowptr) - 1
    ngroups = (lnv + 31) // 32
    nheavy, _ = heavy_info(rowptr, heavy_deg)
    has_heavy = nheavy > 0
    plans = [group_plan(rowptr, g, cap, heavy_deg, has_heavy) for g in range(ngroups)]
    return [[plans[g] for g in gs] for gs in warp_groups(ngroups, ctas)], plans


def pair_coverage(kind_of_group, ngroups, ctas):
    """Ordered pairs (kind of group k, kind of group k + 1) that some warp meets, with their counts."""
    c = Counter()
    for gs in warp_groups(ngroups, ctas):
        for a, b in zip(gs, gs[1:]):
            c[(kind_of_group[a], kind_of_group[b])] += 1
    return c


# ---- k_scan_pq: the gain bound, the ring and its drains ----------------------------------------------------------------
def community_state(rowptr, tails, X):
    """Community degrees and sizes of assignment X (unit weights), indexed by community id."""
    deg = np.diff(np.asarray(rowptr, np.int64))
    n = len(X)
    cdeg = np.bincount(X, weights=deg, minlength=n).astype(np.int64)
    csize = np.bincount(X, minlength=n).astype(np.int64)
    return cdeg, csize


def gain_of(eiy, eix, vdeg, ay, ax, c):
    """kernels.cuh gain_of in fp64, one rounding per operation (Python floats are IEEE doubles, no contraction)."""
    de, da = eiy - eix, ay - ax
    return 2.0 * de - ((2.0 * vdeg) * da) * c


def vertex_pq(v, rowptr, tails, X, cdeg, csize, c, movable=None):
    """k_scan_pq's view of vertex v: m (leftover edges), eix, ax, the gain bound, hard, and the pass-1 decision over
    the candidate communities (best gain, best community, whether the best gain is shared)."""
    a, b = int(rowptr[v]), int(rowptr[v + 1])
    d = b - a
    cc = int(X[v])
    nb = X[tails[a:b]]
    sl = int(np.count_nonzero(tails[a:b] == v))
    m = int(np.count_nonzero(nb != cc))
    eix = float(d - m) - float(sl)
    ax = float(int(cdeg[cc])) - float(d)
    gB = ((2.0 * float(d)) * ax) * c
    bound = 2.0 * (float(m) - eix) + gB
    hard = m > 0 and not (bound <= 0.0) and (movable is None or bool(movable[v]))
    out = {"v": v, "d": d, "m": m, "cc": cc, "eix": eix, "ax": ax, "bound": bound, "hard": hard,
           "best": cc, "best_gain": 0.0, "tie": False}
    if hard:
        ys, cnt = np.unique(nb[nb != cc], return_counts=True)
        best, bg, tie = cc, 0.0, False
        for y, k in zip(ys.tolist(), cnt.tolist()):
            g = gain_of(float(k), eix, float(d), float(int(cdeg[y])), ax, c)
            if g > bg:
                best, bg, tie = y, g, False
            elif g == bg and g != 0.0:
                tie = True
                best = min(best, y)
        if best != cc and best > cc and csize[cc] == 1 and csize[best] == 1:   # singleton veto
            best = cc
        out.update(best=best, best_gain=bg, tie=tie)
    return out


def pq_schedule(rowptr, tails, X, c, ctas, movable=None, heavy_deg=MV_WCAP_UNIT - 4):
    """k_scan_pq over a unit-weight shard with assignment X: per warp, per group, per sub-range whether it ran pass 1
    in place or parked its hard vertices (ring slots), the ring occupancy around every group and every drain
    (size, qhead); plus per vertex the vertex_pq record of every non-heavy vertex with edges."""
    rowptr = np.asarray(rowptr, np.int64)
    tails = np.asarray(tails, np.int64)
    X = np.asarray(X, np.int64)
    cdeg, csize = community_state(rowptr, tails, X)
    warps, _plans = schedule(rowptr, MV_WCAP_UNIT, heavy_deg, ctas)
    verts = {}
    out = []
    for gs in warps:
        qhead, qcount = 0, 0
        recs = []
        for plan in gs:
            rec = {"g": plan["g"], "occ_before": qcount, "subs": [], "drains": []}
            base = 32 * plan["g"]
            for s in plan["subs"]:
                vs = [vertex_pq(base + l, rowptr, tails, X, cdeg, csize, c, movable) for l in range(s["start"], s["end"])]
                for r in vs:
                    if r["d"]:
                        verts[r["v"]] = r
                hard = [r for r in vs if r["hard"]]
                in_place = any(r["m"] > MV_Q_ENT for r in hard)
                slots = []
                if not in_place:
                    for i, r in enumerate(hard):
                        assert r["m"] <= MV_Q_ENT and r["m"] < (1 << 16) and r["d"] < (1 << 15)   # m | d << 16 fits an int
                        slots.append((qhead + qcount + i) % MV_Q_SLOTS)
                        r["parked"] = True
                    qcount += len(hard)
                else:
                    for r in hard:
                        r["parked"] = False
                rec["subs"].append({"start": s["start"], "end": s["end"], "in_place": in_place, "nhard": len(hard),
                                    "slots": slots, "occ": qcount})
                assert qcount <= MV_Q_SLOTS - 1, ("ring overflow", plan["g"], qcount)
            rec["occ_peak"] = qcount
            while qcount >= MV_Q_DRAIN:
                n = min(qcount, 32)
                rec["drains"].append((n, qhead))
                qhead = (qhead + n) % MV_Q_SLOTS
                qcount -= n
            rec["occ_after"] = qcount
            recs.append(rec)
        final = []
        while qcount > 0:
            n = min(qcount, 32)
            final.append((n, qhead))
            qhead = (qhead + n) % MV_Q_SLOTS
            qcount -= n
        out.append({"groups": recs, "final": final})
    return out, verts


def pq_coverage(warps, verts):
    """Counts of the ring and bound cases a k_scan_pq run meets (what the tests claim)."""
    c = Counter()
    for w in warps:
        for rec in w["groups"]:
            c["occ_63"] += rec["occ_peak"] == 63
            for s in rec["subs"]:
                if s["nhard"] and s["in_place"]:
                    c["in_place"] += 1
                    c["in_place_ring_busy"] += rec["occ_before"] > 0
                if s["nhard"] and not s["in_place"]:
                    c["parked_sub"] += 1
                    c["park_wraps"] += any(b < a for a, b in zip(s["slots"], s["slots"][1:]))
            ip = [s["in_place"] for s in rec["subs"] if s["nhard"]]
            c["split_in_place_and_parked"] += (True in ip) and (False in ip)
            for (n, qh) in rec["drains"]:
                c["drain"] += 1
                c["qhead_wraps"] += qh + n >= MV_Q_SLOTS
                c["drain_at_once_32"] += rec["occ_before"] == 0 and n == 32 and len(rec["drains"]) == 1
        for (n, _qh) in w["final"]:
            c[f"final_residue_{n}"] += 1
    for r in verts.values():
        c["parked_m12"] += r.get("parked", False) and r["m"] == MV_Q_ENT
        c["in_place_m13"] += r["hard"] and not r.get("parked", True) and r["m"] == MV_Q_ENT + 1
        c["tie_drained"] += r["hard"] and r.get("parked", False) and r["tie"] and r["best_gain"] > 0.0
        c["tie_in_place"] += r["hard"] and not r.get("parked", True) and r["tie"] and r["best_gain"] > 0.0
        c["bound_zero"] += r["m"] > 0 and r["bound"] == 0.0
        c["bound_pos_gain_zero"] += r["hard"] and r["best_gain"] == 0.0 and r["bound"] > 0.0
    return c


def pq_decisions(rowptr, tails, X, c, movable=None):
    """T(X) as k_scan_pq computes it: every vertex's chosen community (heavy vertices are not covered here)."""
    rowptr = np.asarray(rowptr, np.int64)
    tails = np.asarray(tails, np.int64)
    X = np.asarray(X, np.int64)
    cdeg, csize = community_state(rowptr, tails, X)
    return np.array([vertex_pq(v, rowptr, tails, X, cdeg, csize, c, movable)["best"] for v in range(len(X))], np.int64)
