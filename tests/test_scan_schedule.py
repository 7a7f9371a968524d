"""The host restatement of the persistent scan kernels' group schedule (tests/scan_schedule.py) and the engineered
shards built on it (tests/scan_graphs.py), on the CPU: constants read from the kernel sources, hand cases, the
invariants the kernels rely on without checking them, and every boundary each engineered shard claims to hit."""
import os
import re

import numpy as np
import pytest

import scan_graphs as SG
import scan_schedule as SS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "minivite_b200", "csrc")


def _define(fn, name):
    with open(os.path.join(CSRC, fn)) as f:
        return int(re.search(rf"#define {name} (\d+)", f.read()).group(1))


def test_constants_match_the_kernel_sources():
    assert SS.MV_WCAP_UNIT == _define("scan_pipe.cuh", "MV_WCAP_UNIT")
    assert SS.MV_WCAP_W == _define("scan_pipe.cuh", "MV_WCAP_W")
    assert SS.PW_WARPS == _define("scan_pipe.cuh", "MV_PW_WARPS")
    assert SS.MV_Q_ENT == _define("scan_queue.cuh", "MV_Q_ENT")
    assert SS.MV_Q_SLOTS == _define("scan_queue.cuh", "MV_Q_SLOTS")
    assert SS.MV_Q_DRAIN == _define("scan_queue.cuh", "MV_Q_DRAIN")
    assert SS.K_ECAP == _define("kernels.cuh", "MV_ECAP")
    assert SS.K_TILE_V == _define("kernels.cuh", "MV_TILE_V")


def test_heavy_deg_as_heavy_launch_sets_it():
    assert SS.heavy_deg_of(4, True) == 508 and SS.heavy_deg_of(6, True) == 508
    assert SS.heavy_deg_of(5, False) == 316 and SS.heavy_deg_of(3, True) == 2048
    assert SS.heavy_deg_of(4, True, 16) == 16 and SS.heavy_deg_of(4, True, 5000) == 508
    assert SS.heavy_deg_of(3, False, 5000) == 2048
    assert [SS.heavy_table_size(d) for d in (1, 32, 33, 509, 512, 513, 1025)] == [64, 64, 128, 1024, 1024, 2048, 4096]


def _rowptr(degs):
    rp = np.zeros(len(degs) + 1, np.int64)
    rp[1:] = np.cumsum(degs)
    return rp


def test_hand_cases():
    # 32 x 16 = 512 edges from offset 0: the prefetched block is exactly one buffer, the whole group in one pass
    p = SS.group_plan(_rowptr([16] * 32), 0, 512, 508, False)
    assert p["whole"] and (p["lo4"], p["n4"]) == (0, 512) and len(p["subs"]) == 1
    # one edge more: not whole; lanes 0..30 from the prefetched block, lane 31 by a synchronous copy
    p = SS.group_plan(_rowptr([16] * 31 + [17]), 0, 512, 508, False)
    assert not p["whole"] and [(s["start"], s["end"], s["sync"]) for s in p["subs"]] == [(0, 31, False), (31, 32, True)]
    assert p["subs"][1]["a_sub"] == 496 and p["subs"][1]["copy_n"] == 20
    # an empty group starting at offset 2 still copies one widened 16-byte block; at offset 4 nothing
    assert SS.extent(np.array([2] * 33, np.int64), 0, 512) == (0, 4)
    assert SS.extent(np.array([4] * 33, np.int64), 0, 512) == (4, 0)
    # heavy lanes are skipped one by one and stop the sub-range before them
    p = SS.group_plan(_rowptr([1, 600, 600, 1] + [1] * 28), 0, 512, 508, True)
    assert p["heavy"] == [1, 2] and [(s["start"], s["end"], s["stop"]) for s in p["subs"]] == [(0, 1, "heavy"), (3, 32, None)]
    # a vertex of degree heavy_deg at ra mod 4 = 3 and a degree-1 vertex after it fill the buffer exactly
    p = SS.group_plan(_rowptr([303, 508, 1, 508] + [0] * 28), 0, 512, 508, False)
    assert [(s["start"], s["end"]) for s in p["subs"]] == [(0, 1), (1, 3), (3, 32)]
    assert p["subs"][1]["e_end"] - p["subs"][1]["a_sub"] == 512
    # ragged last group, warps of a one-CTA grid
    assert SS.group_plan(_rowptr([1] * 33), 1, 512, 508, False)["nvalid"] == 1
    assert SS.warp_groups(20, 1)[0] == [0, 8, 16] and len(SS.warp_groups(20, 1)) == 8
    assert len(SS.warp_groups(20, 100)) == 24                   # the grid never exceeds ceil(groups / 8) CTAs


@pytest.mark.parametrize("k", [2, 3, 5, 6])
def test_de_bruijn_has_every_pair(k):
    s = SG.de_bruijn(k)
    assert len(s) == k * k + 1 and {(a, b) for a, b in zip(s, s[1:])} == {(a, b) for a in range(k) for b in range(k)}


def test_start_vertex_always_fits():
    """deg + (ra mod 4) <= CAP for every non-heavy vertex under every force_heavy_deg: a sub-range never comes out
    empty (the kernels would spin: end == start)."""
    for cap in (SS.MV_WCAP_UNIT, SS.MV_WCAP_W):
        for hd in range(1, cap - 3):
            assert hd + 3 <= cap
        assert cap - 4 + 3 < cap
    rp, tl, kinds, _ = SG.unit_heavy()
    for force in (0, 1, 5, 16, 255, 507, 508):
        hd = SS.heavy_deg_of(4, True, force)
        SS.schedule(rp, SS.MV_WCAP_UNIT, hd, 1)              # group_plan asserts the start vertex fits
        SS.schedule(rp, SS.MV_WCAP_W, SS.heavy_deg_of(4, False, force), 1)


LAYOUTS = {
    "unit_heavy": (SG.unit_heavy, SG.UNIT_CAP, SG.UNIT_HD, SG.GROUP_KINDS, True, False),
    "unit_light": (SG.unit_light, SG.UNIT_CAP, SG.UNIT_HD, SG.LIGHT_KINDS, False, True),
    "weighted_heavy": (SG.weighted_heavy, SG.W_CAP, SG.W_HD, SG.GROUP_KINDS, True, False),
}


def report(title, counts, keys):
    print(f"\n{title}: " + ", ".join(f"{k}={counts.get(k, 0)}" for k in keys))


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_layout_hits_every_boundary(name):
    fn, cap, hd, kinds, with_heavy, whole = LAYOUTS[name]
    rp, tl, gk, _ = fn()
    deg = np.diff(rp)
    assert np.all((tl >= 0) & (tl < len(deg)))
    src = np.repeat(np.arange(len(deg)), deg)
    assert not np.any(src == tl)                                # no self loops
    key = src * len(deg) + tl
    assert np.all(np.diff(key) > 0)                             # sorted adjacency, no parallel edges
    assert np.array_equal(np.sort(key), np.sort(tl * len(deg) + src))   # symmetric
    c, req = SG.claims(rp, gk, cap, hd, kinds, with_heavy, whole)
    report(name, c, req)
    assert not [k for k in req if not c.get(k)]
    # the boundaries are tight: one edge less of buffer, or heavy_deg one lower, changes the schedule
    _, a = SS.schedule(rp, cap, hd, 1)
    _, b = SS.schedule(rp, cap - 4, hd - 4, 1)
    assert [p["subs"] for p in a] != [p["subs"] for p in b]
    if with_heavy:
        _, b = SS.schedule(rp, cap, hd + 1, 1)
        assert [p["heavy"] for p in a] != [p["heavy"] for p in b]


PQ_KEYS = ["drain_at_once_32", "parked_m12", "occ_63", "park_wraps", "qhead_wraps", "in_place_m13", "in_place_ring_busy",
           "split_in_place_and_parked", "tie_drained", "tie_in_place"] + [f"final_residue_{t}" for t in range(1, 32)]


def pq_cases():
    rp, tl, kinds = SG.pq_layout()
    X, v0, v1 = SG.pq_bound_assignment(rp, tl)
    return rp, tl, {"identity": (np.arange(len(rp) - 1, dtype=np.int64), PQ_KEYS),
                    "bounds": (X, ["bound_zero", "bound_pos_gain_zero"])}


def test_pq_ring_cases_and_invariants():
    rp, tl, cases = pq_cases()
    c = 1.0 / float(rp[-1])
    assert rp[-1] & (rp[-1] - 1) == 0 and c * float(rp[-1]) == 1.0
    for name, (X, keys) in cases.items():
        warps, verts = SS.pq_schedule(rp, tl, X, c, SG.PQ_CTAS)     # asserts occupancy <= 63, parked m <= MV_Q_ENT
        cov = SS.pq_coverage(warps, verts)
        report(f"pq {name}", cov, keys)
        assert not [k for k in keys if not cov.get(k)]
        for w in warps:
            for rec in w["groups"]:
                assert rec["occ_before"] < SS.MV_Q_DRAIN and rec["occ_peak"] <= SS.MV_Q_SLOTS - 1


def test_pq_decisions_equal_the_oracle():
    """The restatement's bound, gains, tie rule and singleton veto give the C oracle's one-step result T(X)."""
    from oracle import oracle as O
    rp, tl, cases = pq_cases()
    e = SG.edges_of(rp, tl)
    n = len(rp) - 1
    for name, (X, _keys) in cases.items():
        ref = O.louvain(np.array([0, n]), [rp], [e], init_comm=[X], stop_after=1)
        T = SS.pq_decisions(rp, tl, X, 1.0 / float(rp[-1]))
        assert np.array_equal(T, ref["comm"][0]), name
        assert np.count_nonzero(T != X) > 0


def test_default_grid_gives_every_warp_two_groups():
    """With at most 64 resident warps per SM, a shard of 2 x 64 x SMs groups gives every warp of the default grid at
    least two groups; the pairs of group kinds each warp meets, for every CTA count per SM from 1 to 8."""
    sms = 132
    rp, tl, kinds = SG.default_grid_layout(2 * 64 * sms)
    ng = len(kinds)
    for per_sm in range(1, 9):
        wg = SS.warp_groups(ng, per_sm * sms)
        assert min(len(g) for g in wg) >= 2
        pairs = SS.pair_coverage(kinds, ng, per_sm * sms)
        print(f"\nctas/SM {per_sm}: " + ", ".join(f"{a}->{b}={n}" for (a, b), n in sorted(pairs.items())))
        assert len(pairs) == 9
