"""CPU tests of the probe restatement tests/probe_ref.py (DESIGN.md §3.15): against plain per-vertex loops on hand-made
and small random graphs, against step_ref.step and the C oracle's one warm step on every unit and dyadic golden case,
across shard counts, and on the update scenario that motivates the probe."""
import math

import numpy as np
import pytest

import probe_ref as PR
import step_ref as SR
from helpers import case_graph, exact_cases, split_global
from minivite_b200 import hostgraph as hg
from oracle import oracle as O
from scan_graphs import split_at

CASES = exact_cases()


def naive(nv, rowptr, edges, X):
    """Per-vertex dict loops, in the reference's order: k and the counters summed in edge order, a_c in vertex order."""
    k = [0.0] * nv
    for v in range(nv):
        for e in range(rowptr[v], rowptr[v + 1]):
            k[v] += float(edges["weight"][e])
    a, size = [0.0] * nv, [0] * nv
    for v in range(nv):
        a[X[v]] += k[v]
        size[X[v]] += 1
    c = 1.0 / math.fsum(k)
    out = {"target": [], "best": [], "gain": []}
    for v in range(nv):
        x, counter, sl = int(X[v]), {}, 0.0
        for e in range(rowptr[v], rowptr[v + 1]):
            t, w = int(edges["tail"][e]), float(edges["weight"][e])
            y = int(X[t])
            counter[y] = counter.get(y, 0.0) + w
            if t == v:
                sl += w
        eix, ax = counter.get(x, 0.0) - float(math.trunc(sl)), a[x] - k[v]
        best, bg = -1, -math.inf
        for y, e in counter.items():
            if y == x:
                continue
            g = 2.0 * (e - eix) - ((2.0 * k[v]) * (a[y] - ax)) * c
            if g > bg or (g == bg and y < best):
                best, bg = y, g
        t = x
        if bg > 0.0 and not (best > x and size[x] == 1 and size[best] == 1):
            t = best
        out["target"].append(t)
        out["best"].append(best)
        out["gain"].append(bg)
    return {key: np.array(val) for key, val in out.items()}, c


def csr(nv, pairs, loops=()):
    """Symmetric CSR from undirected (u, v, w) pairs (parallel pairs kept) and self loops (v, w), sorted by tail."""
    src, dst, w = [], [], []
    for u, v, wt in pairs:
        src += [u, v]; dst += [v, u]; w += [wt, wt]
    for v, wt in loops:
        src.append(v); dst.append(v); w.append(wt)
    src, dst, w = np.array(src, np.int64), np.array(dst, np.int64), np.array(w, np.float64)
    o = np.lexsort((dst, src))
    rowptr = np.searchsorted(src[o], np.arange(nv + 1)).astype(np.int64)
    edges = np.zeros(len(o), hg.EDGE_DTYPE)
    edges["tail"], edges["weight"] = dst[o], w[o]
    return rowptr, edges


def hand_graphs():
    """(name, nv, rowptr, edges, X): self loops, multi-edges, isolated and interior vertices, a zero-weight edge,
    communities named by outside vertices and by ids of the other half (the other rank on 2 shards)."""
    out = []
    # two triangles and a bridge; vertex 7 isolated, vertex 6 only a self loop
    rp, ed = csr(8, [(0, 1, 1), (1, 2, 1), (0, 2, 1), (3, 4, 1), (4, 5, 1), (3, 5, 1), (2, 3, 1)], loops=[(6, 1.0)])
    out += [("triangles_singletons", 8, rp, ed, np.arange(8)),
            ("triangles_split", 8, rp, ed, np.array([0, 0, 0, 3, 3, 3, 6, 7])),
            ("triangles_named_outside", 8, rp, ed, np.array([7, 7, 7, 6, 6, 6, 0, 1])),
            ("triangles_other_half", 8, rp, ed, np.array([5, 5, 4, 1, 1, 2, 0, 3]))]
    # multi-edges, a zero-weight edge, dyadic weights and a weighted self loop
    rp, ed = csr(6, [(0, 1, 0.5), (0, 1, 0.25), (1, 2, 0.0), (2, 3, 2.0), (3, 4, 1.5), (4, 5, 0.75), (5, 0, 1.0), (2, 4, 0.5)],
                 loops=[(3, 3.5), (3, 1.0)])
    out += [("multi_zero_singletons", 6, rp, ed, np.arange(6)),
            ("multi_zero_pairs", 6, rp, ed, np.array([0, 0, 2, 2, 4, 4])),
            ("multi_zero_one", 6, rp, ed, np.full(6, 3))]
    # a star: every leaf ties with the others; veto both ways among singletons
    rp, ed = csr(7, [(0, v, 1) for v in range(1, 7)])
    out += [("star_singletons", 7, rp, ed, np.arange(7)), ("star_reversed", 7, rp, ed, np.arange(7)[::-1].copy())]
    # a path: ties at zero and negative gain between the two sides
    rp, ed = csr(6, [(0, 1, 1), (1, 2, 1), (2, 3, 1), (3, 4, 1), (4, 5, 1)])
    out += [("path_pairs", 6, rp, ed, np.array([0, 0, 2, 2, 4, 4])), ("path_mid", 6, rp, ed, np.array([1, 1, 3, 3, 3, 5]))]
    return out


def random_small(seed):
    rng = np.random.default_rng(seed)
    nv = int(rng.integers(3, 14))
    m = int(rng.integers(0, 3 * nv))
    pairs = [(int(rng.integers(nv)), int(rng.integers(nv)), float(rng.choice([0.0, 0.5, 1.0, 1.0, 2.0]))) for _ in range(m)]
    pairs = [p for p in pairs if p[0] != p[1]] + [(0, nv - 1, 1.0)]      # 2m > 0
    loops = [(int(rng.integers(nv)), float(rng.choice([0.5, 1.0, 2.5]))) for _ in range(int(rng.integers(0, 3)))]
    rp, ed = csr(nv, pairs, loops)
    X = rng.integers(0, min(nv, int(rng.integers(1, nv + 1))), nv) if seed % 3 else np.arange(nv)
    return nv, rp, ed, X


def check_naive(nv, rp, ed, X, what):
    parts = np.array([0, nv], np.int64)
    got = PR.probe_shards(parts, [rp], [ed], X)
    ref, c = naive(nv, rp, ed, X)
    assert got["constant"] == c, what
    assert np.array_equal(got["best"], ref["best"]), (what, got["best"], ref["best"])
    assert np.array_equal(got["gain"].view(np.int64), ref["gain"].view(np.int64)), (what, got["gain"], ref["gain"])
    assert np.array_equal(got["target"], ref["target"]), what
    assert np.array_equal(got["target"], got["step_target"]), what
    assert got["moves"] == int(np.sum(ref["target"] != X))
    return got


def cases_naive():
    return hand_graphs() + [(f"random{s}",) + random_small(s) for s in range(300)]


def test_against_plain_loops():
    seen = {"tie_pos": 0, "tie_zero": 0, "tie_neg": 0, "veto": 0, "veto_not": 0, "interior": 0, "isolated": 0,
            "zero_weight_best": 0, "named_outside": 0}
    for name, nv, rp, ed, X in cases_naive():
        got = check_naive(nv, rp, ed, X, name)
        X = np.asarray(X)
        G = SR.Graph(np.array([0, nv]), [rp], [ed])
        cv, cy, g = SR.step(G, X, got["constant"])["pairs"]
        for v in range(nv):
            gv = g[(cv == v)]
            if len(gv) >= 2 and np.sum(gv == gv.max()) >= 2:
                seen["tie_pos" if gv.max() > 0 else "tie_zero" if gv.max() == 0 else "tie_neg"] += 1
        size = np.bincount(X, minlength=nv)
        single = (got["gain"] > 0) & (size[X] == 1) & (size[np.maximum(got["best"], 0)] == 1)
        seen["veto"] += int(np.sum(single & (got["best"] > X)))
        seen["veto_not"] += int(np.sum(single & (got["best"] < X)))
        seen["interior"] += got["interior"] - int(np.sum((G.deg > 0) & (G.deg == np.bincount(G.src[G.tail == G.src], minlength=nv))))
        seen["isolated"] += int(np.sum(G.deg == 0))
        zero = G.w == 0.0
        seen["zero_weight_best"] += int(np.sum(got["best"][G.src[zero]] == X[G.tail[zero]]))
        seen["named_outside"] += int(np.sum(X[X] != X))
        assert got["vetoed"] == int(np.sum(single & (got["best"] > X)))
    assert all(v > 0 for v in seen.values()), seen


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_checkpoints_against_step_and_oracle(name):
    """X = C_k, the oracle's checkpoint after k accepted iterations (k = 0: singletons); one warm step of the oracle
    from C_k gives C_{k+1} = target and its trace[0].moved = moves."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    G = SR.Graph(parts, rps, eds)
    nv = G.nv
    iters = case["iters"]
    for k in sorted({0, 1, iters // 2, iters - 1}):
        if k >= iters:
            continue
        X = np.arange(nv, dtype=np.int64) if k == 0 else np.concatenate(O.louvain(parts, rps, eds, stop_after=k)["comm"])
        got = PR.probe(G, X)
        assert np.array_equal(got["target"], got["step_target"]), (name, k)
        init = [X[parts[r]:parts[r + 1]] for r in range(len(rps))]
        one = O.louvain(parts, rps, eds, init_comm=init, stop_after=1)
        assert np.array_equal(got["target"], np.concatenate(one["comm"])), (name, k)
        assert got["moves"] == int(one["trace"][0]["moved"]), (name, k)


def test_shard_counts_and_empty_ranks():
    nv, (rowptr, edges) = 4096, _rgg(4096)
    X = np.random.default_rng(5).integers(0, nv, nv)
    ref = PR.probe_shards(np.array([0, nv]), [rowptr], [edges], X)
    splits = [split_global(nv, rowptr, edges, p)[0] for p in (2, 4, 16)]
    splits.append(np.array([0, 0, 1, 1, 2000, 2001, 2001, nv, nv, nv, nv, nv, nv, nv, nv, nv, nv], np.int64))
    for parts in splits:
        rps, eds = split_at(rowptr, edges, parts)
        got = PR.probe_shards(parts, rps, eds, X)
        for key in ("target", "best"):
            assert np.array_equal(got[key], ref[key]), (key, parts)
        assert np.array_equal(got["gain"].view(np.int64), ref["gain"].view(np.int64)), parts
        assert all(repr(got[f]) == repr(ref[f]) for f in PR.FIELDS), parts


def _rgg(n):
    ss = hg.generate_rgg(n, 1)
    out = ss.shards[0].rowptr.copy(), ss.shards[0].edges.copy()
    ss.close()
    return out


def test_update_leaves_unsettled_vertices_off_the_batch():
    """RGG 65 536 clustered at -p 0, then updated to -p 5: the vertices whose decision from the old result is a move,
    against the batch's endpoints (what LouvainGPU.movable_from_batch seeds).  Many endpoints stay put, and vertices
    that touch no batch record want to move because 1/(2m) and the community degrees changed."""
    import update_ref as U
    ss0, ss5 = hg.generate_rgg(65536, 1), hg.generate_rgg(65536, 1, random_edge_percent=5)
    try:
        s0, s5 = ss0.shards[0], ss5.shards[0]
        parts = np.array([0, 65536], np.int64)
        X0 = np.concatenate(O.louvain(parts, [s0.rowptr], [s0.edges])["comm"])
        src, dst, _w = U.extras(s0, s5)
        seeds = np.zeros(65536, bool)
        seeds[src] = seeds[dst] = True
        got = PR.probe_shards(parts, [s5.rowptr], [s5.edges], X0)
        unsettled = got["target"] != X0
        off_batch = int(np.sum(unsettled & ~seeds))
        assert int(np.sum(unsettled)) == got["moves"]
        # 22 963 seeds, 2 341 unsettled vertices, 1 523 of them off the batch
        assert (int(np.sum(seeds)), got["moves"], off_batch) == (22963, 2341, 1523)
    finally:
        ss0.close()
        ss5.close()
