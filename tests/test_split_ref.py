"""CPU tests of the split definition (DESIGN.md §3.12) and its NumPy / scipy restatement (tests/split_ref.py).

The restatement is held against a plain union-find loop on hand cases.  On the C oracle's results for every unit and
dyadic golden case and both R-MAT fixtures it must keep the intra-community weight exactly, never raise sum(a_c^2) nor
lower the modularity, and be idempotent."""
import numpy as np
import pytest

from helpers import case_graph, split_global
import quality_ref as QR
import split_ref as SR
from oracle import oracle as O
from test_quality_ref import CASES, hand_assignments, hand_graphs

EDGE = np.dtype([("tail", "<i8"), ("weight", "<f8")])


def naive(nv, src, dst, X):
    """The definition as a plain union-find loop over the records."""
    parent = list(range(nv))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a
    for i, j in zip(src, dst):
        if i != j and X[i] == X[j]:
            a, b = find(int(i)), find(int(j))
            if a != b:
                parent[max(a, b)] = min(a, b)
    Y = [0] * nv
    low = {}
    for v in range(nv):
        r = find(v)
        low.setdefault(r, v)                        # v ascends: the first member seen is the smallest
        Y[v] = low[r]
    pieces = {}
    for v in range(nv):
        pieces.setdefault(X[v], set()).add(Y[v])
    return {"Y": Y, "communities": len(pieces), "components": len(set(Y)),
            "disconnected": sum(1 for s in pieces.values() if len(s) > 1)}


def csr(nv, adj, weights=None):
    """rowptr / records of a dict v -> list of tails (weights: dict (v, k) -> weight of v's k-th record)."""
    rowptr = np.zeros(nv + 1, np.int64)
    tails, w = [], []
    for v in range(nv):
        for k, t in enumerate(adj.get(v, [])):
            tails.append(t)
            w.append((weights or {}).get((v, k), 1.0))
        rowptr[v + 1] = len(tails)
    edges = np.zeros(len(tails), EDGE)
    edges["tail"], edges["weight"] = tails, w
    return rowptr, edges


def hand_cases():
    """name -> (nv, rowptr, edges, {assignment name: X})"""
    out = {}
    for gname, (nv, rowptr, edges) in hand_graphs().items():     # isolated vertices, self loops, multi-edges
        out[gname] = (nv, rowptr, edges, hand_assignments(nv))
    # records stored in one direction only: 0 -> 1 on the first half, 7 -> 2 from the second half into the first (a
    # rank boundary on 2 and 4 ranks), 5 -> 5 a self loop; zero-weight records 3 -> 4 and 4 -> 3
    nv = 8
    rowptr, edges = csr(nv, {0: [1], 3: [4], 4: [3], 5: [5], 7: [2]}, {(3, 0): 0.0, (4, 0): 0.0})
    out["one_direction"] = (nv, rowptr, edges, {"one": np.zeros(nv, np.int64), "pairs": np.array([0, 0, 7, 4, 4, 5, 6, 7]),
                                                "outside": np.array([6, 6, 6, 6, 6, 0, 1, 6])})
    # one community spread over 4 ranks whose pieces interleave: even vertices chain 0-2-4-..., odd ones 1-3-5-...
    nv = 64
    adj = {v: [t for t in (v - 2, v + 2) if 0 <= t < nv] for v in range(nv)}
    rowptr, edges = csr(nv, adj)
    v = np.arange(nv, dtype=np.int64)
    out["interleaved"] = (nv, rowptr, edges, {"one": np.full(nv, 9, np.int64), "halves": (v >= 32) * 40})
    # a 2 500-vertex path, and the same path cut into pieces by a community of its own every 100 vertices
    nv = 2500
    adj = {v: [t for t in (v - 1, v + 1) if 0 <= t < nv] for v in range(nv)}
    rowptr, edges = csr(nv, adj)
    v = np.arange(nv, dtype=np.int64)
    out["path2500"] = (nv, rowptr, edges, {"one": np.full(nv, nv - 1, np.int64), "cut": np.where(v % 100 == 50, 1, 0)})
    return out


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_restatement_matches_union_find_on_hand_cases(name):
    nv, rowptr, edges, assigns = hand_cases()[name]
    src = np.repeat(np.arange(nv), np.diff(rowptr))
    for aname, X in assigns.items():
        ref = naive(nv, src, edges["tail"], [int(x) for x in X])
        for p in (1, 2, 4):
            parts, rps, eds = split_global(nv, rowptr, edges, p)
            got = SR.split(parts, rps, eds, [X[parts[r]:parts[r + 1]] for r in range(p)])
            assert list(got["Y"]) == ref["Y"], (name, aname, p)
            for k in ("communities", "components", "disconnected"):
                assert got[k] == ref[k], (name, aname, p, k, got[k], ref[k])


def test_hand_case_values():
    """A few answers written out by hand."""
    nv, rowptr, edges, assigns = hand_cases()["one_direction"]
    parts, rps, eds = split_global(nv, rowptr, edges, 2)
    got = SR.split(parts, rps, eds, assigns["one"])
    assert list(got["Y"]) == [0, 0, 2, 3, 3, 5, 6, 2]            # 7 -> 2 joins across the halves, 5 stays alone
    assert (got["communities"], got["components"], got["disconnected"]) == (1, 5, 1)
    got = SR.split(parts, rps, eds, assigns["outside"])           # community 6 is named by a vertex outside it
    assert list(got["Y"]) == [0, 0, 2, 3, 3, 5, 6, 2]
    nv, rowptr, edges, assigns = hand_cases()["interleaved"]
    parts, rps, eds = split_global(nv, rowptr, edges, 4)
    got = SR.split(parts, rps, eds, assigns["one"])
    assert list(got["Y"]) == [v % 2 for v in range(nv)]
    assert (got["communities"], got["components"], got["disconnected"]) == (1, 2, 1)
    nv, rowptr, edges, assigns = hand_cases()["path2500"]
    parts, rps, eds = split_global(nv, rowptr, edges, 1)
    assert SR.split(parts, rps, eds, assigns["one"])["components"] == 1
    assert SR.split(parts, rps, eds, assigns["cut"])["components"] == 25 + 25 + 1   # 25 cut vertices, 26 runs


# ---- properties on the oracle's results --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_split_of_oracle_results(name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    X = np.concatenate(O.louvain(parts, rps, eds)["comm"])
    s = SR.split(parts, rps, eds, X)
    Y = s["Y"]
    qx, qy = QR.quality(parts, rps, eds, X), QR.quality(parts, rps, eds, Y)
    assert qy["e_in"] == qx["e_in"], name
    assert qy["a2"] <= qx["a2"] and qy["modularity"] >= qx["modularity"], name
    assert qy["communities"] == s["components"] and qx["communities"] == s["communities"]
    assert s["disconnected"] == 0 or s["components"] > s["communities"]
    assert np.all(Y[Y] == Y)                                      # Y names a member of each community
    again = SR.split(parts, rps, eds, Y)
    assert np.array_equal(again["Y"], Y) and again["disconnected"] == 0, name


def test_rmat_fixture_counts():
    """One rank: the counts the oracle's R-MAT results give (roughly one community in twelve is in pieces)."""
    want = {"rmat_s14_p1": (8251, 10500, 759), "rmat_s17_p1": (70303, 86659, 4282)}
    for name, counts in want.items():
        parts, rps, eds, _keep = case_graph(CASES[name])
        X = np.concatenate(O.louvain(parts, rps, eds)["comm"])
        s = SR.split(parts, rps, eds, X)
        assert (s["communities"], s["components"], s["disconnected"]) == counts, name
