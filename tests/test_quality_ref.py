"""CPU tests of the quality definitions (DESIGN.md §3.10) and their NumPy restatement (tests/quality_ref.py).

The modularity the reference reports for iteration k is mixed: e_in is measured on the assignment the scan read (X_{k-1})
and a2 on the one it wrote (X_k).  So for every accepted iteration k of a golden trace
    T[k].modularity == fabs(e_in(X_{k-1})*c - (a2(X_k)*c)*c)   bit for bit
when the sums are exact (unit and dyadic weights).  X_0 is the singleton assignment and X_k comes from the C oracle's
stop points (stop_after).  That pins the restatement -- and through it the device evaluation -- to the
reference's own goldens."""
import numpy as np
import pytest

from helpers import case_graph, exact_cases, random_graph, split_global
import quality_ref as QR
from oracle import oracle as O

CASES = exact_cases()


def small(case):
    return case["kind"] == "hand" or case.get("n", 1 << case.get("scale", 30)) <= 20000


def identity_points(case):
    """Accepted iterations k to check: all of them on small cases, else 1, I/2 and I-1."""
    I = case["iters"]
    if small(case):
        return list(range(1, I))
    return sorted({k for k in (1, I // 2, I - 1) if 1 <= k <= I - 1})


def assignment_after(parts, rps, eds, k):
    if k == 0:
        return np.arange(int(parts[-1]), dtype=np.int64)
    res = O.louvain(parts, rps, eds, stop_after=k)
    assert res["iters"] == k and not res["converged"]
    return np.concatenate(res["comm"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_identity_against_golden_trace(name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    qs = {}

    def q(k):
        if k not in qs:
            qs[k] = QR.quality(parts, rps, eds, assignment_after(parts, rps, eds, k))
        return qs[k]
    for k in identity_points(case):
        want = float(case["trace"][k - 1]["modularity"])
        got = QR.mixed_modularity(q(k - 1), q(k))
        assert repr(got) == repr(want), (name, k, got, want)
    if 1 in qs and 0 in qs:
        assert qs[0]["communities"] == int(parts[-1]) and qs[0]["singletons"] == int(parts[-1])


# ---- hand cases against a per-edge loop ----------------------------------------------------------------------------------
def naive(nv, rowptr, edges, X):
    """The definitions as plain loops (exact with Python integers / fractions for unit and dyadic weights)."""
    from fractions import Fraction
    e_in, deg, vol, internal, size = Fraction(0), [Fraction(0)] * nv, {}, {}, {}
    for i in range(nv):
        for j in range(int(rowptr[i]), int(rowptr[i + 1])):
            w = Fraction(float(edges["weight"][j]))
            deg[i] += w
            if X[int(edges["tail"][j])] == X[i]:
                e_in += w
                internal[X[i]] = internal.get(X[i], Fraction(0)) + w
    for i in range(nv):
        vol[X[i]] = vol.get(X[i], Fraction(0)) + deg[i]
        size[X[i]] = size.get(X[i], 0) + 1
    two_m = sum(deg)
    a2 = sum(v * v for v in vol.values())
    ids = sorted(size)
    return {"e_in": float(e_in), "a2": float(a2), "constant": 1.0 / float(two_m), "communities": len(size),
            "singletons": sum(1 for s in size.values() if s == 1), "max_size": max(size.values()),
            "size": size, "volume": vol, "internal": internal, "compact": [ids.index(X[i]) for i in range(nv)]}


def hand_graphs():
    g = {}
    # isolated vertices 0, 5, 9; self loops on 2 (twice) and 7; a multi-edge 3-4 (three records each way)
    n = 10
    adj = {1: [2, 3], 2: [1, 2, 2, 3], 3: [1, 2, 4, 4, 4], 4: [3, 3, 3, 6], 6: [4, 7, 8], 7: [6, 7, 8], 8: [6, 7]}
    rowptr = np.zeros(n + 1, np.int64)
    tails = []
    for i in range(n):
        tails += adj.get(i, [])
        rowptr[i + 1] = len(tails)
    edges = np.zeros(len(tails), np.dtype([("tail", "<i8"), ("weight", "<f8")]))
    edges["tail"] = tails
    edges["weight"] = 1.0
    g["loops_multi_isolated"] = (n, rowptr, edges)
    rp, ed = random_graph(300, 6, seed=5, self_loops=20, multi=30)
    g["random300"] = (300, rp, ed)
    rp, ed = random_graph(300, 6, seed=6, self_loops=20, multi=30, dyadic=True)
    g["dyadic300"] = (300, rp, ed)
    return g


def hand_assignments(nv):
    v = np.arange(nv, dtype=np.int64)
    rng = np.random.default_rng(nv)
    return {"one_community": np.zeros(nv, np.int64), "singletons": v.copy(),
            "named_outside": (v // 3 * 3 + 3) % nv,                  # community id names a vertex it does not contain
            "other_rank": (v // 4 * 4 + nv // 2 + 1) % nv,           # ids owned by the other half of the vertex range
            "random": rng.integers(0, nv, nv)}


@pytest.mark.parametrize("gname", ["loops_multi_isolated", "random300", "dyadic300"])
def test_restatement_matches_loops_on_hand_cases(gname):
    nv, rowptr, edges = hand_graphs()[gname]
    for aname, X in hand_assignments(nv).items():
        ref = naive(nv, rowptr, edges, [int(x) for x in X])
        for p in (1, 2, 4):
            parts, rps, eds = split_global(nv, rowptr, edges, p)
            q = QR.quality(parts, rps, eds, [X[parts[r]:parts[r + 1]] for r in range(p)])
            what = (gname, aname, p)
            for k in ("e_in", "a2", "constant", "communities", "singletons", "max_size"):
                assert q[k] == ref[k], (what, k, q[k], ref[k])
            assert list(q["compact"]) == ref["compact"], what
            for cid in range(nv):
                assert q["size"][cid] == ref["size"].get(cid, 0), what
                assert q["volume"][cid] == float(ref["volume"].get(cid, 0)), what
                assert q["internal"][cid] == float(ref["internal"].get(cid, 0)), what
            c = q["constant"]
            assert repr(q["modularity"]) == repr(q["e_in"] * c - (q["a2"] * c) * c)
        if aname == "one_community" and gname != "dyadic300":
            assert q["modularity"] == 0.0 and q["communities"] == 1     # e_in = 2m, a2 = (2m)^2: Q = 0 exactly
        if aname == "singletons":
            assert q["communities"] == nv and q["singletons"] == nv


def test_compact_labels_ignore_the_names():
    """Relabelling the communities by any order-preserving map leaves the compact labels unchanged."""
    nv, rowptr, edges = hand_graphs()["random300"]
    X = np.random.default_rng(1).integers(0, 50, nv)
    parts, rps, eds = split_global(nv, rowptr, edges, 1)
    a = QR.quality(parts, rps, eds, [X])
    b = QR.quality(parts, rps, eds, [X * 5 + 7])
    assert np.array_equal(a["compact"], b["compact"]) and a["communities"] == b["communities"]
    assert a["e_in"] == b["e_in"] and a["a2"] == b["a2"]
    assert sorted(set(a["compact"])) == list(range(a["communities"]))
