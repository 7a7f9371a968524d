"""The host restatement of one Louvain step (tests/step_ref.py) against the C oracle, and its certificate against sums
taken in other orders.

fp64 mode must give the oracle's first-iteration targets, moved count and hash from singletons on golden cases of every
kind (unit, dyadic and the three Euclidean ones, whose sums round), and tests/warm_oracle.c's single step from its own
checkpoints and from random assignments.  Certified mode must contain every gain that other summation orders give: the
community degrees in reverse and random vertex order, and the heavy vertices' counters in permuted edge order."""
import json
import os

import numpy as np
import pytest

import step_ref as S
import warm_oracle as W
from helpers import case_graph, random_graph, split_global, weighted_exact_cases
from oracle import oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_cases():
    out = {}
    for fn in ("ref_traces.json", "rmat_traces.json"):
        with open(os.path.join(GOLDEN, fn)) as f:
            for name, c in json.load(f)["cases"].items():
                if c["nv"] <= 65536:
                    out[name] = c
    for name, c in weighted_exact_cases().items():
        if c["nv"] <= 65536:
            out["dyadic_" + name] = c
    return out


CASES = golden_cases()
EUCLIDEAN = ["rgg_n16384_p1_w", "rgg_n16384_p4_w", "file_rgg_n16384_s2_w_p2"]
WARM_CASES = EUCLIDEAN + ["rgg_n16384_p1", "hand_loops_multi_p2", "dyadic_random_n777_d150_self_loops40_multi300",
                          "dyadic_random_n6000_d8_hubs3_hub_deg3000_multi200"]


def chash(parts, T):
    return sum(O.comm_hash(int(parts[r]), T[parts[r]:parts[r + 1]]) for r in range(len(parts) - 1)) & (2 ** 64 - 1)


def one_step(parts, rps, eds, X):
    """warm_oracle's single accepted step from X: (T(X), trace[0], constant)."""
    res = W.louvain(parts, rps, eds, init_comm=[X[parts[r]:parts[r + 1]] for r in range(len(rps))], stop_after=1)
    return np.concatenate(res["comm"]), res["trace"][0], res["constant"]


def general_graphs():
    """Graphs of the GPU step tests that are cheap on the host: non-dyadic weights, self loops of non-integer weight
    above 1, parallel edges, zero weights and a vertex whose edges all weigh 0, weights from 1e-3 to 1e3."""
    out = {}
    for name in EUCLIDEAN:
        parts, rps, eds, keep = case_graph(CASES[name])
        out[name] = (parts.copy(), [r.copy() for r in rps], [e.copy() for e in eds])
        if keep is not None:
            keep.close()
    nv, rowptr, edges = multigraph(3001, seed=5)
    out["multigraph3001_p2"] = split_global(nv, rowptr, edges, 2)
    return out


def multigraph(n, seed):
    """Symmetric random multigraph, adjacency sorted by tail: weights 10^U(-3, 3) (1 % of them 0), a hub of degree 900,
    400 parallel copies of edges with their own weights, 60 self loops of weight in (1, 4), and vertex n-1 with five
    edges of weight 0 only."""
    rng = np.random.default_rng(seed)
    a, b = rng.integers(0, n - 1, 6 * n), rng.integers(0, n - 1, 6 * n)
    a, b = a[a != b], b[a != b]
    hub = rng.choice(np.arange(1, n - 1), 900, replace=False)
    a, b = np.r_[a, np.zeros(900, np.int64)], np.r_[b, hub]
    dup = rng.integers(0, len(a), 400)
    a, b = np.r_[a, a[dup]], np.r_[b, b[dup]]
    w = 10.0 ** rng.uniform(-3.0, 3.0, len(a))
    w[rng.random(len(a)) < 0.01] = 0.0
    z = rng.choice(n - 1, 5, replace=False)
    a, b, w = np.r_[a, np.full(5, n - 1)], np.r_[b, z], np.r_[w, np.zeros(5)]
    s = rng.integers(0, n - 1, 60)
    src, dst = np.r_[a, b, s], np.r_[b, a, s]
    w = np.r_[w, w, 1.0 + 3.0 * rng.random(60)]
    o = np.lexsort((dst, src))                          # stable: parallel edges keep their order in both directions
    rowptr = np.r_[0, np.cumsum(np.bincount(src, minlength=n))].astype(np.int64)
    edges = np.zeros(len(o), O.EDGE_DTYPE)
    edges["tail"], edges["weight"] = dst[o], w[o]
    return n, rowptr, edges


# ---- fp64 mode against the oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_first_step_matches_oracle_and_golden(name):
    case = CASES[name]
    parts, rps, eds, keep = case_graph(case)
    try:
        X0 = np.arange(int(parts[-1]), dtype=np.int64)
        T_or, tr, const = one_step(parts, rps, eds, X0)
        G = S.Graph(parts, rps, eds)
        r = S.step(G, X0, const)
        assert np.array_equal(r["target"], T_or)
        assert r["moved"] == int(tr["moved"]) == case["trace"][0]["moved"]
        assert chash(parts, r["target"]) == int(tr["chash"]) == int(case["trace"][0]["chash"], 16)
        assert repr(const) == repr(float(case["constant"]))
    finally:
        if keep is not None:
            keep.close()


def random_assignments(nv, seed):
    rng = np.random.default_rng(seed)
    v = np.arange(nv, dtype=np.int64)
    return {"random": rng.integers(0, nv, nv), "blocks_other_rank": ((v // 37) * 37 + nv // 2 + 5) % nv,
            "pairs": v ^ 1 if nv % 2 == 0 else np.minimum(v ^ 1, nv - 1)}


def warm_inputs(parts, rps, eds, iters):
    out = {}
    for k in sorted({k for k in (1, iters // 2, iters - 1) if k >= 1}):
        out[f"ck{k}"] = np.concatenate(W.louvain(parts, rps, eds, stop_after=k)["comm"])
    out.update(random_assignments(int(parts[-1]), 3))
    return out


@pytest.mark.parametrize("name", WARM_CASES)
def test_warm_step_matches_warm_oracle(name):
    case = CASES[name]
    parts, rps, eds, keep = case_graph(case)
    try:
        G = S.Graph(parts, rps, eds)
        for xname, X in warm_inputs(parts, rps, eds, case["iters"]).items():
            T_or, tr, const = one_step(parts, rps, eds, X)
            r = S.step(G, X, const)
            assert np.array_equal(r["target"], T_or), xname
            assert r["moved"] == int(tr["moved"]) and chash(parts, r["target"]) == int(tr["chash"]), xname
    finally:
        if keep is not None:
            keep.close()


def test_warm_step_matches_warm_oracle_general_graphs():
    for gname, (parts, rps, eds) in general_graphs().items():
        G = S.Graph(parts, rps, eds)
        res = W.louvain(parts, rps, eds)
        for xname, X in warm_inputs(parts, rps, eds, res["iters"]).items():
            T_or, tr, const = one_step(parts, rps, eds, X)
            r = S.step(G, X, const)
            assert np.array_equal(r["target"], T_or), (gname, xname)
            assert r["moved"] == int(tr["moved"]), (gname, xname)


def test_multigraph_has_the_edges_it_promises():
    n, rowptr, edges = multigraph(3001, seed=5)
    src = np.repeat(np.arange(n), np.diff(rowptr))
    w, dst = edges["weight"], edges["tail"]
    loop = src == dst
    assert np.any(loop & (w > 1.0) & (w != np.floor(w)))
    pair = np.unique(np.stack([src, dst], 1), axis=0, return_counts=True)[1]
    assert np.any(pair > 1)
    pos = w[w > 0]
    assert pos.min() < 2e-3 and pos.max() > 5e2 and np.sum(w == 0.0) > 0
    deg = np.diff(rowptr)
    assert any(deg[v] > 0 and np.all(w[rowptr[v]:rowptr[v + 1]] == 0.0) for v in range(n))
    fwd = np.lexsort((w, dst, src))
    rev = np.lexsort((w, src, dst))
    assert np.array_equal(src[fwd], dst[rev]) and np.array_equal(w[fwd], w[rev])     # symmetric weights


# ---- the certificate against other summation orders -----------------------------------------------------------------
def heavy_edge_permutation(G, heavy, rng=None):
    """Edge order with every heavy vertex's edges shuffled among themselves (rng None: reversed)."""
    o = np.arange(len(G.tail))
    for v in np.flatnonzero(heavy):
        a, b = G.rowptr[v], G.rowptr[v + 1]
        o[a:b] = a + (rng.permutation(b - a) if rng is not None else np.arange(b - a)[::-1])
    return o


def check_certificate(G, X, c, heavy_deg, rng, what):
    cert = S.certify(G, X, c, heavy_deg)
    cv, cy, lo, hi = cert["pairs"]
    assert np.all(lo <= hi), what
    n = G.nv
    heavy = cert["heavy"]
    orders = [(None, None), (None, np.arange(n)[::-1]), (None, rng.permutation(n)),
              (heavy_edge_permutation(G, heavy, rng), rng.permutation(n)), (heavy_edge_permutation(G, heavy), None)]
    for eo, vo in orders:
        r = S.step(G, X, c, edge_order=eo, vertex_order=vo)
        pv, py, g = r["pairs"]
        assert np.array_equal(pv, cv) and np.array_equal(py, cy), what
        bad = (g < lo) | (g > hi)
        assert not bad.any(), (what, np.flatnonzero(bad)[:5], g[bad][:5], lo[bad][:5], hi[bad][:5])
        T = r["target"]
        assert all(S.admits(cert, v, T[v]) for v in range(n)), what
    ex = cert["exact"]
    assert np.all(cert["certified"][ex]), what
    base = S.step(G, X, c)["target"]
    assert np.array_equal(cert["outcome"][ex], base[ex]), what
    frac = 1.0 - cert["certified"].mean()
    print(f"{what}: uncertified {int((~cert['certified']).sum())}/{n} ({100 * frac:.4f} %)")
    return cert


@pytest.mark.parametrize("heavy_deg", [None, 8])
def test_certificate_contains_other_orders(heavy_deg):
    rng = np.random.default_rng(11)
    for gname, (parts, rps, eds) in general_graphs().items():
        G = S.Graph(parts, rps, eds)
        res = W.louvain(parts, rps, eds)
        const = res["constant"]
        inputs = {"X0": np.arange(G.nv, dtype=np.int64)}
        inputs.update(warm_inputs(parts, rps, eds, res["iters"]))
        inputs["final"] = np.concatenate(res["comm"])
        for xname, X in inputs.items():
            check_certificate(G, X, const, heavy_deg, rng, f"{gname} {xname} heavy_deg={heavy_deg}")


def test_certificate_is_exact_on_exact_inputs():
    """All-zero inputs give [0, 0]; with no heavy vertex and singletons every interval has width 0."""
    parts, rps, eds = general_graphs()["multigraph3001_p2"]
    G = S.Graph(parts, rps, eds)
    X0 = np.arange(G.nv, dtype=np.int64)
    cert = S.certify(G, X0, 1.0 / float(np.sum(G.k)))
    cv, cy, lo, hi = cert["pairs"]
    assert np.array_equal(lo, hi) and np.all(cert["exact"])
    zero = np.flatnonzero((G.k == 0.0) & (G.deg > 0))
    assert len(zero) and np.all(lo[np.isin(cv, zero)] == 0.0)
    lo_z, hi_z = S._widen(np.zeros(3), S._radius(np.zeros(3), np.array([0, 5, 100])))
    assert np.all(lo_z == 0.0) and np.all(hi_z == 0.0)


def test_seq_sum_is_sequential():
    """Rounding witnesses for the summation order: 0.1 + 0.2 + 0.3 sequentially is 0.6000000000000001, in reverse 0.6."""
    g = np.array([0, 1, 0, 1, 0, 1])
    v = np.array([0.1, 0.3, 0.2, 0.2, 0.3, 0.1])
    out = S.seq_sum(g, v, 2)
    assert repr(float(out[0])) == "0.6000000000000001" and repr(float(out[1])) == "0.6"
