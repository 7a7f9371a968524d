"""The general-weight Louvain path checked one step at a time, per vertex, on the GPU.

A warm start from any assignment X followed by `stop_after=1` and `lower=-1` returns T(X), the scan's targets (the run
always accepts its one iteration), and a cold `stop_after=1` returns T(X0) through the cold initialisation.  Every step
is compared with tests/step_ref.py on graphs whose weights are not exactly representable sums:
  1. every device target lies in the certified admissible set, and equals the certified outcome where there is one;
  2. at most 0.1 % of the vertices are not certified (the count is printed);
  3. where every input of a decision is exact (not heavy, own and candidate communities with at most 2 members) the
     target equals the fp64 restatement's, computed with the device's 1/(2m); a cold step matches it on every vertex
     that is not heavy;
  4. trace[0].moved counts the moved vertices, trace[0].chash hashes T, and trace[0].modularity is within a rigorous
     bound (step_ref.modularity_bound) of |e_in(X) c - a2(T) c^2| computed with math.fsum;
  5. constant() is within n u relative of 1 / fsum(k_i), and where it equals a golden case's constant, the first
     iteration's moved count and hash equal the golden's.
vDegree is pinned directly too: evaluate() of singletons gives community volumes equal to the host's edge-order k_i bit
for bit, and of pairs the fp64 sum of the two members' k_i."""
import math

import numpy as np
import pytest

import step_ref as S
from helpers import (WITNESS_A, WITNESS_B, WITNESS_V, case_graph, random_graph, rmat_graph, rounding_witness,
                     split_global)
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_warm_start import Ranks
from test_rounding_witness import GOLDEN as WITNESS_GOLDEN, witness_step
from test_step_ref import CASES, EUCLIDEAN, chash, multigraph

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
PW_CAP_W, E_CAP = 320, 2048          # scan_pipe.cuh MV_WCAP_W, kernels.cuh MV_ECAP


def heavy_deg_of(opts):
    """The degree above which a vertex goes to k_scan_heavy (heavy_launch in mvgpu.cu)."""
    cap = PW_CAP_W - 4 if opts.get("scan_variant", 6) >= 4 else E_CAP
    f = opts.get("force_heavy_deg", 0)
    return min(f, cap) if f > 0 else cap


def pair_weights(src, dst, seed, lo=0.01, hi=1.0):
    """One weight uniform in [lo, hi) per undirected pair (both directions agree), from a hash of the pair."""
    a, b = np.minimum(src, dst).astype(np.uint64), np.maximum(src, dst).astype(np.uint64)
    with np.errstate(over="ignore"):                  # arithmetic mod 2^64 on purpose
        z = (a * np.uint64(0x9E3779B97F4A7C15)) ^ (b + np.full_like(b, seed) * np.uint64(0xBF58476D1CE4E5B9))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return lo + (hi - lo) * ((z >> np.uint64(11)).astype(np.float64) / 2.0 ** 53)


def reweighted(rowptr, edges, seed):
    src = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
    e = edges.copy()
    e["weight"] = pair_weights(src, e["tail"], seed)
    return e


def merged(parts, rps, eds):
    rowptr = np.r_[0, np.cumsum(np.concatenate([np.diff(r) for r in rps]))].astype(np.int64)
    return split_global(int(parts[-1]), rowptr, np.concatenate(eds), 1)


NAMES = ["file_rgg_n16384_s2_w_p2", "file_rgg_n16384_s2_w_p2_merged", "rgg_n16384_p1_w", "rgg_n16384_p4_w",
         "rgg_n16384_p4_w_merged", "rgg_n65536_w_p0", "rgg_n65536_w_p5", "rmat_s14_uniform", "multigraph_n20011",
         "planted_n30000"]
_graphs = {}


def graphs():
    """name -> (parts, rowptrs, edge lists, golden case or None), built on first use.  All weights are non-dyadic."""
    if not _graphs:
        _graphs.update(graph_set())
        assert sorted(_graphs) == sorted(NAMES), sorted(_graphs)
    return _graphs


def graph_set():
    from minivite_b200 import hostgraph as hg
    out = {}
    for name in EUCLIDEAN:
        parts, rps, eds, keep = case_graph(CASES[name])
        sh = (parts.copy(), [r.copy() for r in rps], [e.copy() for e in eds])
        if keep is not None:
            keep.close()
        out[name] = sh + (CASES[name],)
        if len(rps) > 1:
            out[name + "_merged"] = merged(*sh) + (None,)
    for pct in (0.0, 5.0):
        ss = hg.generate_rgg(65536, 1, unit_weight=False, random_edge_percent=pct)
        s = ss.shards[0]
        out[f"rgg_n65536_w_p{int(pct)}"] = (s.parts.copy(), [s.rowptr.copy()], [s.edges.copy()], None)
        ss.close()
    n, rowptr, edges = rmat_graph(14, 16, 3)
    out["rmat_s14_uniform"] = split_global(n, rowptr, reweighted(rowptr, edges, 1), 1) + (None,)
    n, rowptr, edges = multigraph(20011, seed=9)
    out["multigraph_n20011"] = split_global(n, rowptr, edges, 1) + (None,)
    rowptr, edges = random_graph(30000, 24, seed=13, blocks=60)
    out["planted_n30000"] = split_global(30000, rowptr, reweighted(rowptr, edges, 2), 1) + (None,)
    return out


def run_step(R, X, k=1):
    """T after k accepted iterations: from X (warm), or cold from singletons when X is None."""
    R.set_initial(X)
    R.set_option("stop_after", k)
    return R.run(lower=-1.0)


def check_step(G, X, res, c, heavy_deg, what, stats, cold=False, uncertified=None):
    """`uncertified`: the exact set of vertices expected uncertified (default: any, at most 0.1 % of them)."""
    T = res["comm"].astype(np.int64)
    tr0 = res["trace"][0]
    n = G.nv
    cert = S.certify(G, X, c, heavy_deg)
    bad = [v for v in range(n) if not S.admits(cert, v, T[v])] if not cert["certified"].all() else \
        np.flatnonzero(cert["outcome"] != T).tolist()
    assert not bad, (what, bad[:5], [(int(X[v]), int(T[v]), cert["outcome"][v]) for v in bad[:5]])
    unc = int((~cert["certified"]).sum())
    stats.append((what, unc, n))
    print(f"{what}: uncertified {unc}/{n}")
    if uncertified is None:
        assert unc <= n // 1000, (what, unc, n)
    else:
        assert set(np.flatnonzero(~cert["certified"]).tolist()) == set(uncertified), what
    ref = S.step(G, X, c)["target"]
    ex = cert["exact"]
    if cold:
        assert np.all(ex == ~cert["heavy"]), what
    assert np.array_equal(T[ex], ref[ex]), (what, np.flatnonzero(T[ex] != ref[ex])[:5])
    assert tr0[1] == int(np.sum(T != X)), what
    assert tr0[2] == chash(G.parts, T), what
    q, B, _e = S.modularity_bound(G, X, T, c)
    assert abs(tr0[0] - q) <= B, (what, tr0[0], q, B)


def check_case(gpu, name, opts, assignments=("x0", "identity", "checkpoints", "final", "final_5pct", "random"),
               stats=None):
    parts, rps, eds, golden = graphs()[name] if "@" not in name else split_ranks(name)
    G = S.Graph(parts, rps, eds)
    hd = heavy_deg_of(opts)
    R = Ranks(parts, rps, eds, **opts)
    stats = [] if stats is None else stats
    tag = f"{name} {opts}"
    try:
        cold = run_step(R, None)
        c = R.g[0].constant()
        assert all(g.constant() == c for g in R.g)
        assert abs(c - 1.0 / math.fsum(G.k)) <= G.nv * U * c, (tag, c)
        nheavy = sum(g.shard_info()["nheavy"] for g in R.g)
        assert nheavy == int(np.sum(G.deg > hd)), (tag, nheavy)
        if name.startswith("rmat"):
            assert nheavy > 0, tag                    # the hubs (degree up to 3684) reach the weighted k_scan_heavy unforced
        X0 = np.arange(G.nv, dtype=np.int64)
        check_step(G, X0, cold, c, hd, f"{tag} cold X0", stats, cold=True)
        if golden is not None and repr(c) == repr(float(golden["constant"])):
            assert cold["trace"][0][1:] == (golden["trace"][0]["moved"], int(golden["trace"][0]["chash"], 16)), tag
        if "identity" in assignments:
            check_step(G, X0, run_step(R, X0), c, hd, f"{tag} warm X0", stats)
        R.set_initial(None)
        R.set_option("stop_after", 0)
        full = R.run()
        inputs = {}
        I = full["iters"]
        if "checkpoints" in assignments:
            for k in sorted({k for k in (1, I // 2, I - 1) if k >= 1}):
                inputs[f"ck{k}"] = run_step(R, None, k)["comm"].astype(np.int64)
        final = full["comm"].astype(np.int64)
        rng = np.random.default_rng(len(name))
        if "final" in assignments:
            inputs["final"] = final
        if "final_5pct" in assignments:
            Y = final.copy()
            pick = rng.choice(G.nv, G.nv // 20, replace=False)
            pick = pick[G.deg[pick] > 0]
            nb = G.tail[G.rowptr[pick] + rng.integers(0, G.deg[pick])]
            Y[pick] = final[nb]
            inputs["final_5pct"] = Y
        if "random" in assignments:
            v = np.arange(G.nv, dtype=np.int64)
            inputs["random"] = rng.integers(0, G.nv, G.nv)
            inputs["blocks_other_rank"] = ((v // 37) * 37 + G.nv // 2 + 5) % G.nv
        for xname, X in inputs.items():
            check_step(G, X, run_step(R, X), c, hd, f"{tag} {xname}", stats)
    finally:
        R.close()
    return stats


# ---- default options on every graph ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_step_default_options(gpu, name):
    check_case(gpu, name, {})


# ---- the run matrix on a subset ---------------------------------------------------------------------------------------
SUBSET = ["rgg_n16384_p1_w", "rmat_s14_uniform", "multigraph_n20011", "planted_n30000"]
OPTS = [{"scan_variant": 3}, {"scan_variant": 4}, {"force_heavy_deg": 8}, {"reorder": 1, "region_size": 32}]


@pytest.mark.parametrize("opts", OPTS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()))
def test_step_under_options(gpu, opts):
    for name in SUBSET:
        check_case(gpu, name, opts, assignments=("x0", "checkpoints", "final_5pct", "random"))


def split_ranks(name):
    """`graph@p`: the one-rank graph split over p ranks."""
    base, p = name.split("@")
    parts, rps, eds, _g = graphs()[base]
    assert len(rps) == 1
    return split_global(int(parts[-1]), rps[0], eds[0], int(p)) + (None,)


@pytest.mark.parametrize("world", [2, 4])
def test_step_thread_ranks(gpu, world):
    for name in ["rgg_n16384_p4_w_merged", "multigraph_n20011", "planted_n30000"]:
        check_case(gpu, f"{name}@{world}", {}, assignments=("x0", "checkpoints", "final_5pct", "random"))


# ---- vDegree directly -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES + ["multigraph_n20011@4"])
def test_volumes_are_edge_order_degrees(gpu, name):
    parts, rps, eds, _g = graphs()[name] if "@" not in name else split_ranks(name)
    G = S.Graph(parts, rps, eds)
    R = Ranks(parts, rps, eds)
    try:
        X0 = np.arange(G.nv, dtype=np.int64)
        pairs = X0 & ~np.int64(1)
        for X, want in ((X0, G.k), (pairs, S.seq_sum(pairs, G.k, G.nv))):
            R.each(lambda r, g: g.evaluate(X[parts[r]:parts[r + 1]]))
            vol = np.concatenate(R.each(lambda r, g: g.community_stats()["volume"].copy()))
            assert np.array_equal(vol, want), (name, np.flatnonzero(vol != want)[:5])
    finally:
        R.close()


# ---- rounding witnesses: one decision that only the edge order of one sum settles --------------------------------------
WITNESS_OPTS = [dict(scan_variant=sv, reorder=ro, **({"region_size": 32} if ro else {})) for sv in (3, 4, 6) for ro in (0, 1)]


@pytest.mark.parametrize("world", [1, 2, 4])
def test_rounding_witnesses_bit_exact(gpu, world):
    """The witness step is bit-exact in its targets, moved count and hash: against the reference's first iteration
    (tests/golden/rounding_traces.json) and the C oracle's X1 for R1, against tests/warm_oracle.c's T(X) for R2."""
    for name in ("r1_ck1", "r1_ck2", "r1_subrange", "r2_own"):
        parts, rps, eds, X, T_or, tr_or, _c = witness_step(name, world)
        gold = [c for c in WITNESS_GOLDEN.values() if c["witness"] == name]
        G = S.Graph(parts, rps, eds)
        for opts in WITNESS_OPTS:
            R = Ranks(parts, rps, eds, **opts)
            try:
                res = run_step(R, None if name.startswith("r1") else X)
                c = R.g[0].constant()
            finally:
                R.close()
            what = f"{name} world={world} {opts}"
            T = res["comm"].astype(np.int64)
            assert np.array_equal(T, T_or), (what, np.flatnonzero(T != T_or))
            assert T[WITNESS_V] == (WITNESS_A if name.startswith("r1") else T_or[WITNESS_V]), what
            assert res["trace"][0][1:] == (int(tr_or["moved"]), int(tr_or["chash"])), what
            for g in gold:
                assert res["trace"][0][1:] == (g["trace"][0]["moved"], int(g["trace"][0]["chash"], 16)), what
            q, B, _e = S.modularity_bound(G, X, T, c)
            assert abs(res["trace"][0][0] - q) <= B, what


def test_rounding_witness_under_forced_heavy(gpu):
    """k_scan_heavy sums the witness's counters with atomics in any order: its target may be A or B (DESIGN §3.2),
    every other vertex is still certified and must match."""
    parts, rps, eds, X, T_or, _tr, _c = witness_step("r1_ck1")
    G = S.Graph(parts, rps, eds)
    R = Ranks(parts, rps, eds, force_heavy_deg=4)
    try:
        res = run_step(R, None)
        c = R.g[0].constant()
    finally:
        R.close()
    T = res["comm"].astype(np.int64)
    assert T[WITNESS_V] in (WITNESS_A, WITNESS_B)
    check_step(G, X, res, c, 4, "r1_ck1 force_heavy_deg=4", [], cold=True, uncertified=[WITNESS_V])
