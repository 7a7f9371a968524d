"""CPU tests of the movable-set oracle (tests/movable_oracle.c, DESIGN.md §3.14) before any GPU run: with everything
movable it is the warm-start oracle; a frozen vertex keeps its community in one step exactly as tests/step_ref.py's step
with that target overwritten; the frontier grows like a plain per-record loop; stop and resume with the returned set
continues the run exactly; and the result does not depend on the shard count."""
import json
import os

import numpy as np
import pytest

from helpers import case_graph, global_csr, split_global, weighted_exact_cases
import movable_oracle as MO
import step_ref as S
import warm_oracle as W
from oracle import oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def exact_cases():
    """name -> case for every golden case whose Comm sums are exact: unit weights, or dyadic weights."""
    out = {}
    for fn in ("ref_traces.json", "rmat_traces.json"):
        with open(os.path.join(GOLDEN, fn)) as f:
            for name, c in json.load(f)["cases"].items():
                if not ("-w" in c.get("args", []) or c.get("unit_weight") is False):
                    out[name] = c
    for name, c in weighted_exact_cases().items():
        out["dyadic_" + name] = c
    return out


CASES = exact_cases()
# graphs that do not depend on the rank count, so that 1, 2 and 4 shards of one graph can be compared
GLOBAL = sorted(n for n, c in CASES.items() if c["kind"] in ("hand", "dyadic_rgg", "dyadic_random", "dyadic_rmat"))


def run_trace(res):
    return [(float(t["modularity"]), int(t["moved"]), int(t["chash"])) for t in res["trace"]]


def random_masks(parts, density, seed):
    rng = np.random.default_rng(seed)
    return [(rng.random(int(parts[r + 1] - parts[r])) < density).astype(np.uint8) for r in range(len(parts) - 1)]


def same_run(a, b):
    assert (a["iters"], repr(a["modularity"]), a["chash_final"], a["converged"]) == \
        (b["iters"], repr(b["modularity"]), b["chash_final"], b["converged"])
    assert run_trace(a) == run_trace(b)
    for x, y in zip(a["comm"], b["comm"]):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("name", sorted(CASES))
def test_all_movable_is_the_warm_oracle(name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    ref = W.louvain(parts, rps, eds)
    ones = [np.ones(int(parts[r + 1] - parts[r]), np.uint8) for r in range(len(rps))]
    for frontier in (0, 1):
        res = MO.louvain(parts, rps, eds, movable=ones, frontier=frontier)
        same_run(res, ref)
        assert all(np.all(m == 1) for m in res["movable"])
    same_run(MO.louvain(parts, rps, eds), ref)


@pytest.mark.parametrize("name", ["rgg_n16384_p1", "hand_loops_multi_p2", "rmat_s14_p2_b"])
def test_all_frozen_moves_nothing(name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    zeros = [np.zeros(int(parts[r + 1] - parts[r]), np.uint8) for r in range(len(rps))]
    res = MO.louvain(parts, rps, eds, movable=zeros, frontier=0)
    # iteration 1 moves nothing and is accepted against lower = -1; iteration 2 repeats it and fails the exit test
    assert res["iters"] == 2 and res["converged"] and [int(t["moved"]) for t in res["trace"]] == [0, 0]
    assert res["trace"][0]["modularity"] == res["trace"][1]["modularity"]
    for r in range(len(rps)):
        assert np.array_equal(res["comm"][r], np.arange(parts[r], parts[r + 1]))


@pytest.mark.parametrize("name", [n for n in GLOBAL if CASES[n]["kind"] == "hand"] + ["rgg_n16384_p2"])
@pytest.mark.parametrize("density", [0.1, 0.5])
def test_one_masked_step_is_step_ref_with_frozen_targets(name, density):
    parts, rps, eds, _keep = case_graph(CASES[name])
    G = S.Graph(parts, rps, eds)
    mask = random_masks(parts, density, 7)
    for X0 in (None, np.random.default_rng(3).integers(0, G.nv, G.nv)):
        init = None if X0 is None else [X0[parts[r]:parts[r + 1]] for r in range(len(rps))]
        res = MO.louvain(parts, rps, eds, movable=mask, init_comm=init, max_trace=1, thresh=-1.0, stop_after=1)
        X = np.arange(G.nv) if X0 is None else X0
        T = S.step(G, X, res["constant"])["target"]
        frozen = np.concatenate(mask) == 0
        T[frozen] = X[frozen]
        assert int(res["trace"][0]["moved"]) == int(np.sum(T != X))
        assert int(res["trace"][0]["chash"]) == O.comm_hash(0, T)
        assert np.array_equal(np.concatenate(res["comm"]), T)


def grow(parts, rps, eds, X, T, mask):
    """M + { u : record v -> u, u != v, T[v] != X[v] }, one record at a time (global arrays)."""
    out = np.concatenate(mask).astype(np.uint8).copy()
    for r in range(len(rps)):
        for i in range(int(parts[r + 1] - parts[r])):
            v = int(parts[r]) + i
            if T[v] == X[v]:
                continue
            for j in range(int(rps[r][i]), int(rps[r][i + 1])):
                u = int(eds[r][j]["tail"])
                if u != v:
                    out[u] = 1
    return out


@pytest.mark.parametrize("name", ["hand_loops_multi_p2", "rgg_n16384_p2", "rmat_s14_p4_b",
                                  "dyadic_random_n777_d150_self_loops40_multi300"])
def test_frontier_growth_is_a_per_record_loop(name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    mask = random_masks(parts, 0.05, 11)
    X = np.arange(int(parts[-1]))
    for k in (1, 2, 3):
        a = MO.louvain(parts, rps, eds, movable=mask, frontier=1, init_comm=[X[parts[r]:parts[r + 1]] for r in range(len(rps))],
                       stop_after=1)
        if a["converged"]:
            break
        T = np.concatenate(a["comm"])
        assert np.array_equal(np.concatenate(a["movable"]), grow(parts, rps, eds, X, T, mask)), (name, k)
        X, mask = T, a["movable"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_stop_and_resume_with_the_returned_set(name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    mask = random_masks(parts, 0.1, 5)
    full = MO.louvain(parts, rps, eds, movable=mask, frontier=1)
    iters = full["iters"]
    for k in sorted({k for k in (1, iters // 2, iters - 1) if 1 <= k <= iters - 1}):
        a = MO.louvain(parts, rps, eds, movable=mask, frontier=1, stop_after=k)
        assert not a["converged"] and run_trace(a) == run_trace(full)[:k], (name, k)
        b = MO.louvain(parts, rps, eds, movable=a["movable"], frontier=1, init_comm=a["comm"], lower=a["modularity"])
        assert k + b["iters"] == iters and run_trace(b) == run_trace(full)[k:], (name, k)
        assert repr(b["modularity"]) == repr(full["modularity"]) and b["chash_final"] == full["chash_final"], (name, k)
        for x, y in zip(b["movable"], full["movable"]):
            assert np.array_equal(x, y), (name, k)


@pytest.mark.parametrize("name", GLOBAL)
@pytest.mark.parametrize("frontier", [0, 1])
def test_same_result_on_1_2_and_4_shards(name, frontier):
    nv, rowptr, edges = global_csr(CASES[name])
    mask = (np.random.default_rng(2).random(nv) < 0.1).astype(np.uint8)
    runs = []
    for p in (1, 2, 4):
        parts, rps, eds = split_global(nv, rowptr, edges, p)
        res = MO.louvain(parts, rps, eds, movable=[mask[parts[r]:parts[r + 1]] for r in range(p)], frontier=frontier)
        runs.append((res["iters"], repr(res["modularity"]), run_trace(res), np.concatenate(res["comm"]).tolist(),
                     np.concatenate(res["movable"]).tolist()))
    assert runs[0] == runs[1] == runs[2]
