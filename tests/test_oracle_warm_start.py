"""CPU tests of the warm-start argument (DESIGN.md §3.9) against the reference goldens.

Only currComm, the Comm aggregates of currComm and prevMod survive one iteration of the reference loop.  So the reference
stopped after its accepted iteration k and resumed from that assignment with lower = prevMod_k must run exactly its
iterations k+1 .. I -- when the recomputed aggregates are exact (unit and dyadic weights) and thresh > 0.  Here the C
oracle's warm start and stop point (init_comm, stop_after) check that on every unit and dyadic golden case, on the case's
own shard count, before any GPU run."""
import numpy as np
import pytest

from helpers import case_graph, exact_cases
from oracle import oracle as O

CASES = exact_cases()


def split_points(iters):
    """k in {1, floor(I/2), I-1}: every accepted iteration the reference ran can be the last one before the stop."""
    return sorted({k for k in (1, iters // 2, iters - 1) if 1 <= k <= iters - 1})


def golden_trace(case):
    return [(float(t["modularity"]), int(t["moved"]), int(t["chash"], 16)) for t in case["trace"]]


def run_trace(res):
    return [(float(t["modularity"]), int(t["moved"]), int(t["chash"])) for t in res["trace"]]


@pytest.mark.parametrize("name", sorted(CASES))
def test_split_and_resume_reproduces_golden(name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    want = golden_trace(case)
    iters = case["iters"]
    for k in split_points(iters):
        a = O.louvain(parts, rps, eds, stop_after=k)
        assert not a["converged"] and a["iters"] == k, (name, k)
        assert run_trace(a) == want[:k], (name, k)
        assert a["modularity"] == want[k - 1][0], (name, k)          # the clamped currMod of iteration k
        b = O.louvain(parts, rps, eds, lower=a["modularity"], init_comm=a["comm"])
        assert b["converged"], (name, k)
        assert k + b["iters"] == iters, (name, k, b["iters"])
        assert run_trace(b) == want[k:], (name, k)
        assert repr(b["modularity"]) == repr(float(case["modularity"])), (name, k)
        assert b["chash_final"] == int(case["final_chash"], 16), (name, k)
        if "comm" in case:
            assert [int(x) for x in np.concatenate(b["comm"])] == case["comm"], (name, k)


@pytest.mark.parametrize("name", ["rgg_n16384_p1", "rgg_n16384_p4", "hand_loops_multi_p2", "rmat_s14_p2_b",
                                  "dyadic_random_n777_d150_self_loops40_multi300"])
def test_identity_start_equals_cold_run(name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    cold = O.louvain(parts, rps, eds)
    ident = [np.arange(parts[r], parts[r + 1], dtype=np.int64) for r in range(len(rps))]
    warm = O.louvain(parts, rps, eds, init_comm=ident)
    assert warm["iters"] == cold["iters"] and warm["modularity"] == cold["modularity"]
    assert run_trace(warm) == run_trace(cold)
    for a, b in zip(warm["comm"], cold["comm"]):
        assert np.array_equal(a, b)


def test_stop_after_past_convergence_is_a_converged_run():
    case = CASES["rgg_n16384_p1"]
    parts, rps, eds, _keep = case_graph(case)
    res = O.louvain(parts, rps, eds, stop_after=case["iters"] + 5)
    assert res["converged"] and res["iters"] == case["iters"]
    assert res["chash_final"] == int(case["final_chash"], 16)


@pytest.mark.parametrize("name", ["rgg_n16384_p2", "hand_weighted20_p2", "rmat_s14_p4_b",
                                  "dyadic_random_n4099_d30_hubs2_hub_deg1000_multi100"])
def test_warm_variant_without_options_is_the_pinned_oracle(name):
    """Started from the singletons it would start from anyway, with a stop point past the end, the warm-start path is the
    pinned oracle, result for result."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    ident = [np.arange(parts[r], parts[r + 1], dtype=np.int64) for r in range(len(rps))]
    a = O.louvain(parts, rps, eds, init_comm=ident, stop_after=case["iters"] + 1)
    b = O.louvain(parts, rps, eds)
    assert a["converged"] and (a["iters"], repr(a["modularity"]), a["chash_final"]) == (b["iters"], repr(b["modularity"]),
                                                                                        b["chash_final"])
    assert run_trace(a) == run_trace(b) and repr(a["constant"]) == repr(b["constant"])
    for x, y in zip(a["comm"], b["comm"]):
        assert np.array_equal(x, y)
