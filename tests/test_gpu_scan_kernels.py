"""Both shipped neighbour-scan kernels -- k_scan_pw (scan_variant 4: persistent warps, TMA-fed double buffer,
scan_pipe.cuh) and k_scan_ws (3: one CTA per 128-vertex tile), k_scan_pq (5: k_scan_pw with a per-warp ring of hard vertices) -- against the reference goldens and the C oracle,
including the paths only unusual graphs reach: groups whose edges overflow one staging buffer (sub-ranges with
synchronous bulk copies), vertices handed to the high-degree kernel, ragged last groups, weights."""
import numpy as np
import pytest

from helpers import assert_trace_matches, dyadic_exponent, random_graph
from test_gpu_parity import as_single, gpu, is_weighted, run_single  # noqa: F401  (gpu is a fixture)

pytestmark = pytest.mark.gpu
VARIANTS = [3, 4, 5, 6]


@pytest.mark.parametrize("variant", VARIANTS)
def test_golden_cases(gpu, golden, variant):
    """Every golden case, bit-exact where the weights are exactly representable (unit, and hand_weighted20's k/4 on 1
    and 2 ranks); the Euclidean -w RGG weights make the last bits depend on the order of the sums, so those 1-rank cases
    keep |dQ| <= 1e-6."""
    for name, case in golden.items():
        nv, parts, rowptr, edges = as_single(case)
        res = run_single(gpu, parts, rowptr, edges, nv, scan_variant=variant)
        if is_weighted(name, case) and dyadic_exponent(edges["weight"]) is None:
            if case["nranks"] == 1:
                assert abs(res["modularity"] - float(case["modularity"])) <= 1e-6, name
        else:
            assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, res["comm"])


@pytest.mark.parametrize("variant", VARIANTS)
def test_options_keep_results(gpu, golden, variant):
    for name in ("rgg_n65536_p1", "hand_loops_multi_p1", "hand_star41_p1", "hand_k66_p1"):
        case = golden[name]
        nv, parts, rowptr, edges = as_single(case)
        for opts in ({"cache_policy": 0}, {"reorder": 1, "region_size": 64}, {"force_weighted": 1}, {"first_iter": 0},
                     {"first_iter": 0, "reorder": 1, "region_size": 128},
                     {"force_heavy_deg": 8, "reorder": 1, "region_size": 32}, {"force_weighted": 1, "reorder": 1, "force_heavy_deg": 5}):
            res = run_single(gpu, parts, rowptr, edges, nv, scan_variant=variant, **opts)
            assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, res["comm"] if "comm" in case else None)


@pytest.mark.parametrize("variant", VARIANTS)
def test_dense_and_skewed_graphs_against_oracle(gpu, variant):
    """Graphs the RGG goldens never produce: 32-vertex groups with thousands of edges (sub-ranges), genuine hubs
    above every tile capacity (high-degree kernel, unforced), self loops, multi-edges, a ragged last group."""
    from oracle import oracle as O
    for (n, deg, kw) in [(1000, 60, {}), (777, 150, {"self_loops": 40, "multi": 300}), (6000, 8, {"hubs": 3, "hub_deg": 3000}),
                         (4099, 30, {"hubs": 2, "hub_deg": 900, "multi": 100}), (33, 20, {}), (2500, 700, {}),
                         (3000, 80, {"blocks": 25}), (20000, 40, {"blocks": 400, "hubs": 1, "hub_deg": 2000})]:
        rowptr, edges = random_graph(n, deg, seed=n + deg, **kw)
        parts = np.array([0, n], np.int64)
        ref = O.louvain(parts, [rowptr], [edges])
        for opts in ({}, {"reorder": 1, "region_size": 64}, {"first_iter": 0}):
            res = run_single(gpu, parts, rowptr, edges, n, scan_variant=variant, **opts)
            assert res["iters"] == ref["iters"] and res["modularity"] == ref["modularity"], (n, deg, kw, opts)
            assert np.array_equal(res["comm"], ref["comm"][0]), (n, deg, kw, opts)
            assert [int(x) for x in res["trace"]["chash"]] == [int(x) for x in ref["trace"]["chash"]]
        if res["info"]["maxdeg"] > 2048:                  # above every tile capacity: the high-degree kernel ran, unforced
            assert res["info"]["nheavy"] > 0


@pytest.mark.parametrize("variant", VARIANTS)
def test_power_law_graphs_reach_the_high_degree_kernel_unforced(gpu, golden_rmat, variant):
    """R-MAT graphs read the way `miniVite -f` reads them: hubs of degree 3 684 / 15 706 are far above every tile
    capacity, so k_scan_heavy runs without the force_heavy_deg test hook; traces equal the unmodified reference's."""
    for name in ("rmat_s14_p1", "rmat_s17_p1"):
        case = golden_rmat[name]
        nv, parts, rowptr, edges = as_single(case)
        for opts in ({}, {"reorder": 1, "region_size": 128}):
            res = run_single(gpu, parts, rowptr, edges, nv, scan_variant=variant, **opts)
            assert res["info"]["maxdeg"] == case["maxdeg"] and res["info"]["nheavy"] > 0
            assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, None)
            assert repr(res["constant"]) == case["constant"]
