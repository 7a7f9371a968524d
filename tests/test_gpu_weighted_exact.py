"""The weighted (fp64) path held to the unit path's bar: bit for bit against the unmodified reference.

The graphs of tests/golden/weighted_exact_traces.json carry dyadic weights (k * 2^-j, j <= 6; tests/helpers.py checks the
precondition).  Every degree, community degree and intra-community sum of such weights is an exact fp64 number, so the
atomics of k_fold_w and k_scan_heavy and the reference's unordered reductions all give the same bits, and the reference
itself gives one trace on every rank and thread count.  Nothing is left to a tolerance: iterations, every (modularity,
moved, hash), the final modularity, 1/(2m) and the final assignment in the caller's numbering must be identical, on every
scan variant, with and without renumbering, through the high-degree kernel, on several ranks and through the CLI.  Unlike
a unit graph run with force_weighted, a weight on the wrong edge changes these results, and the exact gain ties of the
hand-made graphs run the label tie-break and the singleton veto of the weighted path."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import assert_trace_matches, global_csr, weighted_exact_cases
from test_gpu_multirank_one_device import run_threads_case
from test_gpu_parity import gpu, run_single  # noqa: F401  (gpu is a fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = weighted_exact_cases()
VARIANTS = [3, 4, 5, 6]
# a cross-section for the option matrix: auto-renumbered RGGs, random long edges, hubs above every tile capacity,
# parallel edges and self loops, dense groups, R-MAT, and the hand-made graphs with exact ties
OPTION_CASES = ["rgg_n16384_s1", "rgg_n65536_s1", "rgg_n131072_s4", "rgg_n16384_s4_p5",
                "random_n6000_d8_hubs3_hub_deg3000_multi200", "random_n777_d150_self_loops40_multi300",
                "random_n2500_d700", "random_n4099_d30_hubs2_hub_deg1000_multi100", "rmat_s14"] + \
               sorted(k for k in CASES if k.startswith("hand_"))


def graph(name):
    case = CASES[name]
    nv, rowptr, edges = global_csr(case)
    return case, nv, rowptr, edges


def check(case, res, name, opts=None):
    from oracle import oracle as O
    what = (name, opts)
    assert res["timings"]["unit_weight"] == 0, what
    assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], O.comm_hash(0, res["comm"]),
                         res["comm"], exact=True)
    assert repr(res["modularity"]) == repr(float(case["modularity"])), what
    assert repr(res["constant"]) == case["constant"], what


def run(G, name, **opts):
    case, nv, rowptr, edges = graph(name)
    res = run_single(G, np.array([0, nv], np.int64), rowptr, edges, nv, **opts)
    check(case, res, name, opts)
    return res


def test_every_case_matches_reference_and_oracle(gpu):
    """Default options (scan variant 6, auto renumbering): golden and C oracle, bit for bit.  From 65 536 vertices the
    RGG numbering has no locality and the shard is renumbered (k_permute_adj's weight copy); hubs above 2 048 edges
    reach k_scan_heavy without the force_heavy_deg hook."""
    from oracle import oracle as O
    for name, case in CASES.items():
        case, nv, rowptr, edges = graph(name)
        res = run_single(gpu, np.array([0, nv], np.int64), rowptr, edges, nv)
        check(case, res, name)
        ref = O.louvain(np.array([0, nv], np.int64), [rowptr], [edges])
        assert res["iters"] == ref["iters"] and res["modularity"] == ref["modularity"], name
        assert np.array_equal(res["comm"], ref["comm"][0]), name
        assert [int(x) for x in res["trace"]["chash"]] == [int(x) for x in ref["trace"]["chash"]], name
        assert res["info"]["maxdeg"] == case["maxdeg"], name
        if case["maxdeg"] > 2048:
            assert res["info"]["nheavy"] > 0, name
        if case["kind"] == "dyadic_rgg" and nv >= 65536:
            assert res["timings"]["reordered"] == 1, name


@pytest.mark.parametrize("variant", VARIANTS)
def test_scan_variants(gpu, variant):
    """Every shipped neighbour scan on every case, with and without renumbering: the weighted k_scan_pw (12-byte
    records in 316-edge staging buffers, sub-ranges on the dense groups), k_scan_ws, k_scan_pq and the default."""
    for name, case in CASES.items():
        res = run(gpu, name, scan_variant=variant)
        if case["maxdeg"] > 2048:
            assert res["info"]["nheavy"] > 0, (name, variant)
        res = run(gpu, name, scan_variant=variant, reorder=0)
        assert res["timings"]["reordered"] == 0, (name, variant)


@pytest.mark.parametrize("region", [32, 64, 4096])
def test_forced_renumbering(gpu, region):
    """reorder=1 renumbers every shard (k_permute_adj copies the weights next to the tails); results in the caller's
    numbering stay bit-identical, also when the renumbering meets the scan variants that stage weights differently."""
    for name in OPTION_CASES:
        for variant in (3, 6):
            res = run(gpu, name, reorder=1, region_size=region, scan_variant=variant)
            assert res["timings"]["reordered"] == 1, (name, region)


@pytest.mark.parametrize("thr", [2, 8])
def test_forced_high_degree_kernel(gpu, thr):
    """force_heavy_deg sends every vertex above `thr` edges through k_scan_heavy's weighted hash table, alone and after
    a renumbering; with exact sums its fp64 atomics are order-free."""
    for name in OPTION_CASES:
        for opts in ({}, {"reorder": 1, "region_size": 64}, {"reorder": 1, "region_size": 64, "scan_variant": 3}):
            res = run(gpu, name, force_heavy_deg=thr, **opts)
            if res["info"]["maxdeg"] > thr:
                assert res["info"]["nheavy"] > 0, (name, thr, opts)


def test_upload_formats(gpu):
    """Weighted shards always ship the full 16-byte records, whatever compact_upload asks for."""
    for name in ("rgg_n65536_s1", "random_n777_d150_self_loops40_multi300", "hand_self_loops_w", "rmat_s14"):
        case, nv, rowptr, edges = graph(name)
        for cu, extra in ((0, {}), (1, {"host_threads": 4}), (2, {"upload_chunk": 1024, "host_threads": 3})):
            res = run(gpu, name, compact_upload=cu, **extra)
            assert res["timings"]["h2d_bytes"] == 8 * (nv + 1) + 16 * len(edges), (name, cu)


def test_one_call_seam(gpu):
    """mvgpu_dist_louvain_method (distLouvainMethod with host arrays) on weighted graphs."""
    from oracle import oracle as O
    L = gpu.lib()
    for name in ("rgg_n65536_s1", "random_n6000_d8_hubs3_hub_deg3000_multi200", "hand_zero_w", "hand_k66_half"):
        case, nv, rowptr, edges = graph(name)
        iters, mod = ctypes.c_int(0), ctypes.c_double(0)
        comm = np.zeros(nv, np.int64)
        rc = L.mvgpu_dist_louvain_method(0, nv, len(edges), rowptr.ctypes.data, edges.ctypes.data, -1.0, 1e-6,
                                         ctypes.byref(iters), ctypes.byref(mod), comm.ctypes.data)
        assert rc == 0, L.mvgpu_last_error()
        assert iters.value == case["iters"] and repr(mod.value) == repr(float(case["modularity"])), name
        assert "%016x" % O.comm_hash(0, comm) == case["final_chash"], name
        if "comm" in case:
            assert [int(x) for x in comm] == case["comm"], name


@pytest.mark.parametrize("name,world", [("rgg_n16384_s1", 2), ("rgg_n16384_s1", 3), ("rgg_n16384_s1", 4),
                                        ("rmat_s14", 2), ("rmat_s14", 3), ("rmat_s14", 4), ("rgg_n16384_s4_p5", 4),
                                        ("random_n6000_d8_hubs3_hub_deg3000_multi200", 2), ("hand_star40_mixed", 2),
                                        ("hand_self_loops_w", 2), ("hand_k66_half", 3)])
def test_ranks_on_one_device(name, world):
    """Ranks sharing device 0: the 1-rank reference trace on 2, 3 and 4 ranks (partition invariance).  Most RGG edges
    cross the cuts of the 1-strip graph, and R-MAT hubs read their neighbours' communities (cinfo_w) from other ranks."""
    from oracle import oracle as O
    case = CASES[name]
    res = run_threads_case(dict(case, nranks=world))
    assert res["timings"]["unit_weight"] == 0
    assert_trace_matches(case, res["iters"], res["mod"], res["trace"], O.comm_hash(0, res["comm"]), res["comm"])
    assert all(i["nghost"] > 0 for i in res["info"]), res["info"]
    if case["maxdeg"] > 2048:
        assert sum(i["nheavy"] for i in res["info"]) > 0


def test_ranks_on_one_device_with_options():
    case = CASES["rmat_s14"]
    for opts in ({"scan_variant": 3}, {"reorder": 1, "region_size": 64}, {"force_heavy_deg": 8, "reorder": 1},
                 {"compact_upload": 2}):
        res = run_threads_case(dict(case, nranks=2), **opts)
        assert_trace_matches(case, res["iters"], res["mod"], res["trace"], None, None)


def test_cli_reads_weighted_file(tmp_path):
    """bin/miniVite_b200 -f on a written dyadic graph file: trace lines and result equal the reference's."""
    from minivite_b200 import hostgraph as hg
    exe = os.path.join(ROOT, "bin", "miniVite_b200")
    for name in ("rgg_n65536_s4", "random_n4099_d30_hubs2_hub_deg1000_multi100", "hand_self_loops_w"):
        case, nv, rowptr, edges = graph(name)
        path = str(tmp_path / (name + ".bin"))
        hg.write_graph_arrays(path, nv, rowptr, edges["tail"], edges["weight"])
        p = subprocess.run([exe, "-f", path, "-T"], capture_output=True, text=True, timeout=300)
        assert p.returncode == 0, p.stderr[-2000:]
        it = re.findall(r"ITER (\d+) mod=(\S+) moved=(\d+) chash=([0-9a-f]+)", p.stderr)
        assert [(float(a[1]), int(a[2]), a[3]) for a in it] == \
            [(float(g["modularity"]), g["moved"], g["chash"]) for g in case["trace"]], name
        m = re.search(r"RESULT mod=(\S+) iters=(\d+)", p.stderr)
        assert float(m.group(1)) == float(case["modularity"]) and int(m.group(2)) == case["iters"], name
