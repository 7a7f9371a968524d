"""GPU parity tests (run on an H100 with -m gpu): the CUDA path, called through the C ABI,
against the golden traces of the unmodified reference and against the C oracle on the same inputs.
Bar: bit-exact community ids, iteration counts, moved counts and modularity for unit weights and for dyadic weights
(k * 2^-j: every sum exact); |dQ| <= 1e-6 (BASELINE.json north_star tolerance) for the Euclidean weights of the -w RGGs,
whose sums depend on the order of the additions."""
import numpy as np
import pytest

from helpers import assert_trace_matches, case_graph, dyadic_exponent

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    from minivite_b200 import gpu as G
    if G.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on the GPU box")
    return G


def run_single(G, parts, rowptr, edges, nv, **opts):
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        for k, v in opts.items():
            g.set_option(k, v)
        g.upload(nv, parts, rowptr, edges)
        mod, iters = g.louvain(-1.0, 1.0e-6)
        return {"modularity": mod, "iters": iters, "trace": g.trace(), "comm": g.communities(),
                "constant": g.constant(), "timings": g.timings(), "info": g.shard_info()}
    finally:
        g.close()


def as_single(case):
    """Merge a golden case's shards into one rank-0 shard (results are partition invariant for unit weights)."""
    parts, rps, eds, keep = case_graph(case)
    nv = int(parts[-1])
    rowptr = np.concatenate([[0]] + [rp[1:] + off for rp, off in zip(rps, np.cumsum([0] + [len(e) for e in eds[:-1]]))])
    edges = np.concatenate(eds) if len(eds) > 1 else eds[0]
    return nv, np.array([0, nv], np.int64), rowptr.astype(np.int64), edges


def is_weighted(name, case):
    return name.endswith("_w") or "_w_" in name or "weighted" in name or case.get("unit_weight") is False


def test_unit_weight_cases_bit_exact(gpu, golden):
    from oracle import oracle as O
    ran = 0
    for name, case in golden.items():
        if is_weighted(name, case):
            continue
        nv, parts, rowptr, edges = as_single(case)
        res = run_single(gpu, parts, rowptr, edges, nv)
        assert res["timings"]["unit_weight"] == 1, name
        h = O.comm_hash(0, res["comm"])
        assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], h, res["comm"])
        assert repr(res["constant"]) == case["constant"], name
        ran += 1
    assert ran >= 20


def test_weighted_cases(gpu, golden):
    """fp64 path.  Dyadic weights (hand_weighted20: k/4, self loops 2.5 and 0.75) make every sum exact, so the order of
    the additions cannot matter: bit-exact, and the 2-rank golden too (it equals the 1-rank one).  The Euclidean weights
    of the -w RGGs are not exactly representable: community degrees are folded with atomics (any order) and the
    reference's reductions are unordered too (its own results differ in the last bits between rank counts), so those
    keep the 1e-6 modularity tolerance.  tests/test_gpu_weighted_exact.py holds many more dyadic graphs to the exact bar."""
    from oracle import oracle as O
    exact = 0
    for name, case in golden.items():
        if not is_weighted(name, case):
            continue
        nv, parts, rowptr, edges = as_single(case)
        if dyadic_exponent(edges["weight"]) is not None:
            res = run_single(gpu, parts, rowptr, edges, nv)
            assert res["timings"]["unit_weight"] == 0, name
            assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], O.comm_hash(0, res["comm"]), res["comm"])
            assert repr(res["constant"]) == case["constant"], name
            exact += 1
        elif case["nranks"] == 1:
            res = run_single(gpu, parts, rowptr, edges, nv)
            assert res["timings"]["unit_weight"] == 0, name
            assert abs(res["modularity"] - float(case["modularity"])) <= 1e-6, name
            assert abs(res["iters"] - case["iters"]) <= 2, name
    assert exact == 2


def test_fp64_path_on_unit_graph_is_bit_exact(gpu, golden):
    """force_weighted runs the general fp64 kernels on a unit-weight graph: every sum is an exact integer,
    so the trace must again be bit-identical to the reference."""
    case = golden["rgg_n16384_p1"]
    nv, parts, rowptr, edges = as_single(case)
    res = run_single(gpu, parts, rowptr, edges, nv, force_weighted=1)
    assert res["timings"]["unit_weight"] == 0
    assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, None)


def test_high_degree_kernel(gpu, golden):
    """force_heavy_deg routes vertices above a small degree through the high-degree (hash table) kernel."""
    for name, thr in (("hand_star41_p1", 8), ("rgg_n16384_p1", 8), ("hand_k66_p1", 4), ("hand_loops_multi_p1", 2)):
        case = golden[name]
        nv, parts, rowptr, edges = as_single(case)
        res = run_single(gpu, parts, rowptr, edges, nv, force_heavy_deg=thr)
        assert res["info"]["nheavy"] > 0, (name, res["info"])
        assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, res["comm"])
    case = golden["rgg_n16384_p1"]
    nv, parts, rowptr, edges = as_single(case)
    res = run_single(gpu, parts, rowptr, edges, nv, force_heavy_deg=8, force_weighted=1)
    assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, None)


def test_against_oracle_on_fresh_graphs(gpu):
    """Seeded inputs that are not in the golden file: CUDA path vs C oracle, sizes the oracle finishes in seconds."""
    from minivite_b200 import hostgraph as hg
    from oracle import oracle as O
    for n, p, kw in [(8192, 1, {}), (262144, 1, {}), (131072, 4, {}), (65536, 1, {"random_edge_percent": 5.0}),
                     (65536, 2, {"lcg": True})]:
        ss = hg.generate_rgg(n, p, **kw)
        parts = ss.shards[0].parts
        ref = O.louvain(parts, [s.rowptr for s in ss.shards], [s.edges for s in ss.shards])
        rowptr = np.concatenate([[0]] + [s.rowptr[1:] + off for s, off in
                                         zip(ss.shards, np.cumsum([0] + [s.lne for s in ss.shards[:-1]]))])
        edges = np.concatenate([s.edges for s in ss.shards])
        res = run_single(gpu, np.array([0, n], np.int64), rowptr.astype(np.int64), edges, n)
        assert res["iters"] == ref["iters"] and res["modularity"] == ref["modularity"], (n, p, kw)
        assert np.array_equal(res["comm"], np.concatenate(ref["comm"]))
        assert [int(x) for x in res["trace"]["chash"]] == [int(x) for x in ref["trace"]["chash"]]
        assert [int(x) for x in res["trace"]["moved"]] == [int(x) for x in ref["trace"]["moved"]]


def test_edge_cases(gpu):
    from oracle import oracle as O
    EDGE = np.dtype([("tail", "<i8"), ("weight", "<f8")])
    # graph without edges: 1/(2m) is infinite and the modularity NaN, so the reference's exit test
    # (dspl.hpp:1401) never fires and the reference spins forever; we stop at max_iters with an error instead
    from minivite_b200 import gpu as G
    g = G.LouvainGPU(0, 0, 1)
    g.set_option("max_iters", 50)
    g.upload(5, np.array([0, 5], np.int64), np.zeros(6, np.int64), np.zeros(0, EDGE))
    with pytest.raises(G.MvgpuError):
        g.louvain()
    g.close()
    # isolated vertices next to real edges (degree 0 -> target = current community, dspl.hpp:323-324)
    ed = np.zeros(2, EDGE)
    ed["tail"] = [3, 1]
    ed["weight"] = 1.0
    rp = np.array([0, 0, 1, 1, 2, 2], np.int64)
    res = run_single(gpu, np.array([0, 5], np.int64), rp, ed, 5)
    ref = O.louvain(np.array([0, 5], np.int64), [rp], [ed])
    assert res["iters"] == ref["iters"] and res["modularity"] == ref["modularity"]
    assert list(res["comm"]) == list(ref["comm"][0])
    # bad input: tail out of range -> error, not a crash
    g = G.LouvainGPU(0, 0, 1)
    ed = np.zeros(2, EDGE)
    ed["tail"] = [1, 7]
    ed["weight"] = 1.0
    g.upload(2, np.array([0, 2], np.int64), np.array([0, 1, 2], np.int64), ed)
    with pytest.raises(G.MvgpuError):
        g.louvain()
    g.close()


def test_one_call_seam(gpu, golden):
    """mvgpu_dist_louvain_method == distLouvainMethod(me=0, nprocs=1, g, ...) with host arrays."""
    import ctypes
    case = golden["rgg_n16384_p1"]
    nv, parts, rowptr, edges = as_single(case)
    L = gpu.lib()
    iters = ctypes.c_int(0)
    mod = ctypes.c_double(0)
    comm = np.zeros(nv, np.int64)
    rc = L.mvgpu_dist_louvain_method(0, nv, len(edges), rowptr.ctypes.data, edges.ctypes.data, -1.0, 1e-6,
                                     ctypes.byref(iters), ctypes.byref(mod), comm.ctypes.data)
    assert rc == 0, L.mvgpu_last_error()
    assert iters.value == case["iters"] and mod.value == float(case["modularity"])


def test_scan_variants_agree(gpu, golden):
    """k_scan_pw (4, default) and k_scan_ws (3) give the same golden trace; cache-policy settings never change results.
    (tests/test_gpu_scan_kernels.py runs every golden case and the unusual graphs through both.)"""
    case = golden["rgg_n65536_p1"]
    nv, parts, rowptr, edges = as_single(case)
    for opts in ({"scan_variant": 3, "cache_policy": 0}, {"scan_variant": 3}, {"scan_variant": 3, "reorder": 1},
                 {"scan_variant": 3, "force_weighted": 1}, {"scan_variant": 4}, {"scan_variant": 4, "reorder": 1},
                 {"scan_variant": 4, "force_weighted": 1}, {"scan_variant": 3, "force_heavy_deg": 8, "reorder": 1},
                 {"scan_variant": 4, "force_weighted": 1, "reorder": 1}):
        res = run_single(gpu, parts, rowptr, edges, nv, **opts)
        assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, None)
    for name in ("hand_weighted20_p1", "rgg_n16384_p1_w", "hand_loops_multi_p1", "hand_star41_p1", "hand_k66_p1"):
        case = golden[name]
        nv, parts, rowptr, edges = as_single(case)
        for var in (3, 4):
            res = run_single(gpu, parts, rowptr, edges, nv, scan_variant=var)
            if dyadic_exponent(edges["weight"]) is not None:       # unit and dyadic weights: exact sums, exact results
                assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, res["comm"])
            else:
                assert abs(res["modularity"] - float(case["modularity"])) <= 1e-6 and res["iters"] == case["iters"], (name, var)
    g = gpu.LouvainGPU(0, 0, 1)
    with pytest.raises(gpu.MvgpuError):
        g.set_option("scan_variant", 0)              # the first-generation kernel is gone
    g.close()


def test_full_size_config2_matches_reference_trace(gpu):
    """BASELINE.json configs[1]: RGG -n 16777216 on one GPU.  The golden trace was produced by the unmodified
    reference (oracle/_ref, 128 host threads, tools/make_fullsize_golden.py) on the same graph file."""
    import json
    import os
    from minivite_b200 import hostgraph as hg
    from oracle import oracle as O
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_full_16777216_p1.json")))
    ss = hg.generate_rgg(gold["nv"], 1)
    sh = ss.shards[0]
    assert sh.lne == gold["ne"]
    res = run_single(gpu, sh.parts, sh.rowptr, sh.edges, gold["nv"])
    assert res["iters"] == gold["iters"]
    assert repr(res["modularity"]) == repr(float(gold["modularity"]))
    for t, g in zip(res["trace"], gold["trace"]):
        assert float(t["modularity"]) == float(g["modularity"]) and int(t["moved"]) == g["moved"]
        assert int(t["chash"]) == int(g["chash"], 16)
    assert "%016x" % O.comm_hash(0, res["comm"]) == gold["final_chash"]
    # size-independent properties: community ids are vertex ids of members' lineage, sizes add up
    comm = res["comm"]
    assert comm.min() >= 0 and comm.max() < gold["nv"]


def test_locality_renumbering_keeps_results(gpu, golden):
    """reorder=1 renumbers vertices by BFS regions (layout only): traces, final assignment (in the caller's
    numbering, as original ids) and modularity must stay bit-identical to the reference, for every kernel variant."""
    names = ["rgg_n16384_p1", "rgg_n65536_p1", "hand_path16_p1", "hand_two_triangles_p1", "hand_k66_p1",
             "hand_loops_multi_p1", "hand_clique_ring_p1", "hand_star41_p1", "file_rgg_n32768_s8_p1", "rgg_n16384_p2_l"]
    for name in names:
        case = golden[name]
        nv, parts, rowptr, edges = as_single(case)
        for opts in ({"reorder": 1, "region_size": 64}, {"reorder": 1, "region_size": 4096, "scan_variant": 3},
                     {"reorder": 1, "region_size": 32, "force_heavy_deg": 3}):
            res = run_single(gpu, parts, rowptr, edges, nv, **opts)
            assert res["timings"]["reordered"] == 1, (name, opts)
            assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, res["comm"])
    case = golden["rgg_n16384_p1"]
    nv, parts, rowptr, edges = as_single(case)
    res = run_single(gpu, parts, rowptr, edges, nv, reorder=1, force_weighted=1)
    assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, res["comm"] if "comm" in case else None)
    # weighted graph: renumbering keeps the per-vertex edge order, so sums round the same way
    case = golden["rgg_n16384_p1_w"]
    nv, parts, rowptr, edges = as_single(case)
    res = run_single(gpu, parts, rowptr, edges, nv, reorder=1, region_size=128)
    assert abs(res["modularity"] - float(case["modularity"])) <= 1e-6


def test_upload_formats_agree(gpu, golden):
    """mvgpu_upload_shard narrows unit-weight shards to 4-byte tails on the host (compact_upload=1) or ships
    the 16-byte records (0, default); weighted shards always take the full records.  Same results either way."""
    for name in ("rgg_n65536_p1", "hand_loops_multi_p1", "file_balanced_n16384_p4"):
        case = golden[name]
        nv, parts, rowptr, edges = as_single(case)
        for cu in (0, 1):
            res = run_single(gpu, parts, rowptr, edges, nv, compact_upload=cu, host_threads=4)
            assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, None)
            assert res["timings"]["h2d_bytes"] == 8 * (nv + 1) + (4 if cu else 16) * len(edges)
        # compact_upload=2: host threads narrow chunks from the front while the copy engine takes raw chunks from the back
        # (narrowed on the device); small chunks so that both ends are busy on a test-sized graph
        for threads, chunk in ((1, 256), (3, 1024), (8, 4096)):
            res = run_single(gpu, parts, rowptr, edges, nv, compact_upload=2, host_threads=threads, upload_chunk=chunk)
            assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], None, None)
            lo, hi = 8 * (nv + 1) + 4 * len(edges), 8 * (nv + 1) + 16 * len(edges)
            assert lo <= res["timings"]["h2d_bytes"] <= hi
    case = golden["rgg_n16384_p1_w"]
    nv, parts, rowptr, edges = as_single(case)
    for cu, extra in ((1, {}), (2, {"upload_chunk": 1024, "host_threads": 2})):
        res = run_single(gpu, parts, rowptr, edges, nv, compact_upload=cu, **extra)
        assert res["timings"]["h2d_bytes"] == 8 * (nv + 1) + 16 * len(edges) and res["timings"]["unit_weight"] == 0


def test_full_size_config3_random_edges(gpu):
    """BASELINE.json configs[2]: RGG -n 16777216 -p 2 (2 % random long edges, fixed documented seed) on one GPU, against
    the golden trace of the unmodified reference on the same graph file (tools/make_fullsize_golden.py ... 2)."""
    import json
    import os
    from minivite_b200 import hostgraph as hg
    from oracle import oracle as O
    path = os.path.join(os.path.dirname(__file__), "golden", "golden_full_16777216_p1_r2.json")
    if not os.path.exists(path):
        pytest.skip("config-3 golden not generated yet")
    gold = json.load(open(path))
    ss = hg.generate_rgg(gold["nv"], 1, random_edge_percent=gold["random_edge_percent"])
    sh = ss.shards[0]
    assert sh.lne == gold["ne"]
    res = run_single(gpu, sh.parts, sh.rowptr, sh.edges, gold["nv"])
    assert res["iters"] == gold["iters"] and repr(res["modularity"]) == repr(float(gold["modularity"]))
    for t, g in zip(res["trace"], gold["trace"]):
        assert float(t["modularity"]) == float(g["modularity"]) and int(t["moved"]) == g["moved"]
        assert int(t["chash"]) == int(g["chash"], 16)
    assert "%016x" % O.comm_hash(0, res["comm"]) == gold["final_chash"]


def test_full_size_config4_on_one_gpu():
    """BASELINE.json configs[3] (RGG -n 67108864 built on 8 strips) also fits ONE 80 GB H100: unit-weight results are
    partition invariant, so a single GPU must reproduce the 8-rank reference trace
    (tests/golden/golden_full_67108864_p8.json).  12.4 GB of host graph: opt-in with MV_BIG_TESTS=1."""
    import json
    import os
    if os.environ.get("MV_BIG_TESTS") != "1":
        pytest.skip("set MV_BIG_TESTS=1 (12 GB host graph, about a minute)")
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_full_67108864_p8.json")))
    ss = hg.generate_rgg(gold["nv"], gold["strips"])
    offs = np.cumsum([0] + [s.lne for s in ss.shards[:-1]])
    rowptr = np.concatenate([[0]] + [s.rowptr[1:] + off for s, off in zip(ss.shards, offs)]).astype(np.int64)
    edges = np.concatenate([s.edges for s in ss.shards])
    ss.close()
    assert len(edges) == gold["ne"]
    res = run_single(G, np.array([0, gold["nv"]], np.int64), rowptr, edges, gold["nv"])
    assert res["iters"] == gold["iters"] and repr(res["modularity"]) == repr(float(gold["modularity"]))
    for t, g in zip(res["trace"], gold["trace"]):
        assert float(t["modularity"]) == float(g["modularity"]) and int(t["moved"]) == g["moved"]
        assert int(t["chash"]) == int(g["chash"], 16)


@pytest.mark.parametrize("name,ncomm,fnv", [("rgg_n16384_p1", 1953, "2788b5ffe2f49136"),
                                            ("rgg_n65536_p1", 6889, "3cf802502bc50070"),
                                            ("file_rgg_n524288_s1_p1", 48778, "188df44bd1f5b787")])
def test_final_assignment_matches_survey_known_answers(gpu, golden, name, ncomm, fnv):
    """SURVEY.md 8(c): community count and FNV-1a hash of the final currComm as captured from the unmodified reference
    in the survey's own probe session (independent of this repo's hash and hooks)."""
    nv, parts, rowptr, edges = as_single(golden[name])
    comm = run_single(gpu, parts, rowptr, edges, nv)["comm"]
    h = 1469598103934665603
    for v in comm.tolist():
        h = ((h ^ (v & 0xFFFFFFFFFFFFFFFF)) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    assert len(np.unique(comm)) == ncomm and "%016x" % h == fnv
