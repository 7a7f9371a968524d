"""Multi-GPU parity (needs >= 2 GPUs on one box: `python -m pytest tests -m gpu -k multi`).
p GPU ranks must reproduce, bit for bit, the golden traces of the unmodified reference run on p MPI ranks, and
-- partition invariance -- the single-rank trace of the same global graph (SURVEY.md 8(e))."""
import json
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest

from helpers import assert_trace_matches, case_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ngpus():
    from minivite_b200 import gpu as G
    return G.device_count()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, case_name, out_dir, opts):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from minivite_b200 import dist as D
    from minivite_b200 import gpu as G
    R = D.Ranks("gloo")
    if case_name == "keep_order":                # even ranks keep their numbering, odd ranks renumber (test_gpu_layout.py)
        from helpers import split_global
        from test_gpu_layout import keep_order_graph
        nv, parts, rowptr, edges = keep_order_graph(world)
        _, rps, eds = split_global(nv, rowptr, edges, world)
    elif case_name.startswith("empty_first:"):  # every rank but the last owns no vertex (tests/test_gpu_rank_counts.py)
        from helpers import global_csr, rank_cases, split_global
        nv, rowptr, edges = global_csr(rank_cases()[case_name[len("empty_first:"):]])
        parts, rps, eds = split_global(nv, rowptr, edges, 1)
        parts = np.array([0] * world + [nv], np.int64)
        rps, eds = [np.zeros(1, np.int64)] * (world - 1) + rps, [eds[0][:0]] * (world - 1) + eds
    else:
        if case_name.startswith("wexact:"):      # a dyadic-weight case of weighted_exact_traces.json
            from helpers import weighted_exact_cases
            case_name = case_name[len("wexact:"):]
            golden = weighted_exact_cases()
        elif case_name.startswith("ranks:"):     # a case of rank_traces.json (3..16 ranks, uneven splits)
            from helpers import rank_cases
            case_name = case_name[len("ranks:"):]
            golden = rank_cases()
        else:
            golden = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_traces.json")))["cases"]
        case = dict(golden[case_name])
        case["nranks"] = world                   # re-split the same global graph over `world` GPU ranks
        if case["kind"] == "rgg":
            case = dict(case, kind="file_rgg", strips=golden[case_name]["nranks"], unit_weight="-w" not in case["args"])
            if "-l" in golden[case_name]["args"]:
                raise RuntimeError("lcg cases are not re-split here")
        parts, rps, eds, keep = case_graph(case)
    ident = R.broadcast_bytes(G.get_unique_id() if rank == 0 else None, G.UNIQUE_ID_BYTES)
    g = G.LouvainGPU(rank, rank, world)
    g.comm_init(ident)
    g.set_option("trace", 1)
    for k, v in opts.items():
        g.set_option(k, v)
    g.upload(int(parts[-1]), parts, rps[rank], eds[rank])
    mod, iters = g.louvain()
    comm = g.communities()
    tr = g.trace()
    info = g.shard_info()
    allc = R.gather_arrays(comm)
    decided = R.gather_arrays(np.array([g.timings()["reordered"]], np.int64))
    if rank == 0:
        json.dump({"mod": repr(mod), "iters": iters, "trace": [[repr(float(t["modularity"])), int(t["moved"]), int(t["chash"])] for t in tr],
                   "comm": [int(x) for x in np.concatenate(allc)], "info": info, "timings": g.timings(),
                   "reordered": [int(x) for x in np.concatenate(decided)]},
                  open(os.path.join(out_dir, "res.json"), "w"))
    g.close()
    R.shutdown()


def run_ranks(tmp_path, world, case_name, **opts):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(world, _free_port(), case_name, str(tmp_path), opts), nprocs=world, join=True)
    return json.load(open(tmp_path / "res.json"))


def check(res, case, exact=True):
    trace = [{"modularity": float(m), "moved": mv, "chash": h} for m, mv, h in res["trace"]]
    assert_trace_matches(case, res["iters"], float(res["mod"]), trace, None, res["comm"] if "comm" in case else None,
                         exact=exact)


@pytest.mark.parametrize("case_name,world", [("rgg_n16384_p2", 2), ("file_rgg_n16384_s1_p2", 2), ("hand_path16_p2", 2),
                                             ("hand_clique_ring_p2", 2), ("hand_loops_multi_p2", 2), ("hand_k66_p2", 2),
                                             ("rgg_n16384_p4", 4), ("rgg_n131072_p8", 8), ("file_rgg_n32768_s8_p4", 4),
                                             ("file_balanced_n16384_p2", 2), ("file_balanced_n16384_p4", 4),
                                             # SURVEY.md 8(c) known answers of `miniVite -n 524288` (auto renumbering on)
                                             ("file_rgg_n524288_s1_p1", 2), ("file_rgg_n524288_s8_p8", 2),
                                             ("file_rgg_n524288_s8_p8", 8),
                                             # uneven rank counts (tests/golden/rank_traces.json)
                                             ("ranks:file_rgg_n16384_s1_p3", 3), ("ranks:file_rgg_n32768_s8_p5", 5),
                                             ("ranks:file_rgg_n16384_s1_p6", 6), ("ranks:hand_star41_p7", 7),
                                             ("ranks:file_rgg_n32768_s8_p7", 7)])
def test_multi_gpu_matches_reference_ranks(tmp_path, golden, case_name, world):
    if ngpus() < world:
        pytest.skip(f"needs {world} GPUs")
    res = run_ranks(tmp_path, world, case_name)
    if case_name.startswith("ranks:"):
        from helpers import rank_cases
        case = rank_cases()[case_name[len("ranks:"):]]
    else:
        case = golden[case_name]
    check(res, case)
    if world > 1 and case["kind"] not in ("hand",):
        assert res["info"]["nghost"] > 0


def test_multi_gpu_partition_invariance(tmp_path, golden):
    """2 GPUs on the 1-strip graph (most edges cross the cut) == 1-rank reference trace."""
    if ngpus() < 2:
        pytest.skip("needs 2 GPUs")
    res = run_ranks(tmp_path, 2, "rgg_n16384_p1")
    check(res, golden["rgg_n16384_p1"])


def test_multi_gpu_with_renumbering(tmp_path, golden):
    if ngpus() < 2:
        pytest.skip("needs 2 GPUs")
    for name in ("rgg_n16384_p2", "hand_clique_ring_p2", "file_rgg_n16384_s1_p2"):
        res = run_ranks(tmp_path, 2, name, reorder=1, region_size=64)
        assert res["timings"]["reordered"] == 1
        check(res, golden[name])
    res = run_ranks(tmp_path, 2, "rgg_n16384_p2", reorder=1, region_size=64, scan_variant=3)
    check(res, golden["rgg_n16384_p2"])


@pytest.mark.parametrize("world", [2, 4])
def test_multi_gpu_rank_that_keeps_its_numbering(tmp_path, world):
    """Auto mode with mixed decisions (tests/test_gpu_layout.py keep_order_graph): the even ranks keep their numbering
    while the odd ones renumber; bit-exact against the C oracle on the same shards."""
    if ngpus() < world:
        pytest.skip(f"needs {world} GPUs")
    from helpers import split_global
    from oracle import oracle as O
    from test_gpu_layout import keep_order_graph
    res = run_ranks(tmp_path, world, "keep_order")
    assert res["reordered"] == [r % 2 for r in range(world)]
    nv, parts, rowptr, edges = keep_order_graph(world)
    _, rps, eds = split_global(nv, rowptr, edges, world)
    ref = O.louvain(parts, rps, eds)
    assert res["iters"] == ref["iters"] and float(res["mod"]) == ref["modularity"]
    assert [[float(m), mv, h] for m, mv, h in res["trace"]] == \
        [[float(t["modularity"]), int(t["moved"]), int(t["chash"])] for t in ref["trace"]]
    assert res["comm"] == [int(x) for x in np.concatenate(ref["comm"])]


def test_multi_gpu_nccl_collectives_mode(tmp_path, golden):
    """comm_mode=0: the per-iteration exchanges go through NCCL (grouped send/recv all-to-all-v + all-reduce)
    instead of peer-memory stores; results are identical."""
    if ngpus() < 2:
        pytest.skip("needs 2 GPUs")
    for name in ("rgg_n16384_p2", "hand_clique_ring_p2"):
        res = run_ranks(tmp_path, 2, name, comm_mode=0)
        check(res, golden[name])
        res = run_ranks(tmp_path, 2, name, compact_upload=0)
        check(res, golden[name])
        res = run_ranks(tmp_path, 2, name, comm_mode=0, reorder=1, region_size=64)
        check(res, golden[name])
    # rank 0 owns no vertex: empty send and receive counts in every NCCL exchange
    from helpers import rank_cases
    res = run_ranks(tmp_path, 2, "empty_first:hand_clique_ring_p3", comm_mode=0)
    check(res, rank_cases()["hand_clique_ring_p3"])


def test_multi_gpu_weighted_and_heavy(tmp_path, golden):
    if ngpus() < 2:
        pytest.skip("needs 2 GPUs")
    res = run_ranks(tmp_path, 2, "file_rgg_n16384_s2_w_p2")
    assert abs(float(res["mod"]) - float(golden["file_rgg_n16384_s2_w_p2"]["modularity"])) <= 1e-6
    res = run_ranks(tmp_path, 2, "rgg_n16384_p2", force_heavy_deg=8)
    check(res, golden["rgg_n16384_p2"])
    res = run_ranks(tmp_path, 2, "rgg_n16384_p2", force_weighted=1)
    check(res, golden["rgg_n16384_p2"])


@pytest.mark.parametrize("name,world", [("rgg_n16384_s1", 2), ("rgg_n16384_s1", 4), ("rmat_s14", 2), ("rmat_s14", 4),
                                        ("random_n6000_d8_hubs3_hub_deg3000_multi200", 2), ("hand_self_loops_w", 2)])
def test_multi_gpu_weighted_exact(tmp_path, name, world):
    """Dyadic weights (tests/golden/weighted_exact_traces.json): every sum is exact, so p GPUs reproduce the 1-rank
    reference trace bit for bit, weighted remote community reads and hub tables included."""
    if ngpus() < world:
        pytest.skip(f"needs {world} GPUs")
    from helpers import weighted_exact_cases
    case = weighted_exact_cases()[name]
    for opts in ({}, {"reorder": 1, "region_size": 64}):
        res = run_ranks(tmp_path, world, "wexact:" + name, **opts)
        assert res["timings"]["unit_weight"] == 0
        check(res, case)


def test_cli_multi_gpu(tmp_path, golden):
    """bin/miniVite_b200 -g 2 -n 16384: the C++ driver (ranks = forked processes) reproduces `mpirun -n 2 miniVite -n 16384`."""
    if ngpus() < 2:
        pytest.skip("needs 2 GPUs")
    exe = os.path.join(ROOT, "bin", "miniVite_b200")
    p = subprocess.run([exe, "-g", "2", "-n", "16384", "-T", "-o", str(tmp_path / "c")], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    case = golden["rgg_n16384_p2"]
    it = re.findall(r"ITER (\d+) mod=(\S+) moved=(\d+) chash=([0-9a-f]+)", p.stderr)
    assert len(it) == case["iters"]
    for (k, m, mv, h), g in zip(it, case["trace"]):
        assert float(m) == float(g["modularity"]) and int(mv) == g["moved"] and h == g["chash"]
    assert "Modularity, #Iterations: " in p.stdout
    # same run with the graph generated on the GPUs (-D)
    p = subprocess.run([exe, "-g", "2", "-n", "16384", "-T", "-D"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    it = re.findall(r"ITER (\d+) mod=(\S+) moved=(\d+) chash=([0-9a-f]+)", p.stderr)
    assert len(it) == case["iters"] and it[-1][3] == case["trace"][-1]["chash"]


def test_full_size_config4_eight_gpus(tmp_path):
    """BASELINE.json configs[3]: RGG -n 67108864 sharded across 8 GPUs.  Golden trace: the unmodified reference on 8
    ranks reading the same graph (tests/golden/golden_full_67108864_p8.json, tools/make_fullsize_golden.py 67108864 8)."""
    if ngpus() < 8:
        pytest.skip("needs 8 GPUs")
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "golden_full_67108864_p8.json")))
    exe = os.path.join(ROOT, "bin", "miniVite_b200")
    # graph built on the host / on the GPUs; MV_CONFIG4_DEVICE_ONLY=1 skips the minutes-long host generation
    for extra in ([["-D"]] if os.environ.get("MV_CONFIG4_DEVICE_ONLY") else [[], ["-D"]]):
        p = subprocess.run([exe, "-g", "8", "-n", str(gold["nv"]), "-T"] + extra, capture_output=True, text=True, timeout=1500)
        assert p.returncode == 0, p.stderr[-2000:]
        it = re.findall(r"ITER (\d+) mod=(\S+) moved=(\d+) chash=([0-9a-f]+)", p.stderr)
        assert len(it) == gold["iters"]
        for (k, m, mv, h), g in zip(it, gold["trace"]):
            assert float(m) == float(g["modularity"]) and int(mv) == g["moved"] and h == g["chash"], k
        m = re.search(r"Modularity, #Iterations: (\S+), (\d+)", p.stdout)
        assert m and int(m.group(2)) == gold["iters"]
