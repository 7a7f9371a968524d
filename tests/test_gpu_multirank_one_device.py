"""The multi-rank code paths -- ghost discovery (exchangeVertexReqs, dspl.hpp:1106-1272), the per-iteration ghost
vertex->community exchange (fillRemoteCommunities, dspl.hpp:488-952) and the remote community reads / delta pushes
(updateRemoteCommunities, dspl.hpp:978-1103) -- on a box with ONE GPU: p ranks share device 0.  NCCL refuses two ranks
on one device, so the setup exchanges use the library's host transport (option host_transport=1, a shared-memory
segment); the per-iteration data plane is the same peer-memory kernels a multi-GPU run uses (stores into the peers'
ghost slots, flag barrier, flag all-reduce, atomics into the owner's arrays) -- the peers' arrays simply live on the
same device.  p ranks must reproduce the unmodified reference's p-rank golden traces bit for bit.
Ranks are threads of this process (kernels of different ranks run concurrently on their own streams) or, in the
last test, separate processes (arrays mapped through CUDA IPC; the ranks time-slice the GPU)."""
import json
import os
import sys
import threading

import numpy as np
import pytest

from helpers import assert_trace_matches, case_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def resplit(golden, case_name, world):
    case = dict(golden[case_name])
    case["nranks"] = world
    if case["kind"] == "rgg":
        case = dict(case, kind="file_rgg", strips=golden[case_name]["nranks"], unit_weight="-w" not in case["args"])
    return case_graph(case)


def run_threads(golden, case_name, world, **opts):
    from minivite_b200 import gpu as G
    parts, rps, eds, keep = resplit(golden, case_name, world)
    ident = G.get_unique_id()
    out, errs = [None] * world, []

    def work(rank):
        try:
            g = G.LouvainGPU(0, rank, world)
            g.set_option("host_transport", 1)
            g.set_option("trace", 1)
            for k, v in opts.items():
                g.set_option(k, v)
            g.comm_init(ident)
            g.upload(int(parts[-1]), parts, rps[rank], eds[rank])
            mod, iters = g.louvain()
            out[rank] = {"mod": mod, "iters": iters, "trace": g.trace(), "comm": g.communities().copy(), "info": g.shard_info(),
                         "timings": g.timings()}
            g.close()
        except Exception as ex:          # a failing rank must not leave its peers waiting forever: report and bail out
            errs.append((rank, repr(ex)))
    th = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    assert all(o is not None for o in out), "a rank did not finish"
    r0 = out[0]
    for o in out[1:]:
        assert o["iters"] == r0["iters"] and o["mod"] == r0["mod"]
    return {"mod": r0["mod"], "iters": r0["iters"], "trace": r0["trace"], "comm": np.concatenate([o["comm"] for o in out]),
            "info": [o["info"] for o in out], "timings": r0["timings"]}


def check(res, case):
    assert_trace_matches(case, res["iters"], res["mod"], res["trace"], None, res["comm"] if "comm" in case else None)


@pytest.mark.parametrize("case_name,world", [("rgg_n16384_p2", 2), ("file_rgg_n16384_s1_p2", 2), ("hand_path16_p2", 2),
                                             ("hand_clique_ring_p2", 2), ("hand_loops_multi_p2", 2), ("hand_k66_p2", 2),
                                             ("rgg_n16384_p4", 4), ("rgg_n131072_p8", 8), ("file_rgg_n32768_s8_p4", 4),
                                             ("file_balanced_n16384_p2", 2), ("file_balanced_n16384_p4", 4),
                                             ("file_rgg_n524288_s8_p8", 8)])
def test_ranks_on_one_device_match_reference_ranks(golden, case_name, world):
    res = run_threads(golden, case_name, world)
    check(res, golden[case_name])
    if golden[case_name]["kind"] != "hand":
        assert all(i["nghost"] > 0 for i in res["info"])


def test_partition_invariance_on_one_device(golden):
    """4 ranks on the 1-strip graph (most edges cross the cuts) == the 1-rank reference trace."""
    check(run_threads(golden, "rgg_n16384_p1", 4), golden["rgg_n16384_p1"])


def test_options_on_one_device(golden):
    for opts in ({"reorder": 1, "region_size": 64}, {"scan_variant": 3}, {"scan_variant": 4}, {"scan_variant": 3, "reorder": 1, "region_size": 64},
                 {"first_iter": 0}, {"force_heavy_deg": 8}, {"force_weighted": 1}, {"compact_upload": 1}):
        check(run_threads(golden, "rgg_n16384_p2", 2, **opts), golden["rgg_n16384_p2"])
    # dyadic weights (k/4, self loops 2.5 and 0.75): every sum is exact, so the weighted path is bit-exact across ranks
    for name in ("hand_weighted20_p1", "hand_weighted20_p2"):
        for opts in ({}, {"scan_variant": 3}, {"force_heavy_deg": 2}):
            res = run_threads(golden, name, 2, **opts)
            assert res["timings"]["unit_weight"] == 0
            check(res, golden[name])
    # Euclidean weights are not exactly representable: the sums' last bits depend on their order, hence the tolerance
    res = run_threads(golden, "file_rgg_n16384_s2_w_p2", 2)
    assert abs(res["mod"] - float(golden["file_rgg_n16384_s2_w_p2"]["modularity"])) <= 1e-6


def _proc_worker(rank, world, port, case_name, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from minivite_b200 import dist as D
    from minivite_b200 import gpu as G
    R = D.Ranks("gloo")
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_traces.json")))["cases"]
    parts, rps, eds, keep = resplit(golden, case_name, world)
    ident = R.broadcast_bytes(G.get_unique_id() if rank == 0 else None, G.UNIQUE_ID_BYTES)
    g = G.LouvainGPU(0, rank, world)                      # every rank on device 0
    g.set_option("host_transport", 1)
    g.set_option("trace", 1)
    g.comm_init(ident)
    g.upload(int(parts[-1]), parts, rps[rank], eds[rank])
    mod, iters = g.louvain()
    allc = R.gather_arrays(g.communities())
    tr = g.trace()
    if rank == 0:
        json.dump({"mod": repr(mod), "iters": iters, "comm": [int(x) for x in np.concatenate(allc)],
                   "trace": [[repr(float(t["modularity"])), int(t["moved"]), int(t["chash"])] for t in tr]},
                  open(os.path.join(out_dir, "res.json"), "w"))
    g.close()
    R.shutdown()


def test_rank_processes_sharing_one_device(tmp_path, golden):
    """Ranks as separate processes (what torchrun / the CLI start), all on device 0: peers' arrays arrive through CUDA IPC."""
    import torch.multiprocessing as mp
    from test_gpu_multi import _free_port
    mp.spawn(_proc_worker, args=(2, _free_port(), "rgg_n16384_p2", str(tmp_path)), nprocs=2, join=True)
    res = json.load(open(tmp_path / "res.json"))
    trace = [{"modularity": float(m), "moved": mv, "chash": h} for m, mv, h in res["trace"]]
    assert_trace_matches(golden["rgg_n16384_p2"], res["iters"], float(res["mod"]), trace, None, res["comm"])


def run_threads_case(case, **opts):
    """like run_threads, for a case dictionary that is not in ref_traces.json"""
    return run_threads({"_": case}, "_", case["nranks"], **opts)


@pytest.mark.parametrize("name", ["rmat_s14_p2", "rmat_s14_p2_b", "rmat_s17_p4_b"])
def test_power_law_graph_ranks_on_one_device(golden_rmat, name):
    """`-f` R-MAT graph on 2 / 4 ranks, plain and edge-balanced (-b) partitions: hubs whose neighbours live on other
    ranks go through the high-degree kernel with remote community reads."""
    case = golden_rmat[name]
    res = run_threads_case(case)
    assert_trace_matches(case, res["iters"], res["mod"], res["trace"], None, None)
    assert sum(i["nheavy"] for i in res["info"]) > 0
