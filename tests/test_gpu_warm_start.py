"""Warm start and checkpoint / resume of the Louvain phase (mvgpu_set_initial_communities, option stop_after), on the GPU.

A run stopped after its accepted iteration k and resumed from its assignment with lower = its returned modularity must
continue the reference's run exactly (DESIGN.md §3.9; tests/test_oracle_warm_start.py checks that argument on the C
oracle).  So every unit and dyadic golden trace doubles as a split-and-resume test: the stopped run must give the
golden prefix and the oracle's checkpoint assignment C_k array for array, the resumed run the golden suffix, iteration
count, modularity and final hash bit for bit.  Arbitrary starting assignments are checked against the C oracle
started from the same assignment, on 1 rank and on 2 and 4 ranks sharing device 0 (host transport)."""
import json
import os
import re
import subprocess
import sys
import threading

import numpy as np
import pytest

from helpers import case_graph, exact_cases, random_graph, split_global
from oracle import oracle as O
from test_gpu_parity import gpu  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
EXE = os.path.join(ROOT, "bin", "miniVite_b200")
CASES = exact_cases()


def split_points(iters):
    return sorted({k for k in (1, iters // 2, iters - 1) if 1 <= k <= iters - 1})


def golden_trace(case):
    return [(float(t["modularity"]), int(t["moved"]), int(t["chash"], 16)) for t in case["trace"]]


def as_trace(tr):
    return [(float(t["modularity"]), int(t["moved"]), int(t["chash"])) for t in tr]


def layout_info(g):
    """(first_ran, relabel) of the last run, from the library's layout read-back hook."""
    import ctypes
    from minivite_b200 import gpu as G
    f = G.lib().mv_layout_readback
    f.argtypes = [ctypes.c_void_p] * 11
    f.restype = ctypes.c_int
    info = (ctypes.c_int64 * 16)()
    G._ck(f(g._h, info, *[None] * 9))
    return int(info[10]), int(info[1])


class Ranks:
    """`world` ranks of one graph on device 0: world == 1 is a plain context, world > 1 are threads of this process
    whose setup exchanges go through the host transport.  Every call runs on all ranks and returns their results."""

    def __init__(self, parts, rps, eds, **opts):
        from minivite_b200 import gpu as G
        self.world = len(rps)
        self.parts = np.asarray(parts, np.int64)
        self.g = [G.LouvainGPU(0, r, self.world) for r in range(self.world)]
        ident = G.get_unique_id() if self.world > 1 else None
        for r, g in enumerate(self.g):
            if self.world > 1:
                g.set_option("host_transport", 1)
            g.set_option("trace", 1)
            for k, v in opts.items():
                g.set_option(k, v)
        self.each(lambda r, g: self.world > 1 and g.comm_init(ident))
        self.each(lambda r, g: g.upload(int(self.parts[-1]), self.parts, rps[r], eds[r]))

    def each(self, fn):
        if self.world == 1:
            return [fn(0, self.g[0])]
        out, errs = [None] * self.world, []

        def work(r):
            try:
                out[r] = fn(r, self.g[r])
            except Exception as ex:        # a failing rank must not leave its peers waiting: collect and report
                errs.append((r, ex))
        th = [threading.Thread(target=work, args=(r,)) for r in range(self.world)]
        for t in th:
            t.start()
        for t in th:
            t.join(timeout=600)
        if errs:
            raise errs[0][1]
        return out

    def set_option(self, name, value):
        for g in self.g:
            g.set_option(name, value)

    def set_initial(self, comm_global):
        """comm_global: the whole graph's assignment (global ids), or None."""
        for r, g in enumerate(self.g):
            g.set_initial_communities(None if comm_global is None else comm_global[self.parts[r]:self.parts[r + 1]])

    def run(self, lower=-1.0):
        res = self.each(lambda r, g: (g.louvain(lower), g.trace(), g.communities().copy(), g.converged(), layout_info(g)))
        (mod, iters), tr = res[0][0], res[0][1]
        for o in res[1:]:
            assert o[0] == (mod, iters) and as_trace(o[1]) == as_trace(tr) and o[3] == res[0][3]
        return {"mod": mod, "iters": iters, "trace": as_trace(tr), "comm": np.concatenate([o[2] for o in res]),
                "converged": res[0][3], "first_ran": [o[4][0] for o in res], "relabel": res[0][4][1]}

    def close(self):
        for g in self.g:
            g.close()


def oracle_run(parts, rps, eds, init=None, **kw):
    init_slices = None if init is None else [init[parts[r]:parts[r + 1]] for r in range(len(rps))]
    res = O.louvain(parts, rps, eds, init_comm=init_slices, **kw)
    return {"mod": res["modularity"], "iters": res["iters"], "trace": as_trace(res["trace"]),
            "comm": np.concatenate(res["comm"]), "converged": res["converged"]}


def assert_same(res, ref, what):
    assert res["iters"] == ref["iters"], (what, res["iters"], ref["iters"])
    assert res["trace"] == ref["trace"], what
    assert repr(res["mod"]) == repr(ref["mod"]), (what, res["mod"], ref["mod"])
    assert np.array_equal(res["comm"], ref["comm"]), what


def split_and_resume(name, case, R, parts, rps, eds, ks=None, oracle_ck=True):
    """Stop R after k accepted iterations, check against the golden prefix and the oracle's C_k, resume, check the rest."""
    want = golden_trace(case)
    I = case["iters"]
    for k in (ks or split_points(I)):
        R.set_initial(None)
        R.set_option("stop_after", k)
        a = R.run()
        what = f"{name} k={k}"
        assert not a["converged"] and a["iters"] == k, what
        assert a["trace"] == want[:k], what
        assert a["mod"] == want[k - 1][0], what
        if oracle_ck:
            ck = oracle_run(parts, rps, eds, stop_after=k)
            assert np.array_equal(a["comm"], ck["comm"]), what
        R.set_option("stop_after", 0)
        R.set_initial(a["comm"])
        b = R.run(lower=a["mod"])
        assert b["converged"] and k + b["iters"] == I, (what, b["iters"])
        assert b["trace"] == want[k:], what
        assert repr(b["mod"]) == repr(float(case["modularity"])), (what, b["mod"])
        h = sum(O.comm_hash(int(parts[r]), b["comm"][parts[r]:parts[r + 1]]) for r in range(len(rps))) & (2 ** 64 - 1)
        assert h == int(case["final_chash"], 16), what
        if "comm" in case:
            assert [int(x) for x in b["comm"]] == case["comm"], what
        assert not any(b["first_ran"]), what          # the singleton reduction stays off on a warm run
    R.set_initial(None)


# ---- split and resume against the goldens -----------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_split_and_resume_matches_golden(gpu, name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        split_and_resume(name, case, R, parts, rps, eds)
    finally:
        R.close()


VARIANT_CASES = ["rgg_n16384_p1", "rgg_n65536_p1", "rgg_n16384_p4", "rmat_s14_p1", "hand_loops_multi_p2",
                 "dyadic_rgg_n16384_s1", "dyadic_random_n6000_d8_hubs3_hub_deg3000_multi200"]
VARIANTS = [{"scan_variant": 3}, {"scan_variant": 4}, {"scan_variant": 5}, {"scan_variant": 6},
            {"reorder": 0}, {"reorder": 1}, {"reorder": 2}, {"force_heavy_deg": 16}, {"reorder": 1, "force_heavy_deg": 16}]


@pytest.mark.parametrize("opts", VARIANTS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()))
def test_split_and_resume_under_variants(gpu, opts):
    for name in VARIANT_CASES:
        case = CASES[name]
        parts, rps, eds, _keep = case_graph(case)
        R = Ranks(parts, rps, eds, **opts)
        try:
            split_and_resume(name, case, R, parts, rps, eds, ks=[case["iters"] // 2], oracle_ck=False)
        finally:
            R.close()


# ---- identity start == cold run ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [3, 4, 5, 6])
def test_identity_start_equals_cold_run(gpu, variant):
    for name, reorder in (("rgg_n65536_p1", 2), ("rgg_n65536_p1", 1), ("rmat_s17_p1", 2), ("dyadic_rgg_n16384_s4", 1)):
        case = CASES[name]
        parts, rps, eds, _keep = case_graph(case)
        R = Ranks(parts, rps, eds, scan_variant=variant, reorder=reorder)
        try:
            cold = R.run()
            R.set_initial(np.arange(int(parts[-1]), dtype=np.int64))
            warm = R.run()
            again = R.run()                     # the assignment stays in effect: repeated warm runs are identical
        finally:
            R.close()
        assert_same(warm, cold, f"{name} v{variant}")
        assert_same(again, cold, f"{name} v{variant} repeat")
        assert cold["trace"] == golden_trace(case)
        assert not any(warm["first_ran"])
        if variant >= 4 and name.startswith("rgg"):
            assert all(cold["first_ran"])      # FIRST on (cold) and off (warm) give the same bits


# ---- arbitrary starting assignments against the oracle ----------------------------------------------------------------
def assignments(nv, nranks, seed=7):
    rng = np.random.default_rng(seed)
    v = np.arange(nv, dtype=np.int64)
    blk = 37
    nb = (nv + blk - 1) // blk
    return {
        "random": rng.integers(0, nv, nv),
        "all_zero": np.zeros(nv, np.int64),
        # block b is named by the first vertex of block b+1: no community contains its id vertex
        "named_outside": np.minimum(((v // blk + 1) % nb) * blk, nv - 1),
        # blocks named by a vertex half the graph away: on 2 and 4 ranks most ids are owned by another rank
        "other_rank": ((v // blk) * blk + nv // 2 + 5) % nv,
    }


def graphs():
    from minivite_b200 import hostgraph as hg
    out = {}
    ss = hg.generate_rgg(16384, 1)
    out["rgg16384"] = (16384, ss.shards[0].rowptr.copy(), ss.shards[0].edges.copy())
    ss.close()
    rp, ed = random_graph(5000, 12, seed=3, hubs=2, hub_deg=900)
    out["random5000"] = (5000, rp, ed)
    rp, ed = random_graph(4099, 30, seed=11, self_loops=40, multi=100, dyadic=True)
    out["dyadic4099"] = (4099, rp, ed)
    return out


@pytest.mark.parametrize("world", [1, 2, 4])
def test_arbitrary_assignments_match_oracle(gpu, world):
    for gname, (nv, rowptr, edges) in graphs().items():
        parts, rps, eds = split_global(nv, rowptr, edges, world)
        for reorder in (1, 0):
            R = Ranks(parts, rps, eds, reorder=reorder)
            try:
                for aname, init in assignments(nv, world).items():
                    R.set_initial(init)
                    res = R.run()
                    ref = oracle_run(parts, rps, eds, init=init)
                    assert_same(res, ref, f"{gname} {aname} world={world} reorder={reorder}")
                    assert res["relabel"] == (1 if reorder == 1 else 0)
            finally:
                R.close()


@pytest.mark.parametrize("nranks", [2, 4])
def test_keep_order_ranks_with_assignments(gpu, nranks):
    """One rank keeps its numbering while another renumbers (auto mode), so internal ids differ from caller ids on some
    ranks only; the owner's inv is read over the peer mapping."""
    from test_gpu_layout import keep_order_graph
    nv, parts, rowptr, edges = keep_order_graph(nranks)
    _, rps, eds = split_global(nv, rowptr, edges, nranks)
    R = Ranks(parts, rps, eds)
    try:
        for aname, init in assignments(nv, nranks, seed=nranks).items():
            R.set_initial(init)
            res = R.run()
            assert res["relabel"] == 1
            assert_same(res, oracle_run(parts, rps, eds, init=init), f"keep_order {aname} {nranks}")
    finally:
        R.close()


# ---- dynamic graph: re-cluster the -p 5 graph from the -p 0 graph's result ---------------------------------------------
@pytest.mark.parametrize("unit", [True, False])
def test_dynamic_graph_warm_start(gpu, unit):
    from minivite_b200 import hostgraph as hg
    ss0 = hg.generate_rgg(65536, 1, unit_weight=unit)
    ss5 = hg.generate_rgg(65536, 1, unit_weight=unit, random_edge_percent=5)
    s0, s5 = ss0.shards[0], ss5.shards[0]
    g = None
    try:
        from minivite_b200 import gpu as G
        g = G.LouvainGPU(0, 0, 1)
        g.set_option("trace", 1)
        g.upload(s0.nv, s0.parts, s0.rowptr, s0.edges)
        g.louvain()
        prev = g.communities().copy()
        g.upload(s5.nv, s5.parts, s5.rowptr, s5.edges)
        g.set_initial_communities(prev)
        mod, iters = g.louvain()
        comm = g.communities().copy()
        tr = as_trace(g.trace())
        ref = O.louvain(s5.parts, [s5.rowptr], [s5.edges], init_comm=[prev])
        if unit:
            assert (iters, mod) == (ref["iters"], ref["modularity"])
            assert tr == as_trace(ref["trace"])
            assert np.array_equal(comm, ref["comm"][0])
        else:                                   # Euclidean weights: the Comm sums depend on the order of the additions
            assert abs(mod - ref["modularity"]) <= 1e-6
    finally:
        if g is not None:
            g.close()
        ss0.close()
        ss5.close()


# ---- errors -----------------------------------------------------------------------------------------------------------
def test_errors_and_clearing(gpu):
    from minivite_b200 import gpu as G
    case = CASES["rgg_n16384_p1"]
    parts, rps, eds, _keep = case_graph(case)
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        with pytest.raises(G.MvgpuError, match="no shard"):
            G._ck(G.lib().mvgpu_set_initial_communities(g._h, np.zeros(1, np.int64).ctypes.data))
        g.upload(int(parts[-1]), parts, rps[0], eds[0])
        bad = np.zeros(16384, np.int64)
        bad[100] = 16384
        with pytest.raises(G.MvgpuError, match="outside"):
            g.set_initial_communities(bad)
        bad[100] = -1
        with pytest.raises(G.MvgpuError, match="outside"):
            g.set_initial_communities(bad)
        with pytest.raises(ValueError):
            g.set_initial_communities(np.zeros(100, np.int64))
        with pytest.raises(G.MvgpuError):
            g.set_option("stop_after", -1)
        assert as_trace(g.trace()) == [] and g.louvain()[1] == case["iters"]          # still usable: a cold run
        assert as_trace(g.trace()) == golden_trace(case) and g.converged()
        g.set_initial_communities(np.zeros(16384, np.int64))
        g.louvain()
        assert as_trace(g.trace()) != golden_trace(case)
        g.set_initial_communities(None)                                                # NULL clears
        g.louvain()
        assert as_trace(g.trace()) == golden_trace(case) and layout_info(g)[0] == 1
        g.set_initial_communities(np.zeros(16384, np.int64))
        g.upload(int(parts[-1]), parts, rps[0], eds[0])                                 # a new upload clears
        g.louvain()
        assert as_trace(g.trace()) == golden_trace(case)
        g.set_option("stop_after", 3)
        mod, iters = g.louvain()
        assert iters == 3 and not g.converged() and mod == float(case["trace"][2]["modularity"])
        g.set_option("stop_after", case["iters"])                                       # past the exit: a converged run
        mod, iters = g.louvain()
        assert iters == case["iters"] and g.converged() and repr(mod) == repr(float(case["modularity"]))
    finally:
        g.close()


def test_louvain32_refuses_warm_start(gpu):
    from minivite_b200 import gpu as G
    case = CASES["hand_clique_ring_p1"]
    parts, rps, eds, _keep = case_graph(case)
    e32 = np.zeros(len(eds[0]), np.dtype([("tail", "<i4"), ("weight", "<f4")]))
    e32["tail"], e32["weight"] = eds[0]["tail"], eds[0]["weight"]
    g = G.LouvainGPU(0, 0, 1)
    try:
        nv = int(parts[-1])
        g.upload32(nv, parts, rps[0], e32)
        g.set_initial_communities(np.zeros(nv, np.int64))
        with pytest.raises(G.MvgpuError, match="louvain32"):
            g.louvain32()
        g.set_initial_communities(None)
        g.set_option("stop_after", 1)
        with pytest.raises(G.MvgpuError, match="louvain32"):
            g.louvain32()
        g.set_option("stop_after", 0)
        assert g.louvain32()[1] == case["iters"]
    finally:
        g.close()


def test_ranks_that_disagree_fail_together(gpu):
    case = CASES["rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        R.g[0].set_initial_communities(np.arange(int(parts[1]), dtype=np.int64))
        errs = R.each(lambda r, g: _louvain_error(g))
        assert all(e is not None and "disagree" in e for e in errs), errs
        R.set_initial(None)                     # both contexts are still usable
        res = R.run()
        assert res["trace"] == golden_trace(case)
    finally:
        R.close()


def _louvain_error(g):
    from minivite_b200 import gpu as G
    try:
        g.louvain()
    except G.MvgpuError as ex:
        return str(ex)
    return None


# ---- the CLI: -k / -o, then -i / -L -----------------------------------------------------------------------------------
ITER_RE = re.compile(r"ITER (\d+) mod=(\S+) moved=(\d+) chash=([0-9a-f]+)")


def cli(args, env=None):
    p = subprocess.run([EXE] + args, capture_output=True, text=True, timeout=300, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    its = [(int(a[0]), float(a[1]), int(a[2]), int(a[3], 16)) for a in ITER_RE.findall(p.stderr)]
    assert [i for i, *_ in its] == list(range(1, len(its) + 1))          # each run numbers its iterations from 1
    return p, [t[1:] for t in its]


@pytest.mark.parametrize("ranks,extra", [(1, []), (1, ["-D"]), (2, [])])
def test_cli_stop_and_resume(gpu, tmp_path, ranks, extra):
    case = CASES["rgg_n16384_p1" if ranks == 1 else "rgg_n16384_p2"]
    env = dict(os.environ)
    if ranks > 1 and gpu.device_count() < ranks:
        env["MVGPU_OPTIONS"] = "host_transport=1"                        # ranks share device 0
    pre = str(tmp_path / "ck")
    base = ["-n", "16384", "-g", str(ranks), "-T"] + extra
    p1, t1 = cli(base + ["-k", "5", "-o", pre], env)
    m = re.search(r"STOPPED iters=(\d+) prevMod=(\S+)", p1.stderr)
    assert m and int(m.group(1)) == 5
    p2, t2 = cli(base + ["-i", pre, "-L", m.group(2)], env)
    assert "STOPPED" not in p2.stderr
    assert t1 + t2 == golden_trace(case)
    r = re.search(r"RESULT mod=(\S+) iters=(\d+)", p2.stderr)
    assert repr(float(r.group(1))) == repr(float(case["modularity"])) and 5 + int(r.group(2)) == case["iters"]


def test_cli_rejects_mismatched_checkpoint(gpu, tmp_path):
    pre = str(tmp_path / "ck")
    cli(["-n", "16384", "-k", "2", "-o", pre])
    p = subprocess.run([EXE, "-n", "32768", "-i", pre], capture_output=True, text=True, timeout=300)
    assert p.returncode != 0 and "does not match this rank's shard" in p.stderr


# ---- several GPUs: the same split and resume, one process per GPU ------------------------------------------------------
def _multi_worker(rank, world, port, name, k, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from minivite_b200 import dist as D
    from minivite_b200 import gpu as G
    R = D.Ranks("gloo")
    case = dict(CASES[name])
    parts, rps, eds, _keep = case_graph(case)
    ident = R.broadcast_bytes(G.get_unique_id() if rank == 0 else None, G.UNIQUE_ID_BYTES)
    g = G.LouvainGPU(rank, rank, world)
    g.comm_init(ident)
    g.set_option("trace", 1)
    g.upload(int(parts[-1]), parts, rps[rank], eds[rank])
    g.set_option("stop_after", k)
    mod_a, it_a = g.louvain()
    ck = g.communities().copy()
    tr_a = as_trace(g.trace())
    conv_a = g.converged()
    g.set_option("stop_after", 0)
    g.set_initial_communities(ck)
    mod_b, it_b = g.louvain()
    tr_b = as_trace(g.trace())
    allc = R.gather_arrays(g.communities())
    allck = R.gather_arrays(ck)
    if rank == 0:
        json.dump({"a": [repr(mod_a), it_a, tr_a, conv_a], "b": [repr(mod_b), it_b, tr_b, g.converged()],
                   "comm": [int(x) for x in np.concatenate(allc)], "ck": [int(x) for x in np.concatenate(allck)]},
                  open(os.path.join(out_dir, "res.json"), "w"))
    g.close()
    R.shutdown()


@pytest.mark.parametrize("name", ["rgg_n16384_p2", "rgg_n16384_p4", "file_rgg_n524288_s8_p8", "rmat_s17_p2_b",
                                  "hand_loops_multi_p2"])
def test_multi_gpu_split_and_resume(tmp_path, name):
    from minivite_b200 import gpu as G
    import socket
    import torch.multiprocessing as mp
    case = dict(CASES[name])
    world = case["nranks"]
    if G.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    k = case["iters"] // 2
    mp.spawn(_multi_worker, args=(world, port, name, k, str(tmp_path)), nprocs=world, join=True)
    res = json.load(open(tmp_path / "res.json"))
    want = golden_trace(case)
    mod_a, it_a, tr_a, conv_a = res["a"]
    mod_b, it_b, tr_b, conv_b = res["b"]
    assert it_a == k and not conv_a and [tuple(t) for t in tr_a] == want[:k] and float(mod_a) == want[k - 1][0]
    parts, rps, eds, _keep = case_graph(case)
    assert np.array_equal(np.array(res["ck"]), oracle_run(parts, rps, eds, stop_after=k)["comm"])
    assert conv_b and it_a + it_b == case["iters"] and [tuple(t) for t in tr_b] == want[k:]
    assert mod_b == repr(float(case["modularity"]))


# ---- full size ----------------------------------------------------------------------------------------------------------
def test_full_size_config2_split_at_13(gpu):
    """`miniVite -n 16777216` (config 2) stopped after iteration 13 and resumed: the golden trace of the unmodified
    reference, bit for bit (tests/golden/golden_full_16777216_p1.json).  Opt-in with MV_BIG_TESTS=1."""
    if os.environ.get("MV_BIG_TESTS") != "1":
        pytest.skip("set MV_BIG_TESTS=1")
    gold = json.load(open(os.path.join(GOLDEN, "golden_full_16777216_p1.json")))
    want = golden_trace(gold)
    g = gpu.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        g.generate_rgg(gold["nv"])
        g.set_option("stop_after", 13)
        mod_a, it_a = g.louvain()
        assert it_a == 13 and not g.converged() and as_trace(g.trace()) == want[:13] and mod_a == want[12][0]
        ck = g.communities().copy()
        g.set_option("stop_after", 0)
        g.set_initial_communities(ck)
        mod_b, it_b = g.louvain(mod_a)
        assert g.converged() and 13 + it_b == gold["iters"] and as_trace(g.trace()) == want[13:]
        assert repr(mod_b) == repr(float(gold["modularity"]))
        assert "%016x" % O.comm_hash(0, g.communities()) == gold["final_chash"]
    finally:
        g.close()
