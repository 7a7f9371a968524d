"""Splitting disconnected communities on the device (mvgpu_split_communities, DESIGN.md §3.12), against the NumPy /
scipy restatement tests/split_ref.py.

Y and the counts are canonical, so the device must match the restatement exactly: on 1 rank and on 2 and 4 ranks
sharing device 0 (host transport), after runs with every renumbering mode, with every upload mode and on attached,
generated and updated shards.  Y round-trips through evaluate() and the warm start, and a split changes nothing a run
reports or does."""
import ctypes
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from helpers import case_graph, random_graph, split_global
import quality_ref as QR
import split_ref as SR
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_quality import _err, evaluate, snapshot
from test_gpu_warm_start import CASES, Ranks, assert_same, assignments, graphs, oracle_run

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "bin", "miniVite_b200")
COUNTS = ("communities", "components", "disconnected")


def split(R, X=None):
    """Split X (whole-graph assignment, or None = the last run's) on every rank of R; returns (Y, report), the report
    checked to be the same on every rank."""
    res = R.each(lambda r, g: g.split_communities(None if X is None else X[R.parts[r]:R.parts[r + 1]]))
    rep = res[0][1]
    for o in res[1:]:
        assert all(o[1][k] == rep[k] for k in COUNTS + ("rounds",)), (o[1], rep)
    return np.concatenate([o[0] for o in res]), rep


def assert_split(got, ref, what):
    Y, rep = got
    assert np.array_equal(Y, ref["Y"]), what
    assert all(rep[k] == ref[k] for k in COUNTS), (what, rep, {k: ref[k] for k in COUNTS})
    assert rep["rounds"] >= 1 and rep["split_s"] > 0.0, (what, rep)


def path_graph(nv):
    tails = np.stack([np.arange(nv) - 1, np.arange(nv) + 1], 1).reshape(-1)
    tails = tails[(tails >= 0) & (tails < nv)]
    rowptr = np.concatenate([[0], np.cumsum(np.full(nv, 2) - (np.arange(nv) == 0) - (np.arange(nv) == nv - 1))]).astype(np.int64)
    edges = np.zeros(len(tails), np.dtype([("tail", "<i8"), ("weight", "<f8")]))
    edges["tail"], edges["weight"] = tails, 1.0
    return rowptr, edges


# ---- golden graphs: the run's own result, and the round trips --------------------------------------------------------------
GOLDEN = ["rgg_n16384_p1", "rgg_n16384_p2", "rgg_n16384_p4", "rgg_n65536_p1", "rgg_n131072_p8", "file_rgg_n16384_s4_p4",
          "rmat_s14_p1", "rmat_s14_p2", "rmat_s14_p4_b", "rmat_s17_p1", "rmat_s17_p2", "dyadic_rmat_s14",
          "dyadic_random_n20000_d40_blocks400_hubs1_hub_deg2000"]


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_results_and_round_trips(gpu, name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        X = R.run()["comm"]
        ref = SR.split(parts, rps, eds, X)
        got = split(R)
        assert_split(got, ref, name)
        if name == "rmat_s14_p1":
            assert (got[1]["communities"], got[1]["components"], got[1]["disconnected"]) == (8251, 10500, 759)
        if name == "rmat_s17_p1":
            assert (got[1]["communities"], got[1]["components"], got[1]["disconnected"]) == (70303, 86659, 4282)
        assert_split(split(R, X), ref, name + " given")
        Y = got[0]
        qx, qy = evaluate(R, X), evaluate(R, Y)
        assert qy["communities"] == got[1]["components"]
        assert repr(qy["e_in"]) == repr(qx["e_in"]) and qy["a2"] <= qx["a2"] and qy["modularity"] >= qx["modularity"]
        assert repr(qy["modularity"]) == repr(QR.quality(parts, rps, eds, Y)["modularity"])
        assert_split(split(R, Y), SR.split(parts, rps, eds, Y), name + " idempotent")
        assert split(R, Y)[1]["disconnected"] == 0
        R.set_initial(Y)                                 # run -> split -> warm run
        assert_same(R.run(), oracle_run(parts, rps, eds, init=Y), name + " warm from Y")
    finally:
        R.close()


# ---- random and hand-made assignments, 1 / 2 / 4 ranks, every renumbering mode of the run before -----------------------------
def special_graphs():
    out = {}
    rp, ed = path_graph(2500)
    out["path2500"] = (2500, rp, ed)
    rp, ed = random_graph(40000, 3, seed=4, hubs=1, hub_deg=30000)          # the hub is a high-degree vertex of the scan
    out["star40000"] = (40000, rp, ed)
    nv = 4096                                                               # v - v+2 chains: evens and odds interleave
    tails = [[t for t in (v - 2, v + 2) if 0 <= t < nv] for v in range(nv)]
    rp = np.concatenate([[0], np.cumsum([len(t) for t in tails])]).astype(np.int64)
    ed = np.zeros(int(rp[-1]), np.dtype([("tail", "<i8"), ("weight", "<f8")]))
    ed["tail"], ed["weight"] = [t for ts in tails for t in ts], 1.0
    out["interleaved4096"] = (nv, rp, ed)
    return out


@pytest.mark.parametrize("world", [1, 2, 4])
def test_assignments_on_ranks_and_reorder_modes(gpu, world):
    gs = dict(graphs(), **special_graphs())
    for gname, (nv, rowptr, edges) in gs.items():
        parts, rps, eds = split_global(nv, rowptr, edges, world)
        v = np.arange(nv, dtype=np.int64)
        extra = {"one": np.full(nv, nv // 3, np.int64), "thirds": v % 3, "singletons": v}
        for reorder in (0, 1, 2):
            R = Ranks(parts, rps, eds, reorder=reorder)
            try:
                X = R.run()["comm"]                      # a run first: its renumbering must not leak into Y
                assert_split(split(R), SR.split(parts, rps, eds, X), f"{gname} run {world} {reorder}")
                for aname, A in dict(assignments(nv, world), **extra).items():
                    got = split(R, A)
                    assert_split(got, SR.split(parts, rps, eds, A), f"{gname} {aname} {world} {reorder}")
                    if gname == "path2500" and aname == "one":
                        assert got[1]["components"] == 1 and got[1]["rounds"] <= 32, got[1]   # shortcutting works
                    if gname == "interleaved4096" and aname == "one":
                        assert got[1]["components"] == 2 and np.array_equal(got[0], v % 2)
            finally:
                R.close()


def test_hand_cases(gpu):
    from test_split_ref import hand_cases
    for name, (nv, rowptr, edges, assigns) in hand_cases().items():
        for world in (1, 2, 4):
            parts, rps, eds = split_global(nv, rowptr, edges, world)
            R = Ranks(parts, rps, eds)
            try:
                for aname, X in assigns.items():
                    assert_split(split(R, X), SR.split(parts, rps, eds, X), f"{name} {aname} {world}")
            finally:
                R.close()


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_upload_modes(gpu, mode):
    rp, ed = random_graph(20000, 10, seed=2, blocks=64)
    for world in (1, 2):
        parts, rps, eds = split_global(20000, rp, ed, world)
        R = Ranks(parts, rps, eds, compact_upload=mode)
        try:
            X = R.run()["comm"]
            assert_split(split(R), SR.split(parts, rps, eds, X), f"compact_upload={mode} {world}")
        finally:
            R.close()


def test_generated_attached_and_updated_shards(gpu):
    import torch
    from minivite_b200 import gpu as G
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.generate_rgg(65536, random_edge_percent=1.0)
        rowptr, edges = g.download_shard()
        parts = np.array([0, 65536], np.int64)
        g.louvain()
        X = g.communities().copy()
        ref = SR.split(parts, [rowptr], [edges], X)
        assert_split(g.split_communities(), ref, "generated")
        d_rp = torch.from_numpy(rowptr).cuda()
        d_ed = torch.from_numpy(edges.view(np.uint8).copy()).cuda()
        g.attach_device(65536, parts, 65536, len(edges), d_rp.data_ptr(), d_ed.data_ptr(), keepalive=(d_rp, d_ed))
        assert_split(g.split_communities(X), ref, "attached")
        g.louvain()
        # cut every record of 3000 random vertices' lists (both directions) and add 2000 new edges
        rng = np.random.default_rng(9)
        cut = rng.choice(65536, 3000, replace=False)
        src = np.repeat(np.arange(65536), np.diff(rowptr))
        sel = np.isin(src, cut)
        ds, dd = np.concatenate([src[sel], edges["tail"][sel]]), np.concatenate([edges["tail"][sel], src[sel]])
        a, b = rng.integers(0, 65536, 2000), rng.integers(0, 65536, 2000)
        a, b = a[a != b], b[a != b]
        g.update_shard(delete=(ds, dd), insert=(np.concatenate([a, b]), np.concatenate([b, a]), np.ones(2 * len(a))))
        assert _err(lambda: g.split_communities()) is not None      # the run's result belongs to the old shard
        rp2, ed2 = g.download_shard()
        assert_split(g.split_communities(X), SR.split(parts, [rp2], [ed2], X), "updated")
        g.louvain()
        X2 = g.communities().copy()
        assert_split(g.split_communities(), SR.split(parts, [rp2], [ed2], X2), "updated, run")
    finally:
        g.close()


# ---- state rules: a split changes nothing a run reports, and nothing the next run does ---------------------------------------
def test_state_rules(gpu):
    case = CASES["rgg_n65536_p1"]
    parts, rps, eds, _keep = case_graph(case)
    nv = int(parts[-1])
    other = np.random.default_rng(3).integers(0, nv, nv)
    for reorder in (1, 0):
        for warm in (False, True):
            R, plain = Ranks(parts, rps, eds, reorder=reorder), Ranks(parts, rps, eds, reorder=reorder)
            try:
                init = np.arange(nv, dtype=np.int64) // 5 * 5 if warm else None
                R.set_initial(init)
                plain.set_initial(init)
                a = R.run()
                g = R.g[0]
                before = snapshot(g)
                evaluate(R, other)
                split(R, other)
                assert _err(lambda: g.community_stats()) is not None       # the evaluation's arrays are gone
                assert _err(lambda: g.compact_communities()) is not None
                split(R)
                assert snapshot(g) == before, (reorder, warm)
                b = R.run()
                ref = plain.run()
                assert b["trace"] == ref["trace"] == a["trace"] and np.array_equal(b["comm"], ref["comm"])
                assert R.g[0].timings()["kernel_launches"] == plain.g[0].timings()["kernel_launches"]
                R.set_initial(None)
                plain.set_initial(None)
                split(R, other)
                c, cref = R.run(), plain.run()            # a cold run after a split
                assert c["trace"] == cref["trace"] and np.array_equal(c["comm"], cref["comm"])
                assert R.g[0].timings()["kernel_launches"] == plain.g[0].timings()["kernel_launches"]
            finally:
                R.close()
                plain.close()


def test_state_rules_on_two_ranks(gpu):
    case = CASES["rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds, reorder=1)
    try:
        a = R.run()
        comm_before = [g.communities().copy() for g in R.g]
        assert_split(split(R), SR.split(parts, rps, eds, a["comm"]), "2 ranks")
        assert all(np.array_equal(g.communities(), c) for g, c in zip(R.g, comm_before))
        assert R.run()["trace"] == a["trace"]
        q = evaluate(R)
        assert_split(split(R), SR.split(parts, rps, eds, a["comm"]), "2 ranks again")
        assert_split(split(R, a["comm"]), SR.split(parts, rps, eds, a["comm"]), "2 ranks given")
        assert evaluate(R)["modularity"] == q["modularity"]
    finally:
        R.close()


# ---- errors: every rank fails together, and nothing is written ---------------------------------------------------------------
def test_errors(gpu):
    from minivite_b200 import gpu as G
    case = CASES["rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    nv = int(parts[-1])
    R = Ranks(parts, rps, eds)
    try:
        errs = R.each(lambda r, g: _err(lambda: g.split_communities()))        # NULL before any run
        assert all(e and "none" in e for e in errs), errs
        bad = np.zeros(nv, np.int64)
        bad[nv - 1] = nv                                                        # a bad id on rank 1 only
        errs = R.each(lambda r, g: _err(lambda: g.split_communities(bad[parts[r]:parts[r + 1]])))
        assert errs[1] and "outside" in errs[1] and errs[0] and "another rank" in errs[0], errs
        X = np.arange(nv, dtype=np.int64)                                       # a wrong length on rank 1 only
        errs = R.each(lambda r, g: _err(lambda: g.split_communities(X[parts[r]:parts[r + 1]] if r == 0 else X[:5])))
        assert errs[1] and "entries" in errs[1] and errs[0] and "another rank" in errs[0], errs
        a = R.run()
        errs = R.each(lambda r, g: _err(lambda: g.split_communities(None if r == 0 else np.zeros(g.lnv, np.int64))))
        assert all(e and "disagree" in e and "split" in e for e in errs), errs
        assert_split(split(R), SR.split(parts, rps, eds, a["comm"]), "after the failures")   # both contexts still work
    finally:
        R.close()
    g = G.LouvainGPU(0, 0, 1)
    try:
        p1, r1, e1, _k = case_graph(CASES["rgg_n16384_p1"])
        g.upload(int(p1[-1]), p1, r1[0], e1[0])
        g.louvain()
        out = np.full(g.lnv, -5, np.int64)                                       # a failed call writes nothing
        comm = np.zeros(g.lnv, np.int64)
        comm[7] = -1
        rep = G.SplitReport()
        assert G.lib().mvgpu_split_communities(g._h, comm.ctypes.data, out.ctypes.data, ctypes.byref(rep)) != 0
        assert np.all(out == -5) and rep.rounds == 0
        with pytest.raises(G.MvgpuError, match="outside"):
            g.split_communities(comm)
        c32 = CASES["hand_clique_ring_p1"]
        p32, r32, e32s, _k = case_graph(c32)
        e32 = np.zeros(len(e32s[0]), np.dtype([("tail", "<i4"), ("weight", "<f4")]))
        e32["tail"], e32["weight"] = e32s[0]["tail"], e32s[0]["weight"]
        g.upload32(int(p32[-1]), p32, r32[0], e32)
        g.louvain32()
        with pytest.raises(G.MvgpuError, match="upload_shard32"):
            g.split_communities()
        with pytest.raises(G.MvgpuError, match="upload_shard32"):
            g.split_communities(np.zeros(int(p32[-1]), np.int64))
    finally:
        g.close()


# ---- the CLI: -C after a run and on the files -o wrote ---------------------------------------------------------------------
SPLIT_RE = re.compile(r"SPLIT communities=(\d+) components=(\d+) disconnected=(\d+) rounds=(\d+)")


def cli(args, ranks, env):
    p = subprocess.run([EXE, "-n", "16384", "-g", str(ranks)] + args, capture_output=True, text=True, timeout=300, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    return p.stderr


def read_dump(pre, ranks):
    return np.concatenate([np.fromfile(f"{pre}.{r}", np.int64)[2:] for r in range(ranks)])


@pytest.mark.parametrize("ranks", [1, 2])
def test_cli_split(gpu, tmp_path, ranks):
    from test_gpu_quality import parse_quality
    env = dict(os.environ)
    if ranks > 1 and gpu.device_count() < ranks:
        env["MVGPU_OPTIONS"] = "host_transport=1"
    plain, pre = str(tmp_path / "x"), str(tmp_path / "y")
    assert "SPLIT" not in cli(["-o", plain], ranks, env)                 # without -C nothing changes
    err = cli(["-C", "-q", "-o", pre], ranks, env)
    m = SPLIT_RE.search(err)
    assert m, err[-2000:]
    case = CASES["rgg_n16384_p1" if ranks == 1 else "rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    X = read_dump(plain, ranks)
    ref = SR.split(parts, rps, eds, X)
    assert [int(m.group(i)) for i in (1, 2, 3)] == [ref[k] for k in COUNTS] and int(m.group(4)) >= 1
    assert np.array_equal(read_dump(pre, ranks), ref["Y"])                  # -o writes the split assignment
    q = parse_quality(err)                                                  # -q evaluates it
    want = QR.quality(parts, rps, eds, ref["Y"])
    assert q["communities"] == ref["components"] and q["modularity"] == want["modularity"]
    e = cli(["-E", plain, "-C"], ranks, env)                                # -E -C: split the file's assignment
    m2 = SPLIT_RE.search(e)                                                 # (the round count may differ from call to call)
    assert [m2.group(i) for i in (1, 2, 3)] == [m.group(i) for i in (1, 2, 3)] and parse_quality(e) == q and "RESULT" not in e


# ---- several GPUs: one process per GPU ------------------------------------------------------------------------------------
def _multi_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from minivite_b200 import dist as D
    from minivite_b200 import gpu as G
    R = D.Ranks("gloo")
    parts, rps, eds, _keep = case_graph(CASES["rmat_s14_p2"])
    ident = R.broadcast_bytes(G.get_unique_id() if rank == 0 else None, G.UNIQUE_ID_BYTES)
    g = G.LouvainGPU(rank, rank, world)
    g.comm_init(ident)
    g.upload(int(parts[-1]), parts, rps[rank], eds[rank])
    res = {}
    for mode in (1, 0):
        g.set_option("comm_mode", mode)
        g.louvain()
        comm = R.gather_arrays(g.communities())
        Y, rep = g.split_communities()
        Ys = R.gather_arrays(Y)
        if rank == 0:
            res[mode] = {"comm": [int(x) for x in np.concatenate(comm)], "Y": [int(x) for x in np.concatenate(Ys)],
                         "rep": {k: rep[k] for k in COUNTS}}
    if rank == 0:
        json.dump(res, open(os.path.join(out_dir, "res.json"), "w"))
    g.close()
    R.shutdown()


def test_multi_gpu_split(tmp_path):
    from minivite_b200 import gpu as G
    import socket
    import torch.multiprocessing as mp
    if G.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_multi_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    res = json.load(open(tmp_path / "res.json"))
    parts, rps, eds, _keep = case_graph(CASES["rmat_s14_p2"])
    for mode, r in res.items():
        ref = SR.split(parts, rps, eds, np.array(r["comm"], np.int64))
        assert r["Y"] == [int(x) for x in ref["Y"]], mode
        assert r["rep"] == {k: ref[k] for k in COUNTS}, mode
