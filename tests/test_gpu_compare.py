"""Comparing two assignments on the device (mvgpu_compare_communities, mvgpu_get_community_matches; DESIGN.md §3.13),
against the NumPy restatement tests/compare_ref.py.

Every field is exact integer counting, or doubles computed from the merged counts in a fixed order, so the device must
match the restatement bit for bit: on 1 rank and on 2 and 4 ranks sharing device 0 (host transport), after runs with
every renumbering mode.  A comparison reads no edge and changes nothing a run or an evaluation reports."""
import ctypes
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from helpers import case_graph, split_global
import compare_ref as CR
import split_ref as SR
import update_ref as U
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_quality import _err, evaluate, snapshot
from test_gpu_warm_start import CASES, Ranks, assignments, graphs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "bin", "miniVite_b200")


def compare(R, X, Y):
    """Compare X (whole-graph assignment, or None = the last run's) with Y on every rank of R; returns the report
    (checked to be the same on every rank) with the match arrays concatenated over the ranks."""
    def one(r, g):
        sl = slice(int(R.parts[r]), int(R.parts[r + 1]))
        rep = g.compare_communities(Y[sl], None if X is None else X[sl])
        return rep, g.community_matches()
    res = R.each(one)
    rep = res[0][0]
    for o in res[1:]:
        assert all(repr(o[0][k]) == repr(rep[k]) for k in CR.FIELDS), (o[0], rep)
    out = dict(rep)
    for k in CR.MATCHES:
        out[k] = np.concatenate([o[1][k] for o in res])
    return out


def assert_cmp(got, ref, what):
    for k in CR.FIELDS:
        assert repr(got[k]) == repr(ref[k]), (what, k, got[k], ref[k])
    for k in CR.MATCHES:
        assert np.array_equal(got[k], ref[k]), (what, k)
    assert got["compare_s"] > 0.0, what


def check(R, X, Y, what, Xref=None):
    got = compare(R, X, Y)
    assert_cmp(got, CR.compare(X if Xref is None else Xref, Y), what)
    return got


# ---- the pairs a user compares, 1 / 2 / 4 ranks, every renumbering mode of the run before -------------------------------------
@pytest.mark.parametrize("world", [1, 2, 4])
def test_pairs_on_ranks_and_reorder_modes(gpu, world):
    for gname, (nv, rowptr, edges) in graphs().items():
        parts, rps, eds = split_global(nv, rowptr, edges, world)
        v = np.arange(nv, dtype=np.int64)
        for reorder in (0, 1, 2):
            R = Ranks(parts, rps, eds, reorder=reorder)
            try:
                X = R.run()["comm"]                          # a run first: its renumbering must not leak into the result
                Ys = SR.split(parts, rps, eds, X)["Y"]
                check(R, None, Ys, f"{gname} run vs split {world} {reorder}", Xref=X)
                check(R, None, v, f"{gname} run vs singletons {world} {reorder}", Xref=X)
                if reorder != 1:
                    continue
                check(R, X, Ys, f"{gname} given run vs split {world}")
                got = check(R, X, evaluate(R, X)["compact"], f"{gname} run vs compact {world}")
                assert (got["ari"], got["nmi"], got["vi"]) == (1.0, 1.0, 0.0), got
                A = assignments(nv, world)
                one = np.full(nv, nv // 3, np.int64)
                for xa, ya in (("random", "other_rank"), ("named_outside", "random"), ("other_rank", "named_outside"),
                               ("all_zero", "random")):
                    check(R, A[xa], A[ya], f"{gname} {xa} vs {ya} {world}")
                got = check(R, one, X, f"{gname} one vs run {world}")
                assert got["ari"] == 0.0 and got["nmi"] == 0.0 or got["communities_y"] == 1
                check(R, X, one, f"{gname} run vs one {world}")
                check(R, one, one, f"{gname} one vs one {world}")
            finally:
                R.close()


@pytest.mark.parametrize("world", [1, 2, 4])
def test_cold_and_warm_runs_on_an_updated_shard(gpu, world):
    """RGG 65 536: the -p 0 graph's result, the shard updated to -p 5 with the extra records, then a cold and a warm run
    on it; how far apart the two results are."""
    from minivite_b200 import hostgraph as hg
    ss0, ss5 = hg.generate_rgg(65536, world), hg.generate_rgg(65536, world, random_edge_percent=5)
    try:
        parts = np.asarray(ss0.shards[0].parts, np.int64)
        R = Ranks(parts, [s.rowptr for s in ss0.shards], [s.edges for s in ss0.shards])
        try:
            X0 = R.run()["comm"]
            ext = [U.extras(a, b) for a, b in zip(ss0.shards, ss5.shards)]
            R.each(lambda r, g: g.update_shard(insert=ext[r]))
            cold = R.run()["comm"]
            R.set_initial(X0)
            warm = R.run()["comm"]
            got = check(R, None, cold, f"warm vs cold {world}", Xref=warm)
            assert 0.0 < got["ari"] <= 1.0 and 0.0 < got["nmi"] <= 1.0, got
            check(R, cold, warm, f"cold vs warm {world}")
            check(R, X0, warm, f"-p 0 vs warm {world}")
        finally:
            R.close()
    finally:
        ss0.close()
        ss5.close()


def test_golden_results_against_their_splits(gpu):
    for name in ("rmat_s14_p1", "rmat_s14_p2", "rmat_s14_p4_b", "rgg_n131072_p8", "dyadic_rmat_s14"):
        parts, rps, eds, _keep = case_graph(CASES[name])
        R = Ranks(parts, rps, eds)
        try:
            X = R.run()["comm"]
            Y = np.concatenate(R.each(lambda r, g: g.split_communities()[0]))
            got = check(R, None, Y, name, Xref=X)
            s = SR.split(parts, rps, eds, X)
            assert got["pairs_xy"] == got["pairs_y"] and got["cells"] == s["components"], name
        finally:
            R.close()


# ---- state rules: a comparison changes nothing a run or an evaluation reports ----------------------------------------------
@pytest.mark.parametrize("world", [1, 2])
def test_state_rules(gpu, world):
    parts, rps, eds, _keep = case_graph(CASES["rgg_n65536_p1" if world == 1 else "rgg_n16384_p2"])
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
                q = evaluate(R, other)
                before = [snapshot(g) for g in R.g]
                check(R, None, other, f"state {reorder} {warm}", Xref=a["comm"])
                check(R, other, a["comm"], f"state swapped {reorder} {warm}")
                assert [snapshot(g) for g in R.g] == before, (reorder, warm)
                q2 = evaluate_arrays(R)
                for k in ("size", "volume", "internal", "compact"):
                    assert np.array_equal(q2[k], q[k]), k
                b = R.run()
                ref = plain.run()
                assert b["trace"] == ref["trace"] == a["trace"] and np.array_equal(b["comm"], ref["comm"])
                assert [g.timings()["kernel_launches"] for g in R.g] == [g.timings()["kernel_launches"] for g in plain.g]
            finally:
                R.close()
                plain.close()


def evaluate_arrays(R):
    """The last evaluation's per-community arrays and compact labels, read without a new evaluation."""
    res = R.each(lambda r, g: (g.community_stats(), g.compact_communities().copy()))
    out = {k: np.concatenate([o[0][k] for o in res]) for k in ("size", "volume", "internal")}
    out["compact"] = np.concatenate([o[1] for o in res])
    return out


# ---- errors: every rank fails together, nothing is written, and every earlier result stays ----------------------------------
def test_errors(gpu):
    from minivite_b200 import gpu as G
    parts, rps, eds, _keep = case_graph(CASES["rgg_n16384_p2"])
    nv = int(parts[-1])
    v = np.arange(nv, dtype=np.int64)
    R = Ranks(parts, rps, eds)
    try:
        errs = R.each(lambda r, g: _err(lambda: g.community_matches()))          # before the first compare
        assert all(e and "no comparison" in e for e in errs), errs
        errs = R.each(lambda r, g: _err(lambda: g.compare_communities(v[parts[r]:parts[r + 1]])))   # NULL x, no run
        assert all(e and "none" in e for e in errs), errs
        a = R.run()
        q = evaluate(R, v % 7)
        good = check(R, None, v, "first", Xref=a["comm"])
        before = [snapshot(g) for g in R.g]
        bad = v.copy()
        bad[nv - 1] = nv                                                           # a bad id on rank 1 only
        for X, Y in ((bad, v), (v, bad)):
            errs = R.each(lambda r, g: _err(lambda: g.compare_communities(Y[parts[r]:parts[r + 1]], X[parts[r]:parts[r + 1]])))
            assert errs[1] and "outside" in errs[1] and errs[0] and "another rank" in errs[0], errs
            errs = R.each(lambda r, g: _err(lambda: g.community_matches()))      # a failed compare clears the matches
            assert all(e and "no comparison" in e for e in errs), errs
        for which in ("x", "y"):                                                   # a wrong length on rank 1 only
            def one(r, g):
                sl = v[parts[r]:parts[r + 1]]
                short = v[:5] if r == 1 else sl
                return _err(lambda: g.compare_communities(short if which == "y" else sl, short if which == "x" else sl))
            errs = R.each(one)
            assert errs[1] and "entries" in errs[1] and errs[0] and "another rank" in errs[0], errs
        errs = R.each(lambda r, g: _err(lambda: g.compare_communities(v[parts[r]:parts[r + 1]], None if r == 0 else v[parts[r]:parts[r + 1]])))
        assert all(e and "disagree" in e for e in errs), errs
        assert [snapshot(g) for g in R.g] == before
        q2 = evaluate_arrays(R)
        assert all(np.array_equal(q2[k], q[k]) for k in ("size", "volume", "internal", "compact"))
        assert_cmp(compare(R, None, v), CR.compare(a["comm"], v), "after the failures")
        assert good["cells"] == nv
    finally:
        R.close()
    g = G.LouvainGPU(0, 0, 1)
    try:
        p1, r1, e1, _k = case_graph(CASES["rgg_n16384_p1"])
        g.upload(int(p1[-1]), p1, r1[0], e1[0])
        w = np.arange(g.lnv, dtype=np.int64)
        g.compare_communities(w, w)
        assert np.array_equal(g.community_matches()["best"], w)
        bad = w.copy()
        bad[7] = -1
        rep = G.CompareReport()
        rep.ari = -5.0
        assert G.lib().mvgpu_compare_communities(g._h, w.ctypes.data, bad.ctypes.data, ctypes.byref(rep)) != 0
        assert rep.ari == -5.0 and rep.cells == 0                                  # a failed call writes nothing
        assert G.lib().mvgpu_compare_communities(g._h, w.ctypes.data, None, ctypes.byref(rep)) != 0
        assert "NULL" in G.lib().mvgpu_last_error().decode()
        with pytest.raises(G.MvgpuError, match="outside"):
            g.compare_communities(bad, w)
        g.compare_communities(w, w)
        g.upload(int(p1[-1]), p1, r1[0], e1[0])                                   # a new upload clears the matches
        with pytest.raises(G.MvgpuError, match="no comparison"):
            g.community_matches()
        c32 = CASES["hand_clique_ring_p1"]
        p32, r32, e32s, _k = case_graph(c32)
        e32 = np.zeros(len(e32s[0]), np.dtype([("tail", "<i4"), ("weight", "<f4")]))
        e32["tail"], e32["weight"] = e32s[0]["tail"], e32s[0]["weight"]
        g.upload32(int(p32[-1]), p32, r32[0], e32)
        g.louvain32()
        with pytest.raises(G.MvgpuError, match="upload_shard32"):
            g.compare_communities(np.zeros(int(p32[-1]), np.int64))
    finally:
        g.close()


# ---- the CLI: -M with a run, with -C and with -E -----------------------------------------------------------------------------
COMPARE_RE = re.compile(r"COMPARE ari=(\S+) nmi=(\S+) vi=(\S+) rand=(\S+) mi=(\S+) hx=(\S+) hy=(\S+) cells=(\d+) "
                        r"communities_x=(\d+) communities_y=(\d+)")
CLI_FIELDS = ("ari", "nmi", "vi", "rand", "mi", "h_x", "h_y", "cells", "communities_x", "communities_y")


def parse_compare(stderr):
    m = COMPARE_RE.search(stderr)
    assert m, stderr[-2000:]
    return {k: (int if i >= 7 else float)(m.group(i + 1)) for i, k in enumerate(CLI_FIELDS)}


def cli(args, ranks, env):
    p = subprocess.run([EXE, "-n", "16384", "-g", str(ranks)] + args, capture_output=True, text=True, timeout=300, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    return p.stderr


@pytest.mark.parametrize("ranks", [1, 2])
def test_cli_compare(gpu, tmp_path, ranks):
    env = dict(os.environ)
    if ranks > 1 and gpu.device_count() < ranks:
        env["MVGPU_OPTIONS"] = "host_transport=1"
    plain = str(tmp_path / "x")
    assert "COMPARE" not in cli(["-o", plain], ranks, env)
    parts, rps, eds, _keep = case_graph(CASES["rgg_n16384_p1" if ranks == 1 else "rgg_n16384_p2"])
    X = np.concatenate([np.fromfile(f"{plain}.{r}", np.int64)[2:] for r in range(ranks)])
    Y = SR.split(parts, rps, eds, X)["Y"]
    R = Ranks(parts, rps, eds)
    try:
        same = compare(R, X, X)
        py = compare(R, Y, X)                                          # the split against the file, through Python
    finally:
        R.close()
    got = parse_compare(cli(["-M", plain], ranks, env))                # the run's result against itself
    assert all(got[k] == same[k] for k in CLI_FIELDS) and got["ari"] == 1.0
    got = parse_compare(cli(["-C", "-M", plain], ranks, env))          # its split against the run's result
    assert all(got[k] == py[k] for k in CLI_FIELDS), (got, py)
    e = cli(["-E", plain, "-C", "-M", plain], ranks, env)              # the file's split against the file
    assert parse_compare(e) == got and "RESULT" not in e


# ---- full size ------------------------------------------------------------------------------------------------------------------
def test_full_size_config2_against_its_split(gpu):
    """Config 2 (`-n 16777216`) generated on the device: its run result against its split.  Opt-in with MV_BIG_TESTS=1."""
    if os.environ.get("MV_BIG_TESTS") != "1":
        pytest.skip("set MV_BIG_TESTS=1")
    from minivite_b200 import gpu as G
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.generate_rgg(16777216)
        g.louvain()
        Y, rep = g.split_communities()
        got = g.compare_communities(Y)
        assert got["cells"] == rep["components"] == got["communities_y"] and got["pairs_xy"] == got["pairs_y"]
        assert got["communities_x"] == rep["communities"]
    finally:
        g.close()


# ---- several GPUs: one process per GPU ----------------------------------------------------------------------------------------
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
    g.louvain()
    comm = R.gather_arrays(g.communities())
    Y = np.arange(int(parts[rank]), int(parts[rank + 1]), dtype=np.int64) // 3 * 3
    rep = g.compare_communities(Y)
    m = R.gather_arrays(g.community_matches()["best"])
    if rank == 0:
        json.dump({"comm": [int(x) for x in np.concatenate(comm)], "rep": {k: rep[k] for k in CR.FIELDS},
                   "best": [int(x) for x in np.concatenate(m)]}, open(os.path.join(out_dir, "res.json"), "w"))
    g.close()
    R.shutdown()


def test_multi_gpu_compare(tmp_path):
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
    X = np.array(res["comm"], np.int64)
    ref = CR.compare(X, np.arange(len(X), dtype=np.int64) // 3 * 3)
    assert res["rep"] == {k: ref[k] for k in CR.FIELDS}
    assert res["best"] == [int(x) for x in ref["best"]]
