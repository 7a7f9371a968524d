"""Quality of an assignment on the device (mvgpu_evaluate_communities, mvgpu_get_community_stats,
mvgpu_get_compact_communities; DESIGN.md §3.10), against the NumPy restatement tests/quality_ref.py.

Unit and dyadic weights make every sum exact, so the device must match the restatement bit for bit: the global fields,
the per-community arrays and the compact labels, on 1 rank and on 2 and 4 ranks sharing device 0 (host transport), with
every renumbering mode and upload mode.  The same evaluation ties the reported per-iteration modularity to the golden
traces: T[k].modularity == fabs(e_in(X_{k-1})*c - (a2(X_k)*c)*c), with X_k taken from stop_after checkpoints."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from helpers import case_graph, random_graph, split_global
import quality_ref as QR
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_warm_start import CASES, Ranks, assignments, graphs, layout_info
from test_quality_ref import identity_points

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "bin", "miniVite_b200")
GLOBAL_FIELDS = ("modularity", "e_in", "a2", "constant", "communities", "singletons", "max_size")


def evaluate(R, X=None):
    """Evaluate X (whole-graph assignment, or None = the last run's) on every rank of R; returns the global fields (the
    same on every rank) and the concatenated per-community arrays and compact labels."""
    def one(r, g):
        q = g.evaluate(None if X is None else X[R.parts[r]:R.parts[r + 1]])
        return q, g.community_stats(), g.compact_communities().copy()
    res = R.each(one)
    q = res[0][0]
    for o in res[1:]:
        assert all(repr(o[0][k]) == repr(q[k]) for k in GLOBAL_FIELDS), (o[0], q)
    out = dict(q)
    for k in ("size", "volume", "internal"):
        out[k] = np.concatenate([o[1][k] for o in res])
    out["compact"] = np.concatenate([o[2] for o in res])
    return out


def assert_matches(got, ref, what, rel=0.0):
    for k in GLOBAL_FIELDS:
        if rel and isinstance(ref[k], float):
            assert abs(got[k] - ref[k]) <= rel * max(abs(ref[k]), 1e-300), (what, k, got[k], ref[k])
        else:
            assert repr(got[k]) == repr(ref[k]) if isinstance(ref[k], float) else got[k] == ref[k], (what, k, got[k], ref[k])
    assert np.array_equal(got["size"], ref["size"]), what
    assert np.array_equal(got["compact"], ref["compact"]), what
    for k in ("volume", "internal"):
        if rel:
            assert np.allclose(got[k], ref[k], rtol=rel, atol=0.0), (what, k)
        else:
            assert np.array_equal(got[k], ref[k]), (what, k)


# ---- golden cases: X_0, the final assignment and the identity at the split points ----------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_cases_and_identity(gpu, name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    nv = int(parts[-1])
    R = Ranks(parts, rps, eds)
    try:
        X0 = np.arange(nv, dtype=np.int64)
        assert_matches(evaluate(R, X0), QR.quality(parts, rps, eds, X0), f"{name} X_0")
        final = R.run()
        assert final["trace"] == [(float(t["modularity"]), int(t["moved"]), int(t["chash"], 16)) for t in case["trace"]]
        assert_matches(evaluate(R), QR.quality(parts, rps, eds, final["comm"]), f"{name} final")
        qs = {0: evaluate(R, X0)}
        for k in identity_points(case):
            for j in (k - 1, k):
                if j not in qs:
                    R.set_option("stop_after", j)
                    qs[j] = evaluate(R, R.run()["comm"])
            got = QR.mixed_modularity(qs[k - 1], qs[k])
            assert repr(got) == repr(float(case["trace"][k - 1]["modularity"])), (name, k)
        R.set_option("stop_after", 0)
    finally:
        R.close()


# ---- random and hand-made assignments, 1 / 2 / 4 ranks, every renumbering mode ---------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 4])
def test_assignments_on_ranks_and_reorder_modes(gpu, world):
    for gname, (nv, rowptr, edges) in graphs().items():
        parts, rps, eds = split_global(nv, rowptr, edges, world)
        for reorder in (0, 1, 2):
            R = Ranks(parts, rps, eds, reorder=reorder)
            try:
                R.run()                                  # a run first: its renumbering must not leak into the labels
                for aname, X in dict(assignments(nv, world), singletons=np.arange(nv, dtype=np.int64)).items():
                    assert_matches(evaluate(R, X), QR.quality(parts, rps, eds, X), f"{gname} {aname} {world} {reorder}")
            finally:
                R.close()


def test_hand_graph_isolated_loops_multi(gpu):
    from test_quality_ref import hand_assignments, hand_graphs
    for gname, (nv, rowptr, edges) in hand_graphs().items():
        for world in (1, 2):
            parts, rps, eds = split_global(nv, rowptr, edges, world)
            R = Ranks(parts, rps, eds)
            try:
                for aname, X in hand_assignments(nv).items():
                    got = evaluate(R, X)
                    assert_matches(got, QR.quality(parts, rps, eds, X), f"{gname} {aname} {world}")
                    if aname == "one_community" and gname != "dyadic300":
                        assert got["modularity"] == 0.0
            finally:
                R.close()


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_upload_modes(gpu, mode):
    rp, ed = random_graph(20000, 10, seed=2, blocks=64)
    for world in (1, 2):
        parts, rps, eds = split_global(20000, rp, ed, world)
        R = Ranks(parts, rps, eds, compact_upload=mode)
        try:
            res = R.run()
            assert_matches(evaluate(R), QR.quality(parts, rps, eds, res["comm"]), f"compact_upload={mode} {world}")
        finally:
            R.close()


def test_device_generated_and_attached_shards(gpu):
    import torch
    from minivite_b200 import gpu as G
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.generate_rgg(65536)
        rowptr, edges = g.download_shard()
        g.louvain()
        comm = g.communities().copy()
        parts = np.array([0, 65536], np.int64)
        ref = QR.quality(parts, [rowptr], [edges], comm)
        got = g.evaluate()
        assert all(repr(got[k]) == repr(ref[k]) for k in GLOBAL_FIELDS), (got, ref)
        d_rp = torch.from_numpy(rowptr).cuda()
        d_ed = torch.from_numpy(edges.view(np.uint8).copy()).cuda()
        g.attach_device(65536, parts, 65536, len(edges), d_rp.data_ptr(), d_ed.data_ptr(), keepalive=(d_rp, d_ed))
        got = g.evaluate(comm)
        assert all(repr(got[k]) == repr(ref[k]) for k in GLOBAL_FIELDS)
        assert np.array_equal(g.compact_communities(), ref["compact"])
    finally:
        g.close()


def test_euclidean_weights_within_tolerance(gpu):
    """Euclidean -w weights: the device adds the community volumes, the internal weights and 2m with atomics in no fixed
    order, so its sums may differ from the restatement's correctly rounded ones in the last bits.  Held to 1e-12 relative
    (the sums have at most a few hundred thousand terms of one sign)."""
    from minivite_b200 import hostgraph as hg
    for world in (1, 2):
        ss = hg.generate_rgg(65536, world, unit_weight=False)
        parts = ss.shards[0].parts
        rps, eds = [s.rowptr for s in ss.shards], [s.edges for s in ss.shards]
        R = Ranks(parts, rps, eds)
        try:
            res = R.run()
            for X in (res["comm"], np.arange(65536, dtype=np.int64) // 7 * 7):
                assert_matches(evaluate(R, X), QR.quality(parts, rps, eds, X), f"-w {world}", rel=1e-12)
        finally:
            R.close()
            ss.close()


# ---- state rules: an evaluation changes nothing a run reports, and nothing the next run does ----------------------------
def snapshot(g):
    """Everything a context reports about its last run.  communities() is read from the array
    mvgpu_get_communities_device points to, so the pointer and the host copy together pin the device array."""
    import ctypes
    from minivite_b200 import gpu as G
    d = ctypes.c_void_p()
    G._ck(G.lib().mvgpu_get_communities_device(g._h, ctypes.byref(d)))
    return {"comm": g.communities().tolist(), "comm_dev_ptr": d.value, "trace": g.trace().tolist(), "timings": g.timings(),
            "scan": g.scan_times().tolist(), "converged": g.converged(), "constant": repr(g.constant()),
            "layout": layout_info(g)}


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
                evaluate(R)
                assert snapshot(g) == before, (reorder, warm)
                b = R.run()                               # the initial assignment (if any) and the options still hold
                ref = plain.run()
                assert b["trace"] == ref["trace"] == a["trace"] and np.array_equal(b["comm"], ref["comm"])
                assert R.g[0].timings()["kernel_launches"] == plain.g[0].timings()["kernel_launches"]
                evaluate(R, other)
                R.set_initial(None)
                plain.set_initial(None)
                c, cref = R.run(), plain.run()            # a cold run after an evaluation
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
        q = evaluate(R)
        assert_matches(q, QR.quality(parts, rps, eds, a["comm"]), "2 ranks")
        assert all(np.array_equal(g.communities(), c) for g, c in zip(R.g, comm_before))
        assert R.run()["trace"] == a["trace"]
        assert_matches(evaluate(R), q, "2 ranks again")
    finally:
        R.close()


@pytest.mark.parametrize("reorder", [0, 1])
@pytest.mark.parametrize("stop", [1, 2])
def test_evaluation_right_after_a_run_keeps_its_result(gpu, reorder, stop):
    """One rank leaves the run's caller-order labels unresolved until they are asked for, and the run's assignment sits
    in comm_a or comm_b depending on the parity of its iteration count (stop_after 1 and 2 cover both), which an
    evaluation's setup overwrites.  So evaluate an array straight after louvain(), with no communities() in between,
    and only then read the run's result -- communities() copies the array get_communities_device points to -- and
    evaluate it with None."""
    from minivite_b200 import gpu as G
    case = CASES["rgg_n65536_p1"]
    parts, rps, eds, _keep = case_graph(case)
    nv = int(parts[-1])
    other = np.random.default_rng(11).integers(0, nv, nv)
    plain = Ranks(parts, rps, eds, reorder=reorder, stop_after=stop)
    try:
        want = plain.run()["comm"]
    finally:
        plain.close()
    ref_run, ref_other = QR.quality(parts, rps, eds, want), QR.quality(parts, rps, eds, other)
    for none_first in (False, True):
        g = G.LouvainGPU(0, 0, 1)
        try:
            for k, v in (("reorder", reorder), ("stop_after", stop)):
                g.set_option(k, v)
            g.upload(nv, parts, rps[0], eds[0])
            g.louvain()
            got = g.evaluate(other)
            assert all(repr(got[k]) == repr(ref_other[k]) for k in GLOBAL_FIELDS)
            if none_first:
                got = g.evaluate()
                assert np.array_equal(g.communities(), want), (reorder, stop)
            else:
                assert np.array_equal(g.communities(), want), (reorder, stop)
                got = g.evaluate()
            assert all(repr(got[k]) == repr(ref_run[k]) for k in GLOBAL_FIELDS), (reorder, stop, none_first)
            assert np.array_equal(g.compact_communities(), ref_run["compact"])
        finally:
            g.close()


# ---- errors ----------------------------------------------------------------------------------------------------------------
def test_wrong_length_fails_every_rank_and_clears_the_stats(gpu):
    """A rank whose array has the wrong length still enters the collective, so its peer fails with it instead of
    waiting; a failed evaluation leaves no stale per-community arrays behind."""
    case = CASES["rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        X = np.arange(int(parts[-1]), dtype=np.int64)
        evaluate(R, X)
        errs = R.each(lambda r, g: _err(lambda: g.evaluate(X[parts[r]:parts[r + 1]] if r == 0 else X[:5])))
        assert errs[1] and "entries" in errs[1] and errs[0] and "another rank" in errs[0], errs
        errs = R.each(lambda r, g: _err(lambda: g.community_stats()))
        assert all(e and "no evaluation" in e for e in errs), errs
        assert_matches(evaluate(R, X), QR.quality(parts, rps, eds, X), "after the failure")
    finally:
        R.close()



def _err(fn):
    from minivite_b200 import gpu as G
    try:
        fn()
    except G.MvgpuError as ex:
        return str(ex)
    return None


def test_errors(gpu):
    from minivite_b200 import gpu as G
    case = CASES["rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        errs = R.each(lambda r, g: _err(lambda: g.evaluate()))           # NULL before any run
        assert all(e and "no" in e for e in errs), errs
        nv = int(parts[-1])
        bad = np.zeros(nv, np.int64)
        bad[nv - 1] = nv                                                  # a bad id on rank 1 only
        errs = R.each(lambda r, g: _err(lambda: g.evaluate(bad[parts[r]:parts[r + 1]])))
        assert errs[1] and "outside" in errs[1] and errs[0] and "another rank" in errs[0], errs
        R.run()
        errs = R.each(lambda r, g: _err(lambda: g.evaluate(None if r == 0 else np.zeros(g.lnv, np.int64))))
        assert all(e and "disagree" in e for e in errs), errs
        q = evaluate(R)                                                   # both contexts are still usable
        assert q["communities"] >= 1
    finally:
        R.close()
    g = G.LouvainGPU(0, 0, 1)
    try:
        with pytest.raises(G.MvgpuError):
            g.community_stats()
        c32 = CASES["hand_clique_ring_p1"]
        p32, r32, e32s, _k = case_graph(c32)
        e32 = np.zeros(len(e32s[0]), np.dtype([("tail", "<i4"), ("weight", "<f4")]))
        e32["tail"], e32["weight"] = e32s[0]["tail"], e32s[0]["weight"]
        g.upload32(int(p32[-1]), p32, r32[0], e32)
        g.louvain32()
        with pytest.raises(G.MvgpuError, match="upload_shard32"):
            g.evaluate()
        with pytest.raises(G.MvgpuError, match="upload_shard32"):
            g.evaluate(np.zeros(int(p32[-1]), np.int64))
    finally:
        g.close()


# ---- the CLI: -q after a run, -E on the files -o wrote -----------------------------------------------------------------------
QUALITY_RE = re.compile(r"QUALITY mod=(\S+) e=(\S+) a2=(\S+) communities=(\d+) singletons=(\d+) maxsize=(\d+)")


def parse_quality(stderr):
    m = QUALITY_RE.search(stderr)
    assert m, stderr[-2000:]
    return {"modularity": float(m.group(1)), "e_in": float(m.group(2)), "a2": float(m.group(3)),
            "communities": int(m.group(4)), "singletons": int(m.group(5)), "max_size": int(m.group(6))}


@pytest.mark.parametrize("ranks", [1, 2])
def test_cli_quality_and_evaluate_files(gpu, tmp_path, ranks):
    env = dict(os.environ)
    if ranks > 1 and gpu.device_count() < ranks:
        env["MVGPU_OPTIONS"] = "host_transport=1"
    pre = str(tmp_path / "out")
    p = subprocess.run([EXE, "-n", "16384", "-g", str(ranks), "-q", "-o", pre], capture_output=True, text=True, timeout=300, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    q_run = parse_quality(p.stderr)
    e = subprocess.run([EXE, "-n", "16384", "-g", str(ranks), "-E", pre], capture_output=True, text=True, timeout=300, env=env)
    assert e.returncode == 0, e.stderr[-2000:]
    assert "RESULT" not in e.stderr
    assert parse_quality(e.stderr) == q_run
    case = CASES["rgg_n16384_p1" if ranks == 1 else "rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    comm = np.concatenate([np.fromfile(f"{pre}.{r}", np.int64)[2:] for r in range(ranks)])
    R = Ranks(parts, rps, eds)
    try:
        want = evaluate(R, comm)
    finally:
        R.close()
    assert all(q_run[k] == want[k] for k in q_run), (q_run, want)


# ---- several GPUs: one process per GPU ------------------------------------------------------------------------------------
def _multi_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from minivite_b200 import dist as D
    from minivite_b200 import gpu as G
    R = D.Ranks("gloo")
    parts, rps, eds, _keep = case_graph(CASES["rgg_n16384_p2"])
    ident = R.broadcast_bytes(G.get_unique_id() if rank == 0 else None, G.UNIQUE_ID_BYTES)
    g = G.LouvainGPU(rank, rank, world)
    g.comm_init(ident)
    g.upload(int(parts[-1]), parts, rps[rank], eds[rank])
    g.louvain()
    comm = R.gather_arrays(g.communities())
    q = g.evaluate()
    compact = R.gather_arrays(g.compact_communities())
    if rank == 0:
        json.dump({"q": {k: repr(q[k]) for k in GLOBAL_FIELDS}, "comm": [int(x) for x in np.concatenate(comm)],
                   "compact": [int(x) for x in np.concatenate(compact)]}, open(os.path.join(out_dir, "res.json"), "w"))
    g.close()
    R.shutdown()


def test_multi_gpu_evaluate(tmp_path):
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
    parts, rps, eds, _keep = case_graph(CASES["rgg_n16384_p2"])
    ref = QR.quality(parts, rps, eds, np.array(res["comm"], np.int64))
    assert all(res["q"][k] == repr(ref[k]) for k in GLOBAL_FIELDS)
    assert res["compact"] == [int(x) for x in ref["compact"]]
