"""Rank counts up to 16 (the library's limit), uneven splits and ranks that own one vertex or none, on one GPU: ranks are
threads of this process on device 0 whose setup exchanges go through the host transport (host_transport=1), so every
kernel, peer table and mailbox sized by the rank count runs at p = 16.

The bar is the unmodified reference on the same split (tests/golden/rank_traces.json): unit and dyadic cases bit for bit
(iterations, every trace record, modularity, 1/(2m), final hash, assignment where stored), Euclidean weights within 1e-6.
Splits the reference never makes (empty ranks in the middle of a large graph) are held to the C oracle on the same split
and to the partition-invariant trace of the same graph."""
import os
import re
import subprocess

import numpy as np
import pytest

import quality_ref as QR
import split_ref as SR
import update_ref as U
from helpers import assert_trace_matches, case_graph, one_shard, rank_cases
from oracle import oracle as O
from test_gpu_compare import check as check_compare
from test_gpu_movable import oracle as movable_oracle, run as movable_run, set_movable
from test_gpu_multirank_one_device import run_threads_case
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_quality import assert_matches, evaluate
from test_gpu_split import assert_split, split
from test_gpu_update import rank_batch
from test_gpu_warm_start import EXE, Ranks, assert_same, golden_trace, oracle_run, split_and_resume

pytestmark = pytest.mark.gpu
CASES = rank_cases()

# 16 ranks over the 16384-vertex graph: empty ranks first, last and in a row, and ranks of one vertex
PARTS16 = [0, 0, 1000, 1000, 1001, 3000, 3000, 3000, 7000, 7001, 9000, 12000, 12000, 15000, 16383, 16384, 16384]
# 7 ranks, two of them empty, one of one vertex
PARTS7 = [0, 4000, 4000, 4001, 9000, 9000, 12000, 16384]


def exact(case):
    return "-w" not in case.get("args", [])


def shards_on(parts, nv, rowptr, edges):
    parts = np.asarray(parts, np.int64)
    assert parts[0] == 0 and parts[-1] == nv
    rps = [np.ascontiguousarray(rowptr[a:b + 1] - rowptr[a]) for a, b in zip(parts[:-1], parts[1:])]
    eds = [np.ascontiguousarray(edges[rowptr[a]:rowptr[b]]) for a, b in zip(parts[:-1], parts[1:])]
    return parts, rps, eds


def rgg16384(parts):
    """file_rgg_n16384_s1 (our generator, one strip) on `parts`; every split of it has the same reference trace."""
    _, rps, eds, _ = case_graph(dict(CASES["file_rgg_n16384_s1_p3"], nranks=1))
    return shards_on(parts, 16384, rps[0], eds[0])


def final_hash(parts, comm):
    return sum(O.comm_hash(int(parts[r]), comm[parts[r]:parts[r + 1]]) for r in range(len(parts) - 1)) & (2 ** 64 - 1)


def check_golden(res, case, parts, constants):
    if exact(case):
        assert res["trace"] == golden_trace(case) and res["iters"] == case["iters"]
        assert repr(res["mod"]) == repr(float(case["modularity"]))
        assert all(repr(c) == case["constant"] for c in constants), constants
        assert final_hash(parts, res["comm"]) == int(case["final_chash"], 16)
        if "comm" in case:
            assert [int(x) for x in res["comm"]] == case["comm"]
    else:
        tr = [{"modularity": m, "moved": mv, "chash": h} for m, mv, h in res["trace"]]
        assert_trace_matches(case, res["iters"], res["mod"], tr, exact=False)


# ---- the bar: every golden on its own split --------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_rank_count_matches_reference(gpu, name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        res = R.run()
        check_golden(res, case, parts, R.each(lambda r, g: g.constant()))
        info = R.each(lambda r, g: g.shard_info())
    finally:
        R.close()
    assert [i["lnv"] for i in info] == [int(x) for x in np.diff(parts)]
    for r, i in enumerate(info):
        if i["lnv"] == 0:
            assert i == dict.fromkeys(i, 0), (name, r, i)
    if case["nranks"] == 16 and case["nv"] < 16:
        assert sum(i["lnv"] == 0 for i in info) == 16 - case["nv"]          # the split really had empty ranks


# ---- options at p = 16 and on splits with empty ranks ----------------------------------------------------------------------
OPTIONS = [{"scan_variant": 3}, {"scan_variant": 4}, {"scan_variant": 5}, {"scan_variant": 6}, {"reorder": 0},
           {"reorder": 1, "region_size": 64}, {"reorder": 2}, {"first_iter": 0}, {"force_heavy_deg": 8},
           {"force_weighted": 1}, {"compact_upload": 1}, {"compact_upload": 2}, {"scan_ctas": 1}]


@pytest.mark.parametrize("opts", OPTIONS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()))
def test_options_on_uneven_ranks(gpu, opts):
    case = CASES["rgg_n16384_p16"]
    res = run_threads_case(case, **opts)
    assert_trace_matches(case, res["iters"], res["mod"], res["trace"], final_hash(case_graph(case)[0], res["comm"]))
    invariant = CASES["file_rgg_n16384_s1_p16"]              # the 1-rank trace of this graph, on every split
    one = oracle_run(*one_shard(*rgg16384([0, 16384])))
    for layout in (PARTS7, PARTS16):
        parts, rps, eds = rgg16384(layout)
        assert (np.diff(parts) == 0).sum() >= 2 and (np.diff(parts) == 1).any()
        R = Ranks(parts, rps, eds, **opts)
        try:
            got = R.run()
            relabel = R.each(lambda r, g: g.timings()["reordered"])
        finally:
            R.close()
        what = (opts, len(layout) - 1)
        assert_same(got, oracle_run(parts, rps, eds), what)
        assert_same(got, one, what)
        assert got["trace"] == golden_trace(invariant), what
        if opts.get("reorder") == 1:                          # empty ranks keep their (empty) order, the others renumber
            assert relabel == [int(n > 0) for n in np.diff(parts)], what


def test_dyadic_options_at_16_ranks(gpu):
    case = CASES["hand_dyadic52_p16"]
    for opts in ({"scan_variant": 3}, {"force_heavy_deg": 2}, {"reorder": 1, "region_size": 32}):
        res = run_threads_case(case, **opts)
        assert res["timings"]["unit_weight"] == 0
        assert_trace_matches(case, res["iters"], res["mod"], res["trace"], None, res["comm"])


# ---- the other collective calls at p = 16 with empty ranks ---------------------------------------------------------------
def one_vertex_ids(parts, nv):
    owners = [int(parts[r]) for r in range(len(parts) - 1) if parts[r + 1] - parts[r] == 1]
    assert owners
    return np.asarray(owners, np.int64)[np.arange(nv) % len(owners)]


def collective_graphs():
    """(name, parts, rps, eds): the large graph on PARTS16, and hand graphs whose natural 16-rank split has empty ranks."""
    out = [("rgg16384_parts16",) + rgg16384(PARTS16)]
    for name in ("hand_two_triangles_p16", "hand_loops_multi_p16", "hand_k66_p16"):
        parts, rps, eds, _ = case_graph(CASES[name])
        out.append((name, parts, rps, eds))
    return out


@pytest.mark.parametrize("gname", [g[0] for g in collective_graphs()])
def test_collectives_with_empty_ranks(gpu, gname):
    _, parts, rps, eds = [g for g in collective_graphs() if g[0] == gname][0]
    nv = int(parts[-1])
    assert (np.diff(parts) == 0).any() and (np.diff(parts) == 1).any()
    rng = np.random.default_rng(nv)
    R = Ranks(parts, rps, eds)
    try:
        final = R.run()
        assigns = {"final": final["comm"], "random": rng.integers(0, nv, nv), "one_vertex": one_vertex_ids(parts, nv),
                   "singletons": np.arange(nv, dtype=np.int64)}
        for aname, X in assigns.items():
            what = (gname, aname)
            assert_matches(evaluate(R, X), QR.quality(parts, rps, eds, X), what)
            assert_split(split(R, X), SR.split(parts, rps, eds, X), what)
            check_compare(R, X, assigns["random"], what)
            R.set_initial(X)                                   # warm start, ids naming one-vertex ranks' vertices included
            assert_same(R.run(), oracle_run(parts, rps, eds, init=X), what)
        R.set_initial(None)
        assert_same(R.run(), final, (gname, "cold again"))
        # getters on an empty rank: empty arrays, no failure
        empty = [r for r in range(len(rps)) if parts[r + 1] == parts[r]]
        evaluate(R, final["comm"])
        check_compare(R, None, assigns["random"], (gname, "matches"), Xref=final["comm"])
        for r in empty:
            g = R.g[r]
            assert g.shard_info() == dict.fromkeys(g.shard_info(), 0)
            assert g.communities().size == 0 and g.movable().size == 0 and g.compact_communities().size == 0
            assert all(a.size == 0 for a in g.community_stats().values())
            assert all(a.size == 0 for a in g.community_matches().values())
        # stop after k, resume: the partition-invariant golden continues exactly (hand graphs: their own golden)
        case = CASES[gname] if gname in CASES else CASES["file_rgg_n16384_s1_p16"]
        split_and_resume(gname, case, R, parts, rps, eds, ks=[max(1, case["iters"] // 2)])
    finally:
        R.close()


@pytest.mark.parametrize("gname", ["rgg16384_parts16", "hand_two_triangles_p16"])
def test_update_on_some_ranks_only(gpu, gname):
    """Batches whose records live on two ranks only, the first and the last rank that own a vertex: the others (empty
    ranks included) pass nothing.  An insertion of a doubled edge between the two, then its deletion: every shard ==
    update_ref's after each step, the cold run on the changed graph == the C oracle, and the deletion restores the
    graph and its run."""
    _, parts, rps, eds = [g for g in collective_graphs() if g[0] == gname][0]
    live = [r for r in range(len(rps)) if parts[r + 1] > parts[r]]
    v0, v1 = int(parts[live[0]]), int(parts[live[-1]])
    insert = (np.array([v0, v0, v1, v1]), np.array([v1, v1, v0, v0]), np.ones(4))
    delete = (np.array([v0, v1]), np.array([v1, v0]))
    R = Ranks(parts, rps, eds)
    try:
        before = R.run()
        cur = (rps, eds)
        for step, (d, i) in enumerate(((None, insert), (delete, None))):
            batches = [rank_batch(d, i, parts[r], parts[r + 1]) for r in range(len(rps))]
            assert sum(any(t is not None and len(t[0]) for t in bt) for bt in batches) == 2
            R.each(lambda r, g: g.update_shard(*batches[r]))
            nxt = ([], [])
            for r in range(len(rps)):
                want = U.apply(int(parts[r]), cur[0][r], cur[1][r], *batches[r])
                got = R.g[r].download_shard()
                assert np.array_equal(got[0], want[0]) and got[1].tobytes() == want[1].tobytes(), (gname, step, r)
                nxt[0].append(want[0])
                nxt[1].append(want[1])
            cur = nxt
            assert_same(R.run(), oracle_run(parts, *cur), (gname, step))
        assert all(a.tobytes() == b.tobytes() for a, b in zip(cur[1], eds))
        assert_same(R.run(), before, (gname, "restored"))
    finally:
        R.close()


def test_frontier_grows_across_every_rank(gpu):
    """The path with one vertex per rank, every second vertex movable and the frontier on: the set grows from the moved
    vertices into the frozen ranks, as the C oracle grows it."""
    case = CASES["hand_path16_p16"]
    parts, rps, eds, _ = case_graph(case)
    mask = (np.arange(16) % 2 == 0).astype(np.uint8)
    R = Ranks(parts, rps, eds, frontier=1)
    try:
        set_movable(R, mask)
        res = movable_run(R)
    finally:
        R.close()
    ref = movable_oracle(parts, rps, eds, mask, 1)
    assert res["iters"] == ref["iters"] and res["trace"] == ref["trace"] and repr(res["mod"]) == repr(ref["mod"])
    assert np.array_equal(res["comm"], ref["comm"]) and np.array_equal(res["movable"], ref["movable"])
    assert res["movable"][1::2].sum() >= 7                    # odd (frozen) ranks joined the set


# ---- limits -----------------------------------------------------------------------------------------------------------------
def test_rank_limits(gpu):
    from minivite_b200 import gpu as G
    G.LouvainGPU(0, 15, 16).close()
    with pytest.raises(G.MvgpuError, match="rank"):
        G.LouvainGPU(0, 0, 17)
    g = G.LouvainGPU(0, 1, 3)
    try:
        rp = np.zeros(1, np.int64)
        g.upload(10, np.array([0, 4, 4, 10], np.int64), rp, np.zeros(0, O.EDGE_DTYPE))      # an empty range
        assert g.shard_info()["lnv"] == 0
        with pytest.raises(G.MvgpuError, match="monotone"):
            g.upload(10, np.array([0, 6, 4, 10], np.int64), np.zeros(1, np.int64), np.zeros(0, O.EDGE_DTYPE))
    finally:
        g.close()


# ---- the device generator on 16 strips ---------------------------------------------------------------------------------------
def test_device_strips_on_16_ranks_match_reference(gpu):
    """`miniVite -n 16384` on 16 ranks: every strip generated on the device, then the Louvain phase on them."""
    case = CASES["rgg_n16384_p16"]
    parts, rps, eds, _ = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        lne = R.each(lambda r, g: g.generate_rgg(16384))
        assert sum(lne) == case["ne"]
        check_golden(R.run(), case, parts, R.each(lambda r, g: g.constant()))
    finally:
        R.close()


# ---- the CLI: 5 processes on one device ---------------------------------------------------------------------------------
def test_cli_five_processes_on_one_device(gpu, tmp_path):
    """`-g 5 -f`: five forked ranks share device 0 (arrays through CUDA IPC, setup through the host transport) and read
    uneven ranges of the file; trace == the reference's 5-rank run."""
    from minivite_b200 import hostgraph as hg
    case = CASES["file_rgg_n32768_s8_p5"]
    path = str(tmp_path / "g.bin")
    hg.generate_rgg(32768, 8).write(path)
    env = dict(os.environ, MVGPU_OPTIONS="host_transport=1")
    p = subprocess.run([EXE, "-g", "5", "-f", path, "-T"], capture_output=True, text=True, timeout=600, env=env)
    assert p.returncode == 0, p.stderr[-3000:]
    it = re.findall(r"ITER (\d+) mod=(\S+) moved=(\d+) chash=([0-9a-f]+)", p.stderr)
    assert [(float(a[1]), int(a[2]), a[3]) for a in it] == [(float(t["modularity"]), t["moved"], t["chash"])
                                                            for t in case["trace"]]
    m = re.search(r"RESULT mod=(\S+) iters=(\d+)", p.stderr)
    assert repr(float(m.group(1))) == repr(float(case["modularity"])) and int(m.group(2)) == case["iters"]
