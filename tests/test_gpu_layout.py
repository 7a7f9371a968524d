"""The setup decisions and the layout of the locality renumbering, pinned exactly against tests/layout_ref.py.

Tie-breaks compare labels, so any bijective renumbering gives the same traces: the result tests cannot see whether
k_msbfs left a vertex in a non-minimal region or at the wrong level, whether k_bfs_sortkeys ordered the keys differently,
whether the auto decision renumbered, or whether a spurious `unordered` flag kept iteration 1 off the singleton reduction
(FIRST).  mv_layout_readback (a test hook of libmvgpu.so, not in mvgpu.h) returns the decisions and the device arrays of
the last run; every test compares them element for element with the host restatement -- bfs_key itself, not only perm,
since perm hides levels above 255 -- and then checks the run's results against the C oracle or the golden trace.

The rank that keeps its numbering while another renumbers (want = 0, relabel = 1: identity perm from k_bfs_sortkeys, inv
from k_perm_inverse, labels, k_apply_inv on the send list) is built on purpose: rank 0's vertex range is relabelled in
reverse Cuthill-McKee order, so its sampled span is below lnv/64 and rank 1's is above."""
import ctypes
import os
import threading

import numpy as np
import pytest

import layout_ref as LR
from helpers import assert_trace_matches, case_graph, random_graph, rmat_graph, split_global, weighted_exact_cases
from test_gpu_parity import gpu  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
INFO_KEYS = ["want", "relabel", "reordered", "stride", "nregions", "span_sum", "span_cnt", "unordered", "has_self",
             "simple_sorted", "first_ran", "unit", "nlow", "nghost", "lnv", "lne"]
SCALARS = ["want", "relabel", "reordered", "stride", "nregions", "unordered", "has_self", "simple_sorted", "first_ran",
           "nlow", "nghost", "lnv", "lne"]
ARRAYS = ["rowptr", "tails", "bfs_key", "perm", "inv", "lab", "rowptr2", "tails2", "weights2"]


# ---- read-back --------------------------------------------------------------------------------------------------------
def _readback_fn():
    from minivite_b200 import gpu as G
    f = G.lib().mv_layout_readback
    f.argtypes = [ctypes.c_void_p] * 11
    f.restype = ctypes.c_int
    return f


def readback(g):
    from minivite_b200 import gpu as G
    f = _readback_fn()
    info = (ctypes.c_int64 * 16)()
    G._ck(f(g._h, info, *[None] * 9))
    d = dict(zip(INFO_KEYS, [int(x) for x in info]))
    lnv, lne = d["lnv"], d["lne"]
    a = {"rowptr": np.zeros(lnv + 1, np.uint32), "tails": np.zeros(lne, np.int32)}
    if d["want"] and d["relabel"] and lnv:
        a["bfs_key"] = np.zeros(lnv, np.uint32)
    if d["relabel"] and lnv:
        a.update(perm=np.zeros(lnv, np.int32), inv=np.zeros(lnv, np.int32), lab=np.zeros(lnv, np.int32))
    if d["reordered"]:
        a.update(rowptr2=np.zeros(lnv + 1, np.uint32), tails2=np.zeros(lne, np.int32))
        if not d["unit"]:
            a["weights2"] = np.zeros(lne, np.float64)
    G._ck(f(g._h, None, *[a[k].ctypes.data if k in a else None for k in ARRAYS]))
    d.update(a)
    d["span"] = (d["span_sum"], d["span_cnt"])
    return d


def assert_layout(dev, ref, what):
    for k in SCALARS:
        assert dev[k] == ref[k], (what, k, dev[k], ref[k])
    assert dev["span"] == tuple(ref["span"]), (what, dev["span"], ref["span"])
    for k in ARRAYS:
        have = k in ref and ref[k] is not None
        assert (k in dev) == have, (what, k)
        if have:
            assert dev[k].dtype == np.asarray(ref[k]).dtype and np.array_equal(dev[k], ref[k]), (what, k)


# ---- runs ---------------------------------------------------------------------------------------------------------------
def oracle_run(parts, rps, eds):
    from oracle import oracle as O
    ref = O.louvain(parts, rps, eds)
    return {"iters": ref["iters"], "mod": ref["modularity"], "trace": ref["trace"], "comm": np.concatenate(ref["comm"])}


def assert_same_results(res, ref, what):
    assert res["iters"] == ref["iters"] and res["mod"] == ref["mod"], (what, res["iters"], ref["iters"])
    for k in ("modularity", "moved", "chash"):
        assert np.array_equal(res["trace"][k], ref["trace"][k]), (what, k)
    assert np.array_equal(res["comm"], ref["comm"]), what


def run1(G, nv, rowptr, edges, how="upload", repeat=1, **opts):
    """One rank: run, read back; how = upload | attach | generate (device RGG of nv vertices)."""
    g = G.LouvainGPU(0, 0, 1)
    keep = None
    try:
        g.set_option("trace", 1)
        for k, v in opts.items():
            g.set_option(k, v)
        parts = np.array([0, nv], np.int64)
        if how == "upload":
            g.upload(nv, parts, rowptr, edges)
        elif how == "attach":
            import torch
            keep = (torch.from_numpy(np.ascontiguousarray(rowptr, np.int64)).cuda(),
                    torch.from_numpy(np.ascontiguousarray(edges).view(np.uint8)).cuda())
            g.attach_device(nv, parts, nv, len(edges), keep[0].data_ptr(), keep[1].data_ptr())
        else:
            g.generate_rgg(nv)
        out = []
        for _ in range(repeat):
            mod, iters = g.louvain()
            out.append({"mod": mod, "iters": iters, "trace": g.trace(), "comm": g.communities().copy(), "lay": readback(g),
                        "timings": g.timings()})
        return out if repeat > 1 else out[0]
    finally:
        g.close()
        del keep


def ref_layout(nv, rowptr, edges, weighted=False, **opts):
    lo = {k: v for k, v in opts.items() if k in ("reorder", "region_size", "first_iter", "scan_variant")}
    return LR.layout(np.array([0, nv], np.int64), rowptr, edges["tail"], weights=edges["weight"] if weighted else None,
                     unit=not weighted, **lo)


def check1(G, nv, rowptr, edges, oracle=None, what="", **opts):
    """Run one rank, compare the layout with the restatement and the results with the C oracle."""
    res = run1(G, nv, rowptr, edges, **opts)
    assert_layout(res["lay"], ref_layout(nv, rowptr, edges, **opts), (what, opts))
    assert res["timings"]["reordered"] == res["lay"]["reordered"]
    if oracle is None:
        oracle = oracle_run(np.array([0, nv], np.int64), [rowptr], [edges])
    assert_same_results(res, oracle, (what, opts))
    return res


def rgg(n, strips=1):
    """Global CSR of `miniVite -n n` generated on `strips` ranks."""
    from minivite_b200 import hostgraph as hg
    ss = hg.generate_rgg(n, strips)
    rowptr = np.concatenate([[0]] + [s.rowptr[1:] + off for s, off in
                                     zip(ss.shards, np.cumsum([0] + [s.lne for s in ss.shards[:-1]]))]).astype(np.int64)
    edges = np.concatenate([np.array(s.edges) for s in ss.shards])
    ss.close()
    return n, rowptr, edges


def csr(adj):
    from minivite_b200 import hostgraph as hg
    rowptr = np.concatenate([[0], np.cumsum([len(a) for a in adj])]).astype(np.int64)
    edges = np.zeros(int(rowptr[-1]), hg.EDGE_DTYPE)
    edges["tail"] = [t for a in adj for t in a]
    edges["weight"] = 1.0
    return len(adj), rowptr, edges


def path_adj(n, off=0):
    return [[off + v - 1] * (v > 0) + [off + v + 1] * (v + 1 < n) for v in range(n)]


# ---- single rank ------------------------------------------------------------------------------------------------------
def test_rgg_regions(gpu):
    """rgg_n16384_p1 renumbered at region sizes 32 .. 4096 and one region for the whole shard (a single seed)."""
    nv, rowptr, edges = rgg(16384)
    ora = oracle_run(np.array([0, nv], np.int64), [rowptr], [edges])
    for region in (32, 64, 512, 4096, 16384, 100000):
        res = check1(gpu, nv, rowptr, edges, ora, "rgg16384", reorder=1, region_size=region)
        assert res["lay"]["reordered"] == 1 and res["lay"]["first_ran"] == 1


def test_rgg_auto_mode(gpu):
    """Auto mode at 65 536 and 131 072 vertices: the RGG numbering has no locality, so the shard renumbers."""
    for n in (65536, 131072):
        nv, rowptr, edges = rgg(n)
        res = check1(gpu, nv, rowptr, edges, None, "rgg%d" % n)
        assert res["lay"]["want"] == 1 and res["lay"]["span_cnt"] > 0


def test_rmat(gpu):
    """R-MAT hubs spread thousands of edges over many 512-edge batches of one warp (row_of_edge, warp-aggregated
    appends); scale 17 in auto mode."""
    for scale, opts in ((14, {"reorder": 1}), (14, {"reorder": 1, "region_size": 32}), (17, {})):
        nv, rowptr, edges = rmat_graph(scale, 16, 1)
        res = check1(gpu, nv, rowptr, edges, None, "rmat%d" % scale, **opts)
        assert res["lay"]["want"] == 1


def test_unreached_and_clamped_levels(gpu):
    """Components without a seed, isolated vertices, a 2 500-vertex path with one seed (levels above 255 share the
    clamped sort key, levels above 1023 stay unreached and sort last in id order) and a 200 x 200 grid."""
    comps = path_adj(10) + [[] for _ in range(5)] + path_adj(700, 15) + [[] for _ in range(3)] + path_adj(30, 718)
    graphs = {"components": (csr(comps), (64, 512)), "path2500": (csr(path_adj(2500)), (4096,)),
              "path2500_two_seeds": (csr(path_adj(2500)), (2048,))}
    side = 200
    grid = [[u for u in ((v - side) if v >= side else -1, v - 1 if v % side else -1, v + 1 if (v + 1) % side else -1,
                         v + side if v + side < side * side else -1) if u >= 0] for v in range(side * side)]
    graphs["grid200"] = (csr(grid), (32, 512, 40000))
    for name, ((nv, rowptr, edges), regions) in graphs.items():
        ora = oracle_run(np.array([0, nv], np.int64), [rowptr], [edges])
        for region in regions:
            res = check1(gpu, nv, rowptr, edges, ora, name, reorder=1, region_size=region)
            key = res["lay"]["bfs_key"]
            if name == "path2500":
                assert np.all(key[1024:] == LR.UNREACHED) and (int(key[1023]) >> 22) == 1023
            if name == "components":
                assert np.any(key == LR.UNREACHED)


def test_ragged_sizes(gpu):
    """lnv 1, 31, 33, 1000 and 4099: ragged bitmap words and a ragged last region."""
    for n in (1, 31, 33, 1000, 4099):
        if n == 1:
            nv, rowptr, edges = csr([[0]])
        else:
            rowptr, edges = random_graph(n, 4, n)
            nv = n
        for region in (32, 96):
            check1(gpu, nv, rowptr, edges, None, "ragged%d" % n, reorder=1, region_size=region)


def shuffled(rowptr, edges, seed):
    rng = np.random.default_rng(seed)
    e = edges.copy()
    for v in range(len(rowptr) - 1):
        a, b = rowptr[v], rowptr[v + 1]
        e[a:b] = e[a:b][rng.permutation(b - a)]
    return e


def test_unordered_flag_and_first_gate(gpu):
    """`unordered` through k_permute_adj (renumbered) and k_vertex_init (original numbering) on self loops, parallel
    edges and shuffled adjacency lists; on a simple sorted graph FIRST runs exactly for first_iter=1 and scan_variant >= 4."""
    rowptr, edges = random_graph(3000, 6, 11)
    graphs = {"simple": (rowptr, edges), "self_loops": random_graph(3000, 6, 11, self_loops=20),
              "parallel": random_graph(3000, 6, 11, multi=30), "shuffled": (rowptr, shuffled(rowptr, edges, 12))}
    for name, (rp, ed) in graphs.items():
        ora = oracle_run(np.array([0, 3000], np.int64), [rp], [ed])
        for reorder in (0, 1):
            res = check1(gpu, 3000, rp, ed, ora, name, reorder=reorder, region_size=64)
            assert res["lay"]["simple_sorted"] == (name == "simple"), (name, reorder)
    for reorder in (0, 1):
        for first_iter in (0, 1):
            for variant in (3, 4, 6):
                res = check1(gpu, 3000, rowptr, edges, None, "simple", reorder=reorder, first_iter=first_iter,
                             scan_variant=variant)
                assert res["lay"]["first_ran"] == int(first_iter == 1 and variant >= 4)


def test_first_gate_on_32bit_surface(gpu):
    """The USE_32_BIT_GRAPH surface never runs FIRST, even on a simple sorted graph."""
    rowptr, edges = random_graph(3000, 6, 11)
    e32 = np.zeros(len(edges), np.dtype([("tail", "<i4"), ("weight", "<f4")]))
    e32["tail"], e32["weight"] = edges["tail"], 1.0
    for reorder in (0, 1):
        g = gpu.LouvainGPU(0, 0, 1)
        try:
            g.set_option("reorder", reorder)
            g.upload32(3000, np.array([0, 3000], np.int32), rowptr.astype(np.int32), e32)
            g.louvain32()
            lay = readback(g)
        finally:
            g.close()
        ref = LR.layout(np.array([0, 3000], np.int64), rowptr, edges["tail"], reorder=reorder, f32=True)
        assert_layout(lay, ref, ("f32", reorder))
        assert lay["simple_sorted"] == 1 and lay["first_ran"] == 0


def test_weighted_renumbering_carries_weights(gpu):
    """Dyadic weighted cases with reorder=1: weights2 follows tails2, results bit-exact against the golden trace."""
    from oracle import oracle as O
    cases = weighted_exact_cases()
    from helpers import global_csr
    for name in ("rgg_n16384_s1", "random_n777_d150_self_loops40_multi300", "hand_self_loops_w"):
        case = cases[name]
        nv, rowptr, edges = global_csr(case)
        for region in (32, 512):
            res = run1(gpu, nv, rowptr, edges, reorder=1, region_size=region)
            assert_layout(res["lay"], ref_layout(nv, rowptr, edges, weighted=True, reorder=1, region_size=region), name)
            assert res["lay"]["unit"] == 0 and "weights2" in res["lay"]
            assert_trace_matches(case, res["iters"], res["mod"], res["trace"], O.comm_hash(0, res["comm"]), res["comm"])


def test_every_input_path_gives_one_layout(gpu):
    """compact_upload 0 / 1 / 2, mvgpu_attach_shard_device and mvgpu_generate_rgg_shard_ex: one compact CSR, one layout."""
    nv, rowptr, edges = rgg(16384)
    ref = ref_layout(nv, rowptr, edges, reorder=1, region_size=64)
    ora = oracle_run(np.array([0, nv], np.int64), [rowptr], [edges])
    runs = [("compact%d" % cu, dict(compact_upload=cu, upload_chunk=4096)) for cu in (0, 1, 2)]
    runs += [("attach", dict(how="attach")), ("generate", dict(how="generate"))]
    for what, o in runs:
        res = run1(gpu, nv, rowptr, edges, reorder=1, region_size=64, **o)
        assert_layout(res["lay"], ref, what)
        assert_same_results(res, ora, what)


def test_repeated_runs_and_stale_buffers(gpu):
    """mvgpu_louvain twice on one context; then a large graph and a small one through the same context, so the BFS queue
    (in ids), the level bitmaps (in sortkey2) and bfs_level_count start from the previous run's contents."""
    nv, rowptr, edges = rgg(65536)
    ref = ref_layout(nv, rowptr, edges)
    for res in run1(gpu, nv, rowptr, edges, repeat=2):
        assert_layout(res["lay"], ref, "repeat")
    big_n, big_rp, big_ed = rmat_graph(15, 16, 3)
    small_rp, small_ed = random_graph(1000, 5, 13)
    g = gpu.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        g.set_option("reorder", 1)
        for n, rp, ed, region in ((big_n, big_rp, big_ed, 32), (1000, small_rp, small_ed, 512), (big_n, big_rp, big_ed, 512),
                                  (1000, small_rp, small_ed, 32)):
            g.set_option("region_size", region)
            g.upload(n, np.array([0, n], np.int64), rp, ed)
            mod, iters = g.louvain()
            assert_layout(readback(g), ref_layout(n, rp, ed, reorder=1, region_size=region), ("reuse", n, region))
            assert_same_results({"mod": mod, "iters": iters, "trace": g.trace(), "comm": g.communities().copy()},
                                oracle_run(np.array([0, n], np.int64), [rp], [ed]), ("reuse", n))
    finally:
        g.close()


# ---- several ranks on one device -------------------------------------------------------------------------------------
def run_ranks(parts, rps, eds, **opts):
    """Ranks as threads sharing device 0 (host transport, as tests/test_gpu_multirank_one_device.py); per-rank read-back."""
    from minivite_b200 import gpu as G
    world = len(rps)
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
            out[rank] = {"mod": mod, "iters": iters, "trace": g.trace(), "comm": g.communities().copy(), "lay": readback(g)}
            g.close()
        except Exception as ex:
            errs.append((rank, repr(ex)))
    th = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    assert all(o is not None for o in out), "a rank did not finish"
    return {"mod": out[0]["mod"], "iters": out[0]["iters"], "trace": out[0]["trace"],
            "comm": np.concatenate([o["comm"] for o in out]), "lays": [o["lay"] for o in out]}


def assert_rank_layouts(res, parts, rps, eds, what, **opts):
    refs = LR.shard_layouts(parts, rps, [e["tail"] for e in eds], **opts)
    for r, (dev, ref) in enumerate(zip(res["lays"], refs)):
        assert_layout(dev, ref, (what, r))
    return refs


@pytest.mark.parametrize("case_name,world", [("rgg_n16384_p4", 4), ("file_rgg_n32768_s8_p4", 4)])
def test_multirank_shards(golden, case_name, world):
    """Every rank's BFS ignores its ghost slots and tails_ascend puts the nlow lower ghosts first."""
    from test_gpu_multirank_one_device import resplit
    parts, rps, eds, _keep = resplit(golden, case_name, world)
    for region in (32, 512):
        res = run_ranks(parts, rps, eds, reorder=1, region_size=region)
        refs = assert_rank_layouts(res, parts, rps, eds, case_name, reorder=1, region_size=region)
        assert any(r["nlow"] > 0 for r in refs) and all(r["nghost"] > 0 for r in refs)
        assert_trace_matches(golden[case_name], res["iters"], res["mod"], res["trace"], None,
                             res["comm"] if "comm" in golden[case_name] else None)


def keep_order_graph(nranks):
    """An RGG of 65 536 vertices per rank whose even ranks' vertex ranges are relabelled in reverse Cuthill-McKee order of
    their induced subgraphs (adjacency re-sorted, still symmetric): in auto mode the even ranks keep their numbering and
    the odd ranks renumber."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import reverse_cuthill_mckee
    n = 65536 * nranks
    nv, rowptr, edges = rgg(n, nranks)
    parts = np.array([(nv * r) // nranks for r in range(nranks + 1)], np.int64)
    new = np.arange(nv, dtype=np.int64)
    src = np.repeat(np.arange(nv), np.diff(rowptr))
    dst = edges["tail"].astype(np.int64)
    for r in range(0, nranks, 2):
        a, b = parts[r], parts[r + 1]
        m = (src >= a) & (src < b) & (dst >= a) & (dst < b)
        A = sp.csr_matrix((np.ones(int(m.sum())), (src[m] - a, dst[m] - a)), shape=(b - a, b - a))
        order = reverse_cuthill_mckee(A, symmetric_mode=True)
        new[a + order] = a + np.arange(b - a)
    s2, d2 = new[src], new[dst]
    o = np.lexsort((d2, s2))
    rp = np.zeros(nv + 1, np.int64)
    np.add.at(rp, s2 + 1, 1)
    ed = np.zeros(len(d2), edges.dtype)
    ed["tail"], ed["weight"] = d2[o], 1.0
    return nv, parts, np.cumsum(rp), ed


@pytest.mark.parametrize("nranks", [2, 4])
def test_rank_that_keeps_its_numbering(gpu, nranks):
    """Mixed auto decisions: even ranks keep their order (identity perm/inv, lab = base + v, labels still used, send
    list through k_apply_inv), odd ranks renumber.  Bit-exact against the C oracle on the same shards and against a
    1-rank run of the same graph."""
    nv, parts, rowptr, edges = keep_order_graph(nranks)
    _, rps, eds = split_global(nv, rowptr, edges, nranks)
    for r in range(nranks):
        want, (s, c) = LR.rank_want(parts, rps[r], eds[r]["tail"], r)
        lnv = parts[r + 1] - parts[r]
        assert want == (r % 2 == 1), (r, s / c, lnv / 64)
    res = run_ranks(parts, rps, eds)
    refs = assert_rank_layouts(res, parts, rps, eds, "keep_order")
    for r, dev in enumerate(res["lays"]):
        assert dev["want"] == r % 2 and dev["relabel"] == 1 and dev["reordered"] == r % 2
        if r % 2 == 0:
            assert np.array_equal(dev["perm"], np.arange(dev["lnv"])) and np.array_equal(dev["inv"], dev["perm"])
            assert np.array_equal(dev["lab"], parts[r] + np.arange(dev["lnv"]))
    assert refs[0]["want"] == 0 and refs[1]["want"] == 1
    ora = oracle_run(parts, rps, eds)
    assert_same_results(res, ora, "keep_order vs oracle")
    one = run1(gpu, nv, rowptr, edges)
    assert_same_results(one, ora, "keep_order 1 rank")


def threshold_graph(L, lnv=65536):
    """A band graph (v ~ v +- 1, 2) on lnv vertices plus one chord of length L from every vertex 0 mod 64 (the sampled
    rows) and a chord of length 20001 from every vertex 32 mod 64 (never sampled, nor are its partners).  The sampled
    mean span is then about (6 + L) / 5; a sample of every 32nd row would also see the long chords."""
    from minivite_b200 import hostgraph as hg
    v = np.arange(lnv, dtype=np.int64)
    a = [v[:-1], v[:-2]]
    b = [v[1:], v[2:]]
    for start, length in ((0, L), (32, 20001)):
        s = np.arange(start, lnv, 64, dtype=np.int64)
        a.append(s)
        b.append(np.where(s + length < lnv, s + length, s - length))
    a, b = np.concatenate(a), np.concatenate(b)
    key = np.unique(np.minimum(a, b) * lnv + np.maximum(a, b))
    src, dst = np.concatenate([key // lnv, key % lnv]), np.concatenate([key % lnv, key // lnv])
    o = np.lexsort((dst, src))
    rowptr = np.zeros(lnv + 1, np.int64)
    np.add.at(rowptr, src + 1, 1)
    edges = np.zeros(len(dst), hg.EDGE_DTYPE)
    edges["tail"], edges["weight"] = dst[o], 1.0
    return lnv, np.cumsum(rowptr), edges


def test_auto_threshold(gpu):
    """Two graphs whose sampled mean span sits just above and just below lnv/64 = 1024 pin the threshold, the compare
    and the sampling stride of the auto decision: the one above stays below lnv/32, and a sample of every 32nd row
    would put the one below above lnv/64."""
    spans = {}
    for L in range(5100, 5130):
        nv, rowptr, edges = threshold_graph(L)
        spans[L] = LR.span_sample(nv, rowptr, edges["tail"])
    above = min(L for L, (s, c) in spans.items() if s / c > 65536 / 64)
    below = max(L for L, (s, c) in spans.items() if s / c <= 65536 / 64)
    for L, side in ((above, True), (below, False)):
        nv, rowptr, edges = threshold_graph(L)
        s, c = spans[L]
        assert abs(s / c - nv / 64) < 2.0 and s / c < nv / 32, (L, s, c)
        s32, c32 = LR.span_sample(nv, rowptr, edges["tail"], 32)
        assert s32 / c32 > nv / 32, (L, s32, c32)
        res = check1(gpu, nv, rowptr, edges, None, ("threshold", L))
        assert res["lay"]["want"] == int(side) and res["lay"]["span"] == (s, c), (L, side)


@pytest.mark.skipif(os.environ.get("MV_BIG_TESTS") != "1", reason="config-2 layout check (MV_BIG_TESTS=1)")
def test_config2_layout_matches_restatement(gpu):
    """BASELINE.json configs[1] (RGG -n 16777216, one GPU): the device bfs_key and perm equal the restatement's."""
    nv, rowptr, edges = rgg(16777216)
    g = gpu.LouvainGPU(0, 0, 1)
    try:
        g.upload(nv, np.array([0, nv], np.int64), rowptr, edges)
        g.louvain()
        from minivite_b200 import gpu as G
        info = (ctypes.c_int64 * 16)()
        key, perm = np.zeros(nv, np.uint32), np.zeros(nv, np.int32)
        f = _readback_fn()
        G._ck(f(g._h, info, None, None, key.ctypes.data, perm.ctypes.data, None, None, None, None, None))
    finally:
        g.close()
    assert int(info[0]) == 1 and int(info[3]) == 512
    rk = LR.bfs_keys(nv, rowptr, edges["tail"], 512)
    assert np.array_equal(key, rk)
    assert np.array_equal(perm, np.argsort(LR.sort_keys(rk, LR.nregions_of(nv, 512)), kind="stable"))
