"""Shard updates on the device (mvgpu_update_shard, LouvainGPU.update_shard; DESIGN.md §3.11), against the NumPy
restatement tests/update_ref.py element for element, against the device generator (`-p 0` + extras == `-p 5`), and
through the Louvain phase: a cold run on an updated shard equals a cold run on the same graph uploaded fresh, and a warm
run from the pre-update result equals the warm-start oracle started from that assignment."""
import json
import os

import numpy as np
import pytest

import update_ref as U
from helpers import random_graph, reversed_adjacency, rmat_graph, split_global
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_warm_start import Ranks, as_trace, assert_same, oracle_run
from test_update_ref import HAND, HAND_CASES, csr, random_batch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def same(got, ref, what):
    assert np.array_equal(got[0], ref[0]), what
    assert got[1].tobytes() == ref[1].tobytes(), what


def rank_batch(delete, insert, lo, hi):
    """The records of a global batch whose src lies in [lo, hi)."""
    def pick(t):
        if t is None:
            return None
        m = (np.asarray(t[0]) >= lo) & (np.asarray(t[0]) < hi)
        return tuple(np.asarray(a)[m] for a in t)
    return pick(delete), pick(insert)


class Shard:
    """A one-rank context holding (nv, rowptr, edges), uploaded from the host or attached from torch tensors."""

    def __init__(self, mode, nv, rowptr, edges):
        import torch
        from minivite_b200 import gpu as G
        self.g = G.LouvainGPU(0, 0, 1)
        self.mode, self.t = mode, None
        if mode == "upload":
            self.g.upload(nv, np.array([0, nv], np.int64), rowptr, edges)
        elif mode == "attach":
            rp = torch.from_numpy(np.ascontiguousarray(rowptr)).cuda()
            ed = torch.from_numpy(np.ascontiguousarray(edges).view(np.uint8).copy()).cuda()
            if ed.numel() == 0:
                ed = torch.zeros(16, dtype=torch.uint8, device="cuda")
            self.t = (rp, ed, rp.clone(), ed.clone())
            torch.cuda.synchronize()
            self.g.attach_device(nv, np.array([0, nv], np.int64), len(rowptr) - 1, len(edges), rp.data_ptr(), ed.data_ptr(),
                                 keepalive=(rp, ed))
        else:
            raise ValueError(mode)

    def attached_unchanged(self):
        import torch
        if self.t is not None:
            torch.cuda.synchronize()
            assert torch.equal(self.t[0], self.t[2]) and torch.equal(self.t[1], self.t[3]), "attached arrays were written"

    def close(self):
        self.g.close()


MODES = ["upload", "attach"]


def check_update(mode, nv, rowptr, edges, delete, insert, what):
    ref = U.apply(0, rowptr, edges, delete, insert)
    s = Shard(mode, nv, rowptr, edges)
    try:
        lne = s.g.update_shard(delete, insert)
        assert lne == len(ref[1]) == s.g.shard_info()["lne"], what
        same(s.g.download_shard(), ref, (mode, what))
        s.attached_unchanged()
    finally:
        s.close()
    return ref


@pytest.mark.parametrize("mode", MODES)
def test_hand_cases(gpu, mode):
    rowptr, edges = csr([[]] * 10 + HAND + [[]] * 6)          # rows 10..13 of a 20-vertex graph, as in the CPU test
    for name, (d, i) in HAND_CASES.items():
        check_update(mode, 20, rowptr, edges, d, i, name)


@pytest.mark.parametrize("mode", MODES)
def test_random_multigraphs_unsorted_rows(gpu, mode):
    rng = np.random.default_rng(11)
    n = 3000
    rowptr, edges = random_graph(n, 8, 5, hubs=3, hub_deg=900, self_loops=200, multi=400, dyadic=True)
    for v in list(range(3)) + list(rng.integers(0, n, 300)):  # the hubs and more rows reversed
        edges = reversed_adjacency(rowptr, edges, int(v))
    for nd, ni in ((0, 0), (500, 0), (0, 700), (3000, 4000)):
        d, i = random_batch(rng, 0, n, n, rowptr, edges, nd, ni)
        check_update(mode, n, rowptr, edges, d, i, (nd, ni))


@pytest.mark.parametrize("mode", MODES)
def test_delete_everything_and_oversized_batch(gpu, mode):
    rowptr, edges = random_graph(2000, 6, 2, self_loops=30, multi=50)
    row = np.repeat(np.arange(2000), np.diff(rowptr))
    dele = (row, edges["tail"].copy())
    ref = check_update(mode, 2000, rowptr, edges, dele, None, "delete all")
    assert len(ref[1]) == 0
    rng = np.random.default_rng(4)
    k = 3 * len(edges)
    check_update(mode, 2000, rowptr, edges, dele, (rng.integers(0, 2000, k), rng.integers(0, 2000, k), rng.random(k)), "oversized")


@pytest.mark.parametrize("scale,seed,hub_deg", [(14, 3, 3684), (17, 11, 15706)])    # the golden R-MAT graphs
def test_rmat_hub_batches(gpu, scale, seed, hub_deg):
    n, rowptr, edges = rmat_graph(scale, 16, seed)
    deg = np.diff(rowptr)
    hub = int(np.argmax(deg))
    assert int(deg[hub]) == hub_deg
    rng = np.random.default_rng(scale)
    a, b = int(rowptr[hub]), int(rowptr[hub + 1])
    # half the hub's records deleted (both directions), and new pairs on the hub and on the next heaviest vertices
    gone = edges["tail"][a:b][rng.random(b - a) < 0.5]
    heavy = np.argsort(deg)[-8:]
    src = np.repeat(heavy, 500)
    dst = rng.integers(0, n, len(src))
    w = np.ones(len(src))
    dele = (np.concatenate([np.full(len(gone), hub), gone]), np.concatenate([gone, np.full(len(gone), hub)]))
    ins = (np.concatenate([src, dst]), np.concatenate([dst, src]), np.concatenate([w, w]))
    for mode in MODES:
        check_update(mode, n, rowptr, edges, dele, ins, (scale, mode))


def test_rgg_upload_attach_generate(gpu):
    """-p 5's extras inserted into the `-p 0` shard (host generator) through each hand-off mode, then deleted again."""
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    s0 = hg.generate_rgg(65536, 1, unit_weight=False).shards[0]
    s5 = hg.generate_rgg(65536, 1, unit_weight=False, random_edge_percent=5).shards[0]
    src, dst, w = U.extras(s0, s5)
    for mode in MODES:
        check_update(mode, 65536, s0.rowptr, s0.edges, None, (src, dst, w), mode)
        check_update(mode, 65536, s5.rowptr, s5.edges, (src, dst), None, mode)
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.generate_rgg(65536, unit_weight=False)
        rp0, ed0 = g.download_shard()
        assert g.update_shard(None, None) == len(ed0)                # empty batch: byte-identical
        same(g.download_shard(), (rp0, ed0), "empty batch")
        assert g.update_shard(insert=(src, dst, w)) == s5.lne
        same(g.download_shard(), (s5.rowptr, s5.edges), "generated + extras")
    finally:
        g.close()


# ---- the device generator's -p relation, on 1, 2 and 4 ranks ----------------------------------------------------------
def bare_ranks(world):
    """Ranks' per-rank thread runner over `world` new contexts on device 0 (host transport), without a shard."""
    from minivite_b200 import gpu as G
    R = Ranks.__new__(Ranks)
    R.world, R.g = world, [G.LouvainGPU(0, r, world) for r in range(world)]
    if world > 1:
        ident = G.get_unique_id()
        R.set_option("host_transport", 1)
        R.each(lambda r, g: g.comm_init(ident))
    return R


@pytest.mark.parametrize("world,unit", [(1, True), (1, False), (2, True), (4, False)])
def test_device_generator_relation(gpu, world, unit):
    from minivite_b200 import hostgraph as hg
    n = 32768
    s0 = hg.generate_rgg(n, world, unit_weight=unit)
    s5 = hg.generate_rgg(n, world, unit_weight=unit, random_edge_percent=5)
    ext = [U.extras(a, b) for a, b in zip(s0.shards, s5.shards)]
    R = bare_ranks(world)
    try:
        R.each(lambda r, g: g.generate_rgg(n, unit_weight=unit))
        lne = R.each(lambda r, g: g.update_shard(insert=ext[r]))
        for r in range(world):
            assert lne[r] == s5.shards[r].lne
        got = R.each(lambda r, g: g.download_shard())
        for r in range(world):
            same(got[r], (s5.shards[r].rowptr, s5.shards[r].edges), ("p0 + extras", r))
        # and back: the device-generated -p 5 shard minus the extras is the -p 0 shard
        R.each(lambda r, g: g.generate_rgg(n, unit_weight=unit, random_edge_percent=5))
        R.each(lambda r, g: g.update_shard(delete=ext[r][:2]))
        got = R.each(lambda r, g: g.download_shard())
        for r in range(world):
            same(got[r], (s0.shards[r].rowptr, s0.shards[r].edges), ("p5 - extras", r))
    finally:
        R.close()
        s0.close()
        s5.close()


# ---- Louvain on an updated shard --------------------------------------------------------------------------------------
def louvain_graphs():
    """(name, nv, before, after, delete, insert): a unit RGG gaining and losing records, and a dyadic multigraph."""
    from minivite_b200 import hostgraph as hg
    ss0 = hg.generate_rgg(65536, 1)
    ss5 = hg.generate_rgg(65536, 1, random_edge_percent=5)
    s0, s5 = ss0.shards[0], ss5.shards[0]
    src, dst, w = U.extras(s0, s5)
    rng = np.random.default_rng(2)
    row = np.repeat(np.arange(65536), np.diff(s5.rowptr))
    pick = rng.choice(len(row), 2000, replace=False)               # drop some pairs of -p 5, both directions
    ds, dd = row[pick], s5.edges["tail"][pick].copy()
    out = [("rgg_unit", 65536, (s0.rowptr.copy(), s0.edges.copy()), None, (src, dst, w)),
           ("rgg_unit_mixed", 65536, (s0.rowptr.copy(), s0.edges.copy()), (np.concatenate([ds, dd]), np.concatenate([dd, ds])),
            (src, dst, w))]
    ss0.close()
    ss5.close()
    n = 20000
    rp, ed = random_graph(n, 10, 9, blocks=40, dyadic=True, self_loops=50, multi=100)
    d, i = random_batch(rng, 0, n, n, rp, ed, 4000, 4000)
    i = (np.concatenate([i[0], i[1]]), np.concatenate([i[1], i[0]]), np.concatenate([i[2], i[2]]))   # symmetric
    out.append(("dyadic_multigraph", n, (rp, ed), (np.concatenate([d[0], d[1]]), np.concatenate([d[1], d[0]])), i))
    return out


@pytest.mark.parametrize("world", [1, 2, 4])
def test_louvain_after_update(gpu, world):
    """Cold run on the updated shard == cold run on the updated graph uploaded fresh (bit for bit); warm run from the
    pre-update result == the warm-start oracle from that assignment; communities() keeps the pre-update result and the
    initial assignment survives the update."""
    for name, nv, before, dele, ins in louvain_graphs():
        after = U.apply(0, before[0], before[1], dele, ins)
        parts, rps, eds = split_global(nv, before[0], before[1], world)
        R = Ranks(parts, rps, eds)
        try:
            pre = R.run()
            batches = [rank_batch(dele, ins, parts[r], parts[r + 1]) for r in range(world)]
            R.each(lambda r, g: g.update_shard(*batches[r]))
            # the last run's assignment is still there, and a NULL evaluation waits for the next run
            assert np.array_equal(np.concatenate(R.each(lambda r, g: g.communities().copy())), pre["comm"]), name
            cold = R.run()
            _, rps2, eds2 = split_global(nv, after[0], after[1], world)
            F = Ranks(parts, rps2, eds2)
            try:
                assert_same(cold, F.run(), (name, world, "cold"))
            finally:
                F.close()
            R.set_initial(pre["comm"])
            warm = R.run()
            assert_same(warm, oracle_run(parts, rps2, eds2, init=pre["comm"]), (name, world, "warm"))
        finally:
            R.close()


def test_dynamic_graph_warm_start_through_update(gpu):
    """test_gpu_warm_start.py::test_dynamic_graph_warm_start's scenario (-p 0 result, then -p 5) without re-uploading:
    run, update, communities(), set_initial_communities, run."""
    import warm_oracle as W
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    ss0 = hg.generate_rgg(65536, 1)
    ss5 = hg.generate_rgg(65536, 1, random_edge_percent=5)
    s0, s5 = ss0.shards[0], ss5.shards[0]
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        g.upload(s0.nv, s0.parts, s0.rowptr, s0.edges)
        g.louvain()
        g.set_initial_communities(np.arange(65536))                  # replaced below; kept across the update
        g.update_shard(insert=U.extras(s0, s5))
        prev = g.communities().copy()
        g.set_initial_communities(prev)
        mod, iters = g.louvain()
        ref = W.louvain(s5.parts, [s5.rowptr], [s5.edges], init_comm=[prev])
        assert (iters, mod) == (ref["iters"], ref["modularity"])
        assert as_trace(g.trace()) == as_trace(ref["trace"])
        assert np.array_equal(g.communities(), ref["comm"][0])
    finally:
        g.close()
        ss0.close()
        ss5.close()


# ---- state and errors -------------------------------------------------------------------------------------------------
def test_state_rules(gpu):
    from minivite_b200 import gpu as G
    rowptr, edges = random_graph(4000, 8, 1, blocks=20)
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.upload(4000, np.array([0, 4000], np.int64), rowptr, edges)
        init = np.arange(4000) // 7
        g.set_initial_communities(init)
        g.louvain()
        res = g.communities().copy()
        g.evaluate(None)
        g.update_shard(insert=(np.array([0, 1]), np.array([1, 0]), np.array([1.0, 1.0])))
        with pytest.raises(G.MvgpuError, match="NULL evaluates"):
            g.evaluate(None)
        with pytest.raises(G.MvgpuError, match="no evaluation"):
            g.community_stats()
        assert np.array_equal(g.communities(), res)
        warm = g.louvain()                                           # still warm: the initial assignment was kept
        ref_rp, ref_ed = U.apply(0, rowptr, edges, None, (np.array([0, 1]), np.array([1, 0]), np.array([1.0, 1.0])))
        h = G.LouvainGPU(0, 0, 1)
        try:
            h.upload(4000, np.array([0, 4000], np.int64), ref_rp, ref_ed)
            h.set_initial_communities(init)
            assert h.louvain() == warm
            assert np.array_equal(h.communities(), g.communities())
        finally:
            h.close()
        t = g.timings()
        assert t["h2d_s"] == 0.0 and t["h2d_bytes"] == 0
        g.evaluate(None)
    finally:
        g.close()


def test_refusals_leave_the_shard(gpu):
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    g = G.LouvainGPU(0, 0, 1)
    try:
        with pytest.raises(G.MvgpuError, match="no shard"):
            g.update_shard()
        rowptr, edges = random_graph(1000, 6, 3)
        g.upload(1000, np.array([0, 1000], np.int64), rowptr, edges)
        before = g.download_shard()
        one = np.array([1])
        for dele, ins, pat in [((np.array([1000]), one), None, "outside the shard"),
                               ((np.array([-1]), one), None, "outside the shard"),
                               (None, (one, np.array([1000]), np.ones(1)), "outside the shard"),
                               (None, (one, np.array([-5]), np.ones(1)), "outside the shard")]:
            with pytest.raises(G.MvgpuError, match=pat):
                g.update_shard(dele, ins)
            same(g.download_shard(), before, pat)
        with pytest.raises(G.MvgpuError, match="null batch array"):
            G._ck(G.lib().mvgpu_update_shard(g._h, 1, None, None, 0, None, None, None, None))
        with pytest.raises(G.MvgpuError, match="negative"):
            G._ck(G.lib().mvgpu_update_shard(g._h, -1, None, None, 0, None, None, None, None))
        same(g.download_shard(), before, "null / negative")
        # compact upload: no records to update
        g.set_option("compact_upload", 1)
        g.upload(1000, np.array([0, 1000], np.int64), rowptr, edges)
        with pytest.raises(G.MvgpuError, match="compact"):
            g.update_shard(insert=(one, one, np.ones(1)))
        g.set_option("compact_upload", 0)
        # 32-bit shard
        sh = hg.generate_rgg(4096, 1).shards[0]
        e8 = np.zeros(sh.lne, np.dtype([("tail", "<i4"), ("weight", "<f4")]))
        e8["tail"], e8["weight"] = sh.edges["tail"], sh.edges["weight"]
        g.upload32(4096, np.array([0, 4096], np.int32), sh.rowptr.astype(np.int32), e8)
        before32 = g.download_shard()
        with pytest.raises(G.MvgpuError, match="32"):
            g.update_shard(insert=(one, one, np.ones(1)))
        same(g.download_shard(), before32, "32-bit")
    finally:
        g.close()


def test_one_bad_rank_fails_both(gpu):
    rowptr, edges = random_graph(2000, 6, 8)
    parts, rps, eds = split_global(2000, rowptr, edges, 2)
    R = Ranks(parts, rps, eds)
    try:
        before = R.each(lambda r, g: g.download_shard())
        good = (np.array([1500]), np.array([3]), np.ones(1))
        bad = (np.array([5]), np.array([3]), np.ones(1))              # rank 1 does not own vertex 5
        batches = [(None, (np.array([3]), np.array([1500]), np.ones(1))), (None, bad)]
        errs = []

        def one(r, g):
            try:
                g.update_shard(*batches[r])
            except RuntimeError as ex:
                errs.append((r, str(ex)))
        R.each(one)
        assert sorted(r for r, _ in errs) == [0, 1], errs
        assert any("another rank" in m for _, m in errs) and any("outside the shard" in m for _, m in errs)
        after = R.each(lambda r, g: g.download_shard())
        for r in range(2):
            same(after[r], before[r], r)
        # and a good pair of batches goes through on both, as if the failed call had never happened
        batches[1] = (None, good)
        R.each(lambda r, g: g.update_shard(*batches[r]))
        after = R.each(lambda r, g: g.download_shard())
        for r in range(2):
            same(after[r], U.apply(int(parts[r]), rps[r], eds[r], *batches[r]), ("after the failed call", r))
    finally:
        R.close()


@pytest.mark.parametrize("mode", MODES)
def test_malformed_rowptr_is_refused(gpu, mode):
    """Upload and attach do not check edge_indices (the run does): an update of such a shard must fail with the run's
    message before any merge kernel trusts the offsets, and leave the shard as it was -- on one rank, and on the rank
    of two that holds it, with the other rank failing too."""
    import torch
    from minivite_b200 import gpu as G
    rowptr, edges = random_graph(1000, 6, 12)
    lne = len(edges)
    shifted = rowptr + 100                                           # a strip whose offsets were not rebased to 0
    shifted[-1] = lne
    dips = rowptr.copy()
    dips[500] = dips[499] - 1                                        # decreases once
    short = rowptr.copy()
    short[-1] = lne - 1                                              # does not end at lne
    ins = (np.array([1, 2]), np.array([2, 1]), np.ones(2))
    for what, rp in (("not rebased", shifted), ("decreasing", dips), ("short", short)):
        g = G.LouvainGPU(0, 0, 1)
        try:
            parts = np.array([0, 1000], np.int64)
            if mode == "upload":
                G._ck(G.lib().mvgpu_upload_shard(g._h, 1000, parts.ctypes.data, 1000, lne, rp.ctypes.data, edges.ctypes.data))
            else:
                trp = torch.from_numpy(rp.copy()).cuda()
                ted = torch.from_numpy(edges.view(np.uint8).copy()).cuda()
                g.attach_device(1000, parts, 1000, lne, trp.data_ptr(), ted.data_ptr(), keepalive=(trp, ted))
            before = g.download_shard()
            with pytest.raises(G.MvgpuError, match="edge_indices malformed"):
                g.update_shard(insert=ins)
            same(g.download_shard(), before, (mode, what))
            assert g.shard_info()["lne"] == lne
        finally:
            g.close()
    parts, rps, eds = split_global(1000, rowptr, edges, 2)
    R = Ranks(parts, rps, eds)
    try:
        bad_rp = rps[1] + 1
        R.each(lambda r, g: r == 1 and G._ck(G.lib().mvgpu_upload_shard(
            g._h, 1000, parts.ctypes.data, 500, len(eds[1]), bad_rp.ctypes.data, eds[1].ctypes.data)))
        before = R.each(lambda r, g: g.download_shard())
        errs = []

        def one(r, g):
            try:
                g.update_shard()
            except RuntimeError as ex:
                errs.append((r, str(ex)))
        R.each(one)
        assert sorted(r for r, _ in errs) == [0, 1], errs
        assert any("another rank" in m for _, m in errs) and any("edge_indices malformed" in m for _, m in errs)
        after = R.each(lambda r, g: g.download_shard())
        for r in range(2):
            same(after[r], before[r], r)
    finally:
        R.close()


# ---- full size --------------------------------------------------------------------------------------------------------
def test_full_size_config2_to_config3(gpu):
    """Config 2 (`-n 16777216`) generated on the device, updated to config 3 (`-p 2`) with the difference of the
    two host-generated graphs, then run: the unmodified reference's trace on config 3
    (tests/golden/golden_full_16777216_p1_r2.json).  Opt-in with MV_BIG_TESTS=1."""
    if os.environ.get("MV_BIG_TESTS") != "1":
        pytest.skip("set MV_BIG_TESTS=1")
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    from oracle import oracle as O
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "golden_full_16777216_p1_r2.json")))
    n = gold["nv"]
    ss1 = hg.generate_rgg(n, 1)
    ss2 = hg.generate_rgg(n, 1, random_edge_percent=gold["random_edge_percent"])
    batch = U.extras(ss1.shards[0], ss2.shards[0])
    ss1.close()
    ss2.close()
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        g.generate_rgg(n)
        g.louvain()
        assert g.update_shard(insert=batch) == gold["ne"]
        mod, iters = g.louvain()
        assert iters == gold["iters"] and repr(mod) == repr(float(gold["modularity"]))
        for t, ref in zip(g.trace(), gold["trace"]):
            assert float(t["modularity"]) == float(ref["modularity"]) and int(t["moved"]) == ref["moved"]
            assert int(t["chash"]) == int(ref["chash"], 16)
        assert "%016x" % O.comm_hash(0, g.communities()) == gold["final_chash"]
    finally:
        g.close()
