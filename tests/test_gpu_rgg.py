"""Device-side RGG generator (SURVEY.md 8(f) rank 1): byte-identical to the host generator, which is itself
byte-identical to the reference's GenerateRGG (tests/test_oracle.py pins that through the golden traces)."""
import numpy as np
import pytest

from helpers import assert_trace_matches

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,p,ranks,unit,lcg", [(16384, 1, [0], True, False), (16384, 2, [0, 1], True, False),
                                                (16384, 4, [0, 1, 2, 3], True, False), (16384, 8, [0, 3, 7], True, False),
                                                (32768, 4, [1, 2], False, False), (1048576, 1, [0], True, False),
                                                (1048576, 8, [0, 5], True, False),
                                                # -l: the reference's LCG stream, a different point pattern per strip
                                                (16384, 1, [0], True, True), (16384, 2, [0, 1], True, True),
                                                (32768, 4, [0, 1, 2, 3], False, True), (1048576, 8, [0, 4, 7], True, True),
                                                # 16 strips, plain and -l
                                                (16384, 16, [0, 7, 15], True, False), (16384, 16, [0, 9, 15], True, True)])
def test_device_generator_matches_host_generator(n, p, ranks, unit, lcg):
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    for r in ranks:
        ref = hg.generate_rgg(n, p, r, r + 1, unit_weight=unit, lcg=lcg).shards[0]
        g = G.LouvainGPU(0, r, p)          # no communicator needed: generation is local to the rank
        try:
            lne = g.generate_rgg(n, unit_weight=unit, lcg=lcg)
            assert lne == ref.lne, (n, p, r, lne, ref.lne)
            rowptr, edges = g.download_shard()
        finally:
            g.close()
        assert np.array_equal(rowptr, ref.rowptr)
        assert np.array_equal(edges["tail"], ref.edges["tail"])
        assert np.array_equal(edges["weight"], ref.edges["weight"])   # bit-exact, also for Euclidean weights


def test_generate_then_louvain_matches_reference(golden):
    """`miniVite -n 16384` end to end on the device: generator + Louvain phase == reference trace."""
    from minivite_b200 import gpu as G
    case = golden["rgg_n16384_p1"]
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        assert g.generate_rgg(16384) == case["ne"]
        mod, iters = g.louvain()
        assert_trace_matches(case, iters, mod, g.trace(), None, g.communities())
    finally:
        g.close()


def test_generate_lcg_then_louvain_matches_reference(golden):
    """`miniVite -n 16384 -l` on 2 ranks (golden from the reference's own generator), both strips generated on the device
    and run as one shard: generator (-l) + Louvain phase == reference trace."""
    from minivite_b200 import gpu as G
    case = golden["rgg_n16384_p2_l"]
    rps, eds = [], []
    for r in range(2):
        g = G.LouvainGPU(0, r, 2)
        try:
            g.generate_rgg(16384, lcg=True)
            rp, ed = g.download_shard()
        finally:
            g.close()
        rps.append(rp)
        eds.append(ed)
    assert sum(len(e) for e in eds) == case["ne"]
    rowptr = np.concatenate([rps[0], rps[1][1:] + rps[0][-1]])
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        g.upload(16384, np.array([0, 16384], np.int64), rowptr, np.concatenate(eds))
        mod, iters = g.louvain()
        assert_trace_matches(case, iters, mod, g.trace(), None, None)
    finally:
        g.close()


def _same_shard(got, ref, tag):
    rowptr, edges = got
    assert np.array_equal(rowptr, ref.rowptr), tag
    assert np.array_equal(edges["tail"], ref.edges["tail"]), tag
    assert np.array_equal(edges["weight"], ref.edges["weight"]), tag


@pytest.mark.parametrize("n,unit,lcg,pct", [(16384, True, False, 20.0), (16384, False, False, 20.0), (32768, True, True, 7.5),
                                            (2048, True, False, 99.0), (1048576, True, False, 2.0)])
def test_device_generator_random_edges(n, unit, lcg, pct):
    """-p: the random long edges of GenerateRGG (graph.hpp:939-1122) drawn, filtered, de-duplicated and merged on the
    device: byte-identical to the host generator (duplicates within a stream, RGG hits and i == j draws included --
    20 % and 99 % make all of them occur)."""
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    ref = hg.generate_rgg(n, 1, unit_weight=unit, lcg=lcg, random_edge_percent=pct).shards[0]
    base = hg.generate_rgg(n, 1, unit_weight=unit, lcg=lcg).shards[0]
    assert ref.lne > base.lne
    g = G.LouvainGPU(0, 0, 1)
    try:
        assert g.generate_rgg(n, unit_weight=unit, lcg=lcg, random_edge_percent=pct) == ref.lne
        _same_shard(g.download_shard(), ref, (n, pct))
    finally:
        g.close()


@pytest.mark.parametrize("n,p,unit,lcg,pct", [(16384, 2, True, False, 20.0), (32768, 4, False, False, 10.0),
                                              (131072, 8, False, True, 5.0), (16384, 4, True, False, 0.004),
                                              (16384, 16, True, False, 20.0)])
def test_device_generator_random_edges_on_ranks(n, p, unit, lcg, pct):
    """-p on p ranks (threads sharing device 0, host transport): every rank replays all p draw streams and keeps the
    forward edges of its own stream plus the reverse edges the other streams send it; weighted far pairs take the
    hashed-seed weight (graph.hpp:1037-1041).  0.004 % leaves fewer draws than ranks: the last stream gets them all."""
    import threading
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    ss = hg.generate_rgg(n, p, unit_weight=unit, lcg=lcg, random_edge_percent=pct)
    base = hg.generate_rgg(n, p, unit_weight=unit, lcg=lcg)
    assert sum(s.lne for s in ss.shards) > sum(s.lne for s in base.shards)
    ident = G.get_unique_id()
    out, errs = [None] * p, []

    def work(rank):
        try:
            g = G.LouvainGPU(0, rank, p)
            g.set_option("host_transport", 1)
            g.comm_init(ident)
            lne = g.generate_rgg(n, unit_weight=unit, lcg=lcg, random_edge_percent=pct)
            out[rank] = (lne,) + tuple(g.download_shard())
            g.close()
        except Exception as ex:
            errs.append((rank, repr(ex)))
    th = [threading.Thread(target=work, args=(r,)) for r in range(p)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    for r in range(p):
        assert out[r] is not None and out[r][0] == ss.shards[r].lne, r
        _same_shard(out[r][1:], ss.shards[r], (n, p, r))


def test_random_edges_on_ranks_need_the_communicator():
    from minivite_b200 import gpu as G
    g = G.LouvainGPU(0, 1, 2)
    try:
        with pytest.raises(RuntimeError, match="communicator"):
            g.generate_rgg(16384, random_edge_percent=5.0)
        with pytest.raises(RuntimeError, match="random_edge_percent"):
            g.generate_rgg(16384, random_edge_percent=-1.0)
    finally:
        g.close()


def test_generate_config3_then_louvain_matches_reference():
    """BASELINE.json configs[2] (`-n 16777216 -p 2`) without a host graph: generated in HBM, Louvain phase in place,
    trace == the unmodified reference's on that graph (tests/golden/golden_full_16777216_p1_r2.json)."""
    import json
    import os
    from minivite_b200 import gpu as G
    from oracle import oracle as O
    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_full_16777216_p1_r2.json")))
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        assert g.generate_rgg(gold["nv"], random_edge_percent=gold["random_edge_percent"]) == gold["ne"]
        mod, iters = g.louvain()
        assert iters == gold["iters"] and repr(mod) == repr(float(gold["modularity"]))
        for t, ref in zip(g.trace(), gold["trace"]):
            assert float(t["modularity"]) == float(ref["modularity"]) and int(t["moved"]) == ref["moved"]
            assert int(t["chash"]) == int(ref["chash"], 16)
        assert "%016x" % O.comm_hash(0, g.communities()) == gold["final_chash"]
    finally:
        g.close()
