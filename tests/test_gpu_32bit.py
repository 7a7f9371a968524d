"""The reference's USE_32_BIT_GRAPH build (utils.hpp:72-82: int32 ids, float weights) through the mvgpu_*32 entry points.
Goldens: tests/golden/ref32_traces.json, produced by the reference compiled with its own -DUSE_32_BIT_GRAPH switch
(oracle/_ref/miniVite_ref32) on files in that build's format.  Every unit-weight case keeps all sums below 2^24, where
the float build is exact: assignment, iteration count, per-iteration moved / hash and the float modularity must be
bit-identical.  Dyadic weights (k * 2^-j) below 2^24 units keep every sum exact as well and are held to the same bar.
Euclidean weights: the float build accumulates in float, this build in double -> |dQ| <= 1e-4."""
import json
import os
import threading

import numpy as np
import pytest

from helpers import assert_trace_matches, case_graph

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGE32 = np.dtype([("tail", "<i4"), ("weight", "<f4")])


@pytest.fixture(scope="module")
def golden32():
    return json.load(open(os.path.join(ROOT, "tests", "golden", "ref32_traces.json")))["cases"]


def shards32(case):
    parts, rps, eds, keep = case_graph(case)
    out = []
    for rp, ed in zip(rps, eds):
        e = np.zeros(len(ed), EDGE32)
        e["tail"] = ed["tail"]
        e["weight"] = ed["weight"].astype(np.float32)
        out.append((rp.astype(np.int32), e))
    return parts.astype(np.int32), out


def run32(case, thresh=1.0e-6, sharded=None, **opts):
    """One float-build run of case on len(shards) ranks sharing device 0 (threads, host transport); sharded:
    (parts, shards) when the case is not one case_graph rebuilds."""
    from minivite_b200 import gpu as G
    parts, sh = sharded or shards32(case)
    world = len(sh)
    ident = G.get_unique_id()
    out, errs = [None] * world, []

    def work(rank):
        try:
            g = G.LouvainGPU(0, rank, world)
            if world > 1:
                g.set_option("host_transport", 1)
            g.set_option("trace", 1)
            for k, v in opts.items():
                g.set_option(k, v)
            if world > 1:
                g.comm_init(ident)
            g.upload32(int(parts[-1]), parts, sh[rank][0], sh[rank][1])
            mod, iters = g.louvain32(thresh=thresh)
            out[rank] = {"mod": mod, "iters": iters, "trace": g.trace(), "comm": g.communities32().astype(np.int64),
                         "unit": g.timings()["unit_weight"]}
            g.close()
        except Exception as ex:
            errs.append((rank, repr(ex)))
    th = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    return {"mod": out[0]["mod"], "iters": out[0]["iters"], "trace": out[0]["trace"], "unit": out[0]["unit"],
            "comm": np.concatenate([o["comm"] for o in out])}


def test_float_build_unit_weight_cases_are_bit_exact(golden32):
    """Decisions are exact: iteration count, moved counts, community hashes of every iteration and the final assignment
    equal the float build's.  The float modularity is compared bit for bit where the float build's own sum of squared
    degrees is exact (sum < 2^24: the n = 16 384 cases and the hand-made graphs) and within 4 float ulps beyond (the
    reference adds squares sequentially in float there; this build adds exact integers and rounds once)."""
    n = 0
    for name, case in golden32.items():
        if case.get("unit_weight") is False or "weighted" in name or "dyadic" in name:
            continue
        exact_mod = case["nv"] <= 16384
        for opts in ({}, {"scan_variant": 5}, {"scan_variant": 4}, {"scan_variant": 3}, {"reorder": 1, "region_size": 64}):
            res = run32(case, **opts)
            assert res["unit"] == 1, name
            assert res["iters"] == case["iters"], (name, opts)
            mods = [(np.float32(res["mod"]), np.float32(float(case["modularity"])))]
            assert len(res["trace"]) == len(case["trace"])
            for t, g in zip(res["trace"], case["trace"]):
                assert int(t["moved"]) == g["moved"] and int(t["chash"]) == int(g["chash"], 16), (name, opts)
                mods.append((np.float32(t["modularity"]), np.float32(float(g["modularity"]))))
            for a, b in mods:
                if exact_mod:
                    assert a == b, (name, opts, a, b)
                else:
                    assert abs(float(a) - float(b)) <= 4 * float(np.spacing(np.float32(abs(b)))), (name, opts, a, b)
            if "comm" in case:
                assert [int(x) for x in res["comm"]] == case["comm"], (name, opts)
        n += 1
    assert n >= 8


def test_float_build_dyadic_weighted_cases_are_bit_exact(golden32):
    """Dyadic weights (k/4 <= 2 on RGG 16 384 on 1 and 2 ranks, k/8 on a planted partition, the hand-made tie graphs,
    hand_weighted20's k/4): every float sum of the float build stays below 2^24 units and is exact, and so is this
    build's double accumulation, so assignment, iteration count, moved counts and hashes are bit-identical.  The float
    modularity is bit-identical where the float build's sum of squared community degrees is exact too ((2m 2^j)^2 < 2^24:
    the hand-made graphs).  On the RGG and the planted partition that sum exceeds 2^24 units: the float build adds the
    squares one by one in float and its rounding error is absolute, about 8e-9 on the first iteration's modularity of
    1.4e-4 (hundreds of ulps of so small a value; this build adds exactly and rounds once, and the 1- and 2-rank
    references differ from each other too).  There the bar is 4 float ulps or 2^-24, whichever is larger."""
    names = [k for k in golden32 if k.startswith("f32_dyadic_")] + ["f32_hand_weighted20_p1"]
    assert len(names) >= 8
    for name in names:
        case = golden32[name]
        exact_mod = case.get("exact_mod", True)       # hand_weighted20: (2m 4)^2 = 491^2 < 2^24
        for opts in ({}, {"scan_variant": 4}, {"scan_variant": 3}, {"reorder": 1, "region_size": 64}, {"force_heavy_deg": 4}):
            res = run32(case, **opts)
            assert res["unit"] == 0, name
            assert res["iters"] == case["iters"], (name, opts)
            assert len(res["trace"]) == len(case["trace"]), (name, opts)
            mods = [(np.float32(res["mod"]), np.float32(float(case["modularity"])))]
            for t, g in zip(res["trace"], case["trace"]):
                assert int(t["moved"]) == g["moved"] and int(t["chash"]) == int(g["chash"], 16), (name, opts)
                mods.append((np.float32(t["modularity"]), np.float32(float(g["modularity"]))))
            for a, b in mods:
                if exact_mod:
                    assert a == b, (name, opts, a, b)
                else:
                    assert abs(float(a) - float(b)) <= max(4 * float(np.spacing(np.float32(abs(b)))), 2.0 ** -24), \
                        (name, opts, a, b)
            if "comm" in case:
                assert [int(x) for x in res["comm"]] == case["comm"], (name, opts)


def test_float_build_weighted_cases_within_tolerance(golden32):
    """Euclidean weights are not exactly representable: the float build's sums round differently from this build's
    double sums, so the bar is a modularity tolerance (dyadic weights are held bit-exact above)."""
    for name in ("f32_rgg_n16384_s1_w_p1",):
        case = golden32[name]
        res = run32(case)
        assert res["unit"] == 0
        assert abs(res["mod"] - float(case["modularity"])) <= 1e-4, (name, res["mod"], case["modularity"])


def test_entry_points_refuse_mixed_use(golden32):
    from minivite_b200 import gpu as G
    case = golden32["f32_hand_k66_p1"]
    parts, sh = shards32(case)
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.upload32(int(parts[-1]), parts, sh[0][0], sh[0][1])
        mod, iters = g.louvain32()
        assert iters == case["iters"]
        # the same context takes a 64-bit shard afterwards and leaves float mode
        p64, rps, eds, _ = case_graph(case)
        g.upload(int(p64[-1]), p64, rps[0], eds[0])
        with pytest.raises(G.MvgpuError):
            g.louvain32()
        g.louvain()
    finally:
        g.close()
