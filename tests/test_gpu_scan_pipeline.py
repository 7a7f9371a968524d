"""The persistent scan kernels across groups, on the GPU: engineered shards (tests/scan_graphs.py) whose groups land on
every buffer, heavy-vertex and ring boundary, run with the scan_ctas hook so that every warp takes dozens of groups in
an order the host restatement (tests/scan_schedule.py) knows, bit-exact against the C oracle: iterations, every trace
record, the final modularity by repr, constant(), the final assignment, and shard_info()'s nheavy / maxdeg."""
import numpy as np
import pytest

import scan_graphs as SG
import scan_schedule as SS
from oracle import oracle as O
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_warm_start import Ranks, as_trace

pytestmark = pytest.mark.gpu

_cache = {}


def graph(name):
    """(rowptr, edges, unit) of an engineered shard, with the oracle's cold run."""
    if name not in _cache:
        if name == "pq":
            rp, tl, _k = SG.pq_layout()
        elif name == "default_grid":
            rp, tl, _k = SG.default_grid_layout(2 * 64 * num_sms())
        else:
            rp, tl, _k, _n = {"unit_heavy": SG.unit_heavy, "unit_light": SG.unit_light,
                              "weighted_heavy": SG.weighted_heavy}[name]()
        unit = name != "weighted_heavy"
        e = SG.edges_of(rp, tl, dyadic=not unit)
        n = len(rp) - 1
        _cache[name] = (rp, e, unit, O.louvain(np.array([0, n]), [rp], [e]))
    return _cache[name]


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def oracle_as(res):
    return {"mod": res["modularity"], "iters": res["iters"], "trace": as_trace(res["trace"]),
            "comm": np.concatenate(res["comm"]), "constant": res["constant"]}


def run(G, rp, e, init=None, movable=None, **opts):
    n = len(rp) - 1
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        for k, v in opts.items():
            g.set_option(k, v)
        g.upload(n, np.array([0, n], np.int64), rp, e)
        if init is not None:
            g.set_initial_communities(init)
        if movable is not None:
            g.set_movable(movable)
        mod, iters = g.louvain(-1.0, 1.0e-6)
        return {"mod": mod, "iters": iters, "trace": as_trace(g.trace()), "comm": g.communities().copy(),
                "constant": g.constant(), "info": g.shard_info(), "timings": g.timings()}
    finally:
        g.close()


def assert_same(res, ref, what):
    assert res["iters"] == ref["iters"], (what, res["iters"], ref["iters"])
    assert res["trace"] == ref["trace"], what
    assert repr(res["mod"]) == repr(ref["mod"]), (what, res["mod"], ref["mod"])
    assert repr(res["constant"]) == repr(ref["constant"]), what
    assert np.array_equal(res["comm"], ref["comm"]), what


def assert_heavy(res, rp, variant, unit, force=0):
    hd = SS.heavy_deg_of(variant, unit, force)
    assert (res["info"]["nheavy"], res["info"]["maxdeg"]) == SS.heavy_info(rp, hd), (variant, force)


@pytest.mark.parametrize("name", ["unit_heavy", "unit_light"])
@pytest.mark.parametrize("variant", [3, 4, 5, 6])
def test_cold_runs_every_grid(gpu, name, variant):
    rp, e, unit, ref = graph(name)
    ref = oracle_as(ref)
    for ctas in (1, 2, 3, 0):
        for first in (1, 0):
            res = run(gpu, rp, e, scan_variant=variant, scan_ctas=ctas, first_iter=first, reorder=0)
            assert_same(res, ref, (name, variant, ctas, first))
            assert_heavy(res, rp, variant, unit)
    res = run(gpu, rp, e, scan_variant=variant)                     # default options (may renumber): results only
    assert_same(res, ref, (name, variant, "default"))


def test_scan_ctas_is_validated(gpu):
    g = gpu.LouvainGPU(0, 0, 1)
    try:
        with pytest.raises(gpu.MvgpuError):
            g.set_option("scan_ctas", -1)
        g.set_option("scan_ctas", 0)
        g.set_option("scan_ctas", 7)
    finally:
        g.close()


@pytest.mark.parametrize("variant", [4, 5])
def test_pq_one_step_per_assignment(gpu, variant):
    rp, e, _unit, _ref = graph("pq")
    n = len(rp) - 1
    tl = e["tail"].astype(np.int64)
    X_bound, _v0, _v1 = SG.pq_bound_assignment(rp, tl)
    c = 1.0 / float(rp[-1])
    for name, X in (("identity", np.arange(n, dtype=np.int64)), ("bounds", X_bound)):
        warps, verts = SS.pq_schedule(rp, tl, X, c, SG.PQ_CTAS)
        cov = SS.pq_coverage(warps, verts)
        print(f"\npq {name}: " + ", ".join(f"{k}={v}" for k, v in sorted(cov.items())))
        one = O.louvain(np.array([0, n]), [rp], [e], init_comm=[X], stop_after=1)
        assert np.array_equal(SS.pq_decisions(rp, tl, X, c), one["comm"][0])
        res = run(gpu, rp, e, init=X, scan_variant=variant, scan_ctas=SG.PQ_CTAS, reorder=0, stop_after=1)
        assert repr(res["constant"]) == repr(c)
        assert np.array_equal(res["comm"], one["comm"][0]), (variant, name)
        assert res["trace"][:1] == as_trace(one["trace"])[:1], (variant, name)
        full = oracle_as(O.louvain(np.array([0, n]), [rp], [e], init_comm=[X]))
        for ctas in (SG.PQ_CTAS, 1, 0):
            res = run(gpu, rp, e, init=X, scan_variant=variant, scan_ctas=ctas, reorder=0)
            assert_same(res, full, (variant, name, ctas))


@pytest.mark.parametrize("variant", [3, 4, 6])
def test_dyadic_weighted(gpu, variant):
    rp, e, unit, ref = graph("weighted_heavy")
    ref = oracle_as(ref)
    assert not unit
    for ctas in (1, 3, 0):
        for force in (0, 16):
            res = run(gpu, rp, e, scan_variant=variant, scan_ctas=ctas, force_heavy_deg=force, reorder=0)
            assert res["timings"]["unit_weight"] == 0
            assert_same(res, ref, (variant, ctas, force))
            assert_heavy(res, rp, variant, False, force)


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_sharing_device(gpu, world):
    """Shards split at offsets that are not multiples of 32: ragged groups on every rank, ghost candidates."""
    rp, e, _unit, _ref = graph("unit_heavy")
    n = len(rp) - 1
    parts = np.array([0] + [n * r // world + 7 * r for r in range(1, world)] + [n], np.int64)
    assert all(p % 32 for p in parts[1:-1])
    rps, eds = SG.split_at(rp, e, parts)
    ref = O.louvain(parts, rps, eds)
    ref = {"mod": ref["modularity"], "iters": ref["iters"], "trace": as_trace(ref["trace"]),
           "comm": np.concatenate(ref["comm"])}
    for variant in (4, 5, 6):
        R = Ranks(parts, rps, eds, scan_variant=variant, scan_ctas=1, reorder=0)
        try:
            res = R.run()
        finally:
            R.close()
        assert res["iters"] == ref["iters"] and res["trace"] == ref["trace"], (world, variant)
        assert repr(res["mod"]) == repr(ref["mod"]), (world, variant)
        assert np.array_equal(res["comm"], ref["comm"]), (world, variant)


@pytest.mark.parametrize("frontier", [0, 1])
def test_masked_run(gpu, frontier):
    rp, e, _unit, _ref = graph("unit_heavy")
    n = len(rp) - 1
    mask = (np.random.default_rng(11).random(n) < 0.5).astype(np.uint8)
    ref = oracle_as(O.louvain(np.array([0, n]), [rp], [e], movable=[mask], frontier=frontier))
    for variant in (4, 5):
        for ctas in (1, 0):
            res = run(gpu, rp, e, movable=mask, scan_variant=variant, scan_ctas=ctas, reorder=0, frontier=frontier)
            assert_same(res, ref, (frontier, variant, ctas))


def test_default_grid_without_hook(gpu):
    """2 x 64 x SMs groups: every warp of the default grid takes at least two groups at any occupancy."""
    rp, e, _unit, ref = graph("default_grid")
    sms = num_sms()
    ng = (len(rp) - 1) // 32
    kinds = SG.default_grid_layout(ng)[2]
    for per_sm in range(1, 9):
        assert min(len(g) for g in SS.warp_groups(ng, per_sm * sms)) >= 2
        pairs = SS.pair_coverage(kinds, ng, per_sm * sms)
        print(f"\nctas/SM {per_sm}: " + ", ".join(f"{a}->{b}={k}" for (a, b), k in sorted(pairs.items())))
        assert len(pairs) == 9
    ref = oracle_as(ref)
    for variant in (4, 5, 6):
        res = run(gpu, rp, e, scan_variant=variant, reorder=0)
        assert_same(res, ref, ("default grid", variant))
