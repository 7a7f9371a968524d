"""GPU tests of the movable set (mvgpu_set_movable, option "frontier", DESIGN.md §3.14).

Every masked run is held bit for bit to the movable-set oracle (tests/movable_oracle.c): iteration count, every trace
record, the modularity, the final assignment and the returned set.  Covered: every unit and dyadic golden case on its
own rank count (ranks > 1 share device 0 through the host transport) with random sets of density 0.01, 0.1 and 0.5,
frontier 0 and 1, from singletons and warm; scan variants 3-6, renumbering 0/1/2, forced k_scan_heavy and every upload
mode; R-MAT scale 14 with its hubs movable and frozen; all-ones against no set; checkpoint and resume with frontier 1
through the API and the CLI; an update scenario seeded by movable_from_batch; the state rules and refusals; launch
counts."""
import os
import re
import subprocess

import numpy as np
import pytest

from helpers import case_graph, dyadic_rgg, split_global
import movable_oracle as MO
import update_ref as U
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_warm_start import EXE, Ranks, as_trace, cli
from test_movable_oracle import CASES

pytestmark = pytest.mark.gpu

DENSITIES = (0.01, 0.1, 0.5)


def masks_for(nv, density, seed):
    return (np.random.default_rng(seed).random(nv) < density).astype(np.uint8)


def slices(parts, a):
    return [a[parts[r]:parts[r + 1]] for r in range(len(parts) - 1)]


def set_movable(R, mask):
    for r, g in enumerate(R.g):
        g.set_movable(None if mask is None else mask[R.parts[r]:R.parts[r + 1]])


def run(R, lower=-1.0):
    res = R.run(lower)
    res["movable"] = np.concatenate(R.each(lambda r, g: g.movable().copy()))
    return res


def oracle(parts, rps, eds, mask, frontier, init=None, **kw):
    o = MO.louvain(parts, rps, eds, movable=None if mask is None else slices(parts, mask), frontier=frontier,
                   init_comm=None if init is None else slices(parts, init), **kw)
    return {"mod": o["modularity"], "iters": o["iters"], "trace": as_trace(o["trace"]), "comm": np.concatenate(o["comm"]),
            "movable": np.concatenate(o["movable"]), "converged": o["converged"]}


def assert_same(res, ref, what):
    assert res["iters"] == ref["iters"], (what, res["iters"], ref["iters"])
    assert res["trace"] == ref["trace"], what
    assert repr(res["mod"]) == repr(ref["mod"]), (what, res["mod"], ref["mod"])
    assert np.array_equal(res["comm"], ref["comm"]), what
    if "movable" in ref:
        assert np.array_equal(res["movable"], ref["movable"]), what


def check_matrix(name, R, parts, rps, eds, densities=DENSITIES, frontiers=(0, 1), starts=("cold", "warm")):
    nv = int(parts[-1])
    warm0 = None
    for start in starts:
        init = None
        if start == "warm":
            if warm0 is None:
                warm0 = oracle(parts, rps, eds, None, 0, stop_after=2)["comm"]
            init = warm0
        R.set_initial(init)
        for i, density in enumerate(densities):
            mask = masks_for(nv, density, 100 + i)
            set_movable(R, mask)
            for frontier in frontiers:
                R.set_option("frontier", frontier)
                assert_same(run(R), oracle(parts, rps, eds, mask, frontier, init), (name, start, density, frontier))
    set_movable(R, None)
    R.set_initial(None)
    R.set_option("frontier", 0)


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_exact_case_matches_oracle(gpu, name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    big = int(parts[-1]) > 200000          # the host oracle dominates there: one density, both frontiers, cold
    R = Ranks(parts, rps, eds)
    try:
        if big:
            check_matrix(name, R, parts, rps, eds, densities=(0.1,), starts=("cold",))
        else:
            check_matrix(name, R, parts, rps, eds)
    finally:
        R.close()


CONFIGS = [{"scan_variant": v} for v in (3, 4, 5, 6)] + [{"reorder": r} for r in (0, 1, 2)] + \
    [{"force_heavy_deg": 8}, {"force_heavy_deg": 8, "scan_variant": 3}, {"compact_upload": 1}, {"compact_upload": 2}]


@pytest.mark.parametrize("opts", CONFIGS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()))
@pytest.mark.parametrize("name", ["rgg_n65536_p1", "rgg_n16384_p4", "rmat_s14_p2_b",
                                  "dyadic_random_n4099_d30_hubs2_hub_deg1000_multi100"])
def test_configurations_match_oracle(gpu, name, opts):
    parts, rps, eds, _keep = case_graph(CASES[name])
    if opts.get("compact_upload") and name.startswith("dyadic"):
        pytest.skip("the compact upload carries unit-weight shards only")
    R = Ranks(parts, rps, eds, **opts)
    try:
        check_matrix(name, R, parts, rps, eds, densities=(0.1, 0.5))
    finally:
        R.close()


@pytest.mark.parametrize("frozen", [False, True])
def test_rmat_hubs_movable_and_frozen(gpu, frozen):
    parts, rps, eds, _keep = case_graph(CASES["rmat_s14_p2_b"])
    deg = np.concatenate([np.diff(r) for r in rps])
    hubs = deg >= np.sort(deg)[-20]
    mask = masks_for(int(parts[-1]), 0.3, 5)
    mask[hubs] = 0 if frozen else 1
    for opts in ({}, {"force_heavy_deg": 32}):
        R = Ranks(parts, rps, eds, **opts)
        try:
            set_movable(R, mask)
            for frontier in (0, 1):
                R.set_option("frontier", frontier)
                assert_same(run(R), oracle(parts, rps, eds, mask, frontier), (frozen, opts, frontier))
        finally:
            R.close()


@pytest.mark.parametrize("variant", [3, 4, 5, 6])
@pytest.mark.parametrize("name", ["rgg_n16384_p1", "rgg_n16384_p2", "dyadic_rgg_n16384_s4"])
def test_all_ones_is_no_set(gpu, variant, name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    R = Ranks(parts, rps, eds, scan_variant=variant)
    try:
        ref = run(R)
        assert np.all(ref["movable"] == 1)
        set_movable(R, np.ones(int(parts[-1]), np.uint8))
        for frontier in (0, 1):
            R.set_option("frontier", frontier)
            res = run(R)
            assert_same(res, ref, (name, variant, frontier))
            assert res["first_ran"] == [0] * len(rps)        # a masked run never takes the first-iteration reduction
    finally:
        R.close()


@pytest.mark.parametrize("name", ["rgg_n16384_p1", "rgg_n16384_p4", "rmat_s14_p2_b", "dyadic_rgg_n16384_s4_p5"])
def test_checkpoint_and_resume_with_frontier(gpu, name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    mask = masks_for(int(parts[-1]), 0.05, 3)
    R = Ranks(parts, rps, eds, frontier=1)
    try:
        set_movable(R, mask)
        full = run(R)
        assert_same(full, oracle(parts, rps, eds, mask, 1), name)
        I = full["iters"]
        for k in sorted({k for k in (1, I // 2, I - 1) if 1 <= k <= I - 1}):
            R.set_initial(None)
            set_movable(R, mask)
            R.set_option("stop_after", k)
            a = run(R)
            assert not a["converged"] and a["trace"] == full["trace"][:k], (name, k)
            R.set_option("stop_after", 0)
            R.set_initial(a["comm"])
            set_movable(R, a["movable"])
            b = run(R, lower=a["mod"])
            assert b["converged"] and k + b["iters"] == I and b["trace"] == full["trace"][k:], (name, k)
            assert repr(b["mod"]) == repr(full["mod"]) and np.array_equal(b["comm"], full["comm"]), (name, k)
            assert np.array_equal(b["movable"], full["movable"]), (name, k)
    finally:
        R.close()


@pytest.mark.parametrize("ranks", [1, 2])
def test_cli_checkpoint_and_resume_with_frontier(gpu, tmp_path, ranks):
    env = dict(os.environ)
    if ranks > 1 and gpu.device_count() < ranks:
        env["MVGPU_OPTIONS"] = "host_transport=1"                        # ranks share device 0
    nv = 16384
    mask = masks_for(nv, 0.05, 9)
    vp = str(tmp_path / "v")
    for r in range(ranks):
        mask[nv * r // ranks:nv * (r + 1) // ranks].tofile(f"{vp}.{r}")
    base = ["-n", str(nv), "-g", str(ranks), "-T", "-F"]
    full, tf = cli(base + ["-V", vp], env)
    I = int(re.search(r"RESULT mod=\S+ iters=(\d+)", full.stderr).group(1))
    k = I // 2
    ck = str(tmp_path / "ck")
    p1, t1 = cli(base + ["-V", vp, "-k", str(k), "-o", ck], env)
    m = re.search(r"STOPPED iters=(\d+) prevMod=(\S+)", p1.stderr)
    assert m and int(m.group(1)) == k
    p2, t2 = cli(base + ["-i", ck, "-V", ck + ".mask", "-L", m.group(2)], env)
    assert t1 + t2 == tf
    a = re.search(r"RESULT mod=(\S+)", full.stderr).group(1)
    assert re.search(r"RESULT mod=(\S+)", p2.stderr).group(1) == a
    bad = subprocess.run([EXE, "-n", str(nv), "-V", str(tmp_path / "missing")], capture_output=True, text=True, timeout=300)
    assert bad.returncode != 0 and "-V" in bad.stderr


class Rows:
    """The fields update_ref.extras reads, for one whole-graph shard."""

    def __init__(self, nv, rowptr, edges):
        self.nv, self.base, self.rowptr, self.edges = nv, 0, rowptr, edges


def update_graphs(weights):
    """RGG 65536 -p 0 (rowptr, edges) and the insertion batch that turns it into -p 5: unit weights, dyadic weights
    (tests/helpers.py dyadic_rgg: every sum exact) or Euclidean -w weights."""
    from minivite_b200 import hostgraph as hg
    if weights == "dyadic":
        nv, rp0, ed0 = dyadic_rgg(65536, 1)
        _, rp5, ed5 = dyadic_rgg(65536, 1, pct=5)
        return rp0, ed0, U.extras(Rows(nv, rp0, ed0), Rows(nv, rp5, ed5))
    ss0 = hg.generate_rgg(65536, 1, unit_weight=weights == "unit")
    ss5 = hg.generate_rgg(65536, 1, unit_weight=weights == "unit", random_edge_percent=5)
    s0, s5 = ss0.shards[0], ss5.shards[0]
    out = (s0.rowptr.copy(), s0.edges.copy(), U.extras(s0, s5))
    ss0.close()
    ss5.close()
    return out


@pytest.mark.parametrize("weights", ["unit", "dyadic", "euclidean"])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_update_scenario(gpu, world, weights):
    """RGG 65536 -p 0's result, updated to -p 5 with update_shard, re-clustered warm with movable_from_batch's seeds and
    frontier 1: bit-exact against the oracle with unit and dyadic weights; with Euclidean weights within the
    general-weight tolerance (1e-6 on the modularity, iterations within 2)."""
    rowptr, edges, ins = update_graphs(weights)
    nv = 65536
    parts, rps, eds = split_global(nv, rowptr, edges, world)
    R = Ranks(parts, rps, eds, frontier=1)
    try:
        pre = R.run()
        batches = [tuple(a[(ins[0] >= parts[r]) & (ins[0] < parts[r + 1])] for a in ins) for r in range(world)]
        R.each(lambda r, g: g.update_shard(insert=batches[r]))
        seeds = np.concatenate(R.each(lambda r, g: g.movable_from_batch(insert=batches[r])))
        assert np.array_equal(seeds, np.isin(np.arange(nv), ins[0]).astype(np.uint8))
        R.set_initial(pre["comm"])
        set_movable(R, seeds)
        res = run(R)
        after = U.apply(0, rowptr, edges, None, ins)
        _, rps2, eds2 = split_global(nv, after[0], after[1], world)
        ref = oracle(parts, rps2, eds2, seeds, 1, init=pre["comm"])
        if weights == "euclidean":
            assert abs(res["mod"] - ref["mod"]) <= 1e-6 and abs(res["iters"] - ref["iters"]) <= 2
        else:
            assert_same(res, ref, ("update", weights, world))
    finally:
        R.close()


def single_check(g, parts, rps, eds, mask):
    """Masked runs of a one-rank context with frontier 0 and 1 against the oracle; movable() is read straight after
    louvain(), before anything else touches the context."""
    g.set_option("trace", 1)
    g.set_movable(mask)
    for frontier in (0, 1):
        g.set_option("frontier", frontier)
        mod, iters = g.louvain()
        mov = g.movable().copy()
        res = {"mod": mod, "iters": iters, "trace": as_trace(g.trace()), "comm": g.communities().copy(), "movable": mov}
        assert_same(res, oracle(parts, rps, eds, mask, frontier), frontier)


@pytest.mark.parametrize("mode", ["upload", "attach", "generate"])
def test_one_rank_hand_off_modes(gpu, mode):
    """Every way a shard reaches the device (host upload, attached device arrays, the device generator), masked, on
    RGG 65536; movable() right after louvain() returns the run's final set."""
    import torch
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    ss = hg.generate_rgg(65536, 1)
    sh = ss.shards[0]
    parts, rps, eds = sh.parts, [sh.rowptr.copy()], [sh.edges.copy()]
    ss.close()
    g = G.LouvainGPU(0, 0, 1)
    try:
        if mode == "upload":
            g.upload(65536, parts, rps[0], eds[0])
        elif mode == "attach":
            rp = torch.from_numpy(rps[0]).cuda()
            ed = torch.from_numpy(eds[0].view(np.uint8).copy()).cuda()
            torch.cuda.synchronize()
            g.attach_device(65536, parts, 65536, len(eds[0]), rp.data_ptr(), ed.data_ptr(), keepalive=(rp, ed))
        else:
            g.generate_rgg(65536)
        single_check(g, parts, rps, eds, masks_for(65536, 0.05, 21))
    finally:
        g.close()


def test_state_rules_and_refusals(gpu):
    from minivite_b200 import gpu as G
    case = CASES["rgg_n16384_p1"]
    parts, rps, eds, _keep = case_graph(case)
    nv = int(parts[-1])
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        with pytest.raises(G.MvgpuError, match="no shard"):
            G._ck(G.lib().mvgpu_set_movable(g._h, np.zeros(1, np.uint8).ctypes.data))
        g.upload(nv, parts, rps[0], eds[0])
        with pytest.raises(ValueError):
            g.set_movable(np.zeros(nv - 1, np.uint8))
        with pytest.raises(G.MvgpuError):
            g.set_option("frontier", 2)
        assert np.all(g.movable() == 1)                                       # no set: everything movable
        mask = masks_for(nv, 0.2, 1)
        g.set_movable(mask * 7)                                               # nonzero = movable
        assert np.array_equal(g.movable(), mask)
        cold = g.louvain()
        frozen = g.trace()
        assert cold[1] >= 2 and int(frozen["moved"].sum()) > 0
        g.upload(nv, parts, rps[0], eds[0])                                   # a new upload clears the set
        assert np.all(g.movable() == 1)
        assert g.louvain()[1] == case["iters"]
        g.set_movable(mask)
        g.louvain()
        assert as_trace(g.trace()) == as_trace(frozen)
        g.update_shard()                                                      # an (empty) update keeps it
        assert np.array_equal(g.movable(), mask)
        g.louvain()
        assert as_trace(g.trace()) == as_trace(frozen)
        g.set_movable(None)                                                   # NULL clears
        assert g.louvain()[1] == case["iters"]
    finally:
        g.close()
    # the 32-bit surface refuses a set
    g = G.LouvainGPU(0, 0, 1)
    try:
        rp32 = rps[0].astype(np.int32)
        e8 = np.zeros(len(eds[0]), np.dtype([("tail", "<i4"), ("weight", "<f4")]))
        e8["tail"] = eds[0]["tail"]
        e8["weight"] = eds[0]["weight"]
        g.upload32(nv, parts.astype(np.int32), rp32, e8)
        g.set_movable(np.ones(nv, np.uint8))
        with pytest.raises(G.MvgpuError, match="movable"):
            g.louvain32()
    finally:
        g.close()


def test_ranks_that_disagree_fail_together(gpu):
    from minivite_b200 import gpu as G
    parts, rps, eds, _keep = case_graph(CASES["rgg_n16384_p2"])
    R = Ranks(parts, rps, eds)
    try:
        R.g[0].set_movable(np.ones(int(parts[1] - parts[0]), np.uint8))

        def one(r, g):
            try:
                g.louvain()
            except G.MvgpuError as ex:
                return str(ex)
            return None
        errs = R.each(one)
        assert all(e and "movable" in e for e in errs), errs
        R.g[0].set_movable(None)
        assert R.run()["iters"] == CASES["rgg_n16384_p2"]["iters"]            # the ranks are still usable
        set_movable(R, np.ones(int(parts[-1]), np.uint8))                     # a set on both, the frontier on one
        R.g[0].set_option("frontier", 1)
        errs = R.each(one)
        assert all(e and "frontier" in e for e in errs), errs
        R.g[1].set_option("frontier", 1)
        assert R.run()["iters"] == CASES["rgg_n16384_p2"]["iters"]
    finally:
        R.close()


# [kernel_launches, scan_launches, iters] per rank: the unmasked counts of tests/test_gpu_launch_counts.py plus one
# k_movable_in in setup, plus one k_frontier_mark per iteration with the frontier option
LAUNCHES = {(1, 0): [32, 14, 14], (1, 1): [46, 14, 14], (2, 0): [81, 14, 14], (2, 1): [95, 14, 14],
            (4, 0): [81, 14, 14], (4, 1): [95, 14, 14]}


@pytest.mark.parametrize("world,frontier", sorted(LAUNCHES))
def test_launch_counts(gpu, world, frontier):
    from minivite_b200 import hostgraph as hg
    ss = hg.generate_rgg(16384, 1)
    sh = ss.shards[0]
    parts, rps, eds = split_global(16384, sh.rowptr, sh.edges, world)
    R = Ranks(parts, rps, eds, frontier=frontier)
    try:
        set_movable(R, np.ones(16384, np.uint8))
        R.run()
        got = R.each(lambda r, g: [g.timings()[k] for k in ("kernel_launches", "scan_launches", "iters")])
        assert got == [LAUNCHES[(world, frontier)]] * world
    finally:
        R.close()
        ss.close()


@pytest.mark.skipif(os.environ.get("MV_BIG_TESTS") != "1", reason="full-size run: set MV_BIG_TESTS=1")
def test_full_size_config2_to_config3(gpu):
    """Config 2 updated to config 3, re-clustered warm with the batch's seeds and frontier 1: every iteration's trace
    of two masked runs under different scan variants and renumbering modes agree (the host oracle is too slow here)."""
    from minivite_b200 import gpu as G
    from minivite_b200 import hostgraph as hg
    ss1 = hg.generate_rgg(16777216, 1)
    ss2 = hg.generate_rgg(16777216, 1, random_edge_percent=5)
    ins = U.extras(ss1.shards[0], ss2.shards[0])
    ss2.close()
    runs = []
    for opts in ({"scan_variant": 6, "reorder": 2}, {"scan_variant": 4, "reorder": 0}):
        g = G.LouvainGPU(0, 0, 1)
        try:
            g.set_option("trace", 1)
            for k, v in opts.items():
                g.set_option(k, v)
            sh = ss1.shards[0]
            g.upload(sh.nv, sh.parts, sh.rowptr, sh.edges)
            g.louvain()
            pre = g.communities().copy()
            g.update_shard(insert=ins)
            g.set_initial_communities(pre)
            g.set_movable(g.movable_from_batch(insert=ins))
            g.set_option("frontier", 1)
            mod, iters = g.louvain()
            runs.append((iters, repr(mod), as_trace(g.trace()), g.communities().copy(), g.movable().copy()))
        finally:
            g.close()
    ss1.close()
    assert runs[0][:3] == runs[1][:3]
    assert np.array_equal(runs[0][3], runs[1][3]) and np.array_equal(runs[0][4], runs[1][4])
