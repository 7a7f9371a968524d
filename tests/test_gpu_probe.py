"""Probing an assignment on the device (mvgpu_probe_communities; DESIGN.md §3.15), against the NumPy restatement
tests/probe_ref.py.

On unit and dyadic weights every input of the per-vertex rule is exact, so target, best, the bits of gain and every
report field must match the restatement on 1 rank and on 2, 4 and 16 ranks sharing device 0 (host transport), under
every renumbering mode of the run before, forced and unforced high-degree vertices, every upload mode, and attached,
generated and updated shards.  Euclidean weights are held to step_ref.certify.  A probe is iteration 1 of a warm run
from X that moves nothing: its targets and move count are that run's, and it changes nothing a run, an evaluation or a
comparison reports."""
import os
import re
import subprocess

import numpy as np
import pytest

import probe_ref as PR
import split_ref as SRP
import step_ref as SR
import update_ref as U
from helpers import case_graph, split_global
from oracle import oracle as O
from scan_graphs import split_at
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_quality import _err, evaluate, snapshot
from test_gpu_warm_start import CASES, Ranks, assignments

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "bin", "miniVite_b200")


def probe(R, X=None):
    """Probe X (whole-graph assignment, or None = the last run's) on every rank of R; the report (checked to be the same
    on every rank) with target, best and gain concatenated over the ranks."""
    res = R.each(lambda r, g: g.probe(None if X is None else X[R.parts[r]:R.parts[r + 1]]))
    rep = res[0][0]
    for o in res[1:]:
        assert all(repr(o[0][k]) == repr(rep[k]) for k in PR.FIELDS), (o[0], rep)
    out = dict(rep)
    for i, k in enumerate(("target", "best", "gain")):
        out[k] = np.concatenate([o[1 + i] for o in res])
    return out


def assert_probe(got, ref, what):
    for k in PR.FIELDS:
        assert repr(got[k]) == repr(ref[k]), (what, k, got[k], ref[k])
    assert np.array_equal(got["target"], ref["target"]), what
    assert np.array_equal(got["best"], ref["best"]), what
    assert np.array_equal(got["gain"].view(np.int64), ref["gain"].view(np.int64)), what
    assert got["probe_s"] > 0.0, what


def check(R, G, X, what, Xref=None):
    got = probe(R, X)
    assert_probe(got, PR.probe(G, X if Xref is None else Xref), what)
    return got


def probe_points(R, G, parts, rps, eds, what, run=None):
    """Singletons, the checkpoint after one iteration, the final result (NULL form), its split, random and foreign ids,
    and one community."""
    nv = G.nv
    run = R.run() if run is None else run
    check(R, G, None, f"{what} final", Xref=run["comm"])
    check(R, G, np.arange(nv, dtype=np.int64), f"{what} singletons")
    check(R, G, SRP.split(parts, rps, eds, run["comm"])["Y"], f"{what} split")
    A = assignments(nv, R.world)
    for k in ("random", "named_outside", "other_rank"):
        check(R, G, A[k], f"{what} {k}")
    check(R, G, np.full(nv, nv // 3, np.int64), f"{what} one")
    R.set_option("stop_after", 1)
    c1 = R.run()["comm"]
    R.set_option("stop_after", 0)
    check(R, G, c1, f"{what} C_1")


# ---- bit-exact against the restatement --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_cases(gpu, name):
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    G = SR.Graph(parts, rps, eds)
    R = Ranks(parts, rps, eds)
    try:
        probe_points(R, G, parts, rps, eds, name)
    finally:
        R.close()


@pytest.mark.parametrize("world", [2, 4, 16, "empty16"])
def test_rank_counts(gpu, world):
    for name in ("rmat_s14_p1", "dyadic_random_n4099_d30_hubs2_hub_deg1000_multi100", "rgg_n16384_p1"):
        parts1, rps1, eds1, _keep = case_graph(dict(CASES[name], nranks=1))
        nv = int(parts1[-1])
        if world == "empty16":
            parts = np.array([0, 0, 1, 1, 2, nv // 3, nv // 3, nv // 2, nv // 2 + 1] + [nv] * 8, np.int64)
        else:
            parts = split_global(nv, rps1[0], eds1[0], world)[0]
        rps, eds = split_at(rps1[0], eds1[0], parts)
        G = SR.Graph(parts, rps, eds)
        R = Ranks(parts, rps, eds)
        try:
            probe_points(R, G, parts, rps, eds, f"{name} {world}")
        finally:
            R.close()


@pytest.mark.parametrize("opts", [{"reorder": 0}, {"reorder": 1}, {"reorder": 2}, {"force_heavy_deg": 8},
                                  {"force_weighted": 1}, {"compact_upload": 1}, {"compact_upload": 2},
                                  {"scan_variant": 3}])
@pytest.mark.parametrize("world", [1, 2])
def test_options(gpu, opts, world):
    for name in ("rmat_s14_p1", "dyadic_rgg_n16384_s4", "hand_loops_multi_p1"):
        if "compact_upload" in opts and not name.startswith("rmat"):
            continue                                      # the compact format carries unit weights only
        parts1, rps1, eds1, _keep = case_graph(dict(CASES[name], nranks=1))
        nv = int(parts1[-1])
        parts, rps, eds = split_global(nv, rps1[0], eds1[0], world)
        G = SR.Graph(parts, rps, eds)
        R = Ranks(parts, rps, eds, **opts)
        try:
            probe_points(R, G, parts, rps, eds, f"{name} {opts} {world}")
        finally:
            R.close()


@pytest.mark.parametrize("name", ["rmat_s14_p1", "rmat_s17_p1", "rmat_s17_p2"])
def test_rmat_hubs_unforced(gpu, name):
    """R-MAT hubs exceed the tile kernels' capacity, so k_probe_heavy decides them without any option."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    G = SR.Graph(parts, rps, eds)
    R = Ranks(parts, rps, eds)
    try:
        run = R.run()
        assert R.g[0].shard_info()["nheavy"] > 0
        probe_points(R, G, parts, rps, eds, name, run=run)
    finally:
        R.close()


def test_generated_attached_and_updated_shards(gpu):
    import torch
    from minivite_b200 import gpu as Gm
    from minivite_b200 import hostgraph as hg
    parts = np.array([0, 65536], np.int64)
    g = Gm.LouvainGPU(0, 0, 1)
    ss0, ss5 = hg.generate_rgg(65536, 1), hg.generate_rgg(65536, 1, random_edge_percent=5)
    try:
        g.generate_rgg(65536)
        rowptr, edges = g.download_shard()
        G = SR.Graph(parts, [rowptr], [edges])
        g.louvain()
        X0 = g.communities().copy()
        for X in (None, np.arange(65536, dtype=np.int64) // 9 * 9):
            rep, t, b, gn = g.probe(X)
            assert_probe(dict(rep, target=t, best=b, gain=gn), PR.probe(G, X0 if X is None else X), f"generated {X is None}")
        d_rp = torch.from_numpy(rowptr).cuda()
        d_ed = torch.from_numpy(edges.view(np.uint8).copy()).cuda()
        g.attach_device(65536, parts, 65536, len(edges), d_rp.data_ptr(), d_ed.data_ptr(), keepalive=(d_rp, d_ed))
        rep, t, b, gn = g.probe(X0)
        assert_probe(dict(rep, target=t, best=b, gain=gn), PR.probe(G, X0), "attached")
        # updated: -p 0 -> -p 5 with the extra records, probed from the -p 0 result (the NULL form keeps serving it)
        g.upload(65536, parts, ss0.shards[0].rowptr, ss0.shards[0].edges)
        g.louvain()
        X0 = g.communities().copy()
        g.update_shard(insert=U.extras(ss0.shards[0], ss5.shards[0]))
        G5 = SR.Graph(parts, [ss5.shards[0].rowptr], [ss5.shards[0].edges])
        rep, t, b, gn = g.probe(X0)                      # (NULL waits for a run on the changed shard)
        assert_probe(dict(rep, target=t, best=b, gain=gn), PR.probe(G5, X0), "updated")
        assert (rep["moves"], int(np.sum((t != X0)))) == (2341, 2341)
    finally:
        g.close()
        ss0.close()
        ss5.close()


# ---- general weights: the decision inside step_ref.certify's admissible set ---------------------------------------------------
@pytest.mark.parametrize("world", [1, 2])
def test_euclidean_weights_certified(gpu, world):
    from minivite_b200 import hostgraph as hg
    ss = hg.generate_rgg(65536, world, unit_weight=False)
    parts = ss.shards[0].parts
    rps, eds = [s.rowptr for s in ss.shards], [s.edges for s in ss.shards]
    G = SR.Graph(parts, rps, eds)
    R = Ranks(parts, rps, eds)
    try:
        run = R.run()
        for X in (run["comm"], np.arange(65536, dtype=np.int64), np.arange(65536, dtype=np.int64) // 7 * 7):
            got = probe(R, X)
            c = got["constant"]                          # 2m is summed with atomics: the last bits may differ per setup
            assert abs(c - R.g[0].constant()) <= 1e-12 * c
            cert = SR.certify(G, X, c, heavy_deg=None)
            assert all(SR.admits(cert, v, got["target"][v]) for v in range(G.nv)), world
            cv, cy, lo, hi = cert["pairs"]
            key = cv * G.nv + cy
            sel = np.flatnonzero(cert["certified"] & (got["best"] >= 0))
            at = np.searchsorted(key, sel * G.nv + got["best"][sel])
            assert np.all(key[at] == sel * G.nv + got["best"][sel])
            g = got["gain"][sel]
            assert np.all((lo[at] <= g) & (g <= hi[at])), world
            assert np.array_equal(got["best"] < 0, PR.probe(G, X, c)["best"] < 0)
    finally:
        R.close()
        ss.close()


# ---- consistency with a run ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2])
def test_one_warm_step_and_its_movable_set(gpu, world):
    for name in ("rgg_n16384_p1", "dyadic_random_n3000_d80_blocks25", "rmat_s14_p1"):
        parts1, rps1, eds1, _keep = case_graph(dict(CASES[name], nranks=1))
        nv = int(parts1[-1])
        parts, rps, eds = split_global(nv, rps1[0], eds1[0], world)
        R = Ranks(parts, rps, eds)
        try:
            full = R.run()["comm"]
            for X in (np.arange(nv, dtype=np.int64), full, assignments(nv, world)["named_outside"]):
                got = probe(R, X)
                R.set_initial(X)
                R.set_option("stop_after", 1)
                one = R.run()
                assert np.array_equal(one["comm"], got["target"]), name
                assert one["trace"][0][1] == got["moves"], name
                mask = (got["target"] != X).astype(np.uint8)
                R.each(lambda r, g: g.set_movable(mask[parts[r]:parts[r + 1]]))
                masked = R.run()
                assert masked["trace"][0] == one["trace"][0] and np.array_equal(masked["comm"], one["comm"]), name
                R.each(lambda r, g: g.set_movable(None))
                R.set_option("stop_after", 0)
                R.set_initial(None)
        finally:
            R.close()


# ---- state rules --------------------------------------------------------------------------------------------------------------
def test_state_rules(gpu):
    case = CASES["rgg_n65536_p1"]
    parts, rps, eds, _keep = case_graph(case)
    nv = int(parts[-1])
    G = SR.Graph(parts, rps, eds)
    other = np.random.default_rng(3).integers(0, nv, nv)
    for reorder in (1, 0):
        R, plain = Ranks(parts, rps, eds, reorder=reorder), Ranks(parts, rps, eds, reorder=reorder)
        try:
            init = np.arange(nv, dtype=np.int64) // 5 * 5
            mask = (np.arange(nv) % 3 != 0).astype(np.uint8)
            for S in (R, plain):
                S.set_initial(init)
                S.each(lambda r, g: g.set_movable(mask))
            a = R.run()
            g = R.g[0]
            q = evaluate(R, other)
            g.compare_communities(other)
            matches = g.community_matches()
            before = (snapshot(g), g.movable().tolist(), g.community_stats(), g.compact_communities().tolist())
            check(R, G, other, "other")
            check(R, G, None, "final", Xref=a["comm"])
            assert _err(lambda: g.probe(np.zeros(nv + 1, np.int64)))           # refusals change nothing either
            bad = np.zeros(nv, np.int64)
            bad[5] = nv
            assert "outside" in _err(lambda: g.probe(bad))
            after = (snapshot(g), g.movable().tolist(), g.community_stats(), g.compact_communities().tolist())
            assert after[0] == before[0] and after[1] == before[1] and after[3] == before[3], reorder
            assert all(np.array_equal(after[2][k], before[2][k]) for k in before[2]), reorder
            assert all(np.array_equal(g.community_matches()[k], matches[k]) for k in matches), reorder
            assert evaluate(R)["modularity"] == evaluate(R, a["comm"])["modularity"]
            b, ref = R.run(), plain.run()
            assert b["trace"] == ref["trace"] == a["trace"] and np.array_equal(b["comm"], ref["comm"])
            assert g.timings()["kernel_launches"] == plain.g[0].timings()["kernel_launches"]
            assert q["communities"] > 0
        finally:
            R.close()
            plain.close()


def test_errors(gpu):
    from minivite_b200 import gpu as Gm
    case = CASES["rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    R = Ranks(parts, rps, eds)
    try:
        errs = R.each(lambda r, g: _err(lambda: g.probe()))                # NULL before any run
        assert all(e and "no" in e for e in errs), errs
        nv = int(parts[-1])
        bad = np.zeros(nv, np.int64)
        bad[nv - 1] = nv                                                   # a bad id on rank 1 only
        errs = R.each(lambda r, g: _err(lambda: g.probe(bad[parts[r]:parts[r + 1]])))
        assert errs[1] and "outside" in errs[1] and errs[0] and "another rank" in errs[0], errs
        errs = R.each(lambda r, g: _err(lambda: g.probe(np.zeros(g.lnv + r, np.int64))))   # a wrong length on rank 1
        assert errs[1] and "entries" in errs[1] and errs[0] and "another rank" in errs[0], errs
        R.run()
        errs = R.each(lambda r, g: _err(lambda: g.probe(None if r == 0 else np.zeros(g.lnv, np.int64))))
        assert all(e and "disagree on the assignment to probe" in e for e in errs), errs
        assert probe(R)["vertices"] == nv                                  # both contexts are still usable
    finally:
        R.close()
    g = Gm.LouvainGPU(0, 0, 1)
    try:
        c32 = CASES["hand_clique_ring_p1"]
        p32, r32, e32s, _k = case_graph(c32)
        e32 = np.zeros(len(e32s[0]), np.dtype([("tail", "<i4"), ("weight", "<f4")]))
        e32["tail"], e32["weight"] = e32s[0]["tail"], e32s[0]["weight"]
        g.upload32(int(p32[-1]), p32, r32[0], e32)
        g.louvain32()
        with pytest.raises(Gm.MvgpuError, match="upload_shard32"):
            g.probe()
        with pytest.raises(Gm.MvgpuError, match="upload_shard32"):
            g.probe(np.zeros(int(p32[-1]), np.int64))
    finally:
        g.close()


# ---- the CLI: -U after a run, with -C, with -E, and -o's unsettled set as -V -------------------------------------------------
PROBE_RE = re.compile(r"PROBE vertices=(\d+) moves=(\d+) vetoed=(\d+) interior=(\d+) max_gain=(\S+)")


def parse_probe(stderr):
    m = PROBE_RE.search(stderr)
    assert m, stderr[-2000:]
    return {"vertices": int(m.group(1)), "moves": int(m.group(2)), "vetoed": int(m.group(3)), "interior": int(m.group(4)),
            "max_gain": float(m.group(5))}


@pytest.mark.parametrize("ranks", [1, 2])
def test_cli(gpu, tmp_path, ranks):
    env = dict(os.environ)
    if ranks > 1 and gpu.device_count() < ranks:
        env["MVGPU_OPTIONS"] = "host_transport=1"
    case = CASES["rgg_n16384_p1" if ranks == 1 else "rgg_n16384_p2"]
    parts, rps, eds, _keep = case_graph(case)
    G = SR.Graph(parts, rps, eds)

    def cli(*args):
        p = subprocess.run([EXE, "-n", "16384", "-g", str(ranks), *args], capture_output=True, text=True, timeout=300, env=env)
        assert p.returncode == 0, p.stderr[-2000:]
        return p.stderr

    def read(prefix):
        return np.concatenate([np.fromfile(f"{prefix}.{r}", np.int64)[2:] for r in range(ranks)])

    def same(got, X):
        ref = PR.probe(G, X)
        assert all(got[k] == ref[k] for k in got), (got, ref)

    pre, pre2, pre3 = str(tmp_path / "a"), str(tmp_path / "b"), str(tmp_path / "c")
    got = parse_probe(cli("-k", "2", "-U", "-o", pre))                   # a checkpoint: most vertices still want to move
    X = read(pre)
    same(got, X)
    uns = np.concatenate([np.fromfile(f"{pre}.unsettled.{r}", np.uint8) for r in range(ranks)])
    assert np.array_equal(uns, (PR.probe(G, X)["target"] != X).astype(np.uint8)) and got["moves"] == int(uns.sum()) > 0
    same(parse_probe(cli("-E", pre, "-U")), X)
    Y = SRP.split(parts, rps, eds, X)["Y"]
    same(parse_probe(cli("-E", pre, "-C", "-U")), Y)
    got = parse_probe(cli("-i", pre, "-V", f"{pre}.unsettled", "-F", "-C", "-U", "-o", pre2))   # re-cluster from the unsettled
    Z = read(pre2)
    same(got, Z)
    assert np.array_equal(np.concatenate([np.fromfile(f"{pre2}.unsettled.{r}", np.uint8) for r in range(ranks)]),
                          (PR.probe(G, Z)["target"] != Z).astype(np.uint8))
    cli("-i", pre, "-V", f"{pre}.unsettled", "-F", "-o", pre3)
    ref = O.louvain(parts, rps, eds, init_comm=[X[parts[r]:parts[r + 1]] for r in range(ranks)],
                    movable=[uns[parts[r]:parts[r + 1]] for r in range(ranks)], frontier=1)
    assert np.array_equal(read(pre3), np.concatenate(ref["comm"]))
