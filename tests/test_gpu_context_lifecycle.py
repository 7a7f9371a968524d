"""Long-lived contexts (DESIGN.md §4): any sequence of calls on one context gives what fresh contexts give, and a refused
call changes nothing.  The sequences and the shard catalogue are in lifecycle.py; test_lifecycle_scripts.py asserts on
the CPU that they cross the boundaries they claim.  Ranks > 1 are threads sharing device 0 through the host transport,
and, in the last test, two processes that map each other's arrays through CUDA IPC."""
import json
import os
import sys
import threading

import numpy as np
import pytest

import compare_ref
import lifecycle as L
import quality_ref
import split_ref
from test_gpu_parity import gpu  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_RUN = "no run on this shard"
COUNTS = ("unit_weight", "reordered", "scan_launches", "kernel_launches", "iters")


# ---- a context per rank, driven together ------------------------------------------------------------------------------
class Ranks:
    def __init__(self, world, ident=None):
        from minivite_b200 import gpu as G
        self.G, self.world = G, world
        self.g = [G.LouvainGPU(0, r, world) for r in range(world)]
        self.keep = None
        if world > 1:
            ident = ident or G.get_unique_id()
            for g in self.g:
                g.set_option("host_transport", 1)
            self.each(lambda g, r: g.comm_init(ident))

    def each(self, fn):
        """fn(g, rank) on every rank (threads when world > 1); per rank its value or ("error", text)."""
        out = [None] * self.world

        def work(r):
            try:
                out[r] = fn(self.g[r], r)
            except self.G.MvgpuError as ex:
                out[r] = ("error", str(ex))
        if self.world == 1:
            work(0)
            return out
        th = [threading.Thread(target=work, args=(r,)) for r in range(self.world)]
        for t in th:
            t.start()
        for t in th:
            t.join(timeout=300)
        assert not any(t.is_alive() for t in th), "a rank did not return"
        return out

    def close(self):
        for g in self.g:
            g.close()


def load(R, s):
    """Replace the shard through the entry point the spec names."""
    s0 = s["base"] if s["kind"] == "updated" else s
    if s0["via"] == "attach":
        import torch
        t = [(torch.from_numpy(s0["rowptrs"][r].copy()).cuda(), torch.from_numpy(s0["edges"][r].view(np.uint8).copy()).cuda())
             for r in range(R.world)]
        torch.cuda.synchronize()
        R.keep = t
        res = R.each(lambda g, r: g.attach_device(s0["nv"], s0["parts"], len(s0["rowptrs"][r]) - 1, len(s0["edges"][r]),
                                                  t[r][0].data_ptr(), t[r][1].data_ptr(), keepalive=t[r]))
    elif s0["via"] == "generate":
        res = R.each(lambda g, r: g.generate_rgg(s0["nv"], random_edge_percent=s0["pct"]))
    elif s0["via"] == "upload32":
        e8 = [np.zeros(len(e), np.dtype([("tail", "<i4"), ("weight", "<f4")])) for e in s0["edges"]]
        for e, src in zip(e8, s0["edges"]):
            e["tail"], e["weight"] = src["tail"], src["weight"]
        res = R.each(lambda g, r: g.upload32(s0["nv"], s0["parts"], s0["rowptrs"][r], e8[r]))
    else:
        res = R.each(lambda g, r: g.upload(s0["nv"], s0["parts"], s0["rowptrs"][r], s0["edges"][r]))
    if s["kind"] == "updated" and not any(isinstance(x, tuple) for x in res):
        b = L.batch(s0, s["batch_seed"])
        res = R.each(lambda g, r: g.update_shard(*b[r]))
    return res


def python_refusal(fn):
    """A refusal of the binding (before the library is called), as ("error", text)."""
    try:
        fn()
    except ValueError as ex:
        return ("error", str(ex))
    return None


def attempt(fn):
    from minivite_b200 import gpu as G
    try:
        return fn()
    except G.MvgpuError as ex:
        return ("error", str(ex))


def snapshot(g, run_report=True):
    """Everything a context shows (no measured seconds).  run_report: include what describes the last mvgpu_louvain
    call (trace, constant, converged, launch counts), which a shard replacement does not reset."""
    from test_gpu_layout import readback
    s = {"info": g.shard_info(), "movable": attempt(lambda: g.movable().copy()),
         "shard": attempt(lambda: g.download_shard()),
         "comm": attempt(lambda: g.communities().copy()), "comm32": attempt(lambda: g.communities32().copy()),
         "stats": attempt(lambda: g.community_stats()), "compact": attempt(lambda: g.compact_communities().copy()),
         "matches": attempt(lambda: g.community_matches()), "layout": attempt(lambda: readback(g))}
    if run_report:
        t = g.timings()
        s.update(trace=g.trace().copy(), constant=g.constant(), converged=attempt(g.converged),
                 counts={k: t[k] for k in COUNTS})
    return s


def assert_same(a, b, what):
    if isinstance(a, dict):
        assert isinstance(b, dict) and a.keys() == b.keys(), (what, a, b)
        for k in a:
            assert_same(a[k], b[k], f"{what}.{k}")
    elif isinstance(a, (tuple, list)):
        assert isinstance(b, (tuple, list)) and len(a) == len(b), (what, a, b)
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{what}[{i}]")
    elif isinstance(a, np.ndarray):
        assert isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape, (what, a, b)
        assert a.tobytes() == b.tobytes(), what
    elif isinstance(a, float):
        assert repr(a) == repr(b), (what, a, b)
    else:
        assert a == b, (what, a, b)


# ---- the runner: one long-lived context against fresh ones and the references ------------------------------------------
class Runner:
    def __init__(self, world):
        self.world = world
        self.R = Ranks(world)
        self.cur = None                 # the current graph (host arrays)
        self.seg = []                   # the steps since the last shard replacement
        self.opts0 = {}                 # the options in effect when the segment began
        self.opts = {}
        self.last = None                # the last run's assignment (per rank)
        self.ran = False                # a louvain in this segment

    def step(self, st, R=None):
        """Apply one step on R (default: the long-lived ranks); returns per-rank results."""
        R = R or self.R
        op = st[0]
        if op == "load":
            return load(R, st[1])
        if op == "update":
            b = L.batch(self.cur, st[1])
            return R.each(lambda g, r: g.update_shard(*b[r]))
        if op == "opt":
            return R.each(lambda g, r: g.set_option(st[1], st[2]))
        if op == "init":
            a = None if st[1] is None else L.assignment(self.cur, st[1])
            return R.each(lambda g, r: g.set_initial_communities(None if a is None else a[r]))
        if op == "mov":
            m = None if st[1] is None else L.mask(self.cur, st[1])
            return R.each(lambda g, r: g.set_movable(None if m is None else m[r]))
        if op == "run":
            u32 = self.cur["via"] == "upload32"

            def go(g, r):
                if u32:
                    mod, it = g.louvain32()
                    return mod, it, g.communities32().astype(np.int64)
                mod, it = g.louvain()
                return mod, it, g.communities().copy()
            return R.each(go)
        a = None if st[1] is None else L.assignment(self.cur, st[1])
        if op == "eval":
            return R.each(lambda g, r: g.evaluate(None if a is None else a[r]))
        if op == "split":
            return R.each(lambda g, r: g.split_communities(None if a is None else a[r]))
        if op == "compare":
            return R.each(lambda g, r: g.compare_communities(a[r]))
        raise ValueError(op)

    def close(self):
        self.R.close()

    def play(self, steps):
        refused = L.expect_refused(steps)
        for i, st in enumerate(steps):
            if st[0] == "load":
                self.seg, self.opts0, self.ran = [], dict(self.opts), False
            res = self.step(st)                  # an update's batch is drawn from the graph before it
            if st[0] == "load":
                self.cur = L.resolve(st[1])
            elif st[0] == "update":
                self.cur = L.apply_update(self.cur, st[1])
            elif st[0] == "opt":
                self.opts[st[1]] = st[2]
            if st[0] != "load":
                self.seg.append(st)
            if st[0] == "update":
                # the updated shard is what update_ref computes
                for r, g in enumerate(self.R.g):
                    rp, ed = g.download_shard()
                    assert np.array_equal(rp, self.cur["rowptrs"][r]) and ed.tobytes() == self.cur["edges"][r].tobytes(), (i, st)
            self.ran |= st[0] == "run"
            errs = [x for x in res if isinstance(x, tuple) and len(x) == 2 and isinstance(x[0], str) and x[0] == "error"]
            assert len(errs) == (self.world if refused[i] else 0), (i, st, refused[i], errs)
            self.check_refs(i, st, res)
            self.check_fresh(i, st, steps)

    def check_refs(self, i, st, res):
        """Every run against the C oracle, every evaluate / split / compare against its NumPy restatement."""
        from oracle import oracle as O
        errs = [x for x in res if isinstance(x, tuple) and len(x) == 2 and isinstance(x[0], str) and x[0] == "error"]
        cur = self.cur
        if st[0] == "run":
            assert not errs, (i, st, errs)
            mod, it, _c = res[0]
            comm = np.concatenate([x[2] for x in res])
            if cur["via"] == "upload32":
                self.last = [x[2] for x in res]
                return
            stop = self.opts.get("stop_after", 0)
            init = self.init_arrays()
            mov = self.mov_arrays()
            ref = O.louvain(cur["parts"], cur["rowptrs"], cur["edges"], init_comm=init, stop_after=stop, movable=mov,
                            frontier=self.opts.get("frontier", 0) if mov is not None else 0)
            tr = self.R.g[0].trace()
            assert it == ref["iters"] and repr(mod) == repr(ref["modularity"]), (i, st, it, ref["iters"], mod, ref["modularity"])
            assert np.array_equal(comm, np.concatenate(ref["comm"])), (i, st)
            assert repr(self.R.g[0].constant()) == repr(ref["constant"]), (i, st)
            assert len(tr) == len(ref["trace"]) and tr.tobytes() == ref["trace"].tobytes(), (i, st)
            self.last = [x[2] for x in res]
        elif st[0] in ("eval", "split", "compare") and not errs:
            X = self.last if st[1] is None or st[0] == "compare" else L.assignment(cur, st[1])
            if st[0] == "eval":
                q = quality_ref.quality(cur["parts"], cur["rowptrs"], cur["edges"], X)
                for k in ("modularity", "e_in", "a2", "constant", "communities", "singletons", "max_size"):
                    assert repr(res[0][k]) == repr(q[k]), (i, st, k, res[0][k], q[k])
            elif st[0] == "split":
                ref = split_ref.split(cur["parts"], cur["rowptrs"], cur["edges"], X)
                assert np.array_equal(np.concatenate([x[0] for x in res]), ref["Y"]), (i, st)
                for k in ("communities", "components", "disconnected"):
                    assert res[0][1][k] == ref[k], (i, st, k)
            else:
                ref = compare_ref.compare(X, L.assignment(cur, st[1]))
                for k in ("cells", "pairs_xy", "pairs_x", "pairs_y", "ari", "nmi", "vi"):
                    assert repr(res[0][k]) == repr(ref[k]), (i, st, k, res[0][k], ref[k])

    def init_arrays(self):
        for st in reversed(self.seg):
            if st[0] == "init":
                return None if st[1] is None else L.assignment(self.cur, st[1])   # depends on parts only
        return None

    def mov_arrays(self):
        for st in reversed(self.seg):
            if st[0] == "mov":
                return None if st[1] is None else L.mask(self.cur, st[1])
        return None

    def check_fresh(self, i, st, steps):
        """A fresh context given the segment's shard, options and inputs shows the same, bit for bit (launch counts only
        under a fixed scan kernel: scan_variant 6 chooses by timing)."""
        load_step = next((s for s in reversed(steps[:i + 1]) if s[0] == "load"), None)
        if load_step is None:               # options before the first shard: nothing to compare yet
            return
        F = Ranks(self.world)
        try:
            F.each(lambda g, r: [g.set_option(k, v) for k, v in self.opts0.items()])
            saved = self.cur
            base = L.resolve(load_step[1])
            self.cur = base
            load(F, load_step[1])
            for s in self.seg:
                self.step(s, F)
                if s[0] == "update":
                    self.cur = L.apply_update(self.cur, s[1])
            self.cur = saved
            for r in range(self.world):
                a, b = snapshot(self.R.g[r], self.ran), snapshot(F.g[r], self.ran)
                if self.ran and self.opts.get("scan_variant", 6) == 6:
                    for k in ("scan_launches", "kernel_launches"):
                        a["counts"].pop(k), b["counts"].pop(k)
                assert_same(a, b, f"step {i} {st[0]} rank {r}")
        finally:
            F.close()


# ---- 1. getter contract -------------------------------------------------------------------------------------------------
def replace_ops():
    return {"upload": lambda n: L.spec("rgg", n), "upload32": lambda n: L.spec("u32", n),
            "attach": lambda n: L.spec("attach", n), "generate": lambda n: L.spec("gen", n)}


def check_no_result(g, s):
    from test_gpu_layout import readback
    import ctypes
    for fn in (g.communities, g.communities32, lambda: readback(g)):
        r = attempt(fn)
        assert isinstance(r, tuple) and NO_RUN in r[1], r
    from minivite_b200 import gpu as G
    d = ctypes.c_void_p()
    rc = G.lib().mvgpu_get_communities_device(g._h, ctypes.byref(d))
    assert rc != 0 and NO_RUN in G.lib().mvgpu_last_error().decode()
    info = g.shard_info()
    assert info["lnv"] == len(s["rowptrs"][0]) - 1 and info["lne"] == len(s["edges"][0])
    assert [info[k] for k in ("nghost", "nsend", "nheavy", "maxdeg")] == [0, 0, 0, 0], info


@pytest.mark.parametrize("size_b", ["smaller", "larger"])
def test_getter_contract_after_shard_replacement(gpu, size_b):  # noqa: F811
    """Run A (16 384 vertices), replace it by B (4 096 or 65 536) through every replacing entry point, with and without
    a communities() call before: the per-vertex getters refuse with "no run on this shard" and shard_info()[2:6] is 0;
    B's own run then serves B's result."""
    from oracle import oracle as O
    nb = 4096 if size_b == "smaller" else 65536
    for via, mk in replace_ops().items():
        for read_first in (False, True):
            R = Ranks(1)
            try:
                g = R.g[0]
                a = L.spec("rgg", 16384)
                load(R, a)
                g.louvain()
                if read_first:
                    g.communities()
                b = mk(nb)
                assert not isinstance(load(R, b)[0], tuple)
                check_no_result(g, b)
                if via == "upload32":
                    g.louvain32()
                    got = g.communities32().astype(np.int64)
                else:
                    g.louvain()
                    got = g.communities()
                    ref = O.louvain(b["parts"], b["rowptrs"], b["edges"])
                    assert np.array_equal(got, ref["comm"][0]), (via, read_first)
                assert len(got) == nb and g.shard_info()["maxdeg"] > 0
            finally:
                R.close()


def test_update_keeps_serving_the_last_result(gpu):  # noqa: F811
    """mvgpu_update_shard is not a replacement: communities() keeps returning the last run's result."""
    R = Ranks(1)
    try:
        g = R.g[0]
        s = L.spec("rgg", 8192)
        load(R, s)
        g.louvain()
        before = g.communities().copy()
        g.update_shard(*L.batch(s, 3)[0])
        assert np.array_equal(g.communities(), before)
    finally:
        R.close()


# ---- 2. refusals change nothing -----------------------------------------------------------------------------------------
def refusals(world, s):
    """(name, per-rank call) of every refusal of the shard-replacing calls and the setters, for shard s in place."""
    nv, parts = s["nv"], np.asarray(s["parts"], np.int64)
    rp, ed = s["rowptrs"], s["edges"]
    e8 = [np.zeros(len(e), np.dtype([("tail", "<i4"), ("weight", "<f4")])) for e in ed]
    other = L.spec("rgg", 4096, world)
    bad_parts = {"first_not_0": np.r_[1, parts[1:]], "last_not_nv": np.r_[parts[:-1], nv + 1],
                 "lnv_mismatch": None}
    out = []
    for k, p in bad_parts.items():
        if p is None:                                   # every rank hands in another shard's rows with this partition
            out.append(("upload " + k, lambda g, r: g.upload(nv, parts, other["rowptrs"][r], other["edges"][r])))
            out.append(("upload32 " + k, lambda g, r: g.upload32(nv, parts, other["rowptrs"][r].astype(np.int32),
                                                                  np.zeros(len(other["edges"][r]), e8[0].dtype))))
        else:
            out.append(("upload " + k, lambda g, r, p=p: g.upload(nv, p, rp[r], ed[r])))
            out.append(("upload32 " + k, lambda g, r, p=p: g.upload32(nv, p, rp[r].astype(np.int32), e8[r])))
    if world == 1:
        out.append(("upload nv of another graph", lambda g, r: g.upload(2 * nv, np.array([0, 2 * nv], np.int64), rp[0], ed[0])))
        out.append(("upload nv >= 2^31", lambda g, r: g.upload(1 << 31, np.array([0, 1 << 31]), rp[0], ed[0])))
    else:
        mono = np.array(parts, np.int64)
        mono[1], mono[2] = parts[2], parts[1]
        out.append(("upload not monotone", lambda g, r: g.upload(nv, mono, rp[r], ed[r])))

    def attach_bad(g, r):
        import torch
        t = torch.zeros(16, dtype=torch.int64, device="cuda")
        return g.attach_device(nv + 1, parts, len(rp[r]) - 1, 0, t.data_ptr(), t.data_ptr())
    out.append(("attach last_not_nv", attach_bad))
    out.append(("attach misaligned", lambda g, r: g.attach_device(nv, parts, 1, 1, 8, 8)))
    out.append(("generate nv < 1", lambda g, r: g.generate_rgg(0)))
    out.append(("generate pct < 0", lambda g, r: g.generate_rgg(16384, random_edge_percent=-1.0)))
    out.append(("generate too many draws", lambda g, r: g.generate_rgg(16384, random_edge_percent=1e9)))
    if world > 1:
        out.append(("generate not divisible", lambda g, r: g.generate_rgg(world * 1024 + 1)))
    out.append(("init id >= nv", lambda g, r: g.set_initial_communities(np.full(len(rp[r]) - 1, nv, np.int64))))
    out.append(("init id < 0", lambda g, r: g.set_initial_communities(np.full(len(rp[r]) - 1, -1, np.int64))))
    out.append(("movable wrong length", lambda g, r: python_refusal(lambda: g.set_movable(np.ones(len(rp[r]) + 1, np.uint8)))))
    for name, v in (("unknown_option", 1), ("max_iters", 0), ("scan_variant", 7), ("frontier", 2), ("stop_after", -1),
                    ("region_size", 8), ("scan_ctas", -1), ("upload_chunk", 100)):
        out.append((f"option {name}={v}", lambda g, r, name=name, v=v: g.set_option(name, v)))
    return out


@pytest.mark.parametrize("world,base", [(1, "gen"), (1, "rgg"), (2, "gen"), (2, "rgg")])
def test_refusals_change_nothing(gpu, world, base):  # noqa: F811
    """After every refusal: the snapshot equals the one before, and the next louvain equals the run before it bit for
    bit (launch counts included), with the warm start and the movable set still in effect.  The generated base shard is
    the one a refused generate_rgg would overwrite in place."""
    R = Ranks(world)
    try:
        s = L.spec(base, 16384, world)
        load(R, s)
        R.each(lambda g, r: [g.set_option(k, v) for k, v in (("trace", 1), ("scan_variant", 4), ("frontier", 1))])
        init, mov = L.assignment(s, 5), L.mask(s, 6)
        R.each(lambda g, r: g.set_initial_communities(init[r]))
        R.each(lambda g, r: g.set_movable(mov[r]))

        def run_all():
            R.each(lambda g, r: g.louvain())
            return [snapshot(g) for g in R.g]
        run_all()
        first = run_all()
        for name, call in refusals(world, s):
            before = [snapshot(g) for g in R.g]
            res = R.each(call)
            assert all(isinstance(x, tuple) and x[0] == "error" for x in res), (name, res)
            for r in range(world):
                assert_same([snapshot(g) for g in R.g][r], before[r], f"{name} rank {r}")
            again = run_all()
            for r in range(world):
                assert_same(again[r], first[r], f"{name}: the next run, rank {r}")
    finally:
        R.close()


# ---- 3. partition disagreement ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
def test_partition_disagreement_fails_every_rank(gpu, world):  # noqa: F811
    from oracle import oracle as O
    R = Ranks(world)
    try:
        even, skew = L.spec("rgg", 16384, world), L.spec("rgg", 16384, world, parts="skew")
        small = L.spec("rgg", 8192, world)
        for mixed in ((even, skew), (even, small)):      # different parts; a different nv_global
            res = R.each(lambda g, r: load_rank(g, r, mixed[r % 2]))
            assert all(x is None for x in res), res
            res = R.each(lambda g, r: g.louvain())
            assert all(isinstance(x, tuple) and "ranks disagree on the partition" in x[1] for x in res), res
            res = R.each(lambda g, r: g.compare_communities(np.zeros(g.lnv, np.int64), x=np.zeros(g.lnv, np.int64)))
            assert all(isinstance(x, tuple) and "ranks disagree on the partition" in x[1] for x in res), res
        R.each(lambda g, r: g.set_option("trace", 1))
        load(R, even)
        res = R.each(lambda g, r: (g.louvain(), g.communities().copy()))
        ref = O.louvain(even["parts"], even["rowptrs"], even["edges"])
        assert res[0][0] == (ref["modularity"], ref["iters"])
        assert np.array_equal(np.concatenate([x[1] for x in res]), np.concatenate(ref["comm"]))
        assert R.g[0].trace().tobytes() == ref["trace"].tobytes()
    finally:
        R.close()


def load_rank(g, r, s):
    g.upload(s["nv"], s["parts"], s["rowptrs"][r], s["edges"][r])


# ---- 4, 5. differential sequences ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["scripted", "pairs", "walk1", "walk2", "walk3"])
def test_sequences_one_rank(gpu, name):  # noqa: F811
    steps = {"scripted": L.scripted_1rank, "pairs": L.pair_script}.get(name, None)
    steps = steps() if steps else L.walk(L.WALK_SEEDS[int(name[-1]) - 1], 30)
    run = Runner(1)
    try:
        run.play(steps)
    finally:
        run.close()


@pytest.mark.parametrize("world", [2, 4])
def test_sequences_ranks_as_threads(gpu, world):  # noqa: F811
    """The multi-rank script (lifecycle.multirank_script) on ranks that are threads sharing device 0: every run bit-exact
    to the oracle, every step's snapshot equal to fresh contexts given the same inputs."""
    run = Runner(world)
    try:
        run.play(L.multirank_script(world))
    finally:
        run.close()


def test_set_movable_without_a_shard_changes_nothing(gpu):  # noqa: F811
    """The library refuses a movable set on a context without a shard before it touches any state: a later upload and
    run give what a fresh context gives."""
    s = L.spec("rgg", 4096)
    R, F = Ranks(1), Ranks(1)
    try:
        g = R.g[0]
        r = attempt(lambda: g.set_movable(np.zeros(0, np.uint8)))
        assert isinstance(r, tuple) and "no shard yet" in r[1], r
        for X in (R, F):
            X.each(lambda g, r: g.set_option("trace", 1))
            load(X, s)
            X.each(lambda g, r: g.louvain())
        assert_same(snapshot(R.g[0]), snapshot(F.g[0]), "after a refused set_movable")
    finally:
        R.close()
        F.close()


# ---- 6. two rank processes on one device ------------------------------------------------------------------------------
def process_script():
    """A grow on rank 0 only (its exported arrays reallocated while rank 1 keeps its mappings: the collective
    close-before-grow and a re-opened mapping), a shrink and a regrow to the old size (no reallocation: the buffers are
    grow-only, so the mappings stay valid and must not be reopened), unit <-> weighted and a frontier run (arrays
    exported for the first time)."""
    s = lambda k, n, **kw: ("load", L.spec(k, n, 2, **kw))      # noqa: E731
    return [("opt", "trace", 1), s("rgg", 16384), ("run",), s("rgg", 16384, parts="skew"), ("run",),
            s("rgg", 4096), ("run",), s("rgg", 16384), ("run",), s("dyadic", 8192), ("run",),
            s("rgg", 8192), ("mov", 3), ("opt", "frontier", 1), ("run",)]


def _proc_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from minivite_b200 import dist as D
    from minivite_b200 import gpu as G
    import lifecycle as LL
    Rk = D.Ranks("gloo")
    ident = Rk.broadcast_bytes(G.get_unique_id() if rank == 0 else None, G.UNIQUE_ID_BYTES)
    g = G.LouvainGPU(0, rank, world)
    g.set_option("host_transport", 1)
    g.comm_init(ident)
    out, cur = [], None
    for st in process_script():
        if st[0] == "load":
            cur = st[1]
            g.upload(cur["nv"], cur["parts"], cur["rowptrs"][rank], cur["edges"][rank])
        elif st[0] == "opt":
            g.set_option(st[1], st[2])
        elif st[0] == "mov":
            g.set_movable(LL.mask(cur, st[1])[rank])
        else:
            mod, iters = g.louvain()
            allc = Rk.gather_arrays(g.communities())
            if rank == 0:
                out.append({"mod": repr(mod), "iters": iters, "comm": [int(x) for x in np.concatenate(allc)],
                            "trace": g.trace().tobytes().hex()})
    if rank == 0:
        json.dump(out, open(os.path.join(out_dir, "res.json"), "w"))
    g.close()
    Rk.shutdown()


def test_rank_processes_reuse_one_context(tmp_path, gpu):  # noqa: F811
    import torch.multiprocessing as mp
    from oracle import oracle as O
    from test_gpu_multi import _free_port
    mp.spawn(_proc_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    res = json.load(open(tmp_path / "res.json"))
    cur, mov, k = None, None, 0
    for st in process_script():
        if st[0] == "load":
            cur, mov = st[1], None
        elif st[0] == "mov":
            mov = L.mask(cur, st[1])
        elif st[0] == "run":
            ref = O.louvain(cur["parts"], cur["rowptrs"], cur["edges"], movable=mov, frontier=1 if mov else 0)
            got = res[k]
            k += 1
            assert got["iters"] == ref["iters"] and got["mod"] == repr(ref["modularity"]), (k, got["iters"], ref["iters"])
            assert got["comm"] == [int(x) for x in np.concatenate(ref["comm"])], k
            assert bytes.fromhex(got["trace"]) == ref["trace"].tobytes(), k
    assert k == len(res) == 6
