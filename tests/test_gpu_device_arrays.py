"""Per-vertex arrays in device memory (DESIGN.md §3.16).

Every entry point that takes or returns a per-vertex or per-community array takes host memory (pageable or pinned) or
device memory of the context's device, pointer by pointer.  The device form must give the host form's bits: run ->
split -> evaluate -> compare -> probe -> movable set -> warm start -> shard update, on an RGG, an R-MAT shard with
high-degree vertices and a dyadic-weight shard, with and without the locality renumbering, on one rank and on 2, 4
and 16 ranks sharing device 0 with every rank and every pointer choosing its own kind.  A bad id fails every rank with
the host form's message; resuming from device memory continues a run exactly; inputs are copied at call time."""
import json
import os
import socket
import sys

import numpy as np
import pytest

from helpers import case_graph, split_global
from scan_graphs import split_at
from test_gpu_context_lifecycle import assert_same, attempt, snapshot
from test_gpu_parity import gpu  # noqa: F401  (fixture)
from test_gpu_warm_start import CASES, Ranks, as_trace

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

GRAPHS = ["rgg_n65536_p1", "rmat_s17_p1", "dyadic_random_n6000_d8_hubs3_hub_deg3000_multi200"]
FORMS = ("numpy", "pinned", "torch")
TIMES = ("split_s", "eval_s", "compare_s", "probe_s", "rounds")   # rounds: how fast labels spread, timing-dependent


def whole(name):
    """(nv, rowptr, edges) of a one-rank golden case, copied out of the generator's buffers (freed with _keep)."""
    parts, rps, eds, _keep = case_graph(CASES[name])
    assert len(rps) == 1
    return int(parts[-1]), rps[0].copy(), eds[0].copy()


def put(a, form):
    """NumPy array a as the caller would hold it: pageable NumPy, NumPy over pinned memory, or a CUDA tensor."""
    import torch
    a = np.ascontiguousarray(a)
    if form == "numpy":
        return a.copy()
    if form == "pinned":
        return torch.from_numpy(a.copy()).pin_memory().numpy()     # the array keeps its pinned tensor alive
    return torch.from_numpy(a.copy()).cuda()


def get(x):
    """An output as NumPy (a tensor must lie on device 0: outputs come back on the context's device)."""
    if hasattr(x, "is_cuda"):
        assert x.is_cuda and x.device.index == 0
        return x.cpu().numpy()
    assert isinstance(x, np.ndarray)
    return x.copy()


def strip(rep):
    """A report without what depends on the device's timing."""
    return {k: v for k, v in rep.items() if k not in TIMES}


def everywhere(R, fn):
    """fn(r, g) on every rank; per rank, its result or ("error", message)."""
    return R.each(lambda r, g: attempt(lambda: fn(r, g)))


def batch(nv, rowptr, edges, parts, seed=5):
    """Per rank: (delete, insert) of an update batch on the whole graph, both directions of every edge, src owned."""
    rng = np.random.default_rng(seed)
    src = np.repeat(np.arange(nv, dtype=np.int64), np.diff(rowptr))
    dst = edges["tail"].astype(np.int64)
    pick = rng.choice(len(src), min(200, len(src)), replace=False)
    ds, dd = np.concatenate([src[pick], dst[pick]]), np.concatenate([dst[pick], src[pick]])
    a, b = rng.integers(0, nv, 300), rng.integers(0, nv, 300)
    keep = a != b
    a, b = a[keep], b[keep]
    unit = bool(np.all(edges["weight"] == 1.0))
    w = np.ones(len(a)) if unit else rng.integers(1, 17, len(a)) / 8.0
    is_, id_, iw = np.concatenate([a, b]), np.concatenate([b, a]), np.concatenate([w, w])
    out = []
    for r in range(len(parts) - 1):
        md = (ds >= parts[r]) & (ds < parts[r + 1])
        mi = (is_ >= parts[r]) & (is_ < parts[r + 1])
        out.append(((ds[md], dd[md]), (is_[mi], id_[mi], iw[mi])))
    return out


def pipeline(R, form, upd):
    """run -> split -> evaluate -> compare -> probe -> movable set -> warm start -> update on every rank of R; every
    input of rank r named `what` is passed as form(r, what), every output requested as a tensor when that form is
    "torch".  Returns everything the pipeline saw, as NumPy, with the timing fields left out."""
    P, nv = R.parts, int(R.parts[-1])
    dev = lambda r, what: form(r, what) == "torch"                               # noqa: E731
    sl = lambda A, r: A[P[r]:P[r + 1]]                                          # noqa: E731
    cat = lambda xs: np.concatenate([get(x) for x in xs])                       # noqa: E731
    out = {}

    def run(key):
        res = R.each(lambda r, g: (g.louvain(), as_trace(g.trace()), g.communities(device=dev(r, key))))
        out[key] = (res[0][0], res[0][1])
        return cat([o[2] for o in res])

    X = out["X"] = run("run")
    s = R.each(lambda r, g: g.split_communities(put(sl(X, r), form(r, "split_in")), device=dev(r, "split_out")))
    Y = out["Y"] = cat([o[0] for o in s])
    out["split"] = [strip(o[1]) for o in s]
    s = R.each(lambda r, g: g.split_communities(None, device=dev(r, "split_null")))
    out["split_null"] = (cat([o[0] for o in s]), [strip(o[1]) for o in s])
    for key, A in (("eval", Y), ("eval_null", None)):
        q = R.each(lambda r, g: g.evaluate(None if A is None else put(sl(A, r), form(r, key))))
        st = R.each(lambda r, g: g.community_stats(device=dev(r, key + "_stats")))
        cc = R.each(lambda r, g: g.compact_communities(device=dev(r, key + "_compact")))
        out[key] = ([strip(o) for o in q], {k: cat([o[k] for o in st]) for k in st[0]}, cat(cc))
    for key, A in (("cmp", X), ("cmp_null", None)):
        c = R.each(lambda r, g: g.compare_communities(put(sl(Y, r), form(r, key + "_y")),
                                                      None if A is None else put(sl(A, r), form(r, key + "_x"))))
        m = R.each(lambda r, g: g.community_matches(device=dev(r, key + "_matches")))
        out[key] = ([strip(o) for o in c], {k: cat([o[k] for o in m]) for k in m[0]})
    for key, A in (("probe", Y), ("probe_null", None)):
        p = R.each(lambda r, g: g.probe(None if A is None else put(sl(A, r), form(r, key)), device=dev(r, key + "_out")))
        out[key] = ([strip(o[0]) for o in p], [cat([o[i] for o in p]) for i in (1, 2, 3)])
    mask = (np.arange(nv) % 5).astype(np.uint8) * 3                            # 0, 3, 6, 9, 12: normalised to 0 / 1
    R.each(lambda r, g: g.set_movable(put(sl(mask, r), form(r, "mask"))))
    out["movable_given"] = cat(R.each(lambda r, g: g.movable(device=dev(r, "movable_given"))))
    R.each(lambda r, g: g.set_initial_communities(put(sl(Y, r), form(r, "init"))))
    out["warm"] = run("warm")
    out["movable_after"] = cat(R.each(lambda r, g: g.movable(device=dev(r, "movable_after"))))
    R.each(lambda r, g: g.set_movable(None))
    R.each(lambda r, g: g.set_initial_communities(None))
    out["movable_none"] = cat(R.each(lambda r, g: g.movable(device=dev(r, "movable_none"))))

    def update(r, g):
        (ds, dd), (is_, id_, iw) = upd[r]
        lne = g.update_shard(delete=(put(ds, form(r, "del_src")), put(dd, form(r, "del_dst"))),
                             insert=(put(is_, form(r, "ins_src")), put(id_, form(r, "ins_dst")),
                                     put(iw, form(r, "ins_weight"))))
        return lne, g.download_shard()
    u = R.each(update)
    out["update"] = [(o[0], o[1][0], o[1][1].tobytes()) for o in u]
    out["after_update"] = run("after_update")
    return out


def all_host(r, what):
    return "numpy"


def one_form(f):
    return lambda r, what: f


def mixed(r, what):
    return FORMS[(r + sum(map(ord, what))) % 3]


def ranks(nv, rowptr, edges, parts, **opts):
    rps, eds = split_at(rowptr, edges, parts)
    return Ranks(np.asarray(parts, np.int64), rps, eds, **opts)


def compare_forms(nv, rowptr, edges, parts, forms, **opts):
    upd = batch(nv, rowptr, edges, parts)
    res = {}
    for name, form in [("host", all_host)] + forms:
        R = ranks(nv, rowptr, edges, parts, **opts)
        try:
            res[name] = pipeline(R, form, upd)
        finally:
            R.close()
    for name in res:
        assert_same(res[name], res["host"], name)
    return res["host"]


# ---- 1. equality of forms, one rank -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("reorder", [0, 1])
@pytest.mark.parametrize("name", GRAPHS)
def test_forms_give_the_host_bits(gpu, name, reorder):
    nv, rowptr, edges = whole(name)
    host = compare_forms(nv, rowptr, edges, [0, nv], [(f, one_form(f)) for f in FORMS[1:]] + [("mixed", mixed)],
                         reorder=reorder)
    assert host["run"][0][1] > 1
    assert np.array_equal(host["movable_given"], (np.arange(nv) % 5 != 0).astype(np.uint8))
    assert np.all(host["movable_none"] == 1)


# ---- 2. ranks sharing device 0, each rank and each pointer of its own kind ---------------------------------------------------
def parts_with_empty(nv, p):
    parts = [(nv * r) // p for r in range(p + 1)]
    if p > 2:
        parts[2] = parts[1]                                    # rank 1 holds no vertex
    return parts


@pytest.mark.parametrize("p", [2, 4, 16])
def test_mixed_kinds_on_ranks(gpu, p):
    nv, rowptr, edges = whole("rgg_n65536_p1" if p < 16 else "dyadic_random_n6000_d8_hubs3_hub_deg3000_multi200")
    compare_forms(nv, rowptr, edges, parts_with_empty(nv, p),
                  [("mixed", mixed), ("torch", one_form("torch")), ("mixed_shifted", lambda r, w: mixed(r + 1, w))])


def test_bad_id_fails_every_rank_with_the_host_message(gpu):
    nv, rowptr, edges = whole("rgg_n65536_p1")
    parts = parts_with_empty(nv, 4)
    R = ranks(nv, rowptr, edges, parts)
    try:
        first = R.run()
        before = R.each(lambda r, g: snapshot(g))
        base = np.arange(nv, dtype=np.int64)
        bad = base.copy()
        at = parts[2] + 9                                      # rank 2: local 9 and 5 are bad; 5 is named
        bad[at] = nv
        bad[parts[2] + 5] = -3
        sl = lambda A, r: A[parts[r]:parts[r + 1]]             # noqa: E731
        calls = {
            "evaluate": lambda r, g, a: g.evaluate(a),
            "split": lambda r, g, a: g.split_communities(a),
            "probe": lambda r, g, a: g.probe(a),
            "compare_x": lambda r, g, a: g.compare_communities(sl(base, r), a),
            "compare_y": lambda r, g, a: g.compare_communities(a, sl(base, r)),
        }
        for what, fn in calls.items():
            host = everywhere(R, lambda r, g: fn(r, g, sl(bad, r)))
            devf = everywhere(R, lambda r, g: fn(r, g, put(sl(bad, r), "torch" if r == 2 else FORMS[r % 2])))
            assert all(isinstance(h, tuple) and h[0] == "error" for h in host), (what, host)
            assert [h[1] for h in devf] == [h[1] for h in host], (what, devf, host)
            assert "community id -3 of local vertex 5 outside [0, nv)" in host[2][1], (what, host[2])
            assert all("another rank rejected" in h[1] for r, h in enumerate(host) if r != 2), (what, host)
        g = R.g[2]
        msgs = [attempt(lambda: g.set_initial_communities(put(sl(bad, 2), f))) for f in FORMS]
        assert msgs[0][0] == "error" and msgs[1:] == [msgs[0]] * 2, msgs
        assert "mvgpu_set_initial_communities: community id -3 of local vertex 5" in msgs[0][1]
        after = R.each(lambda r, g: snapshot(g))
        for r in range(4):
            assert_same(after[r], before[r], f"rank {r}")
        last = R.run()
        assert last["trace"] == first["trace"] and np.array_equal(last["comm"], first["comm"])
    finally:
        R.close()


# ---- 3. exact resume from device memory --------------------------------------------------------------------------------------
@pytest.mark.parametrize("movable", [False, True])
def test_resume_from_device_memory(gpu, movable):
    import torch
    nv, rowptr, edges = whole("rgg_n65536_p1")
    R = ranks(nv, rowptr, edges, [0, nv], frontier=1 if movable else 0)
    g = R.g[0]
    try:
        mask = torch.from_numpy((np.arange(nv) % 7 < 2).astype(np.uint8)).cuda()
        if movable:
            g.set_movable(mask)
        full = R.run()
        assert full["iters"] > 4
        k = full["iters"] // 2
        R.set_option("stop_after", k)
        if movable:
            g.set_movable(mask)
        a = R.run()
        assert a["trace"] == full["trace"][:k] and not a["converged"]
        comm = g.communities(device=True)
        mov = g.movable(device=True) if movable else None
        assert comm.is_cuda and comm.dtype == torch.int64 and comm.numel() == nv
        R.set_option("stop_after", 0)
        g.set_initial_communities(comm)
        if movable:
            assert mov.is_cuda and mov.dtype == torch.uint8
            g.set_movable(mov)
        b = R.run(lower=a["mod"])
        assert b["converged"] and b["trace"] == full["trace"][k:]
        assert repr(b["mod"]) == repr(full["mod"]) and np.array_equal(b["comm"], full["comm"])
    finally:
        R.close()


# ---- 4. copy at call time ----------------------------------------------------------------------------------------------------
def test_inputs_are_copied_at_call_time(gpu):
    import torch
    nv, rowptr, edges = whole("rgg_n65536_p1")
    R = ranks(nv, rowptr, edges, [0, nv])
    g = R.g[0]
    try:
        R.set_option("stop_after", 3)
        c3 = R.run()["comm"]
        R.set_option("stop_after", 0)
        mask = (np.arange(nv) % 3 != 0).astype(np.uint8)
        g.set_initial_communities(c3)
        g.set_movable(mask)
        want = R.run()
        t, m = torch.from_numpy(c3).cuda(), torch.from_numpy(mask).cuda()
        g.set_initial_communities(t)
        g.set_movable(m)
        t.fill_(0)                                             # overwritten ...
        m.zero_()
        torch.cuda.synchronize()
        assert_same(R.run(), want, "overwritten")
        t, m = torch.from_numpy(c3).cuda(), torch.from_numpy(mask).cuda()
        g.set_initial_communities(t)
        g.set_movable(m)
        del t, m                                               # ... and freed, its memory handed to a new tensor
        torch.cuda.empty_cache()
        junk = torch.full((4 * nv,), 7, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        assert_same(R.run(), want, "freed")
        del junk
    finally:
        R.close()


# ---- 5. refusals -------------------------------------------------------------------------------------------------------------
def test_wrong_length_tensor_is_refused_on_every_rank(gpu):
    import torch
    nv, rowptr, edges = whole("rgg_n65536_p1")
    parts = parts_with_empty(nv, 4)
    R = ranks(nv, rowptr, edges, parts)
    try:
        R.run()
        before = R.each(lambda r, g: snapshot(g))
        short = lambda r, g: torch.zeros(max(g.lnv - 1, 0) if r == 3 else g.lnv, dtype=torch.int64, device="cuda")  # noqa: E731
        for what, fn in (("evaluate", lambda r, g: g.evaluate(short(r, g))),
                         ("split", lambda r, g: g.split_communities(short(r, g), device=True)),
                         ("probe", lambda r, g: g.probe(short(r, g), device=True)),
                         ("compare", lambda r, g: g.compare_communities(short(r, g)))):
            got = everywhere(R, fn)
            assert all(isinstance(h, tuple) and h[0] == "error" for h in got), (what, got)
            assert "entries, the shard has lnv" in got[3][1], (what, got[3])
        with pytest.raises(ValueError):
            R.g[3].set_initial_communities(short(3, R.g[3]))
        with pytest.raises(ValueError):
            R.g[3].set_movable(short(3, R.g[3]).to(torch.uint8))
        after = R.each(lambda r, g: snapshot(g))
        for r in range(4):
            assert_same(after[r], before[r], f"rank {r}")
    finally:
        R.close()


def test_tensor_on_another_device_is_refused(gpu):
    import torch
    if gpu.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    nv, rowptr, edges = whole("rgg_n65536_p1")
    R = ranks(nv, rowptr, edges, split_global(nv, rowptr, edges, 2)[0])
    try:
        R.run()
        before = R.each(lambda r, g: snapshot(g))
        other = lambda r, g: torch.zeros(g.lnv, dtype=torch.int64, device="cuda:1" if r == 1 else "cuda:0")  # noqa: E731
        for what, fn in (("evaluate", lambda r, g: g.evaluate(other(r, g))),
                         ("compare", lambda r, g: g.compare_communities(other(r, g))),
                         ("update", lambda r, g: g.update_shard(insert=(other(r, g)[:4], other(r, g)[:4],
                                                                        other(r, g)[:4].double())))):
            got = everywhere(R, fn)
            assert all(isinstance(h, tuple) and h[0] == "error" for h in got), (what, got)
            assert "is memory of device 1, the context's device is 0" in got[1][1], (what, got[1])
        after = R.each(lambda r, g: snapshot(g))
        for r in range(2):
            assert_same(after[r], before[r], f"rank {r}")
    finally:
        R.close()


def test_pinned_and_pageable_host_arrays_take_the_host_form(gpu):
    import torch
    nv, rowptr, edges = whole("rgg_n65536_p1")
    R = ranks(nv, rowptr, edges, [0, nv])
    g = R.g[0]
    try:
        X = R.run()["comm"]
        pinned = put(X, "pinned")
        assert torch.from_numpy(pinned).is_pinned() and not torch.from_numpy(X).is_pinned()
        reps = [strip(g.evaluate(a)) for a in (X, pinned, put(X, "torch"))]
        assert reps[1] == reps[0] and reps[2] == reps[0]
        out = torch.empty(nv, dtype=torch.int64).pin_memory().numpy()
        assert np.array_equal(g.communities(out=out), X) and np.array_equal(g.communities(), X)
    finally:
        R.close()


# ---- 6. arrays larger than one bounce buffer ---------------------------------------------------------------------------------
def test_arrays_larger_than_one_bounce_buffer(gpu):
    """9 000 000 int64 ids are 72 MB: two full 32 MB chunks and a ragged tail through the pinned bounce buffers, both
    ways.  The split and the warm start give the device form's bits from every input form, into every output form."""
    from minivite_b200 import gpu as G
    nv = 9_000_000
    assert 2 * (4 << 20) < nv < 3 * (4 << 20)
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.generate_rgg(nv)
        g.louvain()
        pinned = put(np.zeros(nv, np.int64), "pinned")

        def communities():
            """The run's result, read into pageable, pinned and device memory: one array."""
            dev = get(g.communities(device=True))
            assert np.array_equal(g.communities(), dev) and np.array_equal(g.communities(out=pinned), dev)
            return dev

        X = communities()
        split = {(f, d): g.split_communities(put(X, f), device=d) for f in FORMS for d in (False, True)}
        Y, rep = get(split["torch", True][0]), strip(split["torch", True][1])
        for key, (y, r) in split.items():
            assert np.array_equal(get(y), Y) and strip(r) == rep, key
        g.set_option("stop_after", 1)
        warm = {}
        for f in FORMS:
            g.set_initial_communities(put(Y, f))
            warm[f] = (g.louvain(), communities())
        for f in FORMS:
            assert warm[f][0] == warm["torch"][0] and np.array_equal(warm[f][1], warm["torch"][1]), f
    finally:
        g.close()


# ---- one process per rank (CUDA IPC between processes), device inputs and outputs -----------------------------------------
def _ipc_worker(rank, world, port, out_dir):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    from minivite_b200 import dist as D
    from minivite_b200 import gpu as G
    D_ = D.Ranks("gloo")
    nv, rowptr, edges = whole("rgg_n65536_p1")
    parts, rps, eds = split_global(nv, rowptr, edges, world)
    ident = D_.broadcast_bytes(G.get_unique_id() if rank == 0 else None, G.UNIQUE_ID_BYTES)
    g = G.LouvainGPU(0, rank, world)
    g.set_option("host_transport", 1)
    g.comm_init(ident)
    g.upload(nv, parts, rps[rank], eds[rank])
    mod, iters = g.louvain()
    X = g.communities(device=True)
    Y, srep = g.split_communities(X, device=True)
    q = g.evaluate(Y)
    c = g.compare_communities(Y, X)
    prep, target, best, gain = g.probe(Y, device=True)
    res = {"run": [mod, iters], "X": X.cpu().tolist(), "Y": Y.cpu().tolist(), "split": strip(srep), "eval": strip(q),
           "cmp": strip(c), "probe": strip(prep), "target": target.cpu().tolist(), "best": best.cpu().tolist(),
           "gain": gain.cpu().numpy().view(np.int64).tolist()}
    torch.cuda.synchronize()
    json.dump(res, open(os.path.join(out_dir, f"rank{rank}.json"), "w"))
    g.close()
    D_.shutdown()


def test_processes_with_device_inputs(gpu, tmp_path):
    import torch.multiprocessing as mp
    nv, rowptr, edges = whole("rgg_n65536_p1")
    parts, rps, eds = split_global(nv, rowptr, edges, 2)
    R = Ranks(parts, rps, eds)
    try:
        mod, iters = R.each(lambda r, g: g.louvain())[0]
        X = np.concatenate(R.each(lambda r, g: g.communities().copy()))
        s = R.each(lambda r, g: g.split_communities(X[parts[r]:parts[r + 1]]))
        Y = np.concatenate([o[0] for o in s])
        sl = lambda A, r: A[parts[r]:parts[r + 1]]             # noqa: E731
        q = R.each(lambda r, g: g.evaluate(sl(Y, r)))[0]
        c = R.each(lambda r, g: g.compare_communities(sl(Y, r), sl(X, r)))[0]
        p = R.each(lambda r, g: g.probe(sl(Y, r)))
    finally:
        R.close()
    sk = socket.socket()
    sk.bind(("127.0.0.1", 0))
    port = sk.getsockname()[1]
    sk.close()
    mp.spawn(_ipc_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    got = [json.load(open(tmp_path / f"rank{r}.json")) for r in range(2)]
    for r, o in enumerate(got):
        assert o["run"] == [mod, iters]
        assert o["X"] == sl(X, r).tolist() and o["Y"] == sl(Y, r).tolist()
        assert o["split"] == strip(s[r][1]) and o["eval"] == strip(q) and o["cmp"] == strip(c)
        assert o["probe"] == strip(p[r][0])
        assert o["target"] == p[r][1].tolist() and o["best"] == p[r][2].tolist()
        assert o["gain"] == p[r][3].view(np.int64).tolist()
