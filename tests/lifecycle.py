"""Long-lived contexts, TEST INFRASTRUCTURE: a catalogue of shard kinds, scripted and seeded sequences of operations on one
context, what a context shows of itself (`snapshot`) and a runner that drives the same sequence on one long-lived context
and on fresh ones.

A sequence is a list of steps; each step is a tuple whose first entry names the operation:
  ("load", spec)            replace the shard: spec["via"] is upload, upload32, attach or generate (`shard`)
  ("update", seed)          mvgpu_update_shard with a batch drawn from the current graph (update_ref restates it)
  ("opt", name, value)      mvgpu_set_option
  ("init", seed | None)     mvgpu_set_initial_communities with `assignment(seed)`, or clear it
  ("mov", seed | None)      mvgpu_set_movable with `mask(seed)`, or clear it
  ("run",)                  mvgpu_louvain (mvgpu_louvain32 on a 32-bit shard)
  ("eval", seed | None)     mvgpu_evaluate_communities of `assignment(seed)` or of the last run (None)
  ("split", seed | None)    mvgpu_split_communities, likewise
  ("compare", seed)         mvgpu_compare_communities of the last run against `assignment(seed)`
Every input is a function of the step and the current graph, so a fresh context can be given the same ones, and the
CPU tests in test_lifecycle_scripts.py can work out from the scripts alone which boundaries the sequences cross.
"""
import itertools

import numpy as np

import layout_ref
import update_ref
from helpers import dyadic_rgg, random_graph, rmat_graph, split_global
from minivite_b200 import hostgraph as hg

# ---- shard kinds (all <= 65 536 vertices) ----------------------------------------------------------------------------
KINDS = ["rgg", "dyadic", "rmat", "multi", "u32", "gen", "gen_p", "attach", "updated"]
UNIT_KINDS = {"rgg", "rmat", "multi", "u32", "gen", "gen_p", "attach"}       # "updated" follows its base
_cache = {}


def _rgg_global(n, pct=0.0, world=1):
    ss = hg.generate_rgg(n, world, random_edge_percent=pct)
    rowptr = np.concatenate([[0]] + [s.rowptr[1:] + off for s, off in
                                     zip(ss.shards, np.cumsum([0] + [s.lne for s in ss.shards[:-1]]))]).astype(np.int64)
    edges = np.concatenate([s.edges for s in ss.shards]).copy()
    ss.close()
    return n, rowptr, edges


def global_graph(kind, n, seed=1):
    """(nv, rowptr, edges) of a kind's whole graph; generated kinds are what the device generator builds on `world` strips
    (the host generator builds the same bytes), and they depend on the strip count, so they are keyed by it."""
    key = (kind, n, seed)
    if key not in _cache:
        if kind in ("rgg", "u32", "attach", "updated"):
            g = _rgg_global(n)
        elif kind == "dyadic":
            g = dyadic_rgg(n, 1)
        elif kind == "rmat":
            g = rmat_graph(14, 8, seed)
        elif kind == "multi":
            rp, ed = random_graph(n, 8, seed, hubs=2, hub_deg=n // 8, self_loops=n // 64, multi=n // 16)
            g = (n, rp, ed)
        else:
            raise ValueError(kind)
        _cache[key] = g
    return _cache[key]


def spec(kind, n, world=1, parts=None, seed=1, batch_seed=7):
    """A shard description: kind, how it reaches the device, the partition and the per-rank host arrays.  parts: None
    = the reference's even split; a list gives uneven or empty ranks."""
    if kind in ("gen", "gen_p"):
        pct = 1.0 if kind == "gen_p" else 0.0
        ss = hg.generate_rgg(n, world, random_edge_percent=pct)
        rps = [s.rowptr.copy() for s in ss.shards]
        eds = [s.edges.copy() for s in ss.shards]
        p = ss.shards[0].parts.copy()
        ss.close()
        return {"kind": kind, "via": "generate", "nv": n, "pct": pct, "parts": p, "rowptrs": rps, "edges": eds,
                "weighted": False}
    if kind == "rmat":
        n = 1 << 14
    nv, rowptr, edges = global_graph(kind, n, seed)
    if parts is None:
        p, rps, eds = split_global(nv, rowptr, edges, world)
    else:
        p = np.asarray(partition(parts, nv, world), np.int64)
        rps = [np.ascontiguousarray(rowptr[a:b + 1] - rowptr[a]) for a, b in zip(p[:-1], p[1:])]
        eds = [np.ascontiguousarray(edges[rowptr[a]:rowptr[b]]) for a, b in zip(p[:-1], p[1:])]
    via = {"u32": "upload32", "attach": "attach"}.get(kind, "upload")
    s = {"kind": kind, "via": via, "nv": nv, "parts": p, "rowptrs": rps, "edges": eds, "weighted": kind == "dyadic"}
    if kind == "updated":
        s = dict(s, kind="rgg")
        return {"kind": "updated", "base": s, "batch_seed": batch_seed}
    return s


def partition(mode, nv, world):
    """"skew": rank 0 holds 3/4 (2 ranks) or 1/2 of the vertices, the rest split evenly; "empty": rank 1 holds none."""
    if mode == "skew":
        first = 3 * nv // 4 if world == 2 else nv // 2
    else:
        first = nv if world == 2 else nv // 2
    rest = [first + (nv - first) * r // (world - 1) for r in range(1, world)]
    if mode == "empty":
        rest = [first] + [first + (nv - first) * r // (world - 2) for r in range(1, world - 1)] if world > 2 else [nv]
    return [0, first] + rest


def batch(cur, seed):
    """An update batch for the current shard `cur` (per rank: delete, insert), both directions of every edge given to their
    owners: deletes k existing undirected edges and inserts k new ones (weight 1, or 1/2 on a weighted graph)."""
    rng = np.random.default_rng(seed)
    parts = cur["parts"]
    world = len(parts) - 1
    nv = int(parts[-1])
    src = np.concatenate([np.repeat(np.arange(parts[r], parts[r + 1]), np.diff(cur["rowptrs"][r])) for r in range(world)])
    dst = np.concatenate([e["tail"] for e in cur["edges"]])
    fwd = np.nonzero(src < dst)[0]
    k = min(24, len(fwd))
    pick = rng.choice(fwd, k, replace=False) if k else fwd[:0]
    du, dv = src[pick], dst[pick]
    iu, iv = rng.integers(0, nv, k), rng.integers(0, nv, k)
    keep = iu != iv
    iu, iv = iu[keep], iv[keep]
    w = 0.5 if cur["weighted"] else 1.0
    ds, dd = np.concatenate([du, dv]), np.concatenate([dv, du])
    is_, id_ = np.concatenate([iu, iv]), np.concatenate([iv, iu])
    out = []
    for r in range(world):
        a, b = parts[r], parts[r + 1]
        md, mi = (ds >= a) & (ds < b), (is_ >= a) & (is_ < b)
        out.append(((ds[md], dd[md]), (is_[mi], id_[mi], np.full(int(mi.sum()), w))))
    return out


def apply_update(cur, seed):
    """The shard after `batch(cur, seed)` (update_ref's restatement of mvgpu_update_shard)."""
    b = batch(cur, seed)
    rps, eds = [], []
    for r, (dl, ins) in enumerate(b):
        rp, ed = update_ref.apply(int(cur["parts"][r]), cur["rowptrs"][r], cur["edges"][r], dl, ins)
        rps.append(rp)
        eds.append(ed)
    return dict(cur, kind="updated", rowptrs=rps, edges=eds)


def assignment(cur, seed):
    """A valid assignment of the current graph (per rank): vertices in blocks of 2..9 of scattered members."""
    nv = int(cur["parts"][-1])
    rng = np.random.default_rng(seed)
    X = (rng.permutation(nv) // int(rng.integers(2, 10))) % max(nv, 1)
    return [X[cur["parts"][r]:cur["parts"][r + 1]].astype(np.int64) for r in range(len(cur["parts"]) - 1)]


def mask(cur, seed):
    rng = np.random.default_rng(seed)
    return [(rng.random(int(cur["parts"][r + 1] - cur["parts"][r])) < 0.4).astype(np.uint8)
            for r in range(len(cur["parts"]) - 1)]


def resolve(s):
    """The shard a ("load", s) step leaves: an "updated" kind is its base after one update."""
    return apply_update(s["base"], s["batch_seed"]) if s["kind"] == "updated" else s


# ---- scripted sequences ---------------------------------------------------------------------------------------------
SIZES = {"rgg": 8192, "dyadic": 8192, "rmat": 16384, "multi": 4096, "u32": 4096, "gen": 16384, "gen_p": 8192,
         "attach": 2048, "updated": 4096}


def pair_order(kinds):
    """A sequence of kinds in which every ordered pair (a, b), a == b included, occurs as consecutive entries (an
    Eulerian circuit of the complete digraph with loops, found greedily)."""
    unused = {a: list(kinds) for a in kinds}
    stack, out = [kinds[0]], []
    while stack:
        v = stack[-1]
        if unused[v]:
            stack.append(unused[v].pop(0))
        else:
            out.append(stack.pop())
    return out[::-1]


def pair_script():
    """1 rank: every ordered pair of shard kinds as consecutive shards, each run once; sizes alternate so that shards
    also shrink below and grow past what the context allocated before."""
    steps = [("opt", "trace", 1), ("opt", "scan_variant", 4)]
    for i, k in enumerate(pair_order(KINDS)):
        n = SIZES[k] * (2 if i % 3 == 2 and k not in ("rmat",) and SIZES[k] <= 16384 else 1)
        steps += [("load", spec(k, n))]
        steps += [("run",)]
    return steps


def scripted_1rank():
    """Option changes, warm starts, movable sets, checkpoints and the assignment calls around shard changes."""
    r = lambda k, n, **kw: ("load", spec(k, n, **kw))       # noqa: E731
    return [("opt", "trace", 1), ("opt", "scan_variant", 5),
            r("rgg", 16384), ("run",), ("eval", None), ("compare", 3),
            ("opt", "reorder", 1), ("run",), ("split", None),
            r("dyadic", 8192), ("init", 4), ("run",), ("opt", "reorder", 0), ("opt", "force_weighted", 1),
            r("rgg", 4096), ("run",), ("opt", "force_weighted", 0), ("mov", 5), ("opt", "frontier", 1), ("run",),
            ("update", 6), ("run",), ("eval", 8),
            r("gen", 65536), ("opt", "stop_after", 2), ("run",), ("opt", "stop_after", 0), ("init", 9), ("run",),
            r("gen_p", 16384), ("opt", "scan_variant", 6), ("run",), ("split", 10), ("compare", 11),
            r("rmat", 16384), ("opt", "scan_variant", 4), ("opt", "reorder", 2), ("run",), ("mov", None),
            r("attach", 8192), ("opt", "frontier", 0), ("run",), ("update", 12), ("run",),
            r("u32", 4096), ("run",), r("multi", 4096), ("run",), ("eval", None)]


WALK_SEEDS = (2, 3, 4)                  # seeds whose 30 steps use every operation (test_lifecycle_scripts.py)
WALK_OPS = ["load", "load", "run", "run", "opt", "init", "mov", "eval", "split", "compare", "update"]
WALK_OPTS = [("reorder", (0, 1, 2)), ("scan_variant", (4, 5, 6)), ("force_weighted", (0, 1)), ("stop_after", (0, 0, 2)),
             ("frontier", (0, 1))]


def walk(seed, steps=30, world=1, kinds=None, sizes=(2048, 4096, 8192, 16384)):
    """A seeded random sequence of about `steps` valid steps (32-bit shards get no warm start, movable set or stop_after:
    louvain32 refuses them; those refusals are covered elsewhere)."""
    rng = np.random.default_rng(seed)
    kinds = kinds or [k for k in KINDS if world == 1 or k != "u32"]
    out = [("opt", "trace", 1), ("load", spec("rgg", 4096, world))]
    cur = out[-1][1]
    opts = {"stop_after": 0}
    have = {"init": False, "mov": False}
    while len(out) < steps:
        op = WALK_OPS[int(rng.integers(len(WALK_OPS)))]
        u32 = cur["via"] == "upload32" if "via" in cur else False
        if op == "load":
            k = kinds[int(rng.integers(len(kinds)))]
            n = int(sizes[int(rng.integers(len(sizes)))])
            if k == "u32" and opts["stop_after"]:
                continue
            cur = spec(k, n, world)
            out.append(("load", cur))
            have = {"init": False, "mov": False}
            if k == "u32":
                out.append(("run",))
        elif op == "run":
            if u32 and (opts["stop_after"] or have["init"] or have["mov"]):
                continue
            out.append(("run",))
        elif op == "opt":
            name, vals = WALK_OPTS[int(rng.integers(len(WALK_OPTS)))]
            v = int(vals[int(rng.integers(len(vals)))])
            if name == "stop_after" and u32 and v:
                continue
            opts[name] = v
            out.append(("opt", name, v))
        elif op in ("init", "mov"):
            if u32:
                continue
            s = None if rng.random() < 0.3 else int(rng.integers(1 << 20))
            have[op] = s is not None
            out.append((op, s))
        elif op in ("eval", "split"):
            if u32:
                continue
            out.append((op, None if rng.random() < 0.5 else int(rng.integers(1 << 20))))
        elif op == "compare":
            if u32:
                continue
            out.append(("compare", int(rng.integers(1 << 20))))
        elif op == "update":
            if u32:
                continue
            out.append(("update", int(rng.integers(1 << 20))))
    return out


def multirank_script(world):
    """2 or 4 ranks as threads: unit <-> weighted, renumbering <-> not, evaluation / split / frontier arrays on and off, one
    rank whose arrays must grow while the others' do not, a rank that goes empty and comes back."""
    n = 16384
    r = lambda k, m=n, **kw: ("load", spec(k, m, world, **kw))     # noqa: E731
    return [("opt", "trace", 1), ("opt", "scan_variant", 4),
            r("rgg"), ("run",), ("eval", None),
            r("dyadic", 8192), ("opt", "reorder", 1), ("run",), ("split", None),
            r("rgg", parts="skew"), ("opt", "reorder", 0), ("run",), ("compare", 2),
            ("mov", 3), ("opt", "frontier", 1), ("run",), ("update", 4), ("run",),
            r("rgg", parts="empty"), ("run",),
            r("gen_p", 8192), ("opt", "reorder", 1), ("run",), ("opt", "frontier", 0), ("split", 5),
            r("dyadic", 8192, parts="empty"), ("opt", "reorder", 0), ("init", 6), ("run",), ("eval", 7),
            r("attach", 4096), ("run",), r("gen", 16384), ("opt", "reorder", 2), ("run",), ("eval", None)]


# ---- what the scripts imply, without a GPU (test_lifecycle_scripts.py) ------------------------------------------------
def shard_states(steps):
    """(step index, op, the current shard after the step, options in effect, movable set present) per step."""
    cur, opts, mov, out = None, {"reorder": 2, "force_weighted": 0, "frontier": 0}, False, []
    for i, st in enumerate(steps):
        if st[0] == "load":
            cur, mov = resolve(st[1]), False
        elif st[0] == "update":
            cur = apply_update(cur, st[1])
        elif st[0] == "opt":
            opts = dict(opts, **{st[1]: st[2]})
        elif st[0] == "mov":
            mov = st[1] is not None
        out.append((i, st, cur, dict(opts), mov))
    return out


def exported(cur, opts, mov, op):
    """The peer-exported arrays (MV_EXPORTS in mvgpu.cu) a setup (run, eval or split) needs."""
    ev = op in ("eval", "split")
    unit = not cur["weighted"] and not opts["force_weighted"]
    relabel = False
    if not ev:
        for rk in range(len(cur["parts"]) - 1):
            relabel |= layout_ref.rank_want(cur["parts"], cur["rowptrs"][rk], cur["edges"][rk]["tail"], rk, opts["reorder"])[0]
    s = {"comm_a", "comm_b", "p2p"}
    s |= {"cdeg", "csize", "upd"} if unit else {"cinfo_w", "usize", "udeg"}
    if relabel:
        s |= {"lab", "inv"}
    if ev:
        s |= {"q_internal", "q_rank"}
    if op == "split":
        s.add("split_lab")
    if not ev and mov and opts["frontier"]:
        s |= {"mov_a", "mov_b"}
    return s


def needs(cur, rank):
    """need_v, need_s of setup_agree: lnv, and lnv + the non-owned edge tails (layout_ref.compact_csr)."""
    lnv = int(cur["parts"][rank + 1] - cur["parts"][rank])
    _rp, slots, _nlow, _g = layout_ref.compact_csr(cur["parts"], cur["rowptrs"][rank], cur["edges"][rank]["tail"], rank)
    return lnv, lnv + int((slots >= lnv).sum())


def expect_refused(steps):
    """Per step: True if the library refuses it by contract -- an eval / split of the last run (None) or a compare
    when no run happened on the shard since its last upload, attach, generate or update."""
    out, ran = [], False
    for st in steps:
        if st[0] in ("load", "update"):
            ran = False
        out.append(st[0] in ("eval", "split", "compare") and (st[1] is None or st[0] == "compare") and not ran)
        ran |= st[0] == "run"
    return out


def all_pairs(kinds):
    return set(itertools.product(kinds, kinds))
