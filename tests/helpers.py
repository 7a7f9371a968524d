"""Shared helpers for the parity tests (test infrastructure)."""
import numpy as np

from minivite_b200 import hostgraph as hg


def case_graph(case):
    """Shards (parts, rowptrs, edge arrays) for a golden case, rebuilt with OUR generator / from the stored graph."""
    kind = case["kind"]
    p = case["nranks"]
    if kind == "rgg":
        args = case["args"]
        ss = hg.generate_rgg(case["n"], p, lcg="-l" in args, unit_weight="-w" not in args)
        return ss.shards[0].parts, [s.rowptr for s in ss.shards], [s.edges for s in ss.shards], ss
    if kind == "file_rgg":
        ss = hg.generate_rgg(case["n"], case["strips"], unit_weight=case["unit_weight"])
        nv = case["n"]
        rowptr = np.concatenate([[0]] + [s.rowptr[1:] + off for s, off in
                                         zip(ss.shards, np.cumsum([0] + [s.lne for s in ss.shards[:-1]]))])
        edges = np.concatenate([s.edges for s in ss.shards])
        return split_global(nv, rowptr.astype(np.int64), edges, p) + (ss,)
    if kind == "file_balanced":
        ss = hg.generate_rgg(case["n"], 1, random_edge_percent=case["pct"])
        sh = ss.shards[0]
        parts = np.array(case["parts"], dtype=np.int64)
        rps, eds = [], []
        for r in range(p):
            a, b = parts[r], parts[r + 1]
            rps.append(np.ascontiguousarray(sh.rowptr[a:b + 1] - sh.rowptr[a]))
            eds.append(np.ascontiguousarray(sh.edges[sh.rowptr[a]:sh.rowptr[b]]))
        return parts, rps, eds, ss
    if kind == "rmat":
        n, rowptr, edges = rmat_graph(case["scale"], case["edge_factor"], case["seed"])
        if case.get("balanced"):
            parts = np.array(case["parts"], dtype=np.int64)     # the reference's own -b bins (graph.hpp:466-572)
            rps = [np.ascontiguousarray(rowptr[a:b + 1] - rowptr[a]) for a, b in zip(parts[:-1], parts[1:])]
            eds = [np.ascontiguousarray(edges[rowptr[a]:rowptr[b]]) for a, b in zip(parts[:-1], parts[1:])]
            return parts, rps, eds, None
        return split_global(n, rowptr, edges, p) + (None,)
    if kind == "hand":
        g = case["graph"]
        edges = np.zeros(len(g["tails"]), hg.EDGE_DTYPE)
        edges["tail"] = g["tails"]
        edges["weight"] = g["weights"]
        return split_global(g["nv"], np.array(g["rowptr"], np.int64), edges, p) + (None,)
    if kind in ("dyadic_rgg", "dyadic_random", "dyadic_rmat"):
        nv, rowptr, edges = dyadic_graph(case)
        return split_global(nv, rowptr, edges, p) + (None,)
    raise ValueError(kind)


def global_csr(case):
    """(nv, rowptr, edges) of a hand-made or dyadic case's whole graph (their graphs do not depend on the rank count)."""
    if case["kind"] == "hand":
        parts, rps, eds, _keep = case_graph(dict(case, nranks=1))
        return int(parts[-1]), rps[0], eds[0]
    return dyadic_graph(case)


# ---- graphs with dyadic weights (k * 2^-j): every fp64 sum of them is exact, so its value does not depend on the order
# ---- of the additions, and the weighted path must reproduce the reference bit for bit (tests/golden/make_golden_weighted.py)

def weighted_exact_cases():
    """name -> case of tests/golden/weighted_exact_traces.json (traces of the unmodified reference, 1 rank, 1 thread)."""
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weighted_exact_traces.json")) as f:
        return json.load(f)["cases"]


def golden_cases():
    """name -> case of every reference trace in ref_traces.json, rmat_traces.json and (prefixed "dyadic_")
    weighted_exact_traces.json."""
    import json
    import os
    out = {}
    for fn in ("ref_traces.json", "rmat_traces.json"):
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", fn)) as f:
            out.update(json.load(f)["cases"])
    for name, c in weighted_exact_cases().items():
        out["dyadic_" + name] = c
    return out


def exact_cases():
    """golden_cases() whose Comm sums are exact: unit weights (hand graphs: unit or k/4 weights), or dyadic weights."""
    return {name: c for name, c in golden_cases().items()
            if not ("-w" in c.get("args", []) or c.get("unit_weight") is False)}


def dyadic_graph(case):
    """Global CSR (nv, rowptr, edges) of a dyadic-weight recipe from tests/golden/weighted_exact_traces.json."""
    kind = case["kind"]
    if kind == "dyadic_rgg":
        return dyadic_rgg(case["n"], case["strips"], case.get("pct", 0.0), case.get("levels", 16), case.get("denom", 16))
    if kind == "dyadic_random":
        rowptr, edges = random_graph(case["n"], case["avg_deg"], case["seed"], dyadic=True, **case.get("kw", {}))
        return case["n"], rowptr, edges
    if kind == "dyadic_rmat":
        return rmat_graph(case["scale"], case["edge_factor"], case["seed"], dyadic=True)
    raise ValueError(kind)


def dyadic_rgg(n, strips, pct=0.0, levels=16, denom=16):
    """`miniVite -n n -w [-p pct]` built on `strips` ranks, each Euclidean weight w replaced by ceil(levels w / rn) / denom
    (rn = the RGG radius; by default 16 distinct weights from 1/16 to 1).  Quantizing on an absolute scale instead would map every
    RGG edge (w <= rn, about 0.01) to one value and leave a uniformly scaled unit graph.  The random long edges of -p
    (w > rn, up to about 1.4) are quantized on their own scale and shifted past the RGG edges' range, 1 + ceil(16 w) / 16,
    so they stay distinct from them."""
    ss = hg.generate_rgg(n, strips, unit_weight=False, random_edge_percent=pct)
    rn = hg.rgg_radius(n, strips)
    nv = ss.shards[0].nv
    rowptr = np.concatenate([[0]] + [s.rowptr[1:] + off for s, off in
                                     zip(ss.shards, np.cumsum([0] + [s.lne for s in ss.shards[:-1]]))]).astype(np.int64)
    edges = np.concatenate([s.edges for s in ss.shards])
    w = edges["weight"]
    edges["weight"] = np.where(w <= rn, np.ceil(levels * w / rn) / denom, 1.0 + np.ceil(16.0 * w) / 16.0)
    ss.close()
    return nv, rowptr, edges


def dyadic_exponent(weights, max_j=6):
    """Smallest j <= max_j with every weight an integer multiple of 2^-j, or None."""
    w = np.asarray(weights, np.float64)
    for j in range(max_j + 1):
        s = w * float(1 << j)
        if np.all(s == np.floor(s)):
            return j
    return None


def assert_dyadic_exact(nv, rowptr, edges, max_j=6):
    """Exactness precondition of the weighted bit-exact goldens: every weight is k * 2^-j (k >= 0 integer, j <= max_j);
    2m * 2^j < 2^53, so every degree, community degree and intra-community sum is an exact fp64 number whatever the order
    of the additions; (2m * 2^j)^2 < 2^53 bounds the sum over communities of the squared community degrees the same way;
    the graph is symmetric with equal weights in both directions (multi-edges compared as multisets)."""
    rowptr = np.asarray(rowptr, np.int64)
    w = np.asarray(edges["weight"], np.float64)
    assert len(w) == rowptr[-1] and np.all(w >= 0)
    j = dyadic_exponent(w, max_j)
    assert j is not None, "weights are not multiples of 2^-%d" % max_j
    two_m = float(np.sum(w))
    units = two_m * float(1 << j)
    assert units < 2.0 ** 53 and units * units < 2.0 ** 53, (two_m, j)
    src = np.repeat(np.arange(nv, dtype=np.int64), np.diff(rowptr))
    dst = np.asarray(edges["tail"], np.int64)
    assert np.all((dst >= 0) & (dst < nv))
    fwd = np.lexsort((w, dst, src))
    rev = np.lexsort((w, src, dst))
    assert np.array_equal(src[fwd], dst[rev]) and np.array_equal(dst[fwd], src[rev]) and np.array_equal(w[fwd], w[rev]), \
        "graph is not symmetric with equal weights"
    return j


def assert_non_degenerate(case, unit_result, min_distinct=4):
    """The weights matter: at least `min_distinct` distinct weight values, and the trace differs from the trace of the same
    graph with every weight set to 1 (`unit_result`: an oracle or reference run of that graph)."""
    _nv, _rowptr, edges = global_csr(case)
    assert len(np.unique(edges["weight"])) >= min_distinct, np.unique(edges["weight"])
    unit = ([(float(t["modularity"]), int(t["moved"]), int(t["chash"])) for t in unit_result["trace"]],
            float(unit_result["modularity"]))
    mine = ([(float(t["modularity"]), int(t["moved"]), int(t["chash"], 16)) for t in case["trace"]],
            float(case["modularity"]))
    assert mine != unit, "trace equals the unit-weight trace"


def random_graph(n, avg_deg, seed, hubs=0, hub_deg=0, self_loops=0, multi=0, blocks=0, dyadic=False):
    """Symmetric random multigraph in the reference's CSR format, adjacency sorted by tail (unit weights unless dyadic).
    blocks > 0: planted partition (90 % of the edges inside `blocks` equal groups of scattered vertex ids).
    dyadic: weight k/8, k in 1..16, drawn per undirected edge before symmetrizing (a second stream, so the graph itself
    is the unit-weight one), so parallel edges between one pair get their own weights and both directions agree."""
    rng = np.random.default_rng(seed)
    m = n * avg_deg // 2
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    if blocks:
        inside = rng.random(m) < 0.9
        b = np.where(inside, (b // blocks) * blocks + a % blocks, b) % n      # same residue class = same block
    keep = a != b
    a, b = a[keep], b[keep]
    for h in range(hubs):
        t = rng.choice(n, hub_deg, replace=False)
        t = t[t != h]
        a, b = np.concatenate([a, np.full(len(t), h)]), np.concatenate([b, t])
    key = np.unique(np.minimum(a, b) * n + np.maximum(a, b))          # simple graph first
    a, b = key // n, key % n
    if multi:
        pick = rng.integers(0, len(a), multi)
        a, b = np.concatenate([a, a[pick]]), np.concatenate([b, b[pick]])
    wrng = np.random.default_rng([seed, 8])
    w = wrng.integers(1, 17, len(a)) / 8.0 if dyadic else np.ones(len(a))
    src, dst, w = np.concatenate([a, b]), np.concatenate([b, a]), np.concatenate([w, w])
    if self_loops:
        s = rng.integers(0, n, self_loops)
        src, dst = np.concatenate([src, s]), np.concatenate([dst, s])
        w = np.concatenate([w, wrng.integers(1, 17, self_loops) / 8.0 if dyadic else np.ones(self_loops)])
    order = np.lexsort((w, dst, src)) if dyadic else np.lexsort((dst, src))
    src, dst, w = src[order], dst[order], w[order]
    rowptr = np.zeros(n + 1, np.int64)
    np.add.at(rowptr, src + 1, 1)
    rowptr = np.cumsum(rowptr)
    edges = np.zeros(len(dst), hg.EDGE_DTYPE)
    edges["tail"] = dst
    edges["weight"] = w
    return rowptr, edges


def split_global(nv, rowptr, edges, p):
    """Vertex-range split parts[r] = nv*r/p of a global CSR (reference graph.hpp:112-113 / 344-355)."""
    parts = np.array([(nv * r) // p for r in range(p + 1)], dtype=np.int64)
    rps, eds = [], []
    for r in range(p):
        a, b = parts[r], parts[r + 1]
        rp = rowptr[a:b + 1] - rowptr[a]
        rps.append(np.ascontiguousarray(rp))
        eds.append(np.ascontiguousarray(edges[rowptr[a]:rowptr[b]]))
    return parts, rps, eds


def assert_trace_matches(case, iters, modularity, trace, final_chash=None, comm=None, exact=True, tol=1e-6):
    """Compare a run (C oracle or CUDA path) with a golden reference record."""
    assert iters == case["iters"], (iters, case["iters"])
    gm = float(case["modularity"])
    if exact:
        assert modularity == gm, (repr(modularity), case["modularity"])
    else:
        assert abs(modularity - gm) <= tol
    assert len(trace) == len(case["trace"])
    for k, (t, g) in enumerate(zip(trace, case["trace"])):
        tm = float(t["modularity"])
        if exact:
            assert tm == float(g["modularity"]), (k, repr(tm), g["modularity"])
            assert int(t["moved"]) == g["moved"], (k, int(t["moved"]), g["moved"])
            assert int(t["chash"]) == int(g["chash"], 16), (k, hex(int(t["chash"])), g["chash"])
        else:
            assert abs(tm - float(g["modularity"])) <= tol
    if final_chash is not None and exact:
        assert final_chash == int(case["final_chash"], 16)
    if comm is not None and "comm" in case and exact:
        assert [int(x) for x in comm] == case["comm"]


def rmat_graph(scale, edge_factor, seed, a=0.57, b=0.19, c=0.19, dyadic=False):
    """Power-law (R-MAT) graph in the reference's CSR format: symmetric, unit weights, no self loops, no parallel
    edges, adjacency sorted by tail.  numpy's legacy RandomState keeps the stream stable across versions, so the graph
    is a function of (scale, edge_factor, seed) and only its golden TRACE needs committing.  dyadic: each undirected
    edge gets weight k/8, k in 1..16, drawn after the graph (the same graph as the unit-weight one)."""
    rng = np.random.RandomState(seed)
    n, m = 1 << scale, edge_factor << scale
    src = np.zeros(m, np.int64)
    dst = np.zeros(m, np.int64)
    for level in range(scale):
        r = rng.random_sample(m)
        right = (r >= a) & (r < a + b) | (r >= a + b + c)          # quadrants b and d set the column bit
        down = r >= a + b                                          # quadrants c and d set the row bit
        src |= down.astype(np.int64) << level
        dst |= right.astype(np.int64) << level
    perm = rng.permutation(n)                                      # scatter the hubs over the id range
    src, dst = perm[src], perm[dst]
    keep = src != dst
    lo, hi = np.minimum(src[keep], dst[keep]), np.maximum(src[keep], dst[keep])
    key = np.unique(lo * n + hi)
    lo, hi = key // n, key % n
    w = rng.randint(1, 17, len(lo)) / 8.0 if dyadic else np.ones(len(lo))
    s2, d2, w2 = np.concatenate([lo, hi]), np.concatenate([hi, lo]), np.concatenate([w, w])
    order = np.lexsort((d2, s2))
    s2, d2, w2 = s2[order], d2[order], w2[order]
    rowptr = np.zeros(n + 1, np.int64)
    np.add.at(rowptr, s2 + 1, 1)
    rowptr = np.cumsum(rowptr)
    edges = np.zeros(len(d2), hg.EDGE_DTYPE)
    edges["tail"] = d2
    edges["weight"] = w2
    return n, rowptr, edges


# ---- rounding witnesses: graphs whose first decision depends on the order of one fp64 sum (tests/golden/make_golden_rounding.py)

WITNESS_NV, WITNESS_V = 64, 40          # the witness vertex sits in the aligned group [32, 64) and on rank 1 of 2 / 2 of 4
WITNESS_B, WITNESS_A, WITNESS_U = 10, 11, 12


def rounding_witness(name):
    """(nv, rowptr, edges, X) of a witness graph; X is the starting assignment (None: singletons).

    R1 ("r1_ck1", "r1_ck2", "r1_subrange"): vertex v has three parallel edges to A of weights 0.1, 0.2, 0.3 and two to
    B of weights 0.5, 0.1, interleaved with three light edges; k_A == k_B bitwise (both 0.6.. + 10 = 10.6) and
    B < A < v, so the gains of A and B differ only in their counter sums.  In edge order A's sum is 0.6000000000000001
    and A wins; summed in reverse (0.6) the gains tie and the smaller id B wins.  ck1 lists A first (the first
    community of pass 1), ck2 lists B first (A is the second community found); subrange adds a dense block around v so
    that its 32-vertex group holds more edges than one staging buffer.
    R2 ("r2_own"): X puts v with u (three parallel edges 0.1, 0.2, 0.3, interleaved); the candidate B has one edge of
    weight 0.6000000000000001 and a_B == a_X - k_v bitwise, so the gain of B is 2 (0.6000000000000001 - counter[0]):
    0 in edge order (v stays), positive with counter[0] summed in reverse (v moves)."""
    nv, v = WITNESS_NV, WITNESS_V
    rng = np.random.default_rng(2024)
    adj = [[] for _ in range(nv)]

    def edge(a, b, w):
        adj[a].append((b, w))
        adj[b].append((a, w))

    light = [50, 51, 52]
    if name.startswith("r1"):
        A, B = WITNESS_A, WITNESS_B
        if name == "r1_ck2":
            order = [(B, 0.5), (A, 0.1), (light[0], 0.01), (A, 0.2), (B, 0.1), (light[1], 0.01), (A, 0.3),
                     (light[2], 0.01)]
        else:
            order = [(A, 0.1), (light[0], 0.01), (B, 0.5), (A, 0.2), (light[1], 0.01), (A, 0.3), (B, 0.1),
                     (light[2], 0.01)]
        pend = {A: 20, B: 21}
    elif name == "r2_own":
        u, B = WITNESS_U, WITNESS_B
        order = [(u, 0.1), (light[0], 0.01), (u, 0.2), (B, 0.6000000000000001), (u, 0.3), (light[1], 0.01)]
        pend = {u: 20, B: 21}
    else:
        raise ValueError(name)
    for t, w in order:                          # v's list in this order; each tail's list gets the edge in this order too
        edge(v, t, w)
    for t, p in pend.items():
        edge(t, p, 10.0)
    special = {v, *pend, *pend.values(), *light}
    others = [x for x in range(nv) if x not in special]
    for x in others:                            # sparse background, general weights
        for y in rng.choice(others, 3, replace=False):
            if y != x:
                edge(x, int(y), float(rng.uniform(0.5, 1.5)))
    for x in light:
        edge(x, int(rng.choice(others)), float(rng.uniform(0.5, 1.5)))
    if name == "r1_subrange":
        block = [x for x in range(32, 64) if x not in special]
        for i, x in enumerate(block):
            for y in block[i + 1:]:
                if rng.random() < 0.6:
                    edge(x, y, float(rng.uniform(0.5, 1.5)))
    rowptr = np.zeros(nv + 1, np.int64)
    rowptr[1:] = np.cumsum([len(a) for a in adj])
    edges = np.zeros(int(rowptr[-1]), hg.EDGE_DTYPE)
    edges["tail"] = [t for a in adj for t, _ in a]
    edges["weight"] = [w for a in adj for _, w in a]
    X = None
    if name == "r2_own":
        X = np.arange(nv, dtype=np.int64)
        X[v] = WITNESS_U
    return nv, rowptr, edges, X


def reversed_adjacency(rowptr, edges, v):
    """The same graph with vertex v's adjacency list in reverse order."""
    e = edges.copy()
    a, b = int(rowptr[v]), int(rowptr[v + 1])
    e[a:b] = edges[a:b][::-1]
    return e
