#!/usr/bin/env python3
"""tests/golden/weighted_exact_traces.json: traces of the UNMODIFIED reference (oracle/_ref/miniVite_ref, `-f`, 1 rank,
1 thread) on graphs with dyadic weights, k * 2^-j with j <= 6.  Every fp64 sum of such weights is exact, so neither the
reference's unordered OpenMP / MPI reductions nor the CUDA path's atomics can change a bit of the result: the weighted
path is held to the same bit-exact bar as the unit-weight path.

Each case is a seeded recipe (tests/helpers.py rebuilds the graph; hand-made graphs are stored whole).  For every case
this script asserts, before writing anything:
  * the exactness precondition (helpers.assert_dyadic_exact): dyadic weights, sums within 53 bits, symmetric weights;
  * that the reference gives the identical trace on another rank count and with 4 OpenMP threads;
  * non-degeneracy (helpers.assert_non_degenerate): at least 4 distinct weights, and a trace that differs from the same
    graph with unit weights.  The uniform K6,6 (all weights 0.5) is the one exemption: it must instead give exactly
    the unit-weight trace, since scaling every weight by a power of two scales every sum and gain exactly.
Run where the reference binary can be built (python oracle/build_ref.py)."""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import assert_dyadic_exact, assert_non_degenerate, global_csr  # noqa: E402
from make_golden import pack  # noqa: E402
from minivite_b200 import hostgraph as hg  # noqa: E402
from oracle import oracle as O  # noqa: E402

OUT = os.path.join(HERE, "weighted_exact_traces.json")
STORE_COMM = 5000          # the full final assignment is stored up to this many vertices, the final hash always


def from_pairs(nv, pairs, w, loops=()):
    """Symmetric CSR from undirected (a, b, weight) pairs; parallel pairs stay separate edges."""
    adj = [[] for _ in range(nv)]
    for (a, b), ww in zip(pairs, w):
        adj[a].append((b, ww))
        adj[b].append((a, ww))
    for (a, ww) in loops:
        adj[a].append((a, ww))
    rowptr, tails, ws = [0], [], []
    for a in range(nv):
        for (b, ww) in sorted(adj[a]):
            tails.append(b)
            ws.append(ww)
        rowptr.append(len(tails))
    return {"nv": nv, "rowptr": rowptr, "tails": tails, "weights": [float(x) for x in ws]}


def handmade():
    """name -> (graph, min distinct weights, scaled_unit).  Exact gain ties everywhere: tie-break by label and the
    singleton veto on the fp64 path."""
    g = {}
    # K6,6, every weight 0.5: uniform but not 1, so the fp64 kernels run with ties everywhere
    g["k66_half"] = (from_pairs(12, [(i, 6 + j) for i in range(6) for j in range(6)], [0.5] * 36), 1, True)
    # path with alternating weights 0.25 / 0.75, two isolated vertices at the end
    g["path_alt"] = (from_pairs(18, [(i, i + 1) for i in range(15)], [0.25 if i % 2 else 0.75 for i in range(15)]), 2, False)
    # star: hub of degree 40 (> 32 lanes), leaves' weights cycle through k/4, three heavier leaf-leaf edges between
    # light leaves (they pull pairs away from the hub only because of their weights), plus one isolated vertex
    g["star40_mixed"] = (from_pairs(42, [(0, i) for i in range(1, 41)] + [(1, 9), (17, 25), (33, 2)],
                                    [(1 + i % 8) / 4.0 for i in range(40)] + [2.0, 2.0, 1.5]), 4, False)
    # parallel edges with different weights between the same pair, next to single edges of the same total
    pairs = [(0, 1), (0, 1), (0, 1), (1, 2), (2, 3), (2, 3), (3, 0), (4, 5), (4, 5), (5, 6), (6, 4), (3, 4), (6, 7), (7, 8),
             (8, 9), (8, 9), (9, 10), (10, 11), (11, 8)]
    w = [0.25, 0.5, 1.25, 2.0, 0.75, 1.25, 2.0, 1.5, 0.5, 2.0, 2.0, 0.125, 1.0, 1.0, 0.375, 1.625, 2.0, 2.0, 2.0]
    g["multi_w"] = (from_pairs(12, pairs, w), 4, False)
    # self loops: 0.75 + 0.75 on one vertex (the reference truncates the SUM to 1, dspl.hpp:285; truncating each loop
    # would give 0), one loop of 2.5 (truncated to 2), one of 0.5 (truncated to 0); two isolated vertices
    pairs = [(0, 1), (1, 2), (2, 0), (2, 3), (3, 4), (4, 5), (5, 3), (5, 6), (6, 7), (7, 8), (8, 6), (1, 7)]
    w = [1.0, 0.75, 1.5, 0.25, 1.0, 1.25, 0.5, 0.25, 1.75, 1.0, 0.5, 0.125]
    g["self_loops_w"] = (from_pairs(12, pairs, w, loops=[(0, 0.75), (0, 0.75), (4, 2.5), (8, 0.5)]), 4, False)
    # a zero-weight edge between two vertices that have other edges (it is a neighbour with gain input 0), two triangles
    # joined by a light edge, two isolated vertices
    pairs = [(0, 1), (1, 2), (2, 0), (3, 4), (4, 5), (5, 3), (2, 3), (1, 4), (6, 7)]
    w = [1.0, 0.5, 1.5, 1.5, 1.0, 0.5, 0.0, 0.25, 1.0]
    g["zero_w"] = (from_pairs(10, pairs, w), 4, False)
    return g


def recipes():
    """name -> (case fields, extra rank count of the cross-check)."""
    r = {}
    for n in (16384, 65536, 131072):
        for s in (1, 4):
            r[f"rgg_n{n}_s{s}"] = ({"kind": "dyadic_rgg", "n": n, "strips": s}, 4)
    for s in (1, 4):
        r[f"rgg_n16384_s{s}_p5"] = ({"kind": "dyadic_rgg", "n": 16384, "strips": s, "pct": 5.0}, 4)
    # tests/test_gpu_scan_kernels.py's shapes: dense 32-vertex groups (staging sub-ranges), a ragged last group (33 and
    # 4 099 vertices), hubs with parallel edges, hubs of degree 3 000 (above every tile capacity: k_scan_heavy unforced
    # on every scan variant), self loops, planted partitions
    for n, deg, kw in [(1000, 60, {}), (777, 150, {"self_loops": 40, "multi": 300}),
                       (6000, 8, {"hubs": 3, "hub_deg": 3000, "multi": 200}),
                       (4099, 30, {"hubs": 2, "hub_deg": 1000, "multi": 100}), (33, 20, {}), (2500, 700, {}),
                       (3000, 80, {"blocks": 25}), (20000, 40, {"blocks": 400, "hubs": 1, "hub_deg": 2000})]:
        tag = "".join(f"_{k}{v}" for k, v in kw.items())
        r[f"random_n{n}_d{deg}{tag}"] = ({"kind": "dyadic_random", "n": n, "avg_deg": deg, "seed": n + deg, "kw": kw}, 2)
    r["rmat_s14"] = ({"kind": "dyadic_rmat", "scale": 14, "edge_factor": 16, "seed": 3}, 4)
    return r


def trace_key(ref):
    return ([(t["mod_repr"], t["moved"], t["chash"]) for t in ref["trace"]], ref["final"]["mod_repr"],
            ref["final"]["chash"], repr(ref["final"]["constant"]), ref["result"]["iters"])


def main():
    if not O.have_reference():
        raise SystemExit("oracle/_ref/miniVite_ref missing: run python oracle/build_ref.py")
    tmp = tempfile.mkdtemp(prefix="mvwgold_")
    gold = {"_comment": "generated by tests/golden/make_golden_weighted.py from the unmodified reference; do not edit",
            "cases": {}}
    todo = {name: (fields, p2, 4, False) for name, (fields, p2) in recipes().items()}
    for name, (graph, min_distinct, scaled_unit) in handmade().items():
        todo["hand_" + name] = ({"kind": "hand", "graph": graph}, 2, min_distinct, scaled_unit)
    for name, (fields, p2, min_distinct, scaled_unit) in todo.items():
        nv, rowptr, edges = global_csr(fields)
        j = assert_dyadic_exact(nv, rowptr, edges)
        path = os.path.join(tmp, name + ".bin")
        hg.write_graph_arrays(path, nv, rowptr, edges["tail"], edges["weight"])
        pre = os.path.join(tmp, name + "_c")
        ref = O.run_reference(["-f", path], nranks=1, threads=1, dump_comm=pre)
        key = trace_key(ref)
        for p, th in ((p2, 1), (1, 4)):
            other = O.run_reference(["-f", path], nranks=p, threads=th)
            assert trace_key(other) == key, (name, p, th)
        case = dict(pack(ref, 1), **fields, dyadic_j=j, checked_ranks=[1, p2], maxdeg=int(np.diff(rowptr).max()))
        if nv <= STORE_COMM:
            case["comm"] = [int(x) for x in np.concatenate([c for _, c in O.read_comm_dump(pre, 1)])]
        unit = edges.copy()
        unit["weight"] = 1.0
        uref = O.louvain(np.array([0, nv], np.int64), [rowptr], [unit])
        if scaled_unit:
            assert [(float(t["modularity"]), int(t["moved"]), int(t["chash"])) for t in uref["trace"]] == \
                [(float(t["modularity"]), t["moved"], int(t["chash"], 16)) for t in case["trace"]], name
        else:
            assert_non_degenerate(case, uref, min_distinct)
        case["scaled_unit"] = scaled_unit
        gold["cases"][name] = case
        print(name, "j=%d" % j, ref["result"], "maxdeg", case["maxdeg"], flush=True)
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0, separators=(",", ":"))
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
