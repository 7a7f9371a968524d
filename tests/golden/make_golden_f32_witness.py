#!/usr/bin/env python3
"""tests/golden/f32_witness_traces.json: traces of the reference's float build (oracle/_ref/miniVite_ref32, -f,
1 thread) on the witness graphs of tests/f32_witness.py, where the float roundings of that build decide a move that
the double build decides the other way.

Every case is checked before it is written:
  * exactness: the weights are k * 2^-j and 2m stays below 2^24 units, so every float sum of the float build is exact
    and its run is reproducible (the bar of ref32_traces.json);
  * liveness: the double reference (oracle/_ref/miniVite_ref) on the same graph and rank count records a different
    community hash; the first iteration where the two differ is printed and stored as `first_diff`;
  * the restatement: tests/step_ref.step with f32=True gives the float build's first iteration, with f32=False the
    double build's, and the two send the witness vertex to different targets (iteration-1 witnesses; the iteration-2
    witness is checked from the float build's assignment after iteration 1).
Exit-test cases run the float build with two -t values a float ulp apart.  At the lower one the float subtraction
Q_k - Q_{k-1} rounds up to exactly -t, so the float test `diff < thresh` fails and the run goes on, while the same test
on the unrounded difference stops at iteration k; the upper one stops at k.  Both runs are recorded.
Run where the reference binaries can be built (python oracle/build_ref.py); the output is byte-identical on every run."""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import f32_witness as W  # noqa: E402
import step_ref as S  # noqa: E402
from helpers import assert_dyadic_exact, split_global  # noqa: E402
from make_golden import pack  # noqa: E402
from minivite_b200 import hostgraph as hg  # noqa: E402
from oracle import oracle as O  # noqa: E402

OUT = os.path.join(HERE, "f32_witness_traces.json")
# name, builder, arguments, rank counts, what the case covers
CASES = [
    ("unit_i1_tile", W.iteration1, dict(k=427, delta=155, mult=1), (1,),
     "iteration 1, unit multigraph, witness degree 427 < heavy_deg; its 32-vertex group fits one k_scan_pw buffer"),
    ("unit_i1_subrange", W.iteration1, dict(k=427, delta=155, mult=100), (1, 2, 4),
     "as unit_i1_tile with pairs of 100 units: the witness's group has more edges than one k_scan_pw buffer takes; "
     "on 2 and 4 ranks y1 and y2 are ghosts of the witness's rank, the last one"),
    ("unit_i1_mid", W.iteration1, dict(k=1295, delta=13, mult=100), (1,),
     "witness degree 1295: k_scan_heavy under k_scan_pw / k_scan_pq, a tile vertex of k_scan_ws"),
    ("unit_i1_heavy", W.iteration1, dict(k=3117, delta=3, mult=100), (1, 2),
     "witness degree 3117 > 2048: k_scan_heavy under every scan kernel; the float constant alone decides here"),
    ("dyadic_i1", W.iteration1, dict(k=427, delta=155, mult=100, denom=4), (1, 2),
     "the unit_i1_subrange graph with every edge one k/4 weight: a simple graph on the weighted path"),
    ("unit_tie", W.iteration1, dict(k=375, delta=6, K=0, mult=100), (1,),
     "K = 0: an exact tie; the double build follows the rounding of 1/(2m), the float build the smaller label"),
    ("unit_i2", W.iteration2, dict(w2=150, s=4, t=154, q1=76, r=306, mult=100), (1, 2),
     "first difference in iteration 2: the witness sits in a two-member community (eix, ax non-zero)"),
]
# exit-test witnesses: (graph case, iteration k whose rounded difference sets -t)
EXIT = [("unit_i2", 1), ("unit_i1_mid", 2)]


def f32_next(x):
    return float(np.nextafter(np.float32(x), np.float32(np.inf)))


def chash(parts, T):
    return sum(O.comm_hash(int(parts[r]), T[parts[r]:parts[r + 1]]) for r in range(len(parts) - 1)) & (2 ** 64 - 1)


def restated(spec, X, f32, f32_constant=True):
    nv, rowptr, edges = W.graph(spec)
    G = S.Graph([0, nv], [rowptr], [edges])
    return S.step(G, X, 1.0 / float(np.sum(G.k)), f32=f32, f32_constant=f32_constant)


def main():
    assert O.have_reference() and os.path.exists(O.REF32_BIN), "reference binaries missing: python oracle/build_ref.py"
    tmp = tempfile.mkdtemp(prefix="mvf32w_")
    cases = {}
    specs = {}
    for name, build, args, ranks, what in CASES:
        spec, v, y1, y2 = build(**args)
        specs[name] = spec
        nv, rowptr, edges = W.graph(spec)
        j = assert_dyadic_exact(nv, rowptr, edges)
        units = float(np.sum(edges["weight"])) * 2.0 ** j
        assert units < 2.0 ** 24 and units == W.units(spec) * 2.0 ** j / spec["denom"], name
        p32, p64 = os.path.join(tmp, name + "32.bin"), os.path.join(tmp, name + "64.bin")
        hg.write_graph_arrays32(p32, nv, rowptr, edges["tail"], edges["weight"].astype(np.float32))
        hg.write_graph_arrays(p64, nv, rowptr, edges["tail"], edges["weight"])
        # the restatement: the step where the witness's decision differs, from the float build's assignment before it
        it = 1 if build is W.iteration1 else 2
        X = np.arange(nv, dtype=np.int64)
        for _ in range(it - 1):
            X = restated(spec, X, True)["target"]
        tf, td = restated(spec, X, True)["target"], restated(spec, X, False)["target"]
        assert tf[v] == y1 and td[v] == y2, (name, tf[v], td[v])
        # does the float constant alone decide?  (float gains with the double 1/(2m) move the witness elsewhere)
        by_constant = bool(restated(spec, X, True, f32_constant=False)["target"][v] != y1)
        for p in ranks:
            pre = os.path.join(tmp, f"{name}_c{p}")
            ref = O.run_reference(["-f", p32], nranks=p, threads=1, binary=O.REF32_BIN, dump_comm=pre)
            dbl = O.run_reference(["-f", p64], nranks=p, threads=1)
            comm = np.concatenate([c for _, c in O.read_comm_dump(pre, p, elem=np.int32)])
            parts = split_global(nv, rowptr, edges, p)[0]
            if p > 1:                          # the witness on the last rank, y1 and y2 owned by another one
                assert v >= parts[p - 1] and y2 < parts[p - 1], name
            diff = [k for k, (a, b) in enumerate(zip(ref["trace"], dbl["trace"])) if a["chash"] != b["chash"]]
            assert diff, (name, p)
            k0 = diff[0] + 1
            assert k0 == it, (name, p, k0)
            if it == 1:
                assert ref["trace"][0]["chash"] == chash(parts, tf) and ref["trace"][0]["moved"] == int(np.sum(tf != X))
                assert dbl["trace"][0]["chash"] == chash(parts, td)
            key = f"{name}_p{p}"
            cases[key] = dict(pack(ref, p, comm if nv <= 5000 else None), spec=spec, witness=int(v), y1=int(y1), y2=int(y2),
                              first_diff=k0, double_iters=dbl["result"]["iters"], constant_decides=by_constant,
                              what=what)
            print(f"{key}: nv {nv} 2m {int(units)} units, witness {v} (degree {int(rowptr[v + 1] - rowptr[v])}) -> "
                  f"float {y1} / double {y2}; float and double first differ in iteration {k0}; "
                  f"iterations {ref['result']['iters']} (float) / {dbl['result']['iters']} (double)"
                  + ("; the float constant alone decides" if by_constant else ""))
    for name, k in EXIT:
        base = cases[f"{name}_p1"]
        q = [np.float32(float(t["modularity"])) for t in base["trace"]]
        prev = np.float32(-1.0) if k == 1 else max(q[k - 2], np.float32(-1.0))
        exact = float(q[k - 1]) - float(prev)                              # exact in double
        assert float(prev) < float(q[k - 1]) / 2, (name, k)
        lo = float(np.float32(q[k - 1]) - prev)                             # the float build's difference
        assert lo > exact, (name, k, lo, exact)                             # rounded up: only a float test goes on
        hi = f32_next(lo)
        p32 = os.path.join(tmp, name + "32.bin")
        runs = {}
        for t in (lo, hi):
            pre = os.path.join(tmp, f"{name}_t{len(runs)}")
            ref = O.run_reference(["-f", p32, "-t", repr(t)], nranks=1, threads=1, binary=O.REF32_BIN, dump_comm=pre)
            comm = np.concatenate([c for _, c in O.read_comm_dump(pre, 1, elem=np.int32)])
            runs[t] = dict(pack(ref, 1, comm), thresh=repr(t))
        assert runs[hi]["iters"] == k and runs[lo]["iters"] > k, (name, runs[lo]["iters"], runs[hi]["iters"])
        for t in (lo, hi):
            cases[f"{name}_exit{k}_{'lo' if t == lo else 'hi'}"] = dict(runs[t], spec=specs[name], exit_iter=k)
        print(f"{name} exit test at iteration {k}: Q_k - Q_k-1 = {exact!r} rounds to {lo!r}; -t {lo!r} runs "
              f"{runs[lo]['iters']} iterations, -t {hi!r} runs {runs[hi]['iters']}")
    gold = {"source": "reference float build (oracle/_ref/miniVite_ref32 -f, 1 thread), "
                      "tests/golden/make_golden_f32_witness.py; do not edit",
            "cases": cases}
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0, separators=(",", ":"), sort_keys=True)
        f.write("\n")
    print("wrote", OUT, len(cases), "cases")


if __name__ == "__main__":
    main()
