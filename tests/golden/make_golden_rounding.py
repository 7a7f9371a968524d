#!/usr/bin/env python3
"""tests/golden/rounding_traces.json: traces of the UNMODIFIED reference (oracle/_ref/miniVite_ref, `-f`, 1 thread) on the
rounding witnesses of tests/helpers.rounding_witness, graphs whose first decision at vertex WITNESS_V turns on the order
of one fp64 counter sum (0.1 + 0.2 + 0.3 = 0.6000000000000001 in edge order, 0.6 in reverse).

R1 cases start from singletons, so the reference itself records them: r1_ck1, r1_ck2 and r1_subrange on 1 rank, and
r1_ck1 split over 2 ranks (A and B are ghosts of v's rank).  The R2 witness needs a warm start, which the reference's
command line does not offer; its tests compare with tests/warm_oracle.c instead, which is pinned to the reference.
Before writing, this script asserts for every case: the reference's first iteration is the same on 1, 2 and 4 ranks,
and the same graph with v's adjacency reversed gives a different first-iteration hash in the reference.
Run where the reference binary can be built (python oracle/build_ref.py); the output is byte-identical on every run."""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import WITNESS_A, WITNESS_B, WITNESS_V, reversed_adjacency, rounding_witness  # noqa: E402
from make_golden import pack  # noqa: E402
from minivite_b200 import hostgraph as hg  # noqa: E402
from oracle import oracle as O  # noqa: E402

OUT = os.path.join(HERE, "rounding_traces.json")
CASES = [("r1_ck1", 1), ("r1_ck2", 1), ("r1_subrange", 1), ("r1_ck1", 2)]


def first(ref):
    t = ref["trace"][0]
    return t["moved"], t["chash"]


def main():
    assert O.have_reference(), "oracle/_ref/miniVite_ref missing: python oracle/build_ref.py"
    tmp = tempfile.mkdtemp(prefix="mvround_")
    cases = {}
    for witness, p in CASES:
        nv, rowptr, edges, X = rounding_witness(witness)
        assert X is None
        path = os.path.join(tmp, witness + ".bin")
        hg.write_graph_arrays(path, nv, rowptr, edges["tail"], edges["weight"])
        ref = O.run_reference(["-f", path], nranks=p, threads=1)
        for q in (1, 2, 4):
            assert first(O.run_reference(["-f", path], nranks=q, threads=1)) == first(ref), (witness, q)
        rev = os.path.join(tmp, witness + "_rev.bin")
        er = reversed_adjacency(rowptr, edges, WITNESS_V)
        hg.write_graph_arrays(rev, nv, rowptr, er["tail"], er["weight"])
        assert first(O.run_reference(["-f", rev], nranks=p, threads=1))[1] != first(ref)[1], witness
        cases[f"{witness}_p{p}"] = dict(pack(ref, p), kind="witness", witness=witness, vertex=WITNESS_V,
                                        edge_order_target=WITNESS_A, reversed_target=WITNESS_B)
    gold = {"source": "unmodified reference (oracle/_ref/miniVite_ref -f, 1 thread), tests/golden/make_golden_rounding.py",
            "cases": cases}
    with open(OUT, "w") as f:
        json.dump(gold, f, indent=0, separators=(",", ":"), sort_keys=True)
        f.write("\n")
    print("wrote", OUT, sorted(cases))


if __name__ == "__main__":
    main()
