"""The float build's step restated (tests/step_ref.step with f32=True), pinned to the reference's USE_32_BIT_GRAPH
build (oracle/_ref/miniVite_ref32) on the witness graphs of tests/golden/f32_witness_traces.json and on every exact
case of tests/golden/ref32_traces.json.  On the witnesses the float step and the double step send the witness vertex
to different communities, so a restatement (or a kernel) that ignored the float roundings would fail here."""
import json
import os

import numpy as np
import pytest

import f32_witness as W
import step_ref as S
from helpers import case_graph, split_global
from oracle import oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    return json.load(open(os.path.join(GOLDEN, name)))["cases"]


WIT = load("f32_witness_traces.json")
REF32 = load("ref32_traces.json")
GRAPHS = sorted(k for k, c in WIT.items() if "witness" in c)
EXACT32 = sorted(k for k, c in REF32.items() if c.get("unit_weight", True) or "dyadic" in k)


def chash(parts, T):
    return sum(O.comm_hash(int(parts[r]), T[parts[r]:parts[r + 1]]) for r in range(len(parts) - 1)) & (2 ** 64 - 1)


def witness_graph(case):
    nv, rowptr, edges = W.graph(case["spec"])
    parts = split_global(nv, rowptr, edges, case["nranks"])[0]
    return parts, S.Graph([0, nv], [rowptr], [edges])


def constant(G):
    return 1.0 / float(np.sum(G.k))


def test_golden_covers_the_issue_cases():
    """Every kind of witness is there, and each one is live: the double build first differs at first_diff."""
    assert {c["first_diff"] for c in WIT.values() if "first_diff" in c} == {1, 2}
    assert any(c["constant_decides"] for c in WIT.values() if "witness" in c)
    assert {c["nranks"] for c in WIT.values()} == {1, 2, 4}
    degs = set()
    for name in GRAPHS:
        nv, rowptr, _ = W.graph(WIT[name]["spec"])
        assert W.units(WIT[name]["spec"]) < 2 ** 24
        v = WIT[name]["witness"]
        degs.add(int(rowptr[v + 1] - rowptr[v]))
    assert min(degs) <= 316 and any(508 < d <= 2048 for d in degs) and max(degs) > 2048


@pytest.mark.parametrize("name", GRAPHS)
def test_restated_float_steps_match_the_float_build(name):
    """The restated float step reproduces every iteration's (moved, chash) of the float build and its final
    assignment (the one before the last iteration, which fails the exit test and is not applied); the restated double
    step moves the witness to y2 where the float one moves it to y1."""
    case = WIT[name]
    parts, G = witness_graph(case)
    c = constant(G)
    X = np.arange(G.nv, dtype=np.int64)
    final = X
    for k, t in enumerate(case["trace"], 1):
        final = X
        r = S.step(G, X, c, f32=True)
        assert r["moved"] == t["moved"] and chash(parts, r["target"]) == int(t["chash"], 16), (name, k)
        if k == case["first_diff"]:
            v = case["witness"]
            d = S.step(G, X, c)
            assert r["target"][v] == case["y1"] and d["target"][v] == case["y2"], name
        X = r["target"]
    if "comm" in case:
        assert [int(x) for x in final] == case["comm"], name
    assert chash(parts, final) == int(case["final_chash"], 16), name


@pytest.mark.parametrize("name", sorted(k for k in WIT if "_exit" in k))
def test_exit_witnesses(name):
    """The two -t values are adjacent floats; the lower one equals the float build's rounded-up difference
    Q_k - Q_{k-1}, so the float build runs past k while a test on the unrounded difference would stop at k."""
    case = WIT[name]
    k = case["exit_iter"]
    pair = WIT[name[:-2] + ("hi" if name.endswith("lo") else "lo")]
    lo, hi = sorted((float(case["thresh"]), float(pair["thresh"])))
    assert np.nextafter(np.float32(lo), np.float32(np.inf)) == np.float32(hi)
    low = case if float(case["thresh"]) == lo else pair
    q = [np.float32(float(t["modularity"])) for t in low["trace"]]
    prev = np.float32(-1.0) if k == 1 else q[k - 2]
    assert np.float32(q[k - 1] - prev) == np.float32(lo) and float(q[k - 1]) - float(prev) < lo
    iters = {float(c["thresh"]): c["iters"] for c in (case, pair)}
    assert iters[hi] == k < iters[lo]


@pytest.mark.parametrize("name", EXACT32)
def test_restated_float_step_matches_ref32_first_iteration(name):
    """The float step restated on every exact case of ref32_traces.json (unit and dyadic weights below 2^24 units)
    gives the float build's trace[0]."""
    case = REF32[name]
    parts, rps, eds, _ = case_graph(case)
    G = S.Graph(parts, rps, eds)
    r = S.step(G, np.arange(G.nv, dtype=np.int64), constant(G), f32=True)
    t = case["trace"][0]
    assert r["moved"] == t["moved"] and chash(parts, r["target"]) == int(t["chash"], 16), name


def test_gain_rounding_example():
    """w1 = 348, w2 = 347 units, 2m = 34 054, d1 = d2 + 49: double gains differ by 2/(2m), float gains are equal."""
    c = 1.0 / 34054
    k, d2 = 695, 348
    g = [S.gain(348.0, 0.0, k, d2 + 49.0, 0.0, c), S.gain(347.0, 0.0, k, float(d2), 0.0, c)]
    g32 = [float(S.gain(348.0, 0.0, k, d2 + 49.0, 0.0, S.constant32(c), True)),
           float(S.gain(347.0, 0.0, k, float(d2), 0.0, S.constant32(c), True))]
    assert g[1] > g[0] and g32[0] == g32[1]
    assert S.constant32(c) == float(np.float32(1.0 / 34054))
