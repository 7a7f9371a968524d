"""The rounding witnesses (tests/helpers.rounding_witness, tests/golden/rounding_traces.json) on the host: the C oracle
reproduces the reference's traces, the witness decision flips when only the order of v's adjacency changes, and the
certificate of tests/step_ref.py decides every vertex (the tie is in the counter sums alone, so neither 1/(2m) nor a
community degree can decide it)."""
import json
import os

import numpy as np
import pytest

import step_ref as S
import warm_oracle as W
from helpers import (WITNESS_A, WITNESS_B, WITNESS_U, WITNESS_V, assert_trace_matches, reversed_adjacency,
                     rounding_witness, split_global)
from oracle import oracle as O

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rounding_traces.json")) as f:
    GOLDEN = json.load(f)["cases"]


def witness_step(name, p=1, reverse=False):
    nv, rowptr, edges, X = rounding_witness(name)
    if reverse:
        edges = reversed_adjacency(rowptr, edges, WITNESS_V)
    parts, rps, eds = split_global(nv, rowptr, edges, p)
    X = np.arange(nv, dtype=np.int64) if X is None else X
    res = W.louvain(parts, rps, eds, init_comm=[X[parts[r]:parts[r + 1]] for r in range(p)], stop_after=1)
    return parts, rps, eds, X, np.concatenate(res["comm"]), res["trace"][0], res["constant"]


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_oracle_reproduces_reference(name):
    case = GOLDEN[name]
    nv, rowptr, edges, _X = rounding_witness(case["witness"])
    parts, rps, eds = split_global(nv, rowptr, edges, case["nranks"])
    res = O.louvain(parts, rps, eds)
    assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], final_chash=res["chash_final"])


@pytest.mark.parametrize("name", ["r1_ck1", "r1_ck2", "r1_subrange", "r2_own"])
@pytest.mark.parametrize("p", [1, 2, 4])
def test_witness_turns_on_the_order(name, p):
    parts, rps, eds, X, T, tr, c = witness_step(name, p)
    _, _, _, _, Tr, trr, _ = witness_step(name, p, reverse=True)
    v = WITNESS_V
    want, flipped = (WITNESS_A, WITNESS_B) if name.startswith("r1") else (WITNESS_U, WITNESS_B)
    assert T[v] == want and Tr[v] == flipped
    assert int(tr["chash"]) != int(trr["chash"])
    assert np.array_equal(np.delete(T, v), np.delete(Tr, v))       # only the witness decision changes
    G = S.Graph(parts, rps, eds)
    r = S.step(G, X, c)
    assert np.array_equal(r["target"], T)
    cert = S.certify(G, X, c, heavy_deg=316)
    assert cert["certified"].all() and np.array_equal(cert["outcome"], T)
    if name.startswith("r1"):
        for case in GOLDEN.values():
            if case["witness"] == name:
                assert (int(tr["moved"]), int(tr["chash"])) == (case["trace"][0]["moved"],
                                                                int(case["trace"][0]["chash"], 16))


def test_witness_shapes():
    for name in ("r1_ck1", "r1_ck2", "r1_subrange", "r2_own"):
        nv, rowptr, edges, _X = rounding_witness(name)
        deg = np.diff(rowptr)
        assert deg.max() <= 316                                       # no heavy vertex by default
        group = int(rowptr[64] - rowptr[32])                          # WITNESS_V's aligned group of 32 vertices
        assert (group > 320) == (name == "r1_subrange"), (name, group)
        G = S.Graph(np.array([0, nv]), [rowptr], [edges])
        if name.startswith("r1"):
            assert G.k[WITNESS_A] == G.k[WITNESS_B]
        else:
            ax = (G.k[WITNESS_V] + G.k[WITNESS_U]) - G.k[WITNESS_V]
            assert ax == G.k[WITNESS_B]


def test_witness_under_forced_heavy_is_admissible_only():
    """With k_scan_heavy summing the witness's counters in any order, A and B are both admissible for v."""
    parts, rps, eds, X, T, tr, c = witness_step("r1_ck1")
    G = S.Graph(parts, rps, eds)
    cert = S.certify(G, X, c, heavy_deg=4)
    assert not cert["certified"][WITNESS_V] and cert["admissible"][WITNESS_V] == {WITNESS_A, WITNESS_B}
