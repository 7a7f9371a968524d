"""CPU tests of the comparison definitions (DESIGN.md §3.13) and their NumPy restatement (tests/compare_ref.py).

The restatement is held against plain loops on small cases: dict counting for the contingency, an O(N^2) walk over the
vertex pairs for the pair counts, entropies and mutual information by their definition with math.fsum (within 1e-12),
and against scikit-learn's scores on random assignments.  The properties DESIGN states as exact hold bit for bit, and
on the C oracle's result of every unit and dyadic golden case, comparing it with its split shows that every piece lies
inside one community."""
import itertools
import math

import numpy as np
import pytest

from helpers import case_graph
import compare_ref as CR
import split_ref as SR
import warm_oracle as W
from test_quality_ref import CASES


def naive(X, Y):
    """The definitions, by plain loops."""
    N = len(X)
    cells, a, b = {}, {}, {}
    for x, y in zip(X, Y):
        cells[(x, y)] = cells.get((x, y), 0) + 1
        a[x] = a.get(x, 0) + 1
        b[y] = b.get(y, 0) + 1
    same_x = same_y = same_both = 0
    for i, j in itertools.combinations(range(N), 2):
        same_x += X[i] == X[j]
        same_y += Y[i] == Y[j]
        same_both += X[i] == X[j] and Y[i] == Y[j]
    h_x = -math.fsum(c / N * math.log(c / N) for c in a.values()) if N else 0.0
    h_y = -math.fsum(c / N * math.log(c / N) for c in b.values()) if N else 0.0
    mi = math.fsum(c / N * math.log(N * c / (a[x] * b[y])) for (x, y), c in cells.items()) if N else 0.0
    best = {}
    for (x, y), c in sorted(cells.items()):
        if x not in best or c > best[x][1]:
            best[x] = (y, c)
    return {"pairs_xy": same_both, "pairs_x": same_x, "pairs_y": same_y, "pairs_all": N * (N - 1) // 2,
            "cells": len(cells), "communities_x": len(a), "communities_y": len(b), "h_x": h_x, "h_y": h_y, "mi": mi,
            "size": [a.get(x, 0) for x in range(N)], "best": [best[x][0] if x in best else -1 for x in range(N)],
            "overlap": [best[x][1] if x in best else 0 for x in range(N)],
            "best_size": [b[best[x][0]] if x in best else 0 for x in range(N)]}


def small_cases():
    rng = np.random.default_rng(5)
    out = {"n1": (np.zeros(1, np.int64), np.zeros(1, np.int64)),
           "singletons_vs_one": (np.arange(9), np.full(9, 4)),
           "singletons_both": (np.arange(7), np.arange(7)[::-1].copy()),
           "one_both": (np.full(8, 3), np.full(8, 0)),
           "ties": (np.array([0, 0, 0, 0, 4, 4]), np.array([5, 5, 2, 2, 1, 3])),        # 0 ties between 2 and 5: 2
           "named_outside": (np.array([3, 3, 3, 0, 0, 1]), np.array([1, 1, 2, 2, 5, 5]))}
    for t in range(6):
        n = int(rng.integers(2, 60))
        out[f"random{t}"] = (rng.integers(0, max(1, n // (t + 1)), n) % n, rng.integers(0, n, n))
    return out


@pytest.mark.parametrize("name", sorted(small_cases()))
def test_restatement_matches_loops(name):
    X, Y = small_cases()[name]
    got, ref = CR.compare(X, Y), naive([int(v) for v in X], [int(v) for v in Y])
    for k in ("pairs_xy", "pairs_x", "pairs_y", "pairs_all", "cells", "communities_x", "communities_y"):
        assert got[k] == ref[k], (name, k, got[k], ref[k])
    for k in ("h_x", "h_y", "mi"):
        assert abs(got[k] - ref[k]) <= 1e-12, (name, k, got[k], ref[k])
    for k in CR.MATCHES:
        assert list(got[k]) == ref[k], (name, k)


def test_against_sklearn():
    sk = pytest.importorskip("sklearn.metrics")
    rng = np.random.default_rng(17)
    for t in range(20):
        n = int(rng.integers(2, 3000))
        X, Y = rng.integers(0, int(rng.integers(1, n + 1)), n), rng.integers(0, int(rng.integers(1, n + 1)), n)
        if t % 4 == 0:
            Y = np.where(rng.random(n) < 0.1, rng.integers(0, n, n), X)               # close to X
        got = CR.compare(X, Y)
        assert abs(got["ari"] - sk.adjusted_rand_score(X, Y)) <= 1e-12, t
        assert abs(got["rand"] - sk.rand_score(X, Y)) <= 1e-12, t
        assert abs(got["mi"] - sk.mutual_info_score(X, Y)) <= 1e-12, t
        assert abs(got["nmi"] - sk.normalized_mutual_info_score(X, Y)) <= 1e-12, t


def same_bits(a, b, keys=CR.FIELDS):
    return all(repr(a[k]) == repr(b[k]) for k in keys)


def test_exact_properties():
    rng = np.random.default_rng(23)
    for n in (1, 2, 5, 100, 4000):
        X, Y = rng.integers(0, max(1, n // 3), n), rng.integers(0, n, n)
        perm = rng.permutation(n)
        for A in (X, Y, np.arange(n), np.zeros(n, np.int64)):
            for B in (A, perm[A]):                            # itself, and any relabelling
                r = CR.compare(A, B)
                assert (r["ari"], r["rand"], r["nmi"], r["vi"]) == (1.0, 1.0, 1.0, 0.0), n
                assert r["mi"] == r["h_x"] == r["h_y"], n
        xy, yx = CR.compare(X, Y), CR.compare(Y, X)
        for k1, k2 in (("h_x", "h_y"), ("pairs_x", "pairs_y"), ("communities_x", "communities_y")):
            assert repr(xy[k1]) == repr(yx[k2]) and repr(xy[k2]) == repr(yx[k1])
        assert same_bits(xy, yx, ("vertices", "cells", "pairs_xy", "pairs_all", "ari", "rand", "nmi", "vi", "mi"))
        if n > 1:
            Z = np.arange(n) % 2                              # anything that is not one community
            for A, B in ((np.zeros(n, np.int64), Z), (Z, np.full(n, n - 1))):
                r = CR.compare(A, B)
                assert r["ari"] == 0.0 and r["nmi"] == 0.0, n


def test_hand_values():
    r = CR.compare(np.zeros(1, np.int64), np.zeros(1, np.int64))                   # N = 1
    assert (r["pairs_all"], r["cells"], r["ari"], r["nmi"], r["vi"]) == (0, 1, 1.0, 1.0, 0.0)
    r = CR.compare(np.arange(6), np.arange(6))                                      # all singletons
    assert (r["pairs_xy"], r["pairs_x"], r["cells"], r["ari"], r["nmi"]) == (0, 0, 6, 1.0, 1.0)
    assert r["h_x"] == math.log(6.0) and list(r["best"]) == list(range(6)) and list(r["best_size"]) == [1] * 6
    r = CR.compare(np.full(6, 2), np.full(6, 5))                                    # one community
    assert (r["pairs_xy"], r["cells"], r["ari"], r["nmi"], r["h_x"]) == (15, 1, 1.0, 1.0, 0.0)
    assert list(r["size"]) == [0, 0, 6, 0, 0, 0] and list(r["best"]) == [-1, -1, 5, -1, -1, -1]
    r = CR.compare(np.array([0, 0, 0, 0, 4, 4]), np.array([5, 5, 2, 2, 1, 3]))     # ties go to the smallest y
    assert list(r["best"][[0, 4]]) == [2, 1] and list(r["overlap"][[0, 4]]) == [2, 1]


# ---- the oracle's results against their splits: every piece lies inside one community -----------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_result_against_its_split(name):
    parts, rps, eds, _keep = case_graph(CASES[name])
    X = np.concatenate(W.louvain(parts, rps, eds)["comm"])
    s = SR.split(parts, rps, eds, X)
    r = CR.compare(X, s["Y"])
    assert r["pairs_xy"] == r["pairs_y"] and r["cells"] == r["communities_y"] == s["components"], name
    assert r["communities_x"] == s["communities"] and np.array_equal(r["size"], np.bincount(X, minlength=len(X)))
    assert r["ari"] == 1.0 if s["disconnected"] == 0 else r["ari"] < 1.0
