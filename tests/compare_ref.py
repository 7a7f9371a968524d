"""NumPy restatement of comparing two assignments (DESIGN.md §3.13; mvgpu_compare_communities,
mvgpu_get_community_matches), TEST INFRASTRUCTURE.

X and Y give each of the N = nv vertices a community id in [0, N).  Cells n_xy, sizes a_x and b_y, pair counts as exact
Python integers, and the doubles from them in the library's order: ARI from the exact integers with one rounding of the
numerator and one of the denominator, entropies from S(h) = sum over the values k > 1 of a histogram, ascending, of
m * (k * log k) with math.log (libm's log, which np.log need not match in the last bit)."""
import math

import numpy as np


def _concat(a):
    return np.concatenate([np.asarray(p, np.int64) for p in a]) if isinstance(a, (list, tuple)) else np.asarray(a, np.int64)


def histogram(counts):
    """(value, multiplicity) of the non-zero values, ascending value (Python ints)."""
    v, m = np.unique(counts[counts > 0], return_counts=True)
    return [(int(k), int(c)) for k, c in zip(v, m)]


def pairs(h):
    return sum(m * (k * (k - 1) // 2) for k, m in h)


def entropy_sum(h):
    s = 0.0
    for k, m in h:
        if k > 1:
            s += float(m) * (float(k) * math.log(float(k)))
    return s


def scores(N, cells_h, a_h, b_h):
    """The report of mvgpu_compare_communities from the three histograms (cells, a, b)."""
    A, P, PX, PY = N * (N - 1) // 2, pairs(cells_h), pairs(a_h), pairs(b_h)
    cx, cy = sum(m for _, m in a_h), sum(m for _, m in b_h)
    num, den = 2 * (A * P - PX * PY), A * (PX + PY) - 2 * PX * PY
    n = float(N)
    sxy, sx, sy = entropy_sum(cells_h), entropy_sum(a_h), entropy_sum(b_h)
    h_x = 0.0 if cx <= 1 else math.log(n) - sx / n
    h_y = 0.0 if cy <= 1 else math.log(n) - sy / n
    mi = 0.0 if (cx <= 1 or cy <= 1) else math.log(n) + (sxy - (sx + sy)) / n
    return {"vertices": N, "communities_x": cx, "communities_y": cy, "cells": sum(m for _, m in cells_h),
            "pairs_xy": P, "pairs_x": PX, "pairs_y": PY, "pairs_all": A,
            "ari": 1.0 if den == 0 else float(num) / float(den),
            "rand": 1.0 if A == 0 else float(A + 2 * P - PX - PY) / float(A),
            "nmi": 1.0 if h_x + h_y == 0.0 else (2.0 * mi) / (h_x + h_y),
            "vi": (h_x + h_y) - 2.0 * mi, "mi": mi, "h_x": h_x, "h_y": h_y}


def compare(X, Y):
    """X, Y: whole-graph assignments (or per-shard lists) -> the report fields and the match arrays of every community
    x in [0, N) (size, best, overlap, best_size; concatenated over the shards, int64)."""
    X, Y = _concat(X), _concat(Y)
    N = len(X)
    assert len(Y) == N and (N == 0 or (min(X.min(), Y.min()) >= 0 and max(X.max(), Y.max()) < N))
    ukey, n = np.unique(X * N + Y, return_counts=True)
    cx, cy = (ukey // N, ukey % N) if N else (ukey, ukey)
    a, b = np.bincount(X, minlength=N), np.bincount(Y, minlength=N)
    out = scores(N, histogram(n), histogram(a), histogram(b))
    order = np.lexsort((cy, -n, cx))                  # per x: the largest n_xy first, ties to the smallest y
    first = order[np.concatenate([[True], cx[order][1:] != cx[order][:-1]])] if len(order) else order
    best = np.full(N, -1, np.int64)
    overlap = np.zeros(N, np.int64)
    best[cx[first]], overlap[cx[first]] = cy[first], n[first]
    out.update(size=a.astype(np.int64), best=best, overlap=overlap,
               best_size=np.where(best >= 0, b[np.maximum(best, 0)], 0).astype(np.int64))
    return out


FIELDS = ("vertices", "communities_x", "communities_y", "cells", "pairs_xy", "pairs_x", "pairs_y", "pairs_all",
          "ari", "rand", "nmi", "vi", "mi", "h_x", "h_y")
MATCHES = ("size", "best", "overlap", "best_size")
