"""NumPy restatement of the quality of an assignment (DESIGN.md §3.10; mvgpu_evaluate_communities), TEST INFRASTRUCTURE.

For an assignment X (global community ids in [0, nv), caller numbering):
  e_in  = sum over vertices i, over the stored edge records (i, j) with X(j) = X(i), of w_ij  (self-loop records once each)
  a_c   = sum of vDegree over the members of c,  a2 = sum_c a_c^2,  c = 1/(2m)
  Q     = e_in*c - (a2*c)*c,  signed.
The sums are taken exactly (Python integers on the unit path, math.fsum otherwise), which is what the device computes
whenever every partial sum is exact: unit weights, and dyadic weights within the bounds of helpers.assert_dyadic_exact."""
import math

import numpy as np


def quality(parts, rowptrs, edge_lists, comm):
    """parts, per-shard rowptrs / edge records (global tails) and per-shard (or concatenated) assignment -> dict with the
    global fields of mvgpu_quality plus the per-community arrays (index = global community id) and the compact labels."""
    parts = np.asarray(parts, np.int64)
    nv = int(parts[-1])
    X = np.concatenate([np.asarray(c, np.int64) for c in comm]) if isinstance(comm, (list, tuple)) else np.asarray(comm, np.int64)
    assert len(X) == nv and (nv == 0 or (X.min() >= 0 and X.max() < nv))
    rowptr = np.concatenate([[0]] + [np.asarray(r[1:], np.int64) + off for r, off in
                                     zip(rowptrs, np.cumsum([0] + [int(r[-1]) for r in rowptrs[:-1]]))]).astype(np.int64)
    edges = np.concatenate(edge_lists) if len(edge_lists) else np.zeros(0, np.dtype([("tail", "<i8"), ("weight", "<f8")]))
    src = np.repeat(np.arange(nv, dtype=np.int64), np.diff(rowptr))
    tail = np.asarray(edges["tail"], np.int64)
    w = np.asarray(edges["weight"], np.float64)
    unit = bool(np.all(w == 1.0))
    same = X[src] == X[tail]
    size = np.bincount(X, minlength=nv).astype(np.int64)
    if unit:
        deg = np.diff(rowptr)                                   # exact integers
        vol_i = np.bincount(X, weights=deg, minlength=nv).astype(np.int64)
        internal_i = np.bincount(X[src[same]], minlength=nv).astype(np.int64)
        e_in = float(int(same.sum()))
        a2 = float(sum(int(v) * int(v) for v in vol_i))
        two_m = float(int(deg.sum()))
        volume, internal = vol_i.astype(np.float64), internal_i.astype(np.float64)
    else:
        deg = np.array([math.fsum(w[rowptr[i]:rowptr[i + 1]]) for i in range(nv)])
        volume = np.zeros(nv)
        internal = np.zeros(nv)
        order = np.argsort(X, kind="stable")
        bounds = np.searchsorted(X[order], np.arange(nv + 1))
        for cid in np.nonzero(size)[0]:
            volume[cid] = math.fsum(deg[order[bounds[cid]:bounds[cid + 1]]])
        sel = np.nonzero(same)[0]
        eorder = sel[np.argsort(X[src[sel]], kind="stable")]
        ebounds = np.searchsorted(X[src[eorder]], np.arange(nv + 1))
        for cid in np.unique(X[src[sel]]):
            internal[cid] = math.fsum(w[eorder[ebounds[cid]:ebounds[cid + 1]]])
        e_in = math.fsum(w[same])
        a2 = math.fsum(v * v for v in volume)
        two_m = math.fsum(deg)
    c = 1.0 / two_m
    Q = e_in * c - (a2 * c) * c                                 # Python floats: IEEE double, no contraction
    nonempty = size > 0
    rank = np.cumsum(nonempty) - nonempty
    return {"modularity": Q, "e_in": e_in, "a2": a2, "constant": c, "communities": int(nonempty.sum()),
            "singletons": int((size == 1).sum()), "max_size": int(size.max()) if nv else 0,
            "size": size, "volume": volume, "internal": internal, "compact": rank[X].astype(np.int64)}


def mixed_modularity(q_read, q_written):
    """The reference's currMod of an iteration: fabs(e_in(read)*c - (a2(written)*c)*c) (dspl.hpp:407-456)."""
    c = q_read["constant"]
    return abs(q_read["e_in"] * c - (q_written["a2"] * c) * c)
