"""Probing an assignment on the host (TEST INFRASTRUCTURE): what every vertex would do under the Louvain rule from X
(mvgpu_probe_communities, DESIGN.md §3.15), restated in NumPy on the whole graph from step_ref.step's candidate pairs.

step_ref.step gives every candidate (v, y != X(v)) of every vertex with its gain in the reference's arithmetic (counter
sums in edge order, a_c in global vertex order from 0.0, the truncated self-loop weight).  From those pairs:
    best[v]    the candidate of largest gain, equal gains (of any value) to the smallest id; -1 without a candidate;
    gain[v]    its gain, -inf without a candidate;
    target[v]  best[v] if gain[v] > 0 and the singleton veto (size X(v) = size best = 1 and best > X(v)) does not fire,
               else X(v) -- step_ref.step's target;
and the report's counts.  On unit and dyadic weights every sum is exact, so the device must match this bit for bit."""
import math

import numpy as np

import step_ref as SR

FIELDS = ("vertices", "moves", "vetoed", "interior", "max_gain", "constant")


def constant(G):
    """1/(2m) as a run computes it, for weights whose sums are exact (unit, dyadic)."""
    return 1.0 / math.fsum(G.k)


def probe(G, X, c=None):
    """Returns dict(target, best, gain, and the report fields of FIELDS) for the assignment X of the whole graph G
    (a step_ref.Graph); c defaults to constant(G)."""
    c = constant(G) if c is None else c
    X = np.asarray(X, np.int64)
    n = G.nv
    st = SR.step(G, X, c)
    cv, cy, g = st["pairs"]
    best, gain = np.full(n, -1, np.int64), np.full(n, -np.inf)
    if len(cv):
        order = np.lexsort((cy, -g, cv))                   # per vertex: largest gain, then smallest id
        first = order[np.r_[True, cv[order][1:] != cv[order][:-1]]]
        best[cv[first]], gain[cv[first]] = cy[first], g[first]
    size = st["size"]
    pos = gain > 0.0
    veto = pos & (best > X) & (size[X] == 1) & (size[np.maximum(best, 0)] == 1)
    target = np.where(pos & ~veto, best, X)
    return {"target": target, "best": best, "gain": gain, "vertices": n, "moves": int(np.sum(target != X)),
            "vetoed": int(np.sum(veto)), "interior": int(np.sum((G.deg > 0) & (best < 0))),
            "max_gain": float(gain.max()) if n else -math.inf, "constant": c, "step_target": st["target"]}


def probe_shards(parts, rowptrs, edge_lists, X, c=None):
    return probe(SR.Graph(parts, rowptrs, edge_lists), X, c)
