"""One Louvain step on the host (TEST INFRASTRUCTURE): the targets T(X) that one `distExecuteLouvainIteration` computes
from an assignment X, for graphs with any fp64 weights.

Two modes, both in caller numbering on the whole graph (the shards only give the vertex ranges):

fp64 mode (`step`) restates the reference's arithmetic with its roundings.  k_i and every counter sum are summed
sequentially in edge order; the self-loop weight is truncated through `long long`; the community degree a_c is summed
in global vertex order from 0.0, as the C oracle does on a warm start (on the singletons of a cold start it is
k_c itself); the gain is `2.0*(eiy-eix) - ((2.0*k)*(ay-ax))*c` in that order; a candidate wins on a gain strictly
above the best so far, starting from 0, and an equal non-zero gain goes to the smaller id (dspl.hpp:214-219); then
the singleton veto (dspl.hpp:224-225).  All sums are sequential by construction (`seq_sum`: vectorised across groups,
one loop step per position inside a group); no pairwise reduction is used.

Certified mode (`certify`) bounds what the device can compute.  The device's inputs to the gain are
    k_i, sl_i        sequential in edge order: the same bits as above (no error);
    c                given (the device's own 1/(2m), read back);
    e_iy, e_ix       sequential in edge order (the same bits) except on heavy vertices (degree > heavy_deg), where
                     k_scan_heavy adds the weights of one community with fp64 atomics in any order;
    a_c              fp64 atomics from 0.0 over the members' k_i in any order (warm start); exact on a cold start.
For s >= 0 non-negative terms with exact sum S, every order of additions (any tree, starting from 0.0 or not) gives a
result within gamma_{s-1} * S of S, gamma_n = n u / (1 - n u), u = 2^-53 (Higham, Accuracy and Stability, Lemma 3.1
and §4.2).  The sequential sum s^ computed here obeys the same bound, so the device value lies within
2 gamma_{s-1} S <= 2 gamma_{s-1} s^ / (1 - gamma_{s-1}) of s^.  This is the radius used, enlarged by a relative 1e-12
and rounded outward, for e_iy / e_ix of heavy vertices (s <= degree) and for a_c of communities with s >= 3 members.
With s <= 2 the sum is exact whatever the order (0 + a = a, and a + b = b + a is one rounding), so the radius is 0;
all-zero inputs therefore give [0, 0].
The gain is then bounded by evaluating the device's own expression on interval end points, with the device's own
fp64 operations: eix = w0 - sl, ax = a_x - k, de = eiy - eix, da = ay - ax, t1 = 2 de, t2 = ((2k) da) c, g = t1 - t2.
Round-to-nearest is monotone (x <= y implies fl(x) <= fl(y)), each operation is monotone in each argument (2k >= 0,
c > 0), so fl(op(lo-end points)) <= fl(op(x)) <= fl(op(hi-end points)) for every x inside the input intervals: the
expression's own roundings are accounted for exactly, and an input interval of width 0 gives the fp64 gain itself.

From the gain intervals [lo_y, hi_y] of the candidates y of v:
    y certainly beats z       lo_y > hi_z, or lo_y >= hi_z and y < z (equal gains go to the smaller id);
    y may win (before veto)   hi_y > 0 and no candidate certainly beats y;
    staying may win           every lo_y <= 0 (a move needs a gain strictly above 0);
`admissible[v]` is the set of these outcomes with the singleton veto applied (sizes are exact integers), and
`certified[v]` holds when that set has one element.
"""
import math

import numpy as np

U = 2.0 ** -53


def gamma(n):
    n = np.maximum(np.asarray(n, np.float64), 0.0)
    return n * U / (1.0 - n * U)


def seq_sum(group, values, ngroups):
    """Per group g in [0, ngroups): 0.0 + the values of g, added one at a time in the order they are given."""
    group = np.asarray(group, np.int64)
    values = np.asarray(values, np.float64)
    out = np.zeros(ngroups, np.float64)
    if len(group) == 0:
        return out
    order = np.argsort(group, kind="stable")            # groups contiguous, given order kept inside each
    g, v = group[order], values[order]
    start = np.flatnonzero(np.r_[True, g[1:] != g[:-1]])
    rank = np.arange(len(g)) - np.repeat(start, np.diff(np.r_[start, len(g)]))
    by_rank = np.argsort(rank, kind="stable")
    pos = 0
    for cnt in np.bincount(rank):                       # position r of every group at once: no group twice per step
        idx = by_rank[pos:pos + cnt]
        out[g[idx]] += v[idx]
        pos += cnt
    return out


class Graph:
    """The whole graph of the shards (parts, rowptrs, edge lists), with k_i and the truncated self-loop weight."""

    def __init__(self, parts, rowptrs, edge_lists):
        self.parts = np.asarray(parts, np.int64)
        self.nv = nv = int(self.parts[-1])
        self.deg = np.concatenate([np.diff(np.asarray(r, np.int64)) for r in rowptrs])
        assert len(self.deg) == nv
        self.rowptr = np.r_[0, np.cumsum(self.deg)].astype(np.int64)
        e = np.concatenate([np.asarray(x) for x in edge_lists]) if len(edge_lists) else np.zeros(0)
        self.tail = np.asarray(e["tail"], np.int64)
        self.w = np.asarray(e["weight"], np.float64)
        self.src = np.repeat(np.arange(nv, dtype=np.int64), self.deg)
        self.k = seq_sum(self.src, self.w, nv)                                    # dspl.hpp:97-100
        loop = self.tail == self.src
        self.sl = np.trunc(seq_sum(self.src[loop], self.w[loop], nv))           # (GraphElem) cast, dspl.hpp:285,315

    def heavy(self, heavy_deg):
        """Vertices whose degree is above heavy_deg (k_scan_heavy's share); heavy_deg None: none."""
        return np.zeros(self.nv, bool) if heavy_deg is None else self.deg > heavy_deg


def gain(eiy, eix, k, ay, ax, c):
    """dspl.hpp:212 with the reference's association, elementwise in fp64 (numpy does not contract to FMA)."""
    return 2.0 * (eiy - eix) - ((2.0 * k) * (ay - ax)) * c


def _pairs(G, X, edge_order=None):
    """(v, community) groups of v's edges, sorted by (v, community): vertex, community, the counter sum (in edge order,
    or in the order of the permutation edge_order of the edges) and the number of edges."""
    key, inv, cnt = np.unique(G.src * G.nv + X[G.tail], return_inverse=True, return_counts=True)
    o = np.arange(len(inv)) if edge_order is None else np.asarray(edge_order)
    e = seq_sum(inv[o], G.w[o], len(key))
    return key // G.nv, key % G.nv, e, cnt


def _comm(G, X, vertex_order=None):
    size = np.bincount(X, minlength=G.nv)
    o = np.arange(G.nv) if vertex_order is None else np.asarray(vertex_order)
    a = seq_sum(X[o], G.k[o], G.nv)                        # global vertex order, from 0.0 (the C oracle's init_comm)
    return size, a


def step(G, X, c, edge_order=None, vertex_order=None):
    """fp64 mode.  edge_order / vertex_order (permutations, default the identity) reorder the counter sums and the
    community degree sums, for checking the certificate against other orders.  Returns dict(target, moved, size, a,
    pairs = (v, y, gain) of every candidate, sorted by (v, y))."""
    X = np.asarray(X, np.int64)
    pv, pc, e, _cnt = _pairs(G, X, edge_order)
    own = pc == X[pv]
    w0 = np.zeros(G.nv)
    w0[pv[own]] = e[own]
    size, a = _comm(G, X, vertex_order)
    eix = w0 - G.sl
    ax = a[X] - G.k
    cv, cy, ce = pv[~own], pc[~own], e[~own]
    g = gain(ce, eix[cv], G.k[cv], a[cy], ax[cv], c)
    pairs = (cv, cy, g)
    T = X.copy()
    pos = g > 0.0
    cv, cy, g = cv[pos], cy[pos], g[pos]
    order = np.lexsort((cy, -g, cv))                       # per vertex: largest gain, then smallest id
    first = order[np.r_[True, cv[order][1:] != cv[order][:-1]]] if len(order) else order
    T[cv[first]] = cy[first]
    veto = (T > X) & (size[X] == 1) & (size[T] == 1)
    T[veto] = X[veto]
    return {"target": T, "moved": int(np.sum(T != X)), "size": size, "a": a, "pairs": pairs}


def _radius(s, n):
    """Rigorous distance between the sequential sum s of n non-negative terms and any other order's sum."""
    gm = gamma(n - 1)
    return np.where(n >= 2, 2.0 * gm * s / (1.0 - gm) * (1.0 + 1e-12), 0.0)


def _widen(x, r):
    lo = np.where(r > 0, np.maximum(np.nextafter(x - r, -np.inf), 0.0), x)
    hi = np.where(r > 0, np.nextafter(x + r, np.inf), x)
    return lo, hi


def certify(G, X, c, heavy_deg=None):
    """Certified mode.  Returns dict(certified (bool per vertex), outcome (the certified target, or -1), admissible
    (v -> set of outcomes, for the vertices that are not certified), heavy, exact (not heavy, and the own and every
    candidate community have at most 2 members: every input of the decision is exact), pairs (the candidates' gain
    intervals))."""
    X = np.asarray(X, np.int64)
    heavy = G.heavy(heavy_deg)
    pv, pc, e, cnt = _pairs(G, X)
    e_lo, e_hi = _widen(e, np.where(heavy[pv], _radius(e, cnt), 0.0))
    own = pc == X[pv]
    w0_lo, w0_hi = np.zeros(G.nv), np.zeros(G.nv)
    w0_lo[pv[own]], w0_hi[pv[own]] = e_lo[own], e_hi[own]
    size, a = _comm(G, X)
    a_lo, a_hi = _widen(a, _radius(a, np.where(size >= 3, size, 0)))
    eix_lo, eix_hi = w0_lo - G.sl, w0_hi - G.sl
    ax_lo, ax_hi = a_lo[X] - G.k, a_hi[X] - G.k
    cv, cy = pv[~own], pc[~own]
    de_lo, de_hi = e_lo[~own] - eix_hi[cv], e_hi[~own] - eix_lo[cv]
    da_lo, da_hi = a_lo[cy] - ax_hi[cv], a_hi[cy] - ax_lo[cv]
    k2 = 2.0 * G.k[cv]
    g_lo = 2.0 * de_lo - (k2 * da_hi) * c
    g_hi = 2.0 * de_hi - (k2 * da_lo) * c
    exact = ~heavy & (size[X] <= 2)
    exact[cv[size[cy] > 2]] = False

    # fast path: the candidate with the largest lo (smallest id among equals) certainly beats every other one
    n = G.nv
    order = np.lexsort((cy, -g_lo, cv))
    head = order[np.r_[True, cv[order][1:] != cv[order][:-1]]] if len(order) else order
    best_y, best_lo = np.full(n, -1), np.full(n, -np.inf)
    best_y[cv[head]], best_lo[cv[head]] = cy[head], g_lo[head]
    other = cy != best_y[cv]
    beaten = (best_lo[cv] > g_hi) | ((best_lo[cv] >= g_hi) & (best_y[cv] < cy))
    fails = np.bincount(cv[other & ~beaten], minlength=n)
    any_pos_hi = np.bincount(cv[g_hi > 0.0], minlength=n) > 0
    move_sure = (best_lo > 0.0) & (fails == 0)
    stay_sure = ~any_pos_hi

    def veto(v, t):
        return int(X[v]) if (t > X[v] and size[X[v]] == 1 and size[t] == 1) else int(t)

    certified = move_sure | stay_sure
    outcome = np.where(stay_sure, X, -1)
    mv = np.flatnonzero(move_sure)
    outcome[mv] = [veto(v, best_y[v]) for v in mv] if len(mv) else outcome[mv]
    admissible = {}
    start = np.searchsorted(cv, np.arange(n + 1))           # cv is sorted: _pairs returns (v, community) in order
    for v in np.flatnonzero(~certified):
        sl_ = slice(start[v], start[v + 1])
        ys, lo, hi = cy[sl_], g_lo[sl_], g_hi[sl_]
        beats = (lo[:, None] > hi[None, :]) | ((lo[:, None] >= hi[None, :]) & (ys[:, None] < ys[None, :]))
        can = (hi > 0.0) & ~beats.any(axis=0)
        outs = {veto(v, y) for y in ys[can]}
        if np.all(lo <= 0.0):
            outs.add(int(X[v]))
        admissible[int(v)] = outs
        if len(outs) == 1:
            certified[v] = True
            outcome[v] = next(iter(outs))
            del admissible[int(v)]
    return {"certified": certified, "outcome": outcome, "admissible": admissible, "heavy": heavy, "exact": exact,
            "pairs": (cv, cy, g_lo, g_hi), "size": size}


def admits(cert, v, t):
    return int(cert["outcome"][v]) == int(t) if cert["certified"][v] else int(t) in cert["admissible"][int(v)]


def fsum_groups(group, values, ngroups):
    """Per group, the correctly rounded sum of its values (math.fsum)."""
    o = np.argsort(group, kind="stable")
    b = np.searchsorted(np.asarray(group)[o], np.arange(ngroups + 1))
    v = np.asarray(values, np.float64)[o]
    return np.array([math.fsum(v[b[i]:b[i + 1]]) if b[i + 1] > b[i] else 0.0 for i in range(ngroups)])


def _q_error(e, err_e, a2, err_a, c, q):
    """Distance between |e c - a2 c^2| and its fp64 evaluation |fl(fl(e^ c) - fl(fl(a2^ c) c))| (the reference's
    association, dspl.hpp:447-448) from inputs with |e^ - e| <= err_e, |a2^ - a2| <= err_a: each product adds one
    rounding (two for the c^2 term: gamma_2), the subtraction one more."""
    E1 = c * err_e + U * (e + err_e) * c
    E2 = c * c * err_a + float(gamma(2)) * (a2 + err_a) * c * c
    return E1 + E2 + U * (q + E1 + E2)


def _a2_error(a, dlt, depth):
    """Error of a sum of the n leaves fl(a^_c^2), |a^_c - a_c| <= dlt_c, added in a tree of the given depth:
    per leaf |a^^2 - a^2| <= 2 a dlt + dlt^2 plus the square's own rounding u (a + dlt)^2, then gamma_depth of the sum."""
    sq = (a + dlt) ** 2
    return math.fsum(2.0 * a * dlt + dlt * dlt + U * sq) + float(gamma(depth)) * math.fsum(sq)


def modularity_bound(G, X, T, c):
    """(q, B, e_in): q = |e_in(X) c - a2(T) c^2| evaluated in fp64 from math.fsum sums, and B bounding |q_dev - q| for
    the device's trace modularity q_dev, as the sum of both evaluations' distances from the exact value.

    Device.  e_in is a sum over the n vertices of counter[0] (leaf v: d_v non-negative terms in edge order, or in any
    order on a heavy vertex: within gamma_{d_v - 1}); the per-thread, warp, CTA, atomic and cross-rank additions form a
    tree over those n leaves, which has depth at most n - 1.  So |e^ - e| <= gamma_{maxdeg + n - 2} e.  a_c(T) is
    fl(a_c(X) + u_c): a_c(X) from the warm-start atomics over s members (within gamma_{s-1} a_c(X); exact for s <= 2
    and on a cold start), u_c the atomic sum from 0.0 of the m movers' +-k_i (within gamma_{m-1} times the sum of their
    k_i), then one rounding of the addition; a2 is a tree over the n squared community degrees (depth n - 1).
    Host.  fsum is correctly rounded: e_in and each a_c within u of the exact value, and the sum of the rounded squares
    within u.
    B itself is a sum of non-negative terms evaluated in fp64 with fewer than 40 roundings of at most u each; the
    factor 1 + 2^-40 (>= (1 + u)^40) covers them and the use of the rounded e_in, a_c as magnitudes."""
    X, T = np.asarray(X, np.int64), np.asarray(T, np.int64)
    n = G.nv
    own = X[G.src] == X[G.tail]
    e_in = math.fsum(G.w[own])
    maxdeg = int(G.deg.max()) if n else 1
    sX = np.bincount(X, minlength=n)
    aX, aT = fsum_groups(X, G.k, n), fsum_groups(T, G.k, n)
    moved = T != X
    flow = np.bincount(T[moved], weights=G.k[moved], minlength=n) + np.bincount(X[moved], weights=G.k[moved], minlength=n)
    nmov = np.bincount(T[moved], minlength=n) + np.bincount(X[moved], minlength=n)
    e1 = np.where(sX >= 3, gamma(sX - 1) * aX, 0.0)
    e2 = gamma(nmov - 1) * flow
    dlt_dev = e1 + e2 + U * (aT + e1 + e2)
    a2 = math.fsum(aT * aT)
    q = abs(e_in * c - a2 * c * c)
    dev = _q_error(e_in, float(gamma(maxdeg + n - 2)) * e_in, a2, _a2_error(aT, dlt_dev, n - 1), c, q)
    host = _q_error(e_in, U * e_in, a2, _a2_error(aT, U * aT, 1), c, q)
    return q, (dev + host) * (1.0 + 2.0 ** -40), e_in
