"""Witness graphs of the float build (TEST INFRASTRUCTURE): small exact graphs on which the reference's
USE_32_BIT_GRAPH build and its double build decide differently, used by tests/golden/make_golden_f32_witness.py and the
tests that read tests/golden/f32_witness_traces.json.

A spec is a dict {nv, denom, edges: [[a, b, m], ...], fill: [first, pairs, mult]}.  Every [a, b, m] is an undirected
edge a - b of m units: m parallel unit edges when denom is 1 (a multigraph on the integer path), one edge of weight
m / denom otherwise (a simple graph on the weighted path).  `fill` appends `pairs` disjoint pairs (first + 2p,
first + 2p + 1) of `mult` units each: they only raise 2m, which the witness conditions are solved for.

The witness vertex i sees two candidates y1 < y2 < i with gains g1 < g2 that float rounds to one value.  Iteration 1
from singletons gives g = 2 w - 2 k_i d c for a candidate of w units and degree d, so
    g2 - g1 = (2 / 2m) K,   K = 2m (w2 - w1) - k_i (d2 - d1).
With K = 1 the double build moves i to y2 and the float build, seeing a tie, to the smaller label y1.  With K = 0 the
two gains are equal and the double build is decided by the rounding of c = 1/(2m) alone."""
import numpy as np

from minivite_b200 import hostgraph as hg


def graph(spec):
    """(nv, rowptr, edges) in caller numbering: edges sorted by (source, tail), both directions of every edge."""
    nv, den = int(spec["nv"]), int(spec["denom"])
    ed = np.asarray(spec["edges"], np.int64).reshape(-1, 3)
    first, pairs, mult = spec.get("fill", (0, 0, 0))
    if pairs:
        a = first + 2 * np.arange(pairs, dtype=np.int64)
        ed = np.concatenate([ed, np.stack([a, a + 1, np.full(pairs, mult, np.int64)], 1)])
    a, b, m = ed[:, 0], ed[:, 1], ed[:, 2]
    assert np.all(a != b) and np.all(m > 0) and max(a.max(), b.max()) < nv
    if den == 1:
        a, b, w = np.repeat(a, m), np.repeat(b, m), np.ones(int(m.sum()))
    else:
        w = m / float(den)
    src, dst, w = np.r_[a, b], np.r_[b, a], np.r_[w, w]
    o = np.lexsort((dst, src))
    edges = np.zeros(len(o), hg.EDGE_DTYPE)
    edges["tail"], edges["weight"] = dst[o], w[o]
    rowptr = np.r_[0, np.cumsum(np.bincount(src, minlength=nv))].astype(np.int64)
    return nv, rowptr, edges


def units(spec):
    """2m in units of 1 / denom."""
    ed = np.asarray(spec["edges"], np.int64).reshape(-1, 3)
    first, pairs, mult = spec.get("fill", (0, 0, 0))
    return 2 * (int(ed[:, 2].sum()) + pairs * mult)


def _fill(spec, total, mult):
    """Pad spec with pairs so that 2m = total units: full pairs of `mult`, then one pair of the rest."""
    rest = total // 2 - units(spec) // 2
    assert total % 2 == 0 and rest >= 0, (total, units(spec))
    pairs, last = divmod(rest, mult)
    first = spec["nv"]
    spec["fill"] = [first, pairs, mult]
    spec["nv"] = first + 2 * pairs
    if last:
        spec["edges"].append([spec["nv"], spec["nv"] + 1, last])
        spec["nv"] += 2
    return spec


def iteration1(k, delta, K=1, mult=100, denom=1):
    """Iteration-1 witness: y1 = 0, y2 = 1, a pad P1 = 2 that gives y1 delta - 1 more units than i does, pairs, and i
    last.  i has w1 = (k + 1) / 2 units to y1 and w2 = w1 - 1 to y2 (k odd), so d1 - d2 = delta and
    K = -2m + k delta: 2m = k delta - K.  y1, y2 and P1 have no choice that a float rounding could change (y1 and y2
    see only larger labels and stay; P1 sees only y1), nor has a pair."""
    assert k % 2 == 1
    w1 = (k + 1) // 2
    assert delta > 1
    spec = {"nv": 3, "denom": denom, "edges": [[0, 2, delta - 1]]}
    spec = _fill(spec, k * delta - K - 2 * k, mult)
    i = spec["nv"]
    spec["nv"] += 1
    spec["edges"] += [[i, 0, w1], [i, 1, w1 - 1]]
    assert units(spec) == k * delta - K
    return spec, i, 0, 1


def iteration2(w2, s, t, q1, r, mult=100, denom=1):
    """Witness in iteration 2: y1 = 0, y2 = 1, P1 = 2 (q1 units to y1 only: joins y1), u = 3 (r units to z only),
    pairs, then i, j (s units to i only: joins i), z (t units to i, r to u: joins u).  In iteration 1 i's best is z,
    a larger singleton, so the singleton veto keeps i in place, and j joins it.  In iteration 2 i sits in {i, j}
    (eix = s, ax = s) and weighs Y1 = {y1, P1} (w1 = w2 + 1 units, degree w1 + 2 q1) against Y2 = {y2} (w2 units,
    degree w2): K = -2m + k_i (1 + 2 q1), so 2m = k_i (1 + 2 q1) - 1."""
    w1 = w2 + 1
    k = w1 + w2 + s + t
    spec = {"nv": 4, "denom": denom, "edges": [[0, 2, q1]]}
    two_m = k * (1 + 2 * q1) - 1
    spec = _fill(spec, two_m - 2 * (k + r), mult)
    i = spec["nv"]
    spec["nv"] += 3
    spec["edges"] += [[i, 0, w1], [i, 1, w2], [i, i + 1, s], [i, i + 2, t], [3, i + 2, r]]
    assert units(spec) == two_m
    return spec, i, 0, 1
