"""CPU tests of the shard-update semantics (tests/update_ref.py, DESIGN.md §3.11): the vectorised restatement equals a
plain per-row loop, and it turns the host generator's `-p 0` shards into its `-p 5` shards and back, byte for byte."""
import numpy as np
import pytest

import update_ref as U
from helpers import random_graph, reversed_adjacency
from minivite_b200 import hostgraph as hg


def csr(rows):
    """rows: list of lists of (tail, weight) -> rowptr, edges."""
    rowptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    e = np.zeros(int(rowptr[-1]), U.EDGE_DTYPE)
    flat = [x for r in rows for x in r]
    if flat:
        e["tail"] = [t for t, _ in flat]
        e["weight"] = [w for _, w in flat]
    return rowptr, e


def same(a, b):
    return np.array_equal(a[0], b[0]) and a[1].tobytes() == b[1].tobytes()


def check(base, rowptr, edges, delete=None, insert=None):
    got = U.apply(base, rowptr, edges, delete, insert)
    ref = U.apply_loop(base, rowptr, edges, delete, insert)
    assert same(got, ref)
    return got


def batch(src, dst, w=None):
    cols = [np.array(src, np.int64), np.array(dst, np.int64)]
    return tuple(cols) if w is None else tuple(cols + [np.array(w, np.float64)])


# rows of vertex 10..13 (base 10) of a 20-vertex graph: row 0 unsorted, row 1 with parallel records and a self loop,
# row 2 empty, row 3 sorted
HAND = [[(5, 1.0), (2, 2.0), (7, 3.0), (2, 4.0)],
        [(3, 1.0), (3, 0.5), (11, 2.0), (15, 1.0)],
        [],
        [(0, 1.0), (4, 1.0), (9, 1.0)]]

HAND_CASES = {
    "empty batch": (None, None),
    "delete parallel records": (batch([11], [3]), None),
    "delete self loop": (batch([11], [11]), None),
    "delete absent pair and duplicates": (batch([10, 10, 10, 13], [2, 2, 19, 5]), None),
    "empty a row": (batch([13, 13, 13], [0, 4, 9]), None),
    "insert into unsorted row": (None, batch([10, 10, 10, 10], [6, 2, 0, 9], [0.1, 0.2, 0.3, 0.4])),
    "insert duplicates keep batch order": (None, batch([11, 11, 11], [3, 3, 11], [7.0, 8.0, 9.0])),
    "insert into empty row": (None, batch([12, 12], [1, 0], [1.0, 2.0])),
    "replace = delete + insert": (batch([13], [4]), batch([13], [4], [0.25])),
    "everything": (batch([10, 11, 12, 13], [2, 3, 0, 9]),
                   batch([13, 10, 11, 12, 10, 13], [9, 2, 11, 5, 5, 1], [1.5, 2.5, 3.5, 4.5, 5.5, 6.5])),
}


@pytest.mark.parametrize("name", list(HAND_CASES))
def test_hand_cases_match_loop(name):
    rowptr, edges = csr(HAND)
    check(10, rowptr, edges, *HAND_CASES[name])


def test_hand_case_values():
    rowptr, edges = csr(HAND)
    rp, e = check(10, rowptr, edges, batch([11], [3]), batch([10, 11, 11], [2, 3, 20 - 1], [9.0, 6.0, 5.0]))
    # row 0 (5,2,7,2) + ins 2: old 5 > 2 -> ins first; row 1 loses both 3s, gains 3 at the front and 19 at the end
    assert rp.tolist() == [0, 5, 9, 9, 12]
    assert e["tail"].tolist() == [2, 5, 2, 7, 2, 3, 11, 15, 19, 0, 4, 9]
    assert e["weight"].tolist() == [9.0, 1.0, 2.0, 3.0, 4.0, 6.0, 2.0, 1.0, 5.0, 1.0, 1.0, 1.0]


def random_batch(rng, base, lnv, nv, rowptr, edges, nd, ni):
    """Deletions half drawn from existing records (so they hit), half at random; insertions at random, with repeats."""
    lne = len(edges)
    row = np.repeat(np.arange(lnv), np.diff(rowptr))
    pick = rng.integers(0, max(lne, 1), nd // 2) if lne else np.zeros(0, np.int64)
    ds = np.concatenate([row[pick] + base, rng.integers(base, base + lnv, nd - len(pick))])
    dd = np.concatenate([edges["tail"][pick], rng.integers(0, nv, nd - len(pick))])
    is_ = rng.integers(base, base + lnv, ni)
    id_ = rng.integers(0, nv, ni)
    rep = rng.integers(0, max(ni, 1), ni // 4) if ni else np.zeros(0, np.int64)
    id_[rep[: len(rep) // 2]] = id_[rep[len(rep) // 2: 2 * (len(rep) // 2)]]    # some repeated pairs
    is_[rep[: len(rep) // 2]] = is_[rep[len(rep) // 2: 2 * (len(rep) // 2)]]
    iw = rng.integers(1, 17, ni) / 8.0
    return (ds, dd), (is_, id_, iw)


@pytest.mark.parametrize("seed", range(6))
def test_random_multigraphs_match_loop(seed):
    rng = np.random.default_rng(seed)
    n = 300
    rowptr, edges = random_graph(n, 6, seed, hubs=2, hub_deg=80, self_loops=20, multi=40, dyadic=True)
    for v in rng.integers(0, n, 30):                       # unsorted rows
        edges = reversed_adjacency(rowptr, edges, int(v))
    base, lnv = 100, 120                                   # a middle strip of the graph
    rp = rowptr[base:base + lnv + 1] - rowptr[base]
    ed = edges[rowptr[base]:rowptr[base + lnv]]
    for nd, ni in ((0, 0), (50, 0), (0, 50), (200, 300), (2000, 10)):
        d, i = random_batch(rng, base, lnv, n, rp, ed, nd, ni)
        check(base, rp, ed, d, i)


def test_delete_everything_and_batch_bigger_than_shard():
    rowptr, edges = random_graph(200, 4, 3, self_loops=5, multi=10)
    row = np.repeat(np.arange(200), np.diff(rowptr))
    rp, e = check(0, rowptr, edges, (row, edges["tail"].copy()))
    assert len(e) == 0 and not rp.any()
    rng = np.random.default_rng(0)
    big = (rng.integers(0, 200, 5 * len(edges)), rng.integers(0, 200, 5 * len(edges)), np.ones(5 * len(edges)))
    rp, e = check(0, rowptr, edges, (row, edges["tail"].copy()), big)
    assert len(e) == len(big[0])


@pytest.mark.parametrize("n,p,unit", [(16384, 1, True), (16384, 1, False), (16384, 2, True), (32768, 2, False),
                                      (16384, 4, True), (32768, 4, False)])
def test_generator_relation(n, p, unit):
    """The host generator's `-p 5` shard is its `-p 0` shard plus the extra records as one insertion batch, and the
    extras as a deletion batch take it back -- on every strip, with unit and Euclidean weights."""
    s0 = hg.generate_rgg(n, p, unit_weight=unit)
    s5 = hg.generate_rgg(n, p, unit_weight=unit, random_edge_percent=5)
    try:
        for a, b in zip(s0.shards, s5.shards):
            src, dst, w = U.extras(a, b)
            assert len(src) == b.lne - a.lne > 0
            # precondition: no extra pair is an RGG pair (so deleting the extras cannot touch an RGG record)
            rs = np.repeat(np.arange(a.lnv, dtype=np.int64), np.diff(a.rowptr)) + a.base
            assert not np.isin(src * (n + 1) + dst, rs * (n + 1) + a.edges["tail"]).any()
            assert same(U.apply(a.base, a.rowptr, a.edges, insert=(src, dst, w)), (b.rowptr, b.edges))
            assert same(U.apply(b.base, b.rowptr, b.edges, delete=(src, dst)), (a.rowptr, a.edges))
    finally:
        s0.close()
        s5.close()


def test_generator_relation_matches_loop():
    s0 = hg.generate_rgg(2048, 2, unit_weight=False)
    s5 = hg.generate_rgg(2048, 2, unit_weight=False, random_edge_percent=20)
    try:
        for a, b in zip(s0.shards, s5.shards):
            src, dst, w = U.extras(a, b)
            check(a.base, a.rowptr, a.edges, None, (src, dst, w))
            check(b.base, b.rowptr, b.edges, (src, dst), None)
    finally:
        s0.close()
        s5.close()
