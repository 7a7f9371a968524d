"""CPU tests of tests/layout_ref.py, the host restatement that pins the device layout (tests/test_gpu_layout.py): its
level-synchronous BFS against a deliberately naive one (one BFS per seed, then the (distance, region) minimum per vertex),
the invariants of the layout it derives, and the arithmetic of the auto decision and of the region-stride clamp."""
from collections import deque

import numpy as np
import pytest

import layout_ref as LR
from helpers import random_graph


def naive_keys(lnv, rowptr, tails, stride, max_level=LR.MAX_LEVELS):
    best = [None] * lnv
    for s in range(0, lnv, stride):
        dist = [-1] * lnv
        dist[s] = 0
        dq = deque([s])
        while dq:
            u = dq.popleft()
            for e in range(int(rowptr[u]), int(rowptr[u + 1])):
                w = int(tails[e])
                if w < lnv and dist[w] < 0:
                    dist[w] = dist[u] + 1
                    dq.append(w)
        for v in range(lnv):
            if dist[v] >= 0 and (best[v] is None or (dist[v], s // stride) < best[v]):
                best[v] = (dist[v], s // stride)
    return np.array([LR.UNREACHED if b is None or b[0] > max_level else (b[0] << LR.REGION_BITS) | b[1] for b in best],
                    np.uint32)


def csr_from_lists(adj):
    rowptr = np.concatenate([[0], np.cumsum([len(a) for a in adj])]).astype(np.int64)
    tails = np.array([t for a in adj for t in a], np.int64)
    return rowptr, tails


def path(n):
    return csr_from_lists([[v - 1] * (v > 0) + [v + 1] * (v + 1 < n) for v in range(n)])


def union(*graphs):
    adj, off = [], 0
    for rowptr, tails in graphs:
        n = len(rowptr) - 1
        adj += [[int(t) + off for t in tails[rowptr[v]:rowptr[v + 1]]] for v in range(n)]
        off += n
    return csr_from_lists(adj)


def with_ghost_tails(rowptr, tails, nghost, seed):
    """Append a random ghost slot (>= lnv) to some rows: the BFS must never follow them."""
    rng = np.random.default_rng(seed)
    n = len(rowptr) - 1
    adj = [list(tails[rowptr[v]:rowptr[v + 1]]) for v in range(n)]
    for v in rng.choice(n, n // 3, replace=False):
        adj[v].append(n + int(rng.integers(0, nghost)))
    return csr_from_lists(adj)


def small_graphs():
    out = {}
    rp, ed = random_graph(600, 3, 1)                              # sparse: isolated vertices, many components
    out["random_sparse"] = (rp, ed["tail"].astype(np.int64))
    rp, ed = random_graph(500, 6, 2, self_loops=30, multi=40)
    out["loops_multi"] = (rp, ed["tail"].astype(np.int64))
    out["path_1100"] = path(1100)                                 # one seed: levels 256 .. 1023 and beyond
    ring = csr_from_lists([[(v + 1) % 90, (v + 7) % 90] for v in range(90)])
    out["components"] = union(path(40), csr_from_lists([[] for _ in range(7)]), path(300), ring)
    out["tiny"] = csr_from_lists([[1], [0, 2], [1], []])          # lnv < stride
    rng = np.random.default_rng(4)                                # directed: out-edges only
    out["directed"] = csr_from_lists([sorted(set(rng.integers(0, 1000, rng.integers(0, 4)).tolist())) for _ in range(1000)])
    rp, ed = random_graph(700, 4, 5)
    out["ghosts"] = with_ghost_tails(rp, ed["tail"].astype(np.int64), 50, 6)
    return out


@pytest.mark.parametrize("name", ["random_sparse", "loops_multi", "path_1100", "components", "tiny", "directed", "ghosts"])
@pytest.mark.parametrize("stride", [32, 96, 512, 100000])
def test_bfs_keys_match_naive_bfs(name, stride):
    rowptr, tails = small_graphs()[name]
    lnv = len(rowptr) - 1
    key = LR.bfs_keys(lnv, rowptr, tails, stride)
    assert np.array_equal(key, naive_keys(lnv, rowptr, tails, stride)), name


def test_path_levels_clamp_and_run_out():
    """One seed on a 2 500-vertex path: levels above 255 share the clamped sort key, levels above 1023 are unreached and
    sort last in id order."""
    rowptr, tails = path(2500)
    key = LR.bfs_keys(2500, rowptr, tails, 4096)
    assert np.array_equal(key[:1024], (np.arange(1024) << LR.REGION_BITS).astype(np.uint32))
    assert np.all(key[1024:] == LR.UNREACHED)
    sk = LR.sort_keys(key, 1)
    assert np.all(sk[255:1024] == 255) and np.all(sk[1024:] == (1 << LR.sort_bits_of(1)) - 1)
    perm = np.argsort(sk, kind="stable")
    assert np.array_equal(perm, np.arange(2500))


@pytest.mark.parametrize("name", ["random_sparse", "loops_multi", "path_1100", "components", "directed", "ghosts"])
@pytest.mark.parametrize("stride", [32, 96, 512])
def test_layout_invariants(name, stride):
    rowptr, tails = small_graphs()[name]
    lnv = len(rowptr) - 1
    parts = np.array([0, lnv], np.int64)
    lay = LR.layout(parts, rowptr, np.where(tails < lnv, tails, 0), reorder=1, region_size=stride)
    perm, inv, key = lay["perm"], lay["inv"], lay["bfs_key"].astype(np.int64)
    assert np.array_equal(np.sort(perm), np.arange(lnv))
    assert np.array_equal(inv[perm], np.arange(lnv)) and np.array_equal(lay["lab"], perm)
    k = key[perm]
    reached = k != LR.UNREACHED
    nreach = int(reached.sum())
    assert np.all(reached[:nreach]) and not np.any(reached[nreach:])  # unreached last ...
    assert np.all(np.diff(perm[nreach:]) > 0)                           # ... in id order
    region, level = k[:nreach] & ((1 << LR.REGION_BITS) - 1), np.minimum(k[:nreach] >> LR.REGION_BITS, 255)
    assert np.all(np.diff(region) >= 0)                                 # regions contiguous, ascending
    same = np.diff(region) == 0
    assert np.all(np.diff(level)[same] >= 0)                            # levels non-decreasing inside a region
    # the renumbered CSR is the old one relabelled: every edge (u, t) appears as (inv u, inv t)
    rp2, t2 = lay["rowptr2"].astype(np.int64), lay["tails2"].astype(np.int64)
    for i in range(0, lnv, 37):
        o = perm[i]
        old = lay["tails"][lay["rowptr"][o]:lay["rowptr"][o + 1]].astype(np.int64)
        assert np.array_equal(t2[rp2[i]:rp2[i + 1]], inv[old])


def test_compact_csr_and_tails_ascend_with_ghosts():
    """Rank 1 of 3 (ids 10..19): ghosts 3, 7 (below base) and 25 (above) get slots 10, 11, 12; nlow = 2.  Rows ordered
    by global id stay in tails_ascend order; a row listing an upper ghost before an own vertex does not."""
    parts = np.array([0, 10, 20, 30], np.int64)
    rowptr = np.concatenate([[0, 4], np.full(9, 4)]).astype(np.int64)
    tails = np.array([3, 7, 12, 25], np.int64)
    rp, slots, nlow, ghosts = LR.compact_csr(parts, rowptr, tails, 1)
    assert list(ghosts) == [3, 7, 25] and nlow == 2 and list(slots) == [10, 11, 2, 12]
    assert not LR.out_of_order(rp, slots, 10, nlow)
    assert LR.out_of_order(rp, np.array([10, 11, 12, 2], np.int32), 10, nlow)
    assert LR.out_of_order(rp, np.array([10, 10, 2, 12], np.int32), 10, nlow)   # parallel edge
    lay = LR.layout(parts, rowptr, tails, rank=1, reorder=1, region_size=32)
    assert list(lay["tails2"]) == [10, 11, int(lay["inv"][2]), 12]


def test_auto_decision_arithmetic():
    """lnv >= 65536, at least one own sampled edge, and mean span > lnv/64 in double."""
    assert not LR.auto_wants(65535, 10 ** 9, 1)
    assert not LR.auto_wants(65536, 0, 0)
    assert LR.auto_wants(65536, 1025, 1) and not LR.auto_wants(65536, 1024, 1)
    assert LR.auto_wants(65536, 5121, 5) and not LR.auto_wants(65536, 5120, 5)
    # the sample: rows 0, 64, ...; only tails < lnv count
    rowptr = np.arange(0, 2 * 65536 + 1, 2, dtype=np.int64)
    tails = np.zeros(2 * 65536, np.int64)
    tails[1::2] = 70000                                          # a ghost slot on every row: ignored
    s, c = LR.span_sample(65536, rowptr, tails)
    assert c == 1024 and s == sum(range(0, 65536, 64))


def test_region_stride_clamp():
    """Region ids have 22 bits.  Without the clamp a shard of more than (2^22 - 1) * region_size vertices would give
    region 2^22 - 1, whose key at level 1023 is the unreached marker; the clamp keeps every region id below it."""
    m = LR.MAX_REGIONS
    assert LR.effective_stride(1000, 32) == 32
    assert LR.effective_stride(32 * m, 32) == 32 and LR.nregions_of(32 * m, 32) == m
    assert LR.effective_stride(32 * m + 1, 32) == 33
    for lnv in (32 * m + 1, 33 * m, 2 ** 31 - 1):
        for region_size in (32, 64, 512):
            st = LR.effective_stride(lnv, region_size)
            nreg = LR.nregions_of(lnv, st)
            assert nreg <= m and (LR.MAX_LEVELS << LR.REGION_BITS) | (nreg - 1) != LR.UNREACHED
            assert LR.sort_bits_of(nreg) <= 32
    unclamped = LR.nregions_of(32 * (m + 1), 32) - 1               # what region_size=32 alone would give
    assert (LR.MAX_LEVELS << LR.REGION_BITS) | unclamped == LR.UNREACHED


def test_keep_order_branch_and_first_gate():
    rowptr, ed = random_graph(3000, 5, 7)
    tails = ed["tail"].astype(np.int64)
    parts = np.array([0, 3000], np.int64)
    lay = LR.layout(parts, rowptr, tails, reorder=0, relabel=True)
    assert lay["want"] == 0 and lay["relabel"] == 1 and lay["reordered"] == 0 and "bfs_key" not in lay
    assert np.array_equal(lay["perm"], np.arange(3000)) and np.array_equal(lay["inv"], np.arange(3000))
    assert lay["simple_sorted"] == 1 and lay["first_ran"] == 1
    assert LR.layout(parts, rowptr, tails, reorder=0, first_iter=0)["first_ran"] == 0
    assert LR.layout(parts, rowptr, tails, reorder=0, scan_variant=3)["first_ran"] == 0
    assert LR.layout(parts, rowptr, tails, reorder=0, f32=True)["first_ran"] == 0
    rp2, ed2 = random_graph(3000, 5, 7, self_loops=1)
    assert LR.layout(parts, rp2, ed2["tail"], reorder=1)["has_self"] == 1
    rp3, ed3 = random_graph(3000, 5, 7, multi=1)
    lay3 = LR.layout(parts, rp3, ed3["tail"], reorder=1)
    assert lay3["unordered"] == 1 and lay3["simple_sorted"] == 0 and lay3["first_ran"] == 0
