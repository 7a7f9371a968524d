"""CPU tests on rank counts up to 16, the library's limit, and on splits parts[r] = nv*r/p that leave ranks with one
vertex or none (tests/golden/rank_traces.json, from the unmodified reference).  The C oracle must reproduce every trace on
the reference's own split and on one shard, and the host restatements the GPU tests compare with (quality, split,
compare, update, layout) must give on these splits, empty shards included, what they give on one shard."""
import numpy as np
import pytest

import compare_ref as CR
import layout_ref as LR
import quality_ref as QR
import split_ref as SR
import update_ref as UR
from helpers import assert_trace_matches, case_graph, one_shard, rank_cases
from oracle import oracle as O

CASES = rank_cases()
SMALL = sorted(k for k, c in CASES.items() if c["kind"] == "hand")


def exact(case):
    return "-w" not in case.get("args", [])


def test_rank_goldens_cover_the_edges():
    """Uneven rank counts from 3 to 16, 16-rank splits with empty ranks, and one vertex per rank."""
    assert {3, 5, 6, 7, 9, 12, 15, 16} <= {c["nranks"] for c in CASES.values()}
    empty16 = [k for k, c in CASES.items() if c["nranks"] == 16 and c["nv"] < 16]
    assert len(empty16) >= 3
    parts, _, _, _ = case_graph(CASES["hand_two_triangles_p16"])
    assert int((np.diff(parts) == 0).sum()) == 8
    parts, _, _, _ = case_graph(CASES["hand_path_scrambled_p16"])
    assert np.all(np.diff(parts) == 1)
    for name in SMALL:
        assert len(CASES[name]["comm"]) == CASES[name]["nv"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_rank_golden(name):
    """Bit for bit on the reference's split and on one shard (Euclidean weights: within 1e-6 on one shard, where the
    sums are taken in another order)."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    assert len(parts) == case["nranks"] + 1 and sum(len(e) for e in eds) == case["ne"], name
    for where, (p, r, e) in (("split", (parts, rps, eds)), ("one shard", one_shard(parts, rps, eds))):
        res = O.louvain(p, r, e)
        ex = exact(case) or where == "split"
        assert_trace_matches(case, res["iters"], res["modularity"], res["trace"], res["chash_final"],
                             np.concatenate(res["comm"]), exact=ex)
        if ex:
            assert repr(res["constant"]) == case["constant"], (name, where)


def _assignments(nv, parts):
    """Assignments whose ids name vertices on other ranks, on one-vertex ranks and on nobody's community."""
    v = np.arange(nv, dtype=np.int64)
    rng = np.random.default_rng(nv)
    owners = [int(parts[r]) for r in range(len(parts) - 1) if parts[r + 1] - parts[r] == 1]
    out = {"random": rng.integers(0, nv, nv), "reversed": nv - 1 - v, "all_last": np.full(nv, nv - 1, np.int64)}
    if owners:
        out["one_vertex_ranks"] = np.asarray(owners, np.int64)[v % len(owners)]
    return out


@pytest.mark.parametrize("name", SMALL)
def test_oracle_extensions_on_empty_ranks(name):
    """Warm start, stop / resume and a growing movable set give the same run on the split as on one shard."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    p1, r1, e1 = one_shard(parts, rps, eds)
    nv = int(parts[-1])
    sl = lambda X: [X[parts[r]:parts[r + 1]] for r in range(len(rps))]  # noqa: E731

    def same(a, b, what):
        assert (a["iters"], repr(a["modularity"]), a["chash_final"], a["converged"]) == \
            (b["iters"], repr(b["modularity"]), b["chash_final"], b["converged"]), what
        assert a["trace"].tobytes() == b["trace"].tobytes(), what
        assert np.array_equal(np.concatenate(a["comm"]), np.concatenate(b["comm"])), what
    for aname, X in _assignments(nv, parts).items():
        same(O.louvain(parts, rps, eds, init_comm=sl(X)), O.louvain(p1, r1, e1, init_comm=[X]), (name, aname))
    k = max(1, case["iters"] // 2)
    same(O.louvain(parts, rps, eds, stop_after=k), O.louvain(p1, r1, e1, stop_after=k), (name, "stop"))
    mov = (np.arange(nv) % 3 == 0).astype(np.uint8)
    a = O.louvain(parts, rps, eds, movable=sl(mov), frontier=1)
    b = O.louvain(p1, r1, e1, movable=[mov], frontier=1)
    same(a, b, (name, "movable"))
    assert np.array_equal(np.concatenate(a["movable"]), b["movable"][0]), name


@pytest.mark.parametrize("name", SMALL)
def test_host_references_on_empty_ranks(name):
    """quality_ref, split_ref and compare_ref on the split == on one shard: every field, every per-community array."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    p1, r1, e1 = one_shard(parts, rps, eds)
    nv = int(parts[-1])
    X = np.asarray(case["comm"], np.int64)
    sl = [X[parts[r]:parts[r + 1]] for r in range(len(rps))]
    for Z in (X, np.arange(nv, dtype=np.int64), np.zeros(nv, np.int64)):
        zs = [Z[parts[r]:parts[r + 1]] for r in range(len(rps))]
        a, b = QR.quality(parts, rps, eds, zs), QR.quality(p1, r1, e1, [Z])
        for k in ("modularity", "e_in", "a2", "constant", "communities", "singletons", "max_size"):
            assert repr(a[k]) == repr(b[k]), (name, k)
        for k in ("size", "volume", "internal", "compact"):
            assert np.array_equal(a[k], b[k]), (name, k)
        a, b = SR.split(parts, rps, eds, zs), SR.split(p1, r1, e1, [Z])
        assert np.array_equal(a["Y"], b["Y"]) and [a[k] for k in ("communities", "components", "disconnected")] == \
            [b[k] for k in ("communities", "components", "disconnected")], name
        a, b = CR.compare(sl, zs), CR.compare(X, Z)
        for k in CR.FIELDS:
            assert repr(a[k]) == repr(b[k]), (name, k)
        for k in CR.MATCHES:
            assert np.array_equal(a[k], b[k]), (name, k)
    # the golden's own final modularity is the quality of its final assignment where the sums are exact
    q = QR.quality(parts, rps, eds, sl)
    assert q["constant"] == float(case["constant"])


@pytest.mark.parametrize("name", SMALL)
def test_update_ref_on_empty_ranks(name):
    """A batch routed to its owners (some ranks get none, empty ranks can get none) and applied shard by shard == the
    batch applied to one shard, for both the vectorised restatement and the plain loop."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    p1, r1, e1 = one_shard(parts, rps, eds)
    nv = int(parts[-1])
    rng = np.random.default_rng(nv + 1)
    src = np.repeat(np.arange(nv, dtype=np.int64), np.diff(r1[0]))
    pick = rng.choice(len(src), min(4, len(src)), replace=False) if len(src) else np.zeros(0, np.int64)
    delete = (src[pick], e1[0]["tail"][pick].astype(np.int64))
    a, b = rng.integers(0, nv, 5), rng.integers(0, nv, 5)
    insert = (np.concatenate([a, b]), np.concatenate([b, a]), np.tile(rng.integers(1, 5, 5) / 4.0, 2))
    whole = UR.apply(0, r1[0], e1[0], delete, insert)
    assert all(np.array_equal(x, y) for x, y in zip((whole[0], whole[1].tobytes()),
                                                    (UR.apply_loop(0, r1[0], e1[0], delete, insert)[0],
                                                     UR.apply_loop(0, r1[0], e1[0], delete, insert)[1].tobytes())))
    rp_out, ed_out = [], []
    for r in range(len(rps)):
        lo, hi = int(parts[r]), int(parts[r + 1])
        md = (delete[0] >= lo) & (delete[0] < hi)
        mi = (insert[0] >= lo) & (insert[0] < hi)
        d = (delete[0][md], delete[1][md])
        i = (insert[0][mi], insert[1][mi], insert[2][mi])
        rp, ed = UR.apply(lo, rps[r], eds[r], d, i)
        rl, el = UR.apply_loop(lo, rps[r], eds[r], d, i)
        assert np.array_equal(rp, rl) and ed.tobytes() == el.tobytes(), (name, r)
        rp_out.append(rp)
        ed_out.append(ed)
    _, (rp1,), (ed1,) = one_shard(parts, rp_out, ed_out)
    assert np.array_equal(rp1, whole[0]) and ed1.tobytes() == whole[1].tobytes(), name


@pytest.mark.parametrize("name", SMALL + ["file_rgg_n16384_s1_p16", "rgg_n16384_p16"])
@pytest.mark.parametrize("reorder", [0, 1, 2])
def test_layout_ref_on_empty_ranks(name, reorder):
    """layout_ref on every rank of the split: an empty rank reports an empty compact CSR, no ghosts, keeps order and
    never runs the singleton reduction; the renumbered ranks' labels together are a permutation of the vertex range."""
    case = CASES[name]
    parts, rps, eds, _keep = case_graph(case)
    unit = bool(all(np.all(e["weight"] == 1.0) for e in eds))
    lays = LR.shard_layouts(parts, rps, [e["tail"] for e in eds], None if unit else [e["weight"] for e in eds],
                            reorder=reorder, region_size=32, unit=unit)
    labs = []
    for r, L in enumerate(lays):
        lnv = int(parts[r + 1] - parts[r])
        assert L["lnv"] == lnv and len(L["rowptr"]) == lnv + 1 and L["lne"] == len(eds[r]), (name, r)
        if lnv == 0:
            assert (L["lne"], L["nghost"], L["reordered"], L["first_ran"], L["nregions"]) == (0, 0, 0, 0, 0), (name, r)
            assert "perm" not in L
        if "lab" in L:
            labs.append(L["lab"].astype(np.int64))
            assert np.array_equal(np.sort(L["perm"]), np.arange(lnv)), (name, r)
            if not L["reordered"]:
                assert np.array_equal(L["perm"], np.arange(lnv)), (name, r)      # the keep-order branch
    relabel = lays[0]["relabel"]
    assert all(L["relabel"] == relabel for L in lays)
    if relabel:
        assert np.array_equal(np.sort(np.concatenate(labs)), np.arange(int(parts[-1]))), name
    if reorder == 1:
        assert relabel == 1 and all(L["reordered"] == int(parts[r + 1] > parts[r]) for r, L in enumerate(lays))
