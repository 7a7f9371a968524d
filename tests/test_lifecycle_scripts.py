"""The sequences of tests/test_gpu_context_lifecycle.py cross the boundaries they claim -- asserted from the scripts and the
host graphs alone, without a GPU (the discipline of test_scan_schedule.py)."""
import pytest

import lifecycle as L


def run_kinds(steps):
    """The kind of each shard a run happened on, consecutive runs on one shard counted once."""
    out, last = [], None
    for i, st, cur, _o, _m in L.shard_states(steps):
        if st[0] == "load":
            last = None
        if st[0] == "run" and last is None:
            kind = "updated" if cur["kind"] == "updated" else next(s[1] for s in reversed(steps[:i]) if s[0] == "load")["kind"]
            out.append(kind)
            last = kind
    return out


def test_every_ordered_pair_of_shard_kinds_on_one_rank():
    kinds = run_kinds(L.pair_script())
    assert set(kinds) == set(L.KINDS)
    assert set(zip(kinds, kinds[1:])) == L.all_pairs(L.KINDS)


@pytest.mark.parametrize("name", ["pairs", "scripted"])
def test_shards_shrink_and_grow_past_capacity(name):
    steps = {"pairs": L.pair_script, "scripted": L.scripted_1rank}[name]()
    cap_v = cap_e = 0
    grew = shrank = False
    for _i, st, cur, _o, _m in L.shard_states(steps):
        if st[0] != "run":
            continue
        lnv, lne = len(cur["rowptrs"][0]) - 1, len(cur["edges"][0])
        if cap_v:
            grew |= lnv > cap_v and lne > cap_e
            shrank |= lnv < cap_v
        cap_v, cap_e = max(cap_v, lnv), max(cap_e, lne)
    assert grew and shrank, name


def test_walks_are_long_and_varied():
    for seed in L.WALK_SEEDS:
        steps = L.walk(seed, 30)
        assert len(steps) >= 30
        ops = {st[0] for st in steps}
        assert {"load", "run", "opt", "init", "mov", "eval", "split", "compare", "update"} <= ops, (seed, ops)


def test_walks_run_most_of_their_assignment_calls():
    """The seeded walks refuse only where the contract says so (checked step by step on the device), and most of their
    evaluate / split / compare steps do run."""
    for seed in L.WALK_SEEDS:
        steps = L.walk(seed, 30)
        ref = L.expect_refused(steps)
        calls = [k for k, st in enumerate(steps) if st[0] in ("eval", "split", "compare")]
        assert sum(not ref[k] for k in calls) >= 2, (seed, [steps[k][0] for k in calls], [ref[k] for k in calls])


def setups(world):
    """(op, exported arrays, per-rank (need_v, need_s), per-rank lnv) of every setup (run, eval, split) of the script."""
    out = []
    for _i, st, cur, opts, mov in L.shard_states(L.multirank_script(world)):
        if st[0] in ("run", "eval", "split"):
            out.append((st[0], L.exported(cur, opts, mov, st[0]), [L.needs(cur, r) for r in range(world)],
                        [int(cur["parts"][r + 1] - cur["parts"][r]) for r in range(world)]))
    return out


@pytest.mark.parametrize("world", [2, 4])
def test_every_exported_array_comes_and_goes(world):
    """Each array of MV_EXPORTS that a setup may or may not need is added and dropped between consecutive setups: unit <->
    weighted, renumbering <-> not, evaluation arrays, split labels, frontier sets."""
    sets = [s[1] for s in setups(world)]
    for a in ("cdeg", "csize", "upd", "cinfo_w", "usize", "udeg", "lab", "inv", "q_internal", "q_rank", "split_lab",
              "mov_a", "mov_b"):
        on = [a in s for s in sets]
        assert any(not x and y for x, y in zip(on, on[1:])), (world, a, "never added")
        assert any(x and not y for x, y in zip(on, on[1:])), (world, a, "never dropped")


@pytest.mark.parametrize("world", [2, 4])
def test_one_rank_alone_outgrows_its_arrays(world):
    """Some setup makes exactly one rank's need_v or need_s exceed what that rank needed before (its grow-only capacity),
    so that rank alone must grow an exported array while its peers keep theirs."""
    caps = [(0, 0)] * world
    alone = False
    for k, (_op, _x, need, _lnv) in enumerate(setups(world)):
        over = [need[r][0] > caps[r][0] or need[r][1] > caps[r][1] for r in range(world)]
        alone |= k > 0 and sum(over) == 1
        caps = [(max(caps[r][0], need[r][0]), max(caps[r][1], need[r][1])) for r in range(world)]
    assert alone


@pytest.mark.parametrize("world", [2, 4])
def test_a_rank_goes_empty_and_comes_back(world):
    lnv1 = [s[3][1] for s in setups(world)]
    first_empty = next(k for k, v in enumerate(lnv1) if v == 0)
    assert lnv1[0] > 0 and any(v > 0 for v in lnv1[first_empty:])


def test_process_script_crosses_its_boundaries():
    """The two-process script: one rank alone must grow an exported array (need_v / need_s past its capacity), a shrink
    is followed by a regrow to the old size, unit <-> weighted, a frontier run."""
    import test_gpu_context_lifecycle as T
    st = [(st, cur, opts, mov) for _i, st, cur, opts, mov in L.shard_states(T.process_script()) if st[0] == "run"]
    lnv = [[int(c["parts"][r + 1] - c["parts"][r]) for r in range(2)] for _s, c, _o, _m in st]
    assert lnv[0] == [8192, 8192] and lnv[1] == [12288, 4096]              # rank 0 alone grows
    need = [[L.needs(c, r) for r in range(2)] for _s, c, _o, _m in st[:2]]
    assert need[1][0][0] > need[0][0][0]                                    # rank 0's need_v passes its capacity
    assert need[1][1][0] <= need[0][1][0] and need[1][1][1] <= need[0][1][1]
    assert lnv[2] == [2048, 2048] and lnv[3] == [8192, 8192]               # shrink, then the old size again
    assert [c["weighted"] for _s, c, _o, _m in st] == [False] * 4 + [True, False]
    assert st[-1][3] and st[-1][2]["frontier"] == 1
