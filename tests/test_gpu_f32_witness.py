"""The mvgpu_*32 entry points on the float-build witnesses of tests/golden/f32_witness_traces.json: graphs where the
reference's USE_32_BIT_GRAPH build and its double build move a vertex differently, because two gains merge when
rounded to float, because the float 1/(2m) decides, or because the exit test subtracts in float.  Every sum stays
below 2^24 units, so the float build is exact and this build must match it decision for decision: iteration count,
every iteration's (moved, chash) and the final assignment, under every scan kernel, the locality renumbering with small
regions (the float tie must go to the smaller label, not the smaller internal id), k_scan_heavy forced below the
witness's degree, and the case's own rank count (ranks as threads on one device).

The float modularity is held bit for bit where the float build's sum of squared community degrees is exact
((2m)^2 < 2^24 units); elsewhere that build adds the squares one by one in float while this build adds exact integers
and rounds once, and the bar is 4 float ulps (as in test_gpu_32bit.py)."""
import json
import os

import numpy as np
import pytest

import f32_witness as W
from helpers import split_global
from oracle import oracle as O
from test_gpu_32bit import EDGE32, run32

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "f32_witness_traces.json")))["cases"]
WITNESSES = sorted(k for k, c in CASES.items() if "witness" in c)
EXITS = sorted(k for k in CASES if "_exit" in k)
OPTS = [{"scan_variant": v} for v in (3, 4, 5, 6)] + [{"reorder": r, "region_size": 32} for r in (0, 1, 2)]


def sharded(case):
    nv, rowptr, edges = W.graph(case["spec"])
    parts, rps, eds = split_global(nv, rowptr, edges, case["nranks"])
    out = []
    for rp, ed in zip(rps, eds):
        e = np.zeros(len(ed), EDGE32)
        e["tail"], e["weight"] = ed["tail"], ed["weight"].astype(np.float32)
        out.append((rp.astype(np.int32), e))
    return parts.astype(np.int32), out


def check(name, case, res, opts):
    tag = (name, opts)
    assert res["unit"] == (1 if case["spec"]["denom"] == 1 else 0), tag
    assert res["iters"] == case["iters"] and len(res["trace"]) == len(case["trace"]), tag
    exact_mod = W.units(case["spec"]) ** 2 < 2 ** 24
    mods = [(np.float32(res["mod"]), np.float32(float(case["modularity"])))]
    for k, (t, g) in enumerate(zip(res["trace"], case["trace"]), 1):
        assert int(t["moved"]) == g["moved"] and int(t["chash"]) == int(g["chash"], 16), tag + (k,)
        mods.append((np.float32(t["modularity"]), np.float32(float(g["modularity"]))))
    for a, b in mods:
        if exact_mod:
            assert a.view(np.uint32) == b.view(np.uint32), tag + (a, b)
        else:
            assert abs(float(a) - float(b)) <= 4 * float(np.spacing(np.float32(abs(b)))), tag + (a, b)
    if "comm" in case:
        assert [int(x) for x in res["comm"]] == case["comm"], tag
    assert O.comm_hash(0, res["comm"]) == int(case["final_chash"], 16), tag


@pytest.mark.parametrize("name", WITNESSES)
def test_witness_bit_exact(name):
    case = CASES[name]
    nv, rowptr, _ = W.graph(case["spec"])
    v = case["witness"]
    deg = int(rowptr[v + 1] - rowptr[v])
    sh = sharded(case)
    for opts in OPTS + [{"force_heavy_deg": max(1, deg - 1)}, {"force_heavy_deg": max(1, deg - 1), "scan_variant": 3}]:
        check(name, case, run32(case, sharded=sh, **opts), opts)


@pytest.mark.parametrize("name", EXITS)
def test_exit_witness(name):
    """The lower -t is the float build's rounded-up difference: the run goes on past exit_iter.  The upper one, a float
    ulp above, stops there.  A test on the unrounded difference would stop at exit_iter for both."""
    case = CASES[name]
    sh = sharded(case)
    for opts in ({}, {"scan_variant": 3}):
        check(name, case, run32(case, thresh=float(case["thresh"]), sharded=sh, **opts), opts)
