"""Absolute kernel-launch counts of the host driver.

`kernel_launches` and `scan_launches` (mvgpu_timings) are counted by hand next to every launch in mvgpu.cu, and the
other tests only compare results: a launch that a change to the host driver adds, drops or moves across a counter goes
unnoticed there.  These tests pin both counters and the iteration count of fixed runs of the RGG n = 16384 graph, on
one rank over the option matrix and on 2 and 4 ranks sharing device 0 (host transport), cold, warm-started and around
an evaluation (whose own launches are not reported: the getters keep describing the last run, which the evaluation
must leave as it was).  Every number is [kernel_launches, scan_launches, iters], per rank."""
import numpy as np
import pytest

from helpers import split_global
from test_gpu_warm_start import Ranks

pytestmark = pytest.mark.gpu

N = 16384

# name -> (world, options, action)
MATRIX = {
    "default": (1, {}, "cold"),
    "scan_variant3": (1, {"scan_variant": 3}, "cold"),
    "scan_variant4": (1, {"scan_variant": 4}, "cold"),
    "scan_variant5": (1, {"scan_variant": 5}, "cold"),
    "reorder0": (1, {"reorder": 0}, "cold"),
    "reorder1": (1, {"reorder": 1}, "cold"),
    "force_weighted": (1, {"force_weighted": 1}, "cold"),
    "force_heavy_deg": (1, {"force_heavy_deg": 8}, "cold"),
    "compact_upload1": (1, {"compact_upload": 1}, "cold"),
    "compact_upload2": (1, {"compact_upload": 2}, "cold"),
    "warm": (1, {}, "warm"),
    "eval": (1, {}, "eval"),
    "p2_cold": (2, {}, "cold"),
    "p2_warm": (2, {}, "warm"),
    "p2_eval": (2, {}, "eval"),
    "p4_cold": (4, {}, "cold"),
    "p4_warm": (4, {}, "warm"),
    "p4_eval": (4, {}, "eval"),
}

# measured on the H100 at the commit before the host driver was restructured; steps of an action in order, each step a
# list over the ranks of [kernel_launches, scan_launches, iters]
EXPECTED = {
    "default": [[[31, 14, 14]]],
    "scan_variant3": [[[31, 14, 14]]],
    "scan_variant4": [[[31, 14, 14]]],
    "scan_variant5": [[[31, 14, 14]]],
    "reorder0": [[[31, 14, 14]]],
    "reorder1": [[[38, 14, 14]]],
    "force_weighted": [[[32, 14, 14]]],
    "force_heavy_deg": [[[46, 28, 14]]],
    "compact_upload1": [[[30, 14, 14]]],
    "compact_upload2": [[[30, 14, 14]]],
    "warm": [[[7, 2, 2]], [[30, 12, 12]]],
    "eval": [[[31, 14, 14]], [[31, 14, 14]], [[31, 14, 14]]],
    "p2_cold": [[[80, 14, 14], [80, 14, 14]]],
    "p2_warm": [[[20, 2, 2], [20, 2, 2]], [[75, 12, 12], [75, 12, 12]]],
    "p2_eval": [[[80, 14, 14], [80, 14, 14]], [[80, 14, 14], [80, 14, 14]], [[80, 14, 14], [80, 14, 14]]],
    "p4_cold": [[[80, 14, 14], [80, 14, 14], [80, 14, 14], [80, 14, 14]]],
    "p4_warm": [[[20, 2, 2]] * 4, [[75, 12, 12]] * 4],
    "p4_eval": [[[80, 14, 14]] * 4] * 3,
}


def counts(R):
    return [[t["kernel_launches"], t["scan_launches"], t["iters"]] for t in R.each(lambda r, g: g.timings())]


def observe(name):
    """The counts of one matrix entry: a list of steps, each a list over the ranks."""
    from minivite_b200 import hostgraph as hg
    world, opts, action = MATRIX[name]
    sh = hg.generate_rgg(N, 1).shards[0]
    parts, rps, eds = split_global(N, np.asarray(sh.rowptr, np.int64), sh.edges, world)
    R = Ranks(parts, rps, eds, **opts)
    try:
        steps = []
        if action == "warm":                   # stop after 2 iterations, resume from there
            R.set_option("stop_after", 2)
            res = R.run()
            steps.append(counts(R))
            R.set_option("stop_after", 0)
            R.set_initial(res["comm"])
            R.run(lower=res["mod"])
            steps.append(counts(R))
        else:
            R.run()
            steps.append(counts(R))
        if action == "eval":
            X = (np.arange(N, dtype=np.int64) // 16) * 16
            R.each(lambda r, g: g.evaluate())
            steps.append(counts(R))
            R.each(lambda r, g: g.evaluate(X[parts[r]:parts[r + 1]]))
            steps.append(counts(R))
        return steps
    finally:
        R.close()


@pytest.mark.parametrize("name", sorted(MATRIX))
def test_launch_counts(name):
    assert observe(name) == EXPECTED[name]
