#!/usr/bin/env python3
"""Re-clustering a changed graph with a movable set (DESIGN.md §3.14) on one GPU.

usage: python tools/movable_bench.py [--nv NV] [--small-frac F] [--out FILE]

Config 2 (`miniVite -n 16777216`) is generated on the device and run.  It is changed two ways: into config 3 (`-p 2`)
by the extras batch (config 3 minus config 2, both directions of every pair, as in tools/update_bench.py), and by a
small batch of random pairs (--small-frac of config 2's edges, both directions, weight 1).  Each changed graph is then
re-clustered three ways: a warm run from config 2's result with everything movable, a warm run with the batch's
endpoints as the movable set and frontier 1, and a cold run.  Per run: iterations, phase time (device events), total
moves (sum of the trace's moved), Q of the result (evaluate), the final size of the movable set, and compare against
config 2's result and against the cold run.  Prints the card name and power limit read in the same call, one line per
run and a JSON summary."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

from minivite_b200 import gpu as G  # noqa: E402
from warm_start_bench import card  # noqa: E402


class Rows:
    """Just the fields update_ref.extras reads, for a downloaded one-rank shard."""

    def __init__(self, nv, rowptr, edges):
        self.nv, self.base, self.rowptr, self.edges = nv, 0, rowptr, edges


def one_run(g, pre, mask, frontier):
    g.set_initial_communities(pre)
    g.set_movable(mask)
    g.set_option("frontier", frontier)
    mod, iters = g.louvain()
    t = g.timings()
    comm = g.communities().copy()
    out = {"iters": iters, "phase_ms": t["total_s"] * 1e3, "moves": int(g.trace()["moved"].sum()),
           "movable_final": int(g.movable().sum()), "mod": mod}
    out["Q"] = g.evaluate(comm)["modularity"]
    return out, comm


def scenario(g, nv, pre, batch):
    """Runs on the shard g holds after `batch` was applied; pre = config 2's result."""
    seeds = g.movable_from_batch(insert=batch)
    runs = {}
    warm_all, c_all = one_run(g, pre, None, 0)
    warm_front, c_front = one_run(g, pre, seeds, 1)
    cold, c_cold = one_run(g, None, None, 0)
    for name, r, c in (("warm_all", warm_all, c_all), ("warm_frontier", warm_front, c_front), ("cold", cold, c_cold)):
        vs_pre = g.compare_communities(pre, c)
        vs_cold = g.compare_communities(c_cold, c)
        r.update({"ari_vs_config2": vs_pre["ari"], "vi_vs_config2": vs_pre["vi"], "ari_vs_cold": vs_cold["ari"],
                  "vi_vs_cold": vs_cold["vi"]})
        runs[name] = r
    runs["seeds"] = int(seeds.sum())
    return runs


def main():
    import update_ref as U
    ap = argparse.ArgumentParser()
    ap.add_argument("--nv", type=int, default=16777216)
    ap.add_argument("--small-frac", type=float, default=0.001)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    g = G.LouvainGPU(0, 0, 1)
    g.set_option("trace", 1)
    summary = {"card": name, "power_limit": power, "nv": a.nv}
    try:
        g.generate_rgg(a.nv, random_edge_percent=2.0)
        rp3, ed3 = g.download_shard()
        lne2 = g.generate_rgg(a.nv)
        rp2, ed2 = g.download_shard()
        extras = U.extras(Rows(a.nv, rp2, ed2), Rows(a.nv, rp3, ed3))
        del rp3, ed3
        g.louvain()                                             # warm-up of every kernel shape, then the real run
        g.louvain()
        pre = g.communities().copy()
        rng = np.random.default_rng(1)
        m = max(1, int(a.small_frac * lne2 / 2))
        s, d = rng.integers(0, a.nv, m), rng.integers(0, a.nv, m)
        keep = s != d
        s, d = s[keep], d[keep]
        small = (np.concatenate([s, d]), np.concatenate([d, s]), np.ones(2 * len(s)))
        for label, batch in (("config3_extras", extras), ("small_random", small)):
            g.generate_rgg(a.nv)
            g.update_shard(insert=batch)
            res = scenario(g, a.nv, pre, batch)
            res["batch_records"] = int(len(batch[0]))
            summary[label] = res
            for k in ("warm_all", "warm_frontier", "cold"):
                r = res[k]
                print(f"{label} {k}: iters {r['iters']}, phase {r['phase_ms']:.2f} ms, moves {r['moves']}, Q {r['Q']:.9f}, "
                      f"|M| final {r['movable_final']}, vs config 2 ARI {r['ari_vs_config2']:.6f} VI {r['vi_vs_config2']:.6f}, "
                      f"vs cold ARI {r['ari_vs_cold']:.6f} VI {r['vi_vs_cold']:.6f}", flush=True)
            print(f"{label}: {res['batch_records']} records, {res['seeds']} seed vertices", flush=True)
    finally:
        g.close()
    print(json.dumps(summary))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
