#!/usr/bin/env python3
"""Probing an assignment on one GPU (mvgpu_probe_communities, DESIGN.md §3.15).

usage: python tools/probe_bench.py [--reps R] [--nv NV] [--scale S] [--out FILE]

  probe   config 2 (`miniVite -n NV`, generated on the device) and R-MAT scale S (edge factor 16, uploaded): the run's
          result probed and evaluated R times each, alternated (probe_s and eval_s: device time from CUDA events), beside
          the renumbering time of a run with reorder = 1 (what a renumbering probe would pay on top);
  update  config 2 -> config 3 (`-p 2`) as one insertion batch on the device: how many vertices are unsettled from
          config 2's result (the probe's moves) against the batch's seeds (its endpoints, movable_from_batch);
  recluster  warm runs from config 2's result on the updated shard with frontier 1, seeded by the probe's unsettled set
          and by the batch's endpoints, alternated R times: iterations, vertices moved (sum of the trace), phase time
          (timings total_s) and modularity.
Prints the card name and power limit read in the same call, one line per measurement, and a JSON summary."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

from minivite_b200 import gpu as G  # noqa: E402
from update_bench import Rows  # noqa: E402
from warm_start_bench import card  # noqa: E402


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "all": [round(x, 4) for x in xs]}


def probe_vs_eval(g, reps):
    g.probe()                                        # warm-up (allocations)
    g.evaluate()
    pt, et = [], []
    for _ in range(reps):
        rep = g.probe()[0]
        pt.append(rep["probe_s"] * 1e3)
        et.append(g.evaluate()["eval_s"] * 1e3)
    return {"probe_ms": spread(pt), "eval_ms": spread(et), "moves": rep["moves"], "vetoed": rep["vetoed"],
            "interior": rep["interior"], "max_gain": rep["max_gain"]}


def reorder_ms(g):
    g.set_option("reorder", 1)
    g.louvain()
    t = g.timings()
    g.set_option("reorder", 2)
    return t["reorder_s"] * 1e3


def show(label, r):
    p, e = r["probe_ms"], r["eval_ms"]
    print(f"{label}: probe {p['median']:.3f} ms [{p['min']:.3f}-{p['max']:.3f}], evaluate {e['median']:.3f} ms "
          f"[{e['min']:.3f}-{e['max']:.3f}]; renumbering in a reorder=1 run {r['reorder_ms']:.3f} ms; moves {r['moves']}, "
          f"vetoed {r['vetoed']}, interior {r['interior']}, max gain {r['max_gain']:.6g}", flush=True)


def main():
    import update_ref as U
    from helpers import rmat_graph
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--nv", type=int, default=16777216)
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if G.device_count() < 1:
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU mode")
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    out = {"card": name, "power_limit": power, "nv": a.nv, "reps": a.reps}
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.set_option("trace", 1)
        g.generate_rgg(a.nv, random_edge_percent=2.0)
        rp3, ed3 = g.download_shard()
        g.generate_rgg(a.nv)
        rp2, ed2 = g.download_shard()
        batch = U.extras(Rows(a.nv, rp2, ed2), Rows(a.nv, rp3, ed3))
        del rp2, ed2, rp3, ed3
        g.louvain()
        X2 = g.communities().copy()
        out["config2"] = dict(probe_vs_eval(g, a.reps), reorder_ms=reorder_ms(g))
        show(f"config 2 ({a.nv} vertices)", out["config2"])

        g.update_shard(insert=batch)
        rep, target, _best, _gain = g.probe(X2)
        unsettled = (target != X2).astype(np.uint8)
        seeds = g.movable_from_batch(insert=batch)
        out["update"] = {"batch_records": len(batch[0]), "seeds": int(seeds.sum()), "unsettled": int(rep["moves"]),
                         "unsettled_off_batch": int(np.sum((unsettled != 0) & (seeds == 0))),
                         "seeds_settled": int(np.sum((seeds != 0) & (unsettled == 0))), "probe_ms": rep["probe_s"] * 1e3}
        u = out["update"]
        print(f"config 2 -> 3: batch {u['batch_records']} records, {u['seeds']} seeds; {u['unsettled']} unsettled vertices, "
              f"{u['unsettled_off_batch']} of them off the batch; {u['seeds_settled']} seeds settled", flush=True)

        g.set_initial_communities(X2)
        g.set_option("frontier", 1)
        runs = {"probe": [], "batch": []}
        for _ in range(a.reps):
            for key, mask in (("probe", unsettled), ("batch", seeds)):
                g.set_movable(mask)
                mod, iters = g.louvain()
                runs[key].append({"ms": g.timings()["total_s"] * 1e3, "iters": iters, "mod": mod,
                                  "moved": int(g.trace()["moved"].sum())})
        g.set_movable(None)
        g.set_option("frontier", 0)
        out["recluster"] = {}
        for key, rs in runs.items():
            r = {"phase_ms": spread([x["ms"] for x in rs]), "iters": rs[-1]["iters"], "moved": rs[-1]["moved"],
                 "modularity": rs[-1]["mod"]}
            assert all((x["iters"], x["moved"], x["mod"]) == (r["iters"], r["moved"], r["modularity"]) for x in rs)
            out["recluster"][key] = r
            print(f"re-cluster from the {key} seeds: {r['iters']} iterations, {r['moved']} moves, phase "
                  f"{r['phase_ms']['median']:.3f} ms [{r['phase_ms']['min']:.3f}-{r['phase_ms']['max']:.3f}], "
                  f"Q {r['modularity']:.17g}", flush=True)
        g.set_initial_communities(None)

        n, rowptr, edges = rmat_graph(a.scale, 16, 1)
        g.upload(n, np.array([0, n], np.int64), rowptr, edges)
        g.louvain()
        out["rmat"] = dict(probe_vs_eval(g, a.reps), reorder_ms=reorder_ms(g), scale=a.scale, nv=n, lne=len(edges),
                           nheavy=g.shard_info()["nheavy"])
        show(f"R-MAT scale {a.scale} ({n} vertices, {out['rmat']['nheavy']} high-degree)", out["rmat"])
    finally:
        g.close()
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
