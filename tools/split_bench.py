#!/usr/bin/env python3
"""Splitting disconnected communities on one GPU (mvgpu_split_communities, DESIGN.md §3.12).

usage: python tools/split_bench.py [--reps R] [--nv NV] [--scale S] [--out FILE]

Two graphs: config 2 (`miniVite -n 16777216`) generated on the device, and an R-MAT graph of scale S (default 20, edge
factor 16, the tests' generator) uploaded from the host.  On each: one Louvain phase gives X, then R splits of X give Y
(split_s: the call's device time from CUDA events, setup included) and X and Y are evaluated.  Every split must return
the same Y and counts.  The k_split_* kernels of one more split are timed separately under torch.profiler.  Prints the card name and power limit read in the same call, one line per graph, and a JSON
summary with medians."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

from minivite_b200 import gpu as G  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        name, power = [x.strip() for x in out.split(",")[:2]]
        return name, power
    except Exception as ex:                  # the numbers are still printed; the card is then unknown
        return f"unknown ({ex!r})", "unknown"


def split_kernel_ms(g):
    """Device time of the k_split_* kernels of one split, from torch.profiler (a call of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.split_communities()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "k_split_" in ev.name:
            key = ev.name.split("(")[0].replace("void ", "").replace("mv::", "")
            per[key] = per.get(key, 0.0) + (ev.time_range.end - ev.time_range.start) / 1e3
    return per


def measure(g, reps):
    """Run once, split the result `reps` times (plus one warm-up), evaluate X and Y."""
    mod, iters = g.louvain()
    run_ms = g.timings()["total_s"] * 1e3
    X = g.communities().copy()
    Y0, rep0 = g.split_communities()                 # warm-up (allocations)
    times, rounds = [], []
    for _ in range(reps):
        Y, rep = g.split_communities()
        # Y and the counts are canonical; the round count depends on the order the device runs the hooks in
        assert np.array_equal(Y, Y0) and all(rep[k] == rep0[k] for k in ("communities", "components", "disconnected"))
        times.append(rep["split_s"] * 1e3)
        rounds.append(rep["rounds"])
    kern = split_kernel_ms(g)
    qx, qy = g.evaluate(X), g.evaluate(Y0)
    assert qy["communities"] == rep0["components"] and qy["modularity"] >= qx["modularity"]
    return {"iters": iters, "run_modularity": mod, "run_ms": run_ms, "split_ms": statistics.median(times),
            "split_ms_all": [round(t, 3) for t in times], "rounds": statistics.median(rounds), "rounds_all": rounds,
            "communities": rep0["communities"], "components": rep0["components"], "disconnected": rep0["disconnected"],
            "Q_X": qx["modularity"], "Q_Y": qy["modularity"], "e_in_equal": qx["e_in"] == qy["e_in"],
            "split_kernels_ms": kern, "split_kernels_total_ms": sum(kern.values())}


def show(label, r):
    print(f"{label}: run {r['iters']} iterations {r['run_ms']:.3f} ms; split {r['split_ms']:.3f} ms (median), "
          f"{r['rounds']} rounds; communities {r['communities']}, disconnected {r['disconnected']}, components "
          f"{r['components']}; Q {r['Q_X']:.17g} -> {r['Q_Y']:.17g}; split kernels {r['split_kernels_total_ms']:.3f} ms "
          + ", ".join(f"{k} {v:.3f}" for k, v in sorted(r["split_kernels_ms"].items())), flush=True)


def main():
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
    out = {"card": name, "power_limit": power, "reps": a.reps}
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.generate_rgg(a.nv)
        out["config2"] = dict(measure(g, a.reps), nv=a.nv, lne=g.shard_info()["lne"])
        show(f"config 2 ({a.nv} vertices, generated on the device)", out["config2"])
        from helpers import rmat_graph
        n, rowptr, edges = rmat_graph(a.scale, 16, 1)
        g.upload(n, np.array([0, n], np.int64), rowptr, edges)
        out["rmat"] = dict(measure(g, a.reps), scale=a.scale, nv=n, lne=len(edges))
        show(f"R-MAT scale {a.scale} ({n} vertices, {len(edges)} records, uploaded)", out["rmat"])
    finally:
        g.close()
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
