#!/usr/bin/env python3
"""Comparing two assignments on one GPU (mvgpu_compare_communities, DESIGN.md §3.13).

usage: python tools/compare_bench.py [--reps R] [--nv NV] [--pct P] [--scale S] [--out FILE]

Three cases:
  split   config 2 (`miniVite -n NV`) generated on the device: the run's result against its split;
  warm    config 3 (`-n NV -p P`, generated on the device): a cold run against a warm run started from config 2's result;
  rmat    an R-MAT graph of scale S (edge factor 16, the tests' generator), uploaded: the run's result against its split.
Each case: one warm-up and R timed compares (compare_s: the call's device time from CUDA events, both arrays already on
the device), which must all give the same report; one more compare under torch.profiler for the kernel breakdown; and
the host alternative, timed on the wall clock: download the run's assignment and compute the NumPy restatement
(tests/compare_ref.py, match arrays included), whose report must equal the device's.  Prints the card name and power
limit read in the same call, one line per case, and a JSON summary."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

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


def kernel_ms(fn):
    """Device time per kernel name of one call of fn, from torch.profiler (a call of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in ev.name and "Memset" not in ev.name:
            name = ev.name.split("(")[0].replace("void ", "").replace("mv::", "")
            name = name.split("<")[0] if "cub::" in name else name
            per[name] = per.get(name, 0.0) + (ev.time_range.end - ev.time_range.start) / 1e3
    return per


def measure(g, Y, reps):
    """Compare the last run's result (x = NULL) with Y on the device, and the same on the host."""
    import compare_ref as CR
    first = g.compare_communities(Y)                 # warm-up (allocations)
    times = []
    for _ in range(reps):
        rep = g.compare_communities(Y)
        assert all(repr(rep[k]) == repr(first[k]) for k in CR.FIELDS)
        times.append(rep["compare_s"] * 1e3)
    kern = kernel_ms(lambda: g.compare_communities(Y))
    t0 = time.perf_counter()
    X = g.communities()
    t1 = time.perf_counter()
    ref = CR.compare(X, Y)
    t2 = time.perf_counter()
    assert all(repr(ref[k]) == repr(first[k]) for k in CR.FIELDS), "device and restatement disagree"
    m = g.community_matches()
    assert all(np.array_equal(m[k], ref[k]) for k in CR.MATCHES)
    return {"compare_ms": statistics.median(times), "compare_ms_all": [round(t, 3) for t in times],
            "ari": first["ari"], "nmi": first["nmi"], "vi": first["vi"], "cells": first["cells"],
            "communities_x": first["communities_x"], "communities_y": first["communities_y"],
            "kernels_ms": kern, "kernels_total_ms": sum(kern.values()),
            "host_download_ms": (t1 - t0) * 1e3, "host_restatement_ms": (t2 - t1) * 1e3}


def show(label, r):
    top = sorted(r["kernels_ms"].items(), key=lambda kv: -kv[1])[:8]
    print(f"{label}: compare {r['compare_ms']:.3f} ms (median of {r['compare_ms_all']}); ARI {r['ari']:.17g}, NMI "
          f"{r['nmi']:.17g}; cells {r['cells']}, communities {r['communities_x']} / {r['communities_y']}; kernels "
          f"{r['kernels_total_ms']:.3f} ms: " + ", ".join(f"{k} {v:.3f}" for k, v in top)
          + f"; host: download {r['host_download_ms']:.1f} ms + NumPy {r['host_restatement_ms']:.1f} ms", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--nv", type=int, default=16777216)
    ap.add_argument("--pct", type=float, default=2.0)
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
        g.louvain()
        X2 = g.communities().copy()
        Y, _ = g.split_communities()
        out["split"] = dict(measure(g, Y, a.reps), nv=a.nv)
        show(f"config 2 ({a.nv} vertices): run vs its split", out["split"])
        g.generate_rgg(a.nv, random_edge_percent=a.pct)
        g.louvain()
        cold = g.communities().copy()
        g.set_initial_communities(X2)
        g.louvain()
        out["warm"] = dict(measure(g, cold, a.reps), nv=a.nv, pct=a.pct)
        show(f"config 3 (-p {a.pct:g}): warm run from config 2's result vs cold run", out["warm"])
        from helpers import rmat_graph
        n, rowptr, edges = rmat_graph(a.scale, 16, 1)
        g.upload(n, np.array([0, n], np.int64), rowptr, edges)
        g.louvain()
        Y, _ = g.split_communities()
        out["rmat"] = dict(measure(g, Y, a.reps), scale=a.scale, nv=n, lne=len(edges))
        show(f"R-MAT scale {a.scale} ({n} vertices): run vs its split", out["rmat"])
    finally:
        g.close()
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
