#!/usr/bin/env python3
"""Warm start and checkpoint / resume on one GPU, with graphs generated on the device.

usage: python tools/warm_start_bench.py [--reps R] [--nv NV] [--stop K] [--out FILE]

Config 2 (`miniVite -n 16777216`): the cold phase, against the same run stopped after K accepted iterations (default 13)
plus its resume from the checkpoint assignment with lower = the stopped run's modularity; the resumed run must end
exactly where the cold run ends.  The warm-start init kernels (k_warm_*) are timed separately under torch.profiler.
Config 3 (the same graph + 2 % random edges, `-p 2`): a cold run against a warm start from config 2's final assignment
(iterations, modularity, phase time).  Phase time = the library's device-event total (setup + all iterations).
Prints the card name and power limit read in the same call, one line per measurement, and a JSON summary."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
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


def run(g, lower=-1.0):
    mod, iters = g.louvain(lower)
    t = g.timings()
    return {"mod": mod, "iters": iters, "total_ms": t["total_s"] * 1e3, "setup_ms": t["setup_s"] * 1e3,
            "launches": t["kernel_launches"], "converged": g.converged()}


def med(xs):
    return statistics.median(xs)


def init_kernel_ms(g, lower):
    """Device time of the k_warm_* kernels of one warm run, from torch.profiler (a run of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.louvain(lower)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "k_warm_" in ev.name:
            key = ev.name.split("(")[0].replace("void ", "").replace("mv::", "")
            per[key] = per.get(key, 0.0) + (ev.time_range.end - ev.time_range.start) / 1e3
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--nv", type=int, default=16777216)
    ap.add_argument("--stop", type=int, default=13)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if G.device_count() < 1:
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU mode")
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    out = {"card": name, "power_limit": power, "nv": a.nv, "stop_after": a.stop, "reps": a.reps}
    g = G.LouvainGPU(0, 0, 1)
    try:
        # ---- config 2: cold vs stop-at-K + resume
        g.generate_rgg(a.nv)
        ref = run(g)                                           # warm-up (module loading, allocations)
        final2 = g.communities().copy()
        cold, stop, resume = [], [], []
        for _ in range(a.reps):                                # alternate the three runs
            g.set_initial_communities(None)
            g.set_option("stop_after", 0)
            cold.append(run(g))
            assert (cold[-1]["iters"], cold[-1]["mod"]) == (ref["iters"], ref["mod"])
            g.set_option("stop_after", a.stop)
            stop.append(run(g))
            assert stop[-1]["iters"] == a.stop and not stop[-1]["converged"]
            ck = g.communities().copy()
            g.set_option("stop_after", 0)
            g.set_initial_communities(ck)
            resume.append(run(g, stop[-1]["mod"]))
            r = resume[-1]
            assert r["converged"] and a.stop + r["iters"] == ref["iters"] and r["mod"] == ref["mod"]
            assert np.array_equal(g.communities(), final2)
        kern = init_kernel_ms(g, stop[-1]["mod"])
        c2 = {"iters": ref["iters"], "modularity": ref["mod"],
              "cold_ms": med([x["total_ms"] for x in cold]), "cold_ms_all": [round(x["total_ms"], 3) for x in cold],
              "cold_launches": cold[-1]["launches"],
              "stop_ms": med([x["total_ms"] for x in stop]), "resume_ms": med([x["total_ms"] for x in resume]),
              "resume_setup_ms": med([x["setup_ms"] for x in resume]), "cold_setup_ms": med([x["setup_ms"] for x in cold]),
              "stop_plus_resume_ms": med([s["total_ms"] + r["total_ms"] for s, r in zip(stop, resume)]),
              "init_kernels_ms": kern, "init_kernels_total_ms": sum(kern.values())}
        out["config2"] = c2
        print(f"config 2 ({a.nv} vertices): {ref['iters']} iterations, modularity {ref['mod']:.17g}", flush=True)
        print(f"  cold phase {c2['cold_ms']:.3f} ms (median of {a.reps}; {c2['cold_launches']} kernel launches; "
              f"setup {c2['cold_setup_ms']:.3f} ms)")
        print(f"  stop after {a.stop}: {c2['stop_ms']:.3f} ms + resume: {c2['resume_ms']:.3f} ms "
              f"(setup {c2['resume_setup_ms']:.3f} ms) = {c2['stop_plus_resume_ms']:.3f} ms")
        print(f"  warm-start init kernels: {c2['init_kernels_total_ms']:.3f} ms "
              + ", ".join(f"{k} {v:.3f}" for k, v in sorted(kern.items())))

        # ---- config 3: cold vs warm start from config 2's final assignment
        g.generate_rgg(a.nv, random_edge_percent=2.0)
        run(g)                                                 # warm-up of the new shard
        cold3, warm3 = [], []
        for _ in range(a.reps):
            g.set_initial_communities(None)
            cold3.append(run(g))
            g.set_initial_communities(final2)
            warm3.append(run(g))
        c3 = {"cold_iters": cold3[-1]["iters"], "cold_modularity": cold3[-1]["mod"], "cold_ms": med([x["total_ms"] for x in cold3]),
              "warm_iters": warm3[-1]["iters"], "warm_modularity": warm3[-1]["mod"], "warm_ms": med([x["total_ms"] for x in warm3]),
              "cold_ms_all": [round(x["total_ms"], 3) for x in cold3], "warm_ms_all": [round(x["total_ms"], 3) for x in warm3]}
        out["config3"] = c3
        print(f"config 3 (+2 % random edges): cold {c3['cold_iters']} iterations, modularity {c3['cold_modularity']:.17g}, "
              f"{c3['cold_ms']:.3f} ms; warm from config 2's result {c3['warm_iters']} iterations, modularity "
              f"{c3['warm_modularity']:.17g}, {c3['warm_ms']:.3f} ms")
    finally:
        g.close()
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
