#!/usr/bin/env python3
"""Evaluation of an assignment (mvgpu_evaluate_communities) against the Louvain phase, on one GPU, graph generated on the
device.

usage: python tools/quality_bench.py [--reps R] [--nv NV] [--rmat SCALE] [--out FILE]

Config 2 (`miniVite -n 16777216`): the phase (device-event total: setup + all iterations) and the evaluation of its
result (eval_s: device events around setup, warm init, the internal-weight pass, the reductions and the compaction),
alternated R times; also an evaluation of the singleton assignment.  The evaluation kernels (k_q_*) are timed separately
under torch.profiler.  --rmat SCALE adds the same measurement on a power-law graph, built on the host and uploaded (the
seeded R-MAT graph of tests/helpers.py, edge factor 16; largest degree 64 837 at scale 20), where one thread per vertex
in the internal-weight pass meets the largest degree.  Prints the card name, power limit and SM clocks read in the same
call, one line per measurement, and a JSON summary."""
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=60).stdout.strip()
        return [x.strip() for x in out.split(",")[:4]]
    except Exception as ex:                  # the numbers are still printed; the card is then unknown
        return [f"unknown ({ex!r})", "unknown", "unknown", "unknown"]


def eval_kernel_ms(g):
    """Device time of the k_q_* kernels of one evaluation, from torch.profiler (a run of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.evaluate()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "k_q_" in ev.name:
            key = ev.name.split("(")[0].replace("void ", "").replace("mv::", "")
            per[key] = per.get(key, 0.0) + (ev.time_range.end - ev.time_range.start) / 1e3
    return per


def rmat_case(g, scale, reps):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from helpers import rmat_graph
    nv, rowptr, edges = rmat_graph(scale, 16, 1)
    g.upload(nv, np.array([0, nv], np.int64), rowptr, edges)
    mod, iters = g.louvain()
    g.evaluate()
    phase, ev = [], []
    for _ in range(reps):
        g.louvain()
        phase.append(g.timings()["total_s"] * 1e3)
        ev.append(g.evaluate()["eval_s"] * 1e3)
    kern = eval_kernel_ms(g)
    res = {"scale": scale, "nv": nv, "lne": len(edges), "max_degree": int(np.diff(rowptr).max()), "iters": iters,
           "phase_ms": statistics.median(phase), "eval_ms": statistics.median(ev), "eval_kernels_ms": kern}
    print(f"R-MAT scale {scale} ({nv} vertices, {len(edges)} edge records, largest degree {res['max_degree']}): "
          f"{iters} iterations, phase {res['phase_ms']:.3f} ms, evaluation {res['eval_ms']:.3f} ms (medians of {reps}); "
          "evaluation kernels " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(kern.items())), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--nv", type=int, default=16777216)
    ap.add_argument("--rmat", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if G.device_count() < 1:
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU mode")
    name, power, clk, clk_max = card()
    print(f"card: {name}, power limit {power}, SM clock {clk} (max {clk_max})", flush=True)
    out = {"card": name, "power_limit": power, "sm_clock": clk, "sm_clock_max": clk_max, "nv": a.nv, "reps": a.reps}
    g = G.LouvainGPU(0, 0, 1)
    try:
        lne = g.generate_rgg(a.nv)
        mod, iters = g.louvain()                               # warm-up (module loading, allocations)
        q0 = g.evaluate()
        phase, ev = [], []
        for _ in range(a.reps):                                # alternate phase and evaluation
            m, i = g.louvain()
            assert (m, i) == (mod, iters)
            phase.append(g.timings()["total_s"] * 1e3)
            q = g.evaluate()
            assert all(q[k] == q0[k] for k in ("modularity", "e_in", "a2", "communities"))
            ev.append(q["eval_s"] * 1e3)
        single = g.evaluate(np.arange(a.nv, dtype=np.int64))
        kern = eval_kernel_ms(g)
        res = {"lne": lne, "iters": iters, "reported_modularity": mod, "Q": q0["modularity"], "e_in": q0["e_in"],
               "a2": q0["a2"], "communities": q0["communities"], "singletons": q0["singletons"], "max_size": q0["max_size"],
               "phase_ms": statistics.median(phase), "phase_ms_all": [round(x, 3) for x in phase],
               "eval_ms": statistics.median(ev), "eval_ms_all": [round(x, 3) for x in ev],
               "eval_singletons_ms": single["eval_s"] * 1e3, "Q_singletons": single["modularity"],
               "eval_kernels_ms": kern, "eval_kernels_total_ms": sum(kern.values())}
        out["config2"] = res
        print(f"config 2 ({a.nv} vertices, {lne} edge records): {iters} iterations, reported modularity {mod:.17g}, "
              f"Q of the returned assignment {q0['modularity']:.17g} ({q0['communities']} communities)")
        print(f"  phase {res['phase_ms']:.3f} ms, evaluation {res['eval_ms']:.3f} ms (medians of {a.reps}); "
              f"singleton assignment {res['eval_singletons_ms']:.3f} ms")
        print(f"  evaluation kernels: {res['eval_kernels_total_ms']:.3f} ms "
              + ", ".join(f"{k} {v:.3f}" for k, v in sorted(kern.items())))
        if a.rmat:
            out["rmat"] = rmat_case(g, a.rmat, a.reps)
    finally:
        g.close()
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
