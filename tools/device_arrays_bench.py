#!/usr/bin/env python3
"""Per-vertex arrays in host or device memory (DESIGN.md §3.16): the pipeline run -> split -> evaluate(Y) ->
compare(X, Y) -> probe(Y) -> set_initial_communities(Y) + warm run on config 2, generated on the device.

usage: python tools/device_arrays_bench.py [--reps R] [--nv NV] [--before-lib PATH] [--out FILE]

The pipeline runs three ways: NumPy pageable arrays, NumPy arrays over pinned memory, and torch CUDA tensors
(device=True outputs, tensors as inputs).  With --before-lib (a libmvgpu.so built from the parent commit, same ABI) it
also runs the host forms on that build in the same process, so that before and after are measured on the same card in
the same call.  Every step is a host-clock wall time around one synchronous call; the ways are alternated R times and
each step's median and range are printed.  The first pipeline of each way is a warm-up and is not counted.  Every way
must give the same bits: X, Y, the reports (timing fields excluded), the probe's arrays and the warm run.
Prints the card name and power limit read in the same call, one line per way, and a JSON summary."""
import argparse
import hashlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

from minivite_b200 import gpu as G  # noqa: E402
from warm_start_bench import card  # noqa: E402

STEPS = ("run", "communities", "split", "evaluate", "compare", "probe", "set_initial", "warm_run")
TIMES = ("split_s", "eval_s", "compare_s", "probe_s", "rounds")   # rounds: how fast labels spread, timing-dependent


def load(path):
    """The binding's library handle for `path` (ctypes keeps two builds apart: RTLD_LOCAL)."""
    G._lib, G._LIB_PATH = None, path
    return G.lib()


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(a.cpu().numpy().tobytes() if hasattr(a, "cpu") else np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


def pipeline(g, way, pinned):
    """One pass; returns (seconds per step, what it computed).  way: pageable / pinned / torch."""
    import torch
    t, res = {}, {}

    def timed(step, fn):
        t0 = time.perf_counter()
        out = fn()
        t[step] = time.perf_counter() - t0
        return out

    dev = way == "torch"
    res["run"] = timed("run", g.louvain)
    if way == "pinned":
        X = timed("communities", lambda: g.communities(out=pinned[0]))
    else:
        X = timed("communities", lambda: g.communities(device=dev))
    Y, srep = timed("split", lambda: g.split_communities(X, device=dev))
    if way == "pinned":                     # the caller keeps Y in pinned memory for the inputs that follow (untimed)
        np.copyto(pinned[1], Y)
        Y = pinned[1]
    q = timed("evaluate", lambda: g.evaluate(Y))
    c = timed("compare", lambda: g.compare_communities(Y, X))
    prep, target, best, gain = timed("probe", lambda: g.probe(Y, device=dev))
    timed("set_initial", lambda: g.set_initial_communities(Y))
    res["warm"] = timed("warm_run", g.louvain)
    g.set_initial_communities(None)
    if dev:
        torch.cuda.synchronize()
    strip = lambda r: {k: v for k, v in r.items() if k not in TIMES}     # noqa: E731
    res.update(split=strip(srep), eval=strip(q), cmp=strip(c), probe=strip(prep),
               arrays=digest(X, Y, target, best, gain), warm_comm=digest(g.communities()))
    return t, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--nv", type=int, default=16777216)
    ap.add_argument("--before-lib", default=None, help="libmvgpu.so of the parent commit: its host forms run too")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    libs = {"after": load(G._LIB_PATH)}
    if a.before_lib:
        libs["before"] = load(a.before_lib)
    G._lib = libs["after"]
    if G.device_count() < 1:
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU mode")
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    ways = [("after", "pageable"), ("after", "pinned"), ("after", "torch")]
    if "before" in libs:
        ways += [("before", "pageable"), ("before", "pinned")]
    ctx = {}
    for lib in libs:
        G._lib = libs[lib]
        g = G.LouvainGPU(0, 0, 1)
        g.generate_rgg(a.nv)
        ctx[lib] = g
    nv = ctx["after"].lnv
    pinned = [torch.empty(nv, dtype=torch.int64).pin_memory().numpy() for _ in range(2)]
    times = {w: [] for w in ways}
    results = {}
    for rep in range(a.reps + 1):                     # rep 0: warm-up of every way
        for w in ways:
            G._lib = libs[w[0]]
            t, res = pipeline(ctx[w[0]], w[1], pinned)
            if rep:
                times[w].append(t)
            results.setdefault(w, res)
            assert res == results[w], (w, "results changed between repetitions")
    ref = results[("after", "pageable")]
    for w, res in results.items():
        assert res == ref, (w, "results differ from the pageable host form")
    out = {"card": name, "power_limit": power, "nv": nv, "reps": a.reps, "iters": ref["run"][1],
           "warm_iters": ref["warm"][1], "ways": {}}
    for w in ways:
        per = {s: [t[s] * 1e3 for t in times[w]] for s in STEPS}
        per["total"] = [sum(t.values()) * 1e3 for t in times[w]]
        summ = {s: {"median": statistics.median(v), "min": min(v), "max": max(v)} for s, v in per.items()}
        out["ways"][f"{w[0]} {w[1]}"] = summ
        print(f"{w[0]:6s} {w[1]:8s} " + ", ".join(f"{s} {summ[s]['median']:.2f} [{summ[s]['min']:.2f}-{summ[s]['max']:.2f}]"
                                                  for s in STEPS + ("total",)) + " ms", flush=True)
    for lib in libs:
        G._lib = libs[lib]
        ctx[lib].close()
    G._lib = libs["after"]
    print(json.dumps(out), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
