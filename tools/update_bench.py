#!/usr/bin/env python3
"""Shard updates on one GPU (mvgpu_update_shard, DESIGN.md §3.11) against the other ways of getting a changed graph
onto the device.

usage: python tools/update_bench.py [--reps R] [--nv NV] [--rmat-scale S] [--out FILE]

Config 2 (`miniVite -n 16777216`) is generated on the device and run.  Config 3 (`-p 2`) differs from it by the random
long edges only, so its extra records (config 3 minus config 2, both directions of every pair) form one insertion batch.
Three ways of turning config 2 into config 3 on the device are timed, alternated, with a host clock around each
synchronous call: update_shard with the batch (host arrays in, the H2D of the batch included), a full upload of config
3's shard from pinned host arrays, and regenerating config 3 on the device.  Then the warm run from config 2's result on
the updated shard, the reverse batch (the extras as deletions, config 3 -> config 2), and R-MAT (edge factor 16) with
batches concentrated on its hubs.  The updated shard is checked against the regenerated one byte for byte, and the cold
run on it against the reference's config-3 trace.  Prints the card name and power limit read in the same call, one line
per measurement, and a JSON summary."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

from minivite_b200 import gpu as G  # noqa: E402
from warm_start_bench import card  # noqa: E402


def med(xs):
    return statistics.median(xs)


def clock(fn):
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


class Rows:
    """Just the fields update_ref.extras reads, for a downloaded one-rank shard."""

    def __init__(self, nv, rowptr, edges):
        self.nv, self.base, self.rowptr, self.edges = nv, 0, rowptr, edges


def breakdown(fn):
    """One call of fn under torch.profiler (a run of its own, not timed otherwise): wall time, and the device time of
    every kernel, copy and memset it issued, summed by name.  Wall minus device is host work: allocation and release of
    the temporaries and the new shard, pageable staging of the batch, synchronisations."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        ms, _ = clock(fn)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            key = ev.name.split("(")[0].replace("void ", "").replace("mv::", "")
            key = key.split("<")[0] if key.startswith("cub::") else key
            per[key] = per.get(key, 0.0) + (ev.time_range.end - ev.time_range.start) / 1e3
    dev = sum(per.values())
    return {"wall_ms": ms, "device_ms": dev, "host_ms": ms - dev,
            "top": {k: round(v, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:12]}}


def main():
    import torch
    import update_ref as U
    from helpers import rmat_graph
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--nv", type=int, default=16777216)
    ap.add_argument("--rmat-scale", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if G.device_count() < 1:
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU mode")
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    out = {"card": name, "power_limit": power, "nv": a.nv, "reps": a.reps}
    g = G.LouvainGPU(0, 0, 1)
    try:
        g.generate_rgg(a.nv, random_edge_percent=2.0)
        rp3, ed3 = g.download_shard()
        lne2 = g.generate_rgg(a.nv)
        rp2, ed2 = g.download_shard()
        batch = U.extras(Rows(a.nv, rp2, ed2), Rows(a.nv, rp3, ed3))
        nrec = len(batch[0])
        del rp2, ed2
        print(f"config 2: lne {lne2}; config 3: lne {len(ed3)}; batch {nrec} records "
              f"({nrec * 24 / 1e6:.1f} MB of host arrays)", flush=True)
        # pinned host copies of config 3 for the upload path
        prp = torch.empty(len(rp3), dtype=torch.int64, pin_memory=True).numpy()
        ped = torch.empty(len(ed3) * 16, dtype=torch.uint8, pin_memory=True).numpy().view(ed3.dtype)
        prp[:] = rp3
        ped[:] = ed3
        parts = np.array([0, a.nv], np.int64)

        mod2, it2 = g.louvain()
        final2 = g.communities().copy()
        print(f"config 2 run: {it2} iterations, modularity {mod2:.17g}", flush=True)

        # warm-up of every path, and the correctness checks
        g.update_shard(insert=batch)
        up = g.download_shard()
        assert np.array_equal(up[0], rp3) and up[1].tobytes() == ed3.tobytes(), "updated shard != regenerated config 3"
        del up
        g.set_initial_communities(None)
        cold = g.louvain()
        gold = json.load(open(os.path.join(ROOT, "tests", "golden", "golden_full_16777216_p1_r2.json")))
        if a.nv == gold["nv"]:
            assert cold == (float(gold["modularity"]), gold["iters"]), (cold, gold["iters"], gold["modularity"])
        g.upload(a.nv, parts, prp, ped)
        g.generate_rgg(a.nv, random_edge_percent=2.0)

        upd, upl, regen, warm = [], [], [], []
        for _ in range(a.reps):
            g.generate_rgg(a.nv)                                   # back to config 2 (untimed)
            ms, lne = clock(lambda: g.update_shard(insert=batch))
            assert lne == len(ed3)
            upd.append(ms)
            g.set_initial_communities(final2)
            mod, iters = g.louvain()
            warm.append({"ms": g.timings()["total_s"] * 1e3, "iters": iters, "mod": mod})
            g.set_initial_communities(None)
            upl.append(clock(lambda: g.upload(a.nv, parts, prp, ped))[0])
            ms, _ = clock(lambda: g.generate_rgg(a.nv, random_edge_percent=2.0))
            regen.append(ms)
        rev = []
        for _ in range(a.reps):
            g.generate_rgg(a.nv, random_edge_percent=2.0)
            ms, lne = clock(lambda: g.update_shard(delete=batch[:2]))
            assert lne == lne2
            rev.append(ms)
        g.generate_rgg(a.nv)
        prof = breakdown(lambda: g.update_shard(insert=batch))
        print(f"  one profiled update_shard: wall {prof['wall_ms']:.3f} ms, device (kernels + copies + memsets) "
              f"{prof['device_ms']:.3f} ms, the rest {prof['host_ms']:.3f} ms; largest: "
              + ", ".join(f"{k} {v:.3f}" for k, v in prof["top"].items()), flush=True)
        c3 = {"batch_records": nrec, "profiled_update": prof, "lne2": lne2, "lne3": len(ed3),
              "update_ms": med(upd), "update_ms_all": [round(x, 3) for x in upd],
              "upload_ms": med(upl), "upload_ms_all": [round(x, 3) for x in upl],
              "regenerate_ms": med(regen), "regenerate_ms_all": [round(x, 3) for x in regen],
              "reverse_update_ms": med(rev), "reverse_update_ms_all": [round(x, 3) for x in rev],
              "warm_ms": med([x["ms"] for x in warm]), "warm_iters": warm[-1]["iters"], "warm_modularity": warm[-1]["mod"],
              "cold_iters": cold[1], "cold_modularity": cold[0]}
        out["config3"] = c3
        print(f"config 2 -> 3 (median of {a.reps}, alternated): update_shard {c3['update_ms']:.3f} ms; "
              f"upload from pinned host arrays {c3['upload_ms']:.3f} ms; "
              f"regenerate on the device {c3['regenerate_ms']:.3f} ms")
        print(f"  warm run on the updated shard from config 2's result: {c3['warm_iters']} iterations, modularity "
              f"{c3['warm_modularity']:.17g}, {c3['warm_ms']:.3f} ms (cold: {cold[1]} iterations, modularity {cold[0]:.17g})")
        print(f"  reverse batch (the extras deleted, config 3 -> 2): {c3['reverse_update_ms']:.3f} ms", flush=True)
        del prp, ped, rp3, ed3

        # ---- R-MAT: batches on the hubs
        n, rowptr, edges = rmat_graph(a.rmat_scale, 16, 1)
        deg = np.diff(rowptr)
        hubs = np.argsort(deg)[-16:]
        rng = np.random.default_rng(0)
        ds, dd = [], []
        for h in hubs:                                             # half of every hub's pairs deleted, both directions
            t = edges["tail"][rowptr[h]:rowptr[h + 1]]
            t = t[rng.random(len(t)) < 0.5]
            ds += [np.full(len(t), h), t]
            dd += [t, np.full(len(t), h)]
        dele = (np.concatenate(ds), np.concatenate(dd))
        src = np.repeat(hubs, 1 << 15)                             # 32 Ki new pairs on every hub, both directions
        dst = rng.integers(0, n, len(src))
        ins = (np.concatenate([src, dst]), np.concatenate([dst, src]), np.ones(2 * len(src)))
        ref = U.apply(0, rowptr, edges, dele, ins)
        rparts = np.array([0, n], np.int64)
        g.upload(n, rparts, rowptr, edges)
        g.update_shard(dele, ins)
        got = g.download_shard()
        assert np.array_equal(got[0], ref[0]) and got[1].tobytes() == ref[1].tobytes(), "R-MAT update != update_ref"
        rm = []
        for _ in range(a.reps):
            g.upload(n, rparts, rowptr, edges)
            rm.append(clock(lambda: g.update_shard(dele, ins))[0])
        r = {"scale": a.rmat_scale, "lne": len(edges), "max_degree": int(deg.max()), "deletions": len(dele[0]),
             "insertions": len(ins[0]), "update_ms": med(rm), "update_ms_all": [round(x, 3) for x in rm]}
        out["rmat"] = r
        print(f"R-MAT scale {a.rmat_scale} (lne {len(edges)}, max degree {r['max_degree']}): {r['deletions']} deletions + "
              f"{r['insertions']} insertions on the 16 largest hubs: update_shard {r['update_ms']:.3f} ms")
    finally:
        g.close()
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
