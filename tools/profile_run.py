#!/usr/bin/env python3
"""Minimal profiling driver: one RGG, device-resident inputs, N Louvain phases, nothing else.
usage: python tools/profile_run.py [nv] [runs] [pct_random_edges] [--split]

--split records the last phase (the earlier ones warm it up) under torch.profiler with CUDA activities and prints the
device time of every kernel in it, the locality renumbering's stages first (k_msbfs, k_bfs_sortkeys, the CUB radix
sort by (region, level), k_perm_inverse, the CUB radix sort that builds inv, the CUB exclusive sum, k_permute_adj)."""
import argparse
import collections
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from minivite_b200 import gpu as G  # noqa: E402
from minivite_b200 import hostgraph as hg  # noqa: E402

# renumbering stages in launch order: (label, substring of the kernel name).  The two CUB radix sorts launch the same
# kernels; the one before k_perm_inverse sorts by (region, level), the one after it builds inv.
RENUMBER_STAGES = [("k_msbfs", "k_msbfs"), ("k_bfs_sortkeys", "k_bfs_sortkeys"),
                   ("cub sort (region, level)", "DeviceRadixSort"), ("k_perm_inverse", "k_perm_inverse"),
                   ("cub sort (inv)", "DeviceRadixSort"), ("cub exclusive sum", "DeviceScan"),
                   ("k_permute_adj", "k_permute_adj")]


def kernel_events(prof):
    """[(start us, kernel name, device us)] of the CUDA kernels of a finished profile, in launch order."""
    evs = [(ev.time_range.start, ev.name, ev.time_range.end - ev.time_range.start) for ev in prof.events()
           if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.name.startswith(("Memcpy", "Memset"))]
    return sorted(evs)


def print_split(evs, reorder_ms):
    stages = {label: [0, 0.0] for label, _ in RENUMBER_STAGES}
    others = collections.defaultdict(lambda: [0, 0.0])
    after_inverse = False
    for _, name, us in evs:
        after_inverse |= "k_perm_inverse" in name
        label = next((lb for lb, pat in RENUMBER_STAGES if pat in name
                      and (pat != "DeviceRadixSort" or after_inverse == (lb == "cub sort (inv)"))), None)
        a = stages[label] if label else others[name]
        a[0] += 1
        a[1] += us
    print(f"renumbering stages (device time, one phase; library events put the renumbering at {reorder_ms:.3f} ms):")
    for label, _ in RENUMBER_STAGES:
        n, us = stages[label]
        print(f"  {label:26s} {n:3d} launches {us / 1e3:8.3f} ms")
    print(f"  {'sum':26s}              {sum(v[1] for v in stages.values()) / 1e3:8.3f} ms")
    print("all other kernels of the phase:")
    for name, (n, us) in sorted(others.items(), key=lambda kv: -kv[1][1]):
        print(f"  {n:4d} launches {us / 1e3:8.3f} ms  {name[:110]}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("nv", nargs="?", type=int, default=16777216)
    ap.add_argument("runs", nargs="?", type=int, default=1)
    ap.add_argument("pct", nargs="?", type=float, default=0.0)
    ap.add_argument("--split", action="store_true", help="per-kernel device times of the last phase (torch.profiler)")
    args = ap.parse_args()
    runs = max(args.runs, 2) if args.split else args.runs
    t = time.time()
    ss = hg.generate_rgg(args.nv, 1, random_edge_percent=args.pct)
    sh = ss.shards[0]
    print(f"generated nv={args.nv} ne={sh.lne} in {time.time() - t:.1f}s", flush=True)
    d_rowptr = torch.from_numpy(np.ascontiguousarray(sh.rowptr)).cuda()
    d_edges = torch.from_numpy(np.ascontiguousarray(sh.edges).view(np.uint8)).cuda()
    torch.cuda.synchronize()
    ctx = G.LouvainGPU(0, 0, 1)
    ctx.attach_device(args.nv, sh.parts, sh.lnv, sh.lne, d_rowptr.data_ptr(), d_edges.data_ptr())
    prof = None
    for r in range(runs):
        if args.split and r == runs - 1:
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                mod, iters = ctx.louvain()
                torch.cuda.synchronize()
        else:
            mod, iters = ctx.louvain()
        tm = ctx.timings()
        print(f"run {r}: mod={mod:.17g} iters={iters} total={tm['total_s']*1e3:.3f}ms setup={tm['setup_s']*1e3:.3f}ms "
              f"(renumbering {tm['reorder_s']*1e3:.3f}ms) scan={tm['scan_s']*1e3:.3f}ms ({tm['scan_s']/iters*1e3:.3f} ms/iter) "
              f"fold={tm['fold_s']*1e3:.3f}ms edges/s={sh.lne*iters/tm['total_s']:.4g}", flush=True)
        if r == runs - 1:
            print("scan ms per iteration:", " ".join(f"{x*1e3:.2f}" for x in ctx.scan_times()), flush=True)
    if prof is not None:
        print_split(kernel_events(prof), tm["reorder_s"] * 1e3)
    ctx.close()


if __name__ == "__main__":
    main()
