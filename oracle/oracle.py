"""oracle/oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Python access to the two CPU checkers:
  * `louvain()`       -> the plain-C restatement in oracle/louvain_oracle.c (built into oracle/_build/)
  * `run_reference()` -> the UNMODIFIED reference binary oracle/_ref/miniVite_ref (built by build_ref.py
                         where /root/reference exists; the prebuilt binary travels to the GPU box)
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
"""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "louvain_oracle.c")
LIB = os.path.join(HERE, "_build", "liblouvain_oracle.so")
REF_BIN = os.path.join(HERE, "_ref", "miniVite_ref")
REF32_BIN = os.path.join(HERE, "_ref", "miniVite_ref32")       # the reference compiled with -DUSE_32_BIT_GRAPH
REF_GPU_BIN = os.path.join(HERE, "_ref", "miniVite_ref_gpu")   # reference main.cpp + INTEGRATION.md patch (build_ref.py --gpu)

TRACE_DTYPE = np.dtype([("modularity", "<f8"), ("moved", "<i8"), ("chash", "<u8")])
EDGE_DTYPE = np.dtype([("tail", "<i8"), ("weight", "<f8")])


def build(force=False):
    """Compile the C restatement (gcc, no FMA contraction) and, if the reference tree is present, oracle/_ref."""
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        subprocess.check_call(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall",
                               "-o", LIB, SRC, "-lm"])
    if os.path.isdir("/root/reference"):
        subprocess.check_call([sys.executable, os.path.join(HERE, "build_ref.py")])


_lib = None


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
            build()
        L = ctypes.CDLL(LIB)
        vp = ctypes.c_void_p
        L.mvo_louvain.restype = ctypes.c_double
        L.mvo_louvain.argtypes = [ctypes.c_int, vp, vp, vp, ctypes.c_double, ctypes.c_double, ctypes.POINTER(ctypes.c_int),
                                  vp, vp, ctypes.c_int, ctypes.POINTER(ctypes.c_double), vp, ctypes.c_int,
                                  ctypes.POINTER(ctypes.c_int), vp, ctypes.c_int, vp]
        L.mvo_comm_hash.restype = ctypes.c_uint64
        L.mvo_comm_hash.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p]
        _lib = L
    return _lib


def comm_hash(base, comm):
    comm = np.ascontiguousarray(comm, dtype=np.int64)
    return int(_load().mvo_comm_hash(int(base), len(comm), comm.ctypes.data))


def louvain(parts, rowptrs, edge_lists, lower=-1.0, thresh=1.0e-6, max_trace=512, init_comm=None, stop_after=0,
            movable=None, frontier=0):
    """Run the C restatement on shards (parts[r]..parts[r+1]).  init_comm: per-shard starting assignments in global
    community ids (None = singletons); stop_after > 0: stop after that many accepted iterations; movable: per-shard byte
    masks, nonzero = movable (None = every vertex movable); frontier 0 / 1 (louvain_oracle.c's header).  Returns a dict
    with modularity, iters, trace (structured array), comm (list of int64 arrays, currComm at exit), constant,
    chash_final, converged (False when stop_after ended the run) and movable (per shard, the set, uint8 0 / 1, the next
    iteration would use)."""
    L = _load()
    n = len(rowptrs)
    parts = np.ascontiguousarray(parts, dtype=np.int64)
    assert len(parts) == n + 1
    sizes = [int(parts[r + 1] - parts[r]) for r in range(n)]
    rps = [np.ascontiguousarray(r, dtype=np.int64) for r in rowptrs]
    eds = [np.ascontiguousarray(e) for e in edge_lists]
    assert all(e.dtype.itemsize == 16 for e in eds)
    comm = [np.zeros(s, dtype=np.int64) for s in sizes]
    mov_out = [np.zeros(s, dtype=np.uint8) for s in sizes]
    PtrArr = ctypes.c_void_p * n

    def arr(xs):
        return ctypes.cast(PtrArr(*[x.ctypes.data if len(x) else None for x in xs]), ctypes.c_void_p)
    init = mov = None
    if init_comm is not None:
        assert len(init_comm) == n
        init = [np.ascontiguousarray(c, dtype=np.int64) for c in init_comm]
        for r in range(n):
            assert len(init[r]) == sizes[r]
            assert len(init[r]) == 0 or (init[r].min() >= 0 and init[r].max() < parts[n])
    if movable is not None:
        assert len(movable) == n
        mov = [np.ascontiguousarray(m, dtype=np.uint8) for m in movable]
        assert all(len(mov[r]) == sizes[r] for r in range(n))
    trace = np.zeros(max_trace, dtype=TRACE_DTYPE)
    iters = ctypes.c_int(0)
    const = ctypes.c_double(0)
    converged = ctypes.c_int(1)
    mod = L.mvo_louvain(n, parts.ctypes.data, arr(rps), arr(eds), lower, thresh, ctypes.byref(iters), arr(comm),
                        trace.ctypes.data, max_trace, ctypes.byref(const), None if init is None else arr(init),
                        int(stop_after), ctypes.byref(converged), None if mov is None else arr(mov), int(frontier),
                        arr(mov_out))
    h = 0
    for r in range(n):
        h = (h + comm_hash(int(parts[r]), comm[r])) & 0xFFFFFFFFFFFFFFFF
    return {"modularity": mod, "iters": iters.value, "trace": trace[:min(iters.value, max_trace)].copy(),
            "comm": comm, "constant": const.value, "chash_final": h, "converged": bool(converged.value),
            "movable": mov_out}


def have_reference():
    return os.path.exists(REF_BIN) and os.access(REF_BIN, os.X_OK)


_ITER_RE = re.compile(r"ITER (\d+) mod=(\S+) moved=(\d+) chash=([0-9a-f]+)")
_FINAL_RE = re.compile(r"FINAL prevMod=(\S+) chashCurr=([0-9a-f]+) constant=(\S+)")
_RESULT_RE = re.compile(r"RESULT mod=(\S+) iters=(\d+) time=(\S+) nv=(\d+) ne=(\d+) nprocs=(\d+) threads=(\d+)")


def run_reference(args, nranks=1, threads=1, trace=True, dump_comm=None, dump_graph=None, cwd=None, timeout=None,
                  arena_gb=None, binary=None, extra_env=None):
    """Run oracle/_ref/miniVite_ref with the reference's own command line (`args`, e.g. ["-n","16384"] or
    ["-f", path]); `nranks` processes (fork shim) x `threads` OpenMP threads.  Returns parsed results."""
    binary = binary or REF_BIN
    if not (os.path.exists(binary) and os.access(binary, os.X_OK)):
        raise RuntimeError(f"{binary} missing (run oracle/build_ref.py where /root/reference exists)")
    env = dict(os.environ, MVSHIM_NP=str(nranks), OMP_NUM_THREADS=str(threads))
    env.update(extra_env or {})
    env.pop("MV_TRACE", None)
    if trace:
        env["MV_TRACE"] = "1"
    if dump_comm:
        env["MV_DUMP_COMM"] = dump_comm
    if dump_graph:
        env["MV_DUMP_GRAPH"] = dump_graph
    if arena_gb:
        env["MVSHIM_ARENA_GB"] = str(arena_gb)
    p = subprocess.run([binary] + [str(a) for a in args], env=env, capture_output=True, text=True, cwd=cwd,
                       timeout=timeout)
    if p.returncode != 0:
        raise RuntimeError(f"reference failed rc={p.returncode}: {p.stderr[-2000:]}")
    out = {"stdout": p.stdout, "stderr": p.stderr, "trace": []}
    for m in _ITER_RE.finditer(p.stderr):
        out["trace"].append({"iter": int(m.group(1)), "modularity": float(m.group(2)), "mod_repr": m.group(2),
                             "moved": int(m.group(3)), "chash": int(m.group(4), 16)})
    m = _FINAL_RE.search(p.stderr)
    if m:
        out["final"] = {"modularity": float(m.group(1)), "mod_repr": m.group(1), "chash": int(m.group(2), 16),
                        "constant": float(m.group(3))}
    m = _RESULT_RE.search(p.stderr)
    if m:
        out["result"] = {"modularity": float(m.group(1)), "iters": int(m.group(2)), "time": float(m.group(3)),
                         "nv": int(m.group(4)), "ne": int(m.group(5)), "nprocs": int(m.group(6)),
                         "threads": int(m.group(7))}
    return out


def read_comm_dump(prefix, nranks, elem=np.int64):
    """currComm slices written by MV_DUMP_COMM (16-byte header, then GraphElem entries: int64, or int32 for the
    USE_32_BIT_GRAPH build); returns list of (base, int64 array)."""
    out = []
    for r in range(nranks):
        hdr = np.fromfile(f"{prefix}.{r}", dtype=np.int64, count=2)
        base, nv = int(hdr[0]), int(hdr[1])
        body = np.fromfile(f"{prefix}.{r}", dtype=elem, offset=16, count=nv)
        out.append((base, body.astype(np.int64)))
    return out
