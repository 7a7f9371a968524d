"""Python access to tests/movable_oracle.c (TEST INFRASTRUCTURE): the warm-start oracle's Louvain phase with a movable
set and the frontier rule (DESIGN.md §3.14).  Compiled on first use with the oracle's own flags into the temporary
directory (keyed by the sources' contents), so the tree is never written."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "movable_oracle.c")
_lib = None


def _load():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in (SRC, O.SRC):
            with open(f, "rb") as fh:
                h.update(fh.read())
        lib = os.path.join(tempfile.gettempdir(), f"mv_movable_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(lib):
            tmp = f"{lib}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall",
                                   "-o", tmp, SRC, "-lm"])
            os.replace(tmp, lib)
        L = ctypes.CDLL(lib)
        vp = ctypes.c_void_p
        L.mvo_louvain_movable.restype = ctypes.c_double
        L.mvo_louvain_movable.argtypes = [ctypes.c_int, vp, vp, vp, ctypes.c_double, ctypes.c_double,
                                          ctypes.POINTER(ctypes.c_int), vp, vp, ctypes.c_int,
                                          ctypes.POINTER(ctypes.c_double), vp, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                          vp, ctypes.c_int, vp]
        _lib = L
    return _lib


def louvain(parts, rowptrs, edge_lists, lower=-1.0, thresh=1.0e-6, max_trace=512, init_comm=None, stop_after=0,
            movable=None, frontier=0):
    """warm_oracle.louvain() with `movable` (per-shard byte masks, nonzero = movable; None = everything movable) and
    `frontier` (0 / 1).  Returns warm_oracle.louvain()'s dict plus `movable`: per shard, the set (uint8 0 / 1) the next
    iteration would use."""
    L = _load()
    n = len(rowptrs)
    parts = np.ascontiguousarray(parts, dtype=np.int64)
    assert len(parts) == n + 1
    sizes = [int(parts[r + 1] - parts[r]) for r in range(n)]
    rps = [np.ascontiguousarray(r, dtype=np.int64) for r in rowptrs]
    eds = [np.ascontiguousarray(e) for e in edge_lists]
    assert all(e.dtype.itemsize == 16 for e in eds)
    comm = [np.zeros(s, dtype=np.int64) for s in sizes]
    mov_out = [np.zeros(s + 1, dtype=np.uint8) for s in sizes]
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
    trace = np.zeros(max_trace, dtype=O.TRACE_DTYPE)
    iters = ctypes.c_int(0)
    const = ctypes.c_double(0)
    converged = ctypes.c_int(1)
    mod = L.mvo_louvain_movable(n, parts.ctypes.data, arr(rps), arr(eds), lower, thresh, ctypes.byref(iters), arr(comm),
                                trace.ctypes.data, max_trace, ctypes.byref(const),
                                arr(init) if init is not None else None, int(stop_after), ctypes.byref(converged),
                                arr(mov) if mov is not None else None, int(frontier), arr(mov_out))
    h = 0
    for r in range(n):
        h = (h + O.comm_hash(int(parts[r]), comm[r])) & 0xFFFFFFFFFFFFFFFF
    return {"modularity": mod, "iters": iters.value, "trace": trace[:min(iters.value, max_trace)].copy(),
            "comm": comm, "constant": const.value, "chash_final": h, "converged": bool(converged.value),
            "movable": [m[:s].copy() for m, s in zip(mov_out, sizes)]}
