"""Python access to tests/warm_oracle.c (TEST INFRASTRUCTURE): the C oracle's Louvain phase started from a given
assignment and / or stopped after k accepted iterations.  The library is compiled on first use with the oracle's own
flags into the temporary directory (keyed by the sources' contents), so the tree is never written."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "warm_oracle.c")
_lib = None


def _load():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in (SRC, O.SRC):
            with open(f, "rb") as fh:
                h.update(fh.read())
        lib = os.path.join(tempfile.gettempdir(), f"mv_warm_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(lib):
            tmp = f"{lib}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall",
                                   "-o", tmp, SRC, "-lm"])
            os.replace(tmp, lib)
        L = ctypes.CDLL(lib)
        L.mvo_louvain_warm.restype = ctypes.c_double
        L.mvo_louvain_warm.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_double,
                                       ctypes.c_double, ctypes.POINTER(ctypes.c_int), ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.c_void_p, ctypes.c_int,
                                       ctypes.POINTER(ctypes.c_int)]
        _lib = L
    return _lib


def louvain(parts, rowptrs, edge_lists, lower=-1.0, thresh=1.0e-6, max_trace=512, init_comm=None, stop_after=0):
    """oracle.louvain() with init_comm (per-shard starting assignments, global community ids; None = singletons) and
    stop_after (> 0: stop after that many accepted iterations).  Returns oracle.louvain()'s dict plus `converged`
    (False when stop_after ended the run)."""
    L = _load()
    n = len(rowptrs)
    parts = np.ascontiguousarray(parts, dtype=np.int64)
    assert len(parts) == n + 1
    rps = [np.ascontiguousarray(r, dtype=np.int64) for r in rowptrs]
    eds = [np.ascontiguousarray(e) for e in edge_lists]
    assert all(e.dtype.itemsize == 16 for e in eds)
    comm = [np.zeros(int(parts[r + 1] - parts[r]), dtype=np.int64) for r in range(n)]
    PtrArr = ctypes.c_void_p * n
    rp_ptrs = PtrArr(*[r.ctypes.data for r in rps])
    ed_ptrs = PtrArr(*[e.ctypes.data if len(e) else None for e in eds])
    cm_ptrs = PtrArr(*[c.ctypes.data if len(c) else None for c in comm])
    init_ptrs = None
    if init_comm is not None:
        assert len(init_comm) == n
        init = [np.ascontiguousarray(c, dtype=np.int64) for c in init_comm]
        for r in range(n):
            assert len(init[r]) == parts[r + 1] - parts[r]
            assert len(init[r]) == 0 or (init[r].min() >= 0 and init[r].max() < parts[n])
        init_ptrs = PtrArr(*[c.ctypes.data if len(c) else None for c in init])
    trace = np.zeros(max_trace, dtype=O.TRACE_DTYPE)
    iters = ctypes.c_int(0)
    const = ctypes.c_double(0)
    converged = ctypes.c_int(1)
    mod = L.mvo_louvain_warm(n, parts.ctypes.data, ctypes.cast(rp_ptrs, ctypes.c_void_p),
                             ctypes.cast(ed_ptrs, ctypes.c_void_p), lower, thresh, ctypes.byref(iters),
                             ctypes.cast(cm_ptrs, ctypes.c_void_p), trace.ctypes.data, max_trace, ctypes.byref(const),
                             ctypes.cast(init_ptrs, ctypes.c_void_p) if init_ptrs is not None else None,
                             int(stop_after), ctypes.byref(converged))
    h = 0
    for r in range(n):
        h = (h + O.comm_hash(int(parts[r]), comm[r])) & 0xFFFFFFFFFFFFFFFF
    return {"modularity": mod, "iters": iters.value, "trace": trace[:min(iters.value, max_trace)].copy(),
            "comm": comm, "constant": const.value, "chash_final": h, "converged": bool(converged.value)}
