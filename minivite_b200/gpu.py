"""ctypes binding of libmvgpu.so (include/mvgpu.h) + the host-side mirror of the reference seam.

`dist_louvain_method(me, nprocs, shard, lower, thresh)` has the argument meaning of the reference's
`distLouvainMethod` (dspl.hpp:1280-1283): it returns (modularity, iters).  There is NO CPU fallback:
if the CUDA library is missing or no GPU is usable every call raises.

Per-vertex inputs (assignments, masks, update batches) may be NumPy arrays or torch tensors; a CUDA tensor is read
where it lies (DESIGN.md §3.16).  Per-vertex outputs are NumPy arrays, or torch tensors on the context's device with
device=True.  torch is imported only when a tensor is passed or device=True.
"""
import ctypes
import os
import sys

import numpy as np

_LIB_PATH = os.environ.get("MVGPU_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libmvgpu.so")
UNIQUE_ID_BYTES = 128

TRACE_DTYPE = np.dtype([("modularity", "<f8"), ("moved", "<i8"), ("chash", "<u8")])


class Timings(ctypes.Structure):
    _fields_ = [("total_s", ctypes.c_double), ("setup_s", ctypes.c_double), ("scan_s", ctypes.c_double),
                ("fold_s", ctypes.c_double), ("exchange_s", ctypes.c_double), ("h2d_s", ctypes.c_double),
                ("scan_launches", ctypes.c_int64), ("kernel_launches", ctypes.c_int64),
                ("iters", ctypes.c_int32), ("unit_weight", ctypes.c_int32), ("reorder_s", ctypes.c_double),
                ("reordered", ctypes.c_int32), ("scan_kernel_chosen", ctypes.c_int32), ("h2d_bytes", ctypes.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Quality(ctypes.Structure):
    _fields_ = [("modularity", ctypes.c_double), ("e_in", ctypes.c_double), ("a2", ctypes.c_double),
                ("constant", ctypes.c_double), ("communities", ctypes.c_int64), ("singletons", ctypes.c_int64),
                ("max_size", ctypes.c_int64), ("eval_s", ctypes.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SplitReport(ctypes.Structure):
    _fields_ = [("communities", ctypes.c_int64), ("components", ctypes.c_int64), ("disconnected", ctypes.c_int64),
                ("rounds", ctypes.c_int32), ("split_s", ctypes.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class CompareReport(ctypes.Structure):
    _fields_ = [("vertices", ctypes.c_int64), ("communities_x", ctypes.c_int64), ("communities_y", ctypes.c_int64),
                ("cells", ctypes.c_int64), ("pairs_xy", ctypes.c_uint64), ("pairs_x", ctypes.c_uint64),
                ("pairs_y", ctypes.c_uint64), ("pairs_all", ctypes.c_uint64), ("ari", ctypes.c_double),
                ("rand", ctypes.c_double), ("nmi", ctypes.c_double), ("vi", ctypes.c_double), ("mi", ctypes.c_double),
                ("h_x", ctypes.c_double), ("h_y", ctypes.c_double), ("compare_s", ctypes.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class ProbeReport(ctypes.Structure):
    _fields_ = [("vertices", ctypes.c_int64), ("moves", ctypes.c_int64), ("vetoed", ctypes.c_int64),
                ("interior", ctypes.c_int64), ("max_gain", ctypes.c_double), ("constant", ctypes.c_double),
                ("probe_s", ctypes.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


EXPORTS = ["mvgpu_last_error", "mvgpu_device_count", "mvgpu_create", "mvgpu_destroy", "mvgpu_get_unique_id",
           "mvgpu_comm_init", "mvgpu_upload_shard", "mvgpu_attach_shard_device", "mvgpu_generate_rgg_shard", "mvgpu_generate_rgg_shard_ex",
           "mvgpu_download_shard", "mvgpu_louvain",
           "mvgpu_get_communities", "mvgpu_get_communities_device", "mvgpu_upload_shard32", "mvgpu_louvain32", "mvgpu_get_communities32", "mvgpu_set_option", "mvgpu_get_trace",
           "mvgpu_get_timings", "mvgpu_get_scan_times", "mvgpu_get_constant", "mvgpu_get_shard_info", "mvgpu_dist_louvain_method",
           "mvgpu_set_initial_communities", "mvgpu_get_converged", "mvgpu_evaluate_communities",
           "mvgpu_get_community_stats", "mvgpu_get_compact_communities", "mvgpu_update_shard", "mvgpu_split_communities",
           "mvgpu_compare_communities", "mvgpu_get_community_matches", "mvgpu_set_movable", "mvgpu_get_movable",
           "mvgpu_probe_communities"]

_lib = None


def lib():
    """Load libmvgpu.so (fails loudly if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise RuntimeError(f"{_LIB_PATH} missing: the CUDA extension is not built "
                               "(python -c 'import __graft_entry__ as g; g.build()'); there is no CPU fallback")
        L = ctypes.CDLL(_LIB_PATH)
        vp, i64, dbl, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_double, ctypes.c_int
        L.mvgpu_last_error.restype = ctypes.c_char_p
        L.mvgpu_create.argtypes = [ctypes.POINTER(vp), ci, ci, ci]
        L.mvgpu_destroy.argtypes = [vp]
        L.mvgpu_get_unique_id.argtypes = [vp]
        L.mvgpu_comm_init.argtypes = [vp, vp]
        L.mvgpu_upload_shard.argtypes = [vp, i64, vp, i64, i64, vp, vp]
        L.mvgpu_attach_shard_device.argtypes = [vp, i64, vp, i64, i64, vp, vp]
        L.mvgpu_generate_rgg_shard.argtypes = [vp, i64, ci, ctypes.POINTER(i64)]
        L.mvgpu_generate_rgg_shard_ex.argtypes = [vp, i64, ci, ci, ctypes.c_double, ctypes.POINTER(i64)]
        L.mvgpu_download_shard.argtypes = [vp, vp, vp]
        L.mvgpu_update_shard.argtypes = [vp, i64, vp, vp, i64, vp, vp, vp, ctypes.POINTER(i64)]
        L.mvgpu_louvain.argtypes = [vp, dbl, dbl, ctypes.POINTER(ci), ctypes.POINTER(dbl)]
        L.mvgpu_get_communities.argtypes = [vp, vp]
        L.mvgpu_set_initial_communities.argtypes = [vp, vp]
        L.mvgpu_get_converged.argtypes = [vp, ctypes.POINTER(ci)]
        L.mvgpu_set_movable.argtypes = [vp, vp]
        L.mvgpu_get_movable.argtypes = [vp, vp]
        L.mvgpu_evaluate_communities.argtypes = [vp, vp, ctypes.POINTER(Quality)]
        L.mv_evaluate_refused.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(Quality)]
        L.mvgpu_get_community_stats.argtypes = [vp, vp, vp, vp]
        L.mvgpu_split_communities.argtypes = [vp, vp, vp, ctypes.POINTER(SplitReport)]
        L.mv_split_refused.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(SplitReport)]
        L.mvgpu_compare_communities.argtypes = [vp, vp, vp, ctypes.POINTER(CompareReport)]
        L.mv_compare_refused.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(CompareReport)]
        L.mvgpu_probe_communities.argtypes = [vp, vp, vp, vp, vp, ctypes.POINTER(ProbeReport)]
        L.mv_probe_refused.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(ProbeReport)]
        L.mvgpu_get_community_matches.argtypes = [vp, vp, vp, vp, vp]
        L.mvgpu_get_compact_communities.argtypes = [vp, vp]
        L.mvgpu_upload_shard32.argtypes = [vp, ctypes.c_int32, vp, ctypes.c_int32, ctypes.c_int32, vp, vp]
        L.mvgpu_louvain32.argtypes = [vp, ctypes.c_float, ctypes.c_float, ctypes.POINTER(ci), ctypes.POINTER(ctypes.c_float)]
        L.mvgpu_get_communities32.argtypes = [vp, vp]
        L.mvgpu_get_communities_device.argtypes = [vp, ctypes.POINTER(vp)]
        L.mvgpu_set_option.argtypes = [vp, ctypes.c_char_p, i64]
        L.mvgpu_get_trace.argtypes = [vp, ci, vp, ctypes.POINTER(ci)]
        L.mvgpu_get_timings.argtypes = [vp, ctypes.POINTER(Timings)]
        L.mvgpu_get_scan_times.argtypes = [vp, ci, vp, ctypes.POINTER(ci)]
        L.mvgpu_get_constant.argtypes = [vp, ctypes.POINTER(dbl)]
        L.mvgpu_get_shard_info.argtypes = [vp, vp]
        L.mvgpu_dist_louvain_method.argtypes = [ci, i64, i64, vp, vp, dbl, dbl, ctypes.POINTER(ci),
                                                ctypes.POINTER(dbl), vp]
        _lib = L
    return _lib


class MvgpuError(RuntimeError):
    pass


def _ck(rc):
    if rc != 0:
        raise MvgpuError(lib().mvgpu_last_error().decode(errors="replace"))


_NP = {"i8": np.int64, "u1": np.uint8, "f8": np.float64}
_TORCH = {"i8": "int64", "u1": "uint8", "f8": "float64"}


def _cuda_tensor(a):
    t = sys.modules.get("torch")         # a caller holding a tensor has imported torch
    return t is not None and isinstance(a, t.Tensor) and a.is_cuda


class _Input:
    """An input array as the C ABI reads it.  kind: "i8" (int64 ids), "u1" (a mask: nonzero = 1) or "f8" (float64).
    A CUDA tensor is converted on its own device and passed as a device pointer once its current stream has been
    synchronised (the library reads it on its own stream); a tensor on another device than the context's is passed
    as well, and the library refuses it.  Anything else becomes a C-contiguous NumPy array.  An empty array passes a
    one-element dummy of the same kind: a zero-length array has no address, and NULL means "no array"."""

    def __init__(self, a, kind, flat=False):
        if _cuda_tensor(a):
            import torch
            t = a.reshape(-1) if flat else a
            t = (t != 0).to(torch.uint8) if kind == "u1" and t.dtype != torch.uint8 else t.to(getattr(torch, _TORCH[kind]))
            t = t.contiguous()
            self.ndim, self.size = t.dim(), t.numel()
            self.arr = t if self.size else torch.zeros(1, dtype=t.dtype, device=t.device)
            torch.cuda.current_stream(t.device).synchronize()
            self.ptr = self.arr.data_ptr()
        else:
            x = np.ascontiguousarray(a)
            x = x.reshape(-1) if flat else x
            x = (x != 0).astype(np.uint8) if kind == "u1" and x.dtype != np.uint8 else np.ascontiguousarray(x, _NP[kind])
            self.ndim, self.size = x.ndim, x.size
            self.arr = x if x.size else np.zeros(1, _NP[kind])
            self.ptr = self.arr.ctypes.data


def _outputs(device, ctx_device, n, kinds):
    """Output arrays of n entries (at least one, so that a pointer is never NULL on an empty rank): NumPy, or torch
    tensors on the context's device (device=True), whose allocation the library's stream is ordered after."""
    if not device:
        out = [np.zeros(max(n, 1), _NP[k]) for k in kinds]
        return out, [o.ctypes.data for o in out]
    import torch
    dev = torch.device("cuda", ctx_device)
    out = [torch.empty(max(n, 1), dtype=getattr(torch, _TORCH[k]), device=dev) for k in kinds]
    torch.cuda.current_stream(dev).synchronize()
    return out, [o.data_ptr() for o in out]


def device_count():
    n = lib().mvgpu_device_count()
    if n < 0:
        raise MvgpuError(lib().mvgpu_last_error().decode(errors="replace"))
    return n


def get_unique_id():
    buf = ctypes.create_string_buffer(UNIQUE_ID_BYTES)
    _ck(lib().mvgpu_get_unique_id(buf))
    return buf.raw


class LouvainGPU:
    """One rank == one GPU (the per-process state of the reference's distLouvainMethod)."""

    def __init__(self, device=0, rank=0, nranks=1):
        self._h = ctypes.c_void_p()
        self.rank, self.nranks, self.device = rank, nranks, device
        _ck(lib().mvgpu_create(ctypes.byref(self._h), device, rank, nranks))
        self.lnv = 0
        self.base = 0                # global id of this rank's first vertex
        self._keep = None

    def comm_init(self, unique_id: bytes):
        assert len(unique_id) == UNIQUE_ID_BYTES
        _ck(lib().mvgpu_comm_init(self._h, ctypes.c_char_p(unique_id)))

    def upload(self, nv_global, parts, rowptr, edges):
        """Host arrays of a reference Graph shard (graph.hpp:289-293) -> HBM."""
        parts = np.ascontiguousarray(parts, dtype=np.int64)
        rowptr = np.ascontiguousarray(rowptr, dtype=np.int64)
        edges = np.ascontiguousarray(edges)
        assert edges.dtype.itemsize == 16, "edge records must be {int64 tail; double weight}"
        lnv, lne = len(rowptr) - 1, len(edges)
        assert int(rowptr[-1]) == lne
        _ck(lib().mvgpu_upload_shard(self._h, int(nv_global), parts.ctypes.data, lnv, lne, rowptr.ctypes.data,
                                     edges.ctypes.data if lne else None))
        self.lnv, self.base = lnv, int(parts[self.rank])

    # ---- the reference's USE_32_BIT_GRAPH build: int32 ids, float weights, float results (include/mvgpu.h)
    def upload32(self, nv_global, parts, rowptr, edges):
        parts = np.ascontiguousarray(parts, dtype=np.int32)
        rowptr = np.ascontiguousarray(rowptr, dtype=np.int32)
        edges = np.ascontiguousarray(edges)
        assert edges.dtype.itemsize == 8, "edge records must be {int32 tail; float weight}"
        lnv, lne = len(rowptr) - 1, len(edges)
        assert int(rowptr[-1]) == lne
        _ck(lib().mvgpu_upload_shard32(self._h, int(nv_global), parts.ctypes.data, lnv, lne, rowptr.ctypes.data,
                                       edges.ctypes.data if lne else None))
        self.lnv, self.base = lnv, int(parts[self.rank])

    def louvain32(self, lower=-1.0, thresh=1.0e-6):
        iters = ctypes.c_int(0)
        mod = ctypes.c_float(0.0)
        _ck(lib().mvgpu_louvain32(self._h, lower, thresh, ctypes.byref(iters), ctypes.byref(mod)))
        return mod.value, iters.value

    def communities32(self):
        out = np.empty(self.lnv, dtype=np.int32)
        _ck(lib().mvgpu_get_communities32(self._h, out.ctypes.data))
        return out

    def attach_device(self, nv_global, parts, lnv, lne, d_rowptr_ptr, d_edges_ptr, keepalive=None):
        """Arrays already resident in this GPU's memory (raw device pointers)."""
        parts = np.ascontiguousarray(parts, dtype=np.int64)
        _ck(lib().mvgpu_attach_shard_device(self._h, int(nv_global), parts.ctypes.data, int(lnv), int(lne),
                                            ctypes.c_void_p(d_rowptr_ptr), ctypes.c_void_p(d_edges_ptr)))
        self.lnv, self.base = int(lnv), int(parts[self.rank])
        self._keep = keepalive

    def generate_rgg(self, nv_global, unit_weight=True, lcg=False, random_edge_percent=0.0):
        """Build this rank's strip of `miniVite -n nv_global [-w] [-l] [-p pct]` on the device (reference GenerateRGG);
        returns lne.  With several ranks and random_edge_percent > 0 the call is collective (after comm_init)."""
        lne = ctypes.c_int64(0)
        _ck(lib().mvgpu_generate_rgg_shard_ex(self._h, int(nv_global), int(bool(unit_weight)), int(bool(lcg)),
                                              float(random_edge_percent), ctypes.byref(lne)))
        self.lnv = int(nv_global) // self.nranks
        self.base = self.rank * self.lnv
        self._lne = lne.value
        return lne.value

    def download_shard(self):
        """The shard's reference-format arrays (int64 rowptr, {tail, weight} records) as numpy arrays."""
        info = self.shard_info()
        rowptr = np.zeros(info["lnv"] + 1, dtype=np.int64)
        edges = np.zeros(info["lne"], dtype=np.dtype([("tail", "<i8"), ("weight", "<f8")]))
        _ck(lib().mvgpu_download_shard(self._h, rowptr.ctypes.data, edges.ctypes.data if info["lne"] else None))
        return rowptr, edges

    def update_shard(self, delete=None, insert=None):
        """Change the shard in place on the device (DESIGN.md §3.11): delete=(src, dst) drops every record (src, dst) of
        the shard, insert=(src, dst, w) merges new records in; global ids, src owned by this rank, both directions of an
        undirected edge given by the caller.  Collective with several ranks (pass None, None when a rank has no
        changes).  Returns the new lne.  Each array may be a NumPy array or a torch tensor (CUDA tensors are read on the
        device)."""
        def cols(t, kinds, what):
            if t is None:
                return 0, [None] * len(kinds), []
            if len(t) != len(kinds):
                raise ValueError(f"{what} takes {len(kinds)} arrays")
            arrs = [_Input(a, k, flat=True) for a, k in zip(t, kinds)]
            if any(a.size != arrs[0].size for a in arrs):
                raise ValueError(f"{what}: arrays of different lengths")
            n = arrs[0].size
            return n, [a.ptr if n else None for a in arrs], arrs
        n_del, (ds, dd), keep_del = cols(delete, ("i8", "i8"), "delete")
        n_ins, (is_, id_, iw), keep_ins = cols(insert, ("i8", "i8", "f8"), "insert")
        lne = ctypes.c_int64(0)
        _ck(lib().mvgpu_update_shard(self._h, n_del, ds, dd, n_ins, is_, id_, iw, ctypes.byref(lne)))
        del keep_del, keep_ins
        self._keep = None            # an attached shard's arrays are no longer read
        return lne.value

    def set_option(self, name, value):
        _ck(lib().mvgpu_set_option(self._h, name.encode(), int(value)))

    def louvain(self, lower=-1.0, thresh=1.0e-6):
        iters = ctypes.c_int(0)
        mod = ctypes.c_double(0.0)
        _ck(lib().mvgpu_louvain(self._h, lower, thresh, ctypes.byref(iters), ctypes.byref(mod)))
        return mod.value, iters.value

    def set_initial_communities(self, comm):
        """Start every later louvain() on this shard from `comm` (lnv global community ids in [0, nv), caller's vertex
        numbering, e.g. what communities() returned; a NumPy array or a torch tensor) instead of singletons; None clears
        it.  The array is copied at call time.  A new upload / attach / generate clears it too.  Resuming a run stopped by
        the stop_after option from its communities() with lower = its modularity continues that run exactly."""
        if comm is None:
            _ck(lib().mvgpu_set_initial_communities(self._h, None))
            return
        a = _Input(comm, "i8")
        if a.ndim != 1 or a.size != self.lnv:
            raise ValueError(f"initial assignment has {a.size} entries, the shard has lnv = {self.lnv}")
        _ck(lib().mvgpu_set_initial_communities(self._h, a.ptr))

    def set_movable(self, mask):
        """Hold vertices in place (DESIGN.md §3.14): every later louvain() on this shard lets only the vertices with a
        nonzero entry in `mask` (lnv entries, caller's vertex numbering, a NumPy array or a torch tensor) move; with the
        option frontier = 1 the set grows from the vertices that move.  The mask is copied at call time.  None clears it
        (everything movable); a new upload / attach / generate clears it too, update_shard keeps it.  With several ranks
        every rank or none must set one."""
        if mask is None:
            _ck(lib().mvgpu_set_movable(self._h, None))
            return
        a = _Input(mask, "u1")
        if a.ndim != 1 or a.size != self.lnv:
            raise ValueError(f"movable set has {a.size} entries, the shard has lnv = {self.lnv}")
        _ck(lib().mvgpu_set_movable(self._h, a.ptr))

    def movable(self, device=False):
        """The set the next iteration would use (uint8 0 / 1, lnv entries): after a run with a set, the set after its last
        accepted iteration -- resume a stop_after checkpoint with it; otherwise the set as given, all ones without one.
        device=True: a torch tensor on the context's device."""
        (out,), (p,) = _outputs(device, self.device, self.lnv, ("u1",))
        _ck(lib().mvgpu_get_movable(self._h, p))
        return out[:self.lnv]

    def movable_from_batch(self, delete=None, insert=None):
        """The lnv mask (uint8) of this rank's `src` endpoints of an update_shard batch: delete = (src, dst), insert =
        (src, dst, w) as update_shard takes them.  The caller gives both directions of every edge, so every endpoint is
        covered on its owner without communication.  Endpoints outside this rank raise ValueError."""
        mask = np.zeros(self.lnv, np.uint8)
        for t in (delete, insert):
            if t is None:
                continue
            src = np.ascontiguousarray(t[0], dtype=np.int64).reshape(-1) - self.base
            if src.size and (src.min() < 0 or src.max() >= self.lnv):
                raise ValueError("batch src outside this rank's vertices")
            mask[src] = 1
        return mask

    def converged(self):
        """True if the last louvain() ended on the exit test, False if the stop_after option ended it first."""
        v = ctypes.c_int(0)
        _ck(lib().mvgpu_get_converged(self._h, ctypes.byref(v)))
        return bool(v.value)

    def _assignment(self, comm, refuse, rep):
        """comm as the collective entry points take it: None, or an _Input of lnv ids.  A wrong shape still enters the
        collective through `refuse`, flagged, so that the other ranks fail with this one instead of waiting for it."""
        if comm is None:
            return None
        a = _Input(comm, "i8")
        if a.ndim != 1 or a.size != self.lnv:
            why = f"assignment has {a.size} entries, the shard has lnv = {self.lnv}"
            _ck(refuse(self._h, why.encode(), ctypes.byref(rep)))
            raise AssertionError("unreachable: a refused call fails")
        return a

    def evaluate(self, comm=None):
        """Modularity Q and community counts of an assignment (lnv global community ids in [0, nv), caller's vertex
        numbering, the form set_initial_communities takes; a NumPy array or a torch tensor); None evaluates what the last
        louvain() returned.  Collective: every rank passes an array or every rank None; a bad id or an array whose length
        is not lnv on any rank raises MvgpuError on every rank.  Returns mvgpu_quality as a dict (DESIGN.md §3.10)."""
        q = Quality()
        a = self._assignment(comm, lib().mv_evaluate_refused, q)
        _ck(lib().mvgpu_evaluate_communities(self._h, a and a.ptr, ctypes.byref(q)))
        return q.as_dict()

    def split_communities(self, comm=None, device=False):
        """Split every community of an assignment into its connected pieces (DESIGN.md §3.12): Y gives each vertex the
        smallest global id of its component, where two vertices are joined when they share a community and the shard
        stores a record between them.  `comm` takes the form evaluate() takes; None splits what the last louvain()
        returned.  Collective, with evaluate()'s error rules.  Returns (Y, report): Y is this rank's lnv entries (int64,
        a valid input to set_initial_communities and evaluate; a torch tensor on the context's device with device=True),
        report the global counts of mvgpu_split_report as a dict."""
        rep = SplitReport()
        a = self._assignment(comm, lib().mv_split_refused, rep)
        (out,), (p,) = _outputs(device, self.device, self.lnv, ("i8",))
        _ck(lib().mvgpu_split_communities(self._h, a and a.ptr, p, ctypes.byref(rep)))
        return out[:self.lnv], rep.as_dict()

    def compare_communities(self, y, x=None):
        """Compare two assignments (DESIGN.md §3.13): contingency counts, pair counts, ARI, Rand index, NMI, VI and the
        entropies, exact and the same on every rank count.  `y` and `x` take the form evaluate() takes (each a NumPy array
        or a torch tensor, of either kind); x = None compares what the last louvain() returned.  Collective: every rank
        passes x or every rank None; a bad id or a wrong length on any rank raises MvgpuError on every rank.  Returns
        mvgpu_compare_report as a dict; community_matches() then gives the best match of every community of x."""
        rep = CompareReport()
        arrs = [None if a is None else _Input(a, "i8") for a in (x, y)]
        bad = [a for a in arrs if a is not None and (a.ndim != 1 or a.size != self.lnv)]
        if y is None or bad:
            # still enter the collective, flagged, so that the other ranks fail with this one instead of waiting for it
            why = ("y must not be None" if y is None else
                   f"assignment has {bad[0].size} entries, the shard has lnv = {self.lnv}")
            _ck(lib().mv_compare_refused(self._h, why.encode(), ctypes.byref(rep)))
            raise AssertionError("unreachable: a refused comparison fails")
        _ck(lib().mvgpu_compare_communities(self._h, arrs[0] and arrs[0].ptr, arrs[1].ptr, ctypes.byref(rep)))
        return rep.as_dict()

    def probe(self, comm=None, device=False):
        """What every vertex would do under the Louvain rule from an assignment (DESIGN.md §3.15), without moving anything.
        `comm` takes the form evaluate() takes; None probes what the last louvain() returned.  Collective, with
        evaluate()'s error rules.  Returns (report, target, best, gain): mvgpu_probe_report as a dict (global counts), and
        this rank's lnv entries of the decision (int64), the best candidate community (int64, -1 without one) and its
        gain (float64, -inf without one); torch tensors on the context's device with device=True."""
        rep = ProbeReport()
        a = self._assignment(comm, lib().mv_probe_refused, rep)
        (target, best, gain), outs = _outputs(device, self.device, self.lnv, ("i8", "i8", "f8"))
        _ck(lib().mvgpu_probe_communities(self._h, a and a.ptr, *outs, ctypes.byref(rep)))
        return rep.as_dict(), target[:self.lnv], best[:self.lnv], gain[:self.lnv]

    def community_matches(self, device=False):
        """Per community of x in the last compare_communities(): entry s describes community parts[rank] + s.  Returns a
        dict of int64 arrays `size`, `best`, `overlap` and `best_size`, lnv entries each (best = -1 for an empty x);
        torch tensors on the context's device with device=True."""
        names = ("size", "best", "overlap", "best_size")
        out, ptrs = _outputs(device, self.device, self.lnv, ("i8",) * 4)
        _ck(lib().mvgpu_get_community_matches(self._h, *ptrs))
        return {k: a[:self.lnv] for k, a in zip(names, out)}

    def community_stats(self, device=False):
        """Per community of the last evaluate(): entry s describes community parts[rank] + s.  Returns a dict of
        `size` (int64), `volume` and `internal` (float64), lnv entries each; torch tensors on the context's device with
        device=True."""
        (size, vol, internal), ptrs = _outputs(device, self.device, self.lnv, ("i8", "f8", "f8"))
        _ck(lib().mvgpu_get_community_stats(self._h, *ptrs))
        return {"size": size[:self.lnv], "volume": vol[:self.lnv], "internal": internal[:self.lnv]}

    def compact_communities(self, device=False):
        """Per vertex of the last evaluate(): its community's rank among the non-empty ids in ascending id (int64); a
        torch tensor on the context's device with device=True."""
        (out,), (p,) = _outputs(device, self.device, self.lnv, ("i8",))
        _ck(lib().mvgpu_get_compact_communities(self._h, p))
        return out[:self.lnv]

    def communities(self, out=None, device=False):
        """currComm of this rank's vertices (global community ids).  `out`: optional preallocated int64 array
        (pinned or pageable: a pinned one is filled by one copy, a pageable one in chunks through the library's pinned
        bounce buffers, so neither takes the driver's staged pageable copy).  device=True: a torch tensor on the context's
        device instead."""
        if device:
            assert out is None, "device=True allocates its own tensor"
            (t,), (p,) = _outputs(True, self.device, self.lnv, ("i8",))
            _ck(lib().mvgpu_get_communities(self._h, p))
            return t[:self.lnv]
        if out is None:
            out = np.empty(self.lnv, dtype=np.int64)
        assert out.dtype == np.int64 and out.size >= self.lnv and out.flags["C_CONTIGUOUS"]
        _ck(lib().mvgpu_get_communities(self._h, out.ctypes.data))
        return out[:self.lnv]

    def trace(self):
        n = ctypes.c_int(0)
        _ck(lib().mvgpu_get_trace(self._h, 0, None, ctypes.byref(n)))
        out = np.zeros(n.value, dtype=TRACE_DTYPE)
        if n.value:
            _ck(lib().mvgpu_get_trace(self._h, n.value, out.ctypes.data, ctypes.byref(n)))
        return out

    def timings(self):
        t = Timings()
        _ck(lib().mvgpu_get_timings(self._h, ctypes.byref(t)))
        return t.as_dict()

    def scan_times(self):
        n = ctypes.c_int(0)
        _ck(lib().mvgpu_get_scan_times(self._h, 0, None, ctypes.byref(n)))
        out = np.zeros(n.value, dtype=np.float64)
        if n.value:
            _ck(lib().mvgpu_get_scan_times(self._h, n.value, out.ctypes.data, ctypes.byref(n)))
        return out

    def constant(self):
        v = ctypes.c_double(0)
        _ck(lib().mvgpu_get_constant(self._h, ctypes.byref(v)))
        return v.value

    def shard_info(self):
        info = (ctypes.c_int64 * 6)()
        _ck(lib().mvgpu_get_shard_info(self._h, info))
        return dict(zip(["lnv", "lne", "nghost", "nsend", "nheavy", "maxdeg"], [int(x) for x in info]))

    def close(self):
        if self._h:
            lib().mvgpu_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def dist_louvain_method(me, nprocs, shard, lower=-1.0, thresh=1.0e-6, device=None, unique_id=None, want_comm=False):
    """Mirror of the reference call `distLouvainMethod(me, nprocs, g, ..., lower, thresh, iters)`
    (dspl.hpp:1280-1283, called from main.cpp:168).  `shard` is a hostgraph.Shard (the arrays of the
    reference's Graph).  Returns (modularity, iters[, communities])."""
    g = LouvainGPU(device if device is not None else me, me, nprocs)
    try:
        if nprocs > 1:
            g.comm_init(unique_id)
        g.upload(shard.nv, shard.parts, shard.rowptr, shard.edges)
        mod, iters = g.louvain(lower, thresh)
        if want_comm:
            return mod, iters, g.communities()
        return mod, iters
    finally:
        g.close()
