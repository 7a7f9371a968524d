"""NumPy / scipy restatement of splitting an assignment into its connected pieces (DESIGN.md §3.12;
mvgpu_split_communities), TEST INFRASTRUCTURE.

For an assignment X (global community ids in [0, nv), caller numbering) two vertices i and j are joined when
X(i) = X(j) and some shard stores a record i -> j or j -> i: any weight (zero included), either direction (weak
connectivity on the records as stored), self loops join nothing.  Y(v) is the smallest vertex id of v's component.
The report counts the non-empty communities of X, the components (= the communities of Y) and the communities of X
with more than one component."""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components


def global_records(parts, rowptrs, edge_lists):
    """(nv, src, dst) of every stored record of the shards, global ids."""
    parts = np.asarray(parts, np.int64)
    nv = int(parts[-1])
    src = np.concatenate([int(parts[r]) + np.repeat(np.arange(len(rp) - 1, dtype=np.int64), np.diff(np.asarray(rp, np.int64)))
                          for r, rp in enumerate(rowptrs)] + [np.zeros(0, np.int64)])
    dst = np.concatenate([np.asarray(e["tail"], np.int64) for e in edge_lists] + [np.zeros(0, np.int64)])
    return nv, src, dst


def split(parts, rowptrs, edge_lists, comm):
    """parts, per-shard rowptrs / edge records (global tails) and per-shard (or concatenated) assignment -> dict with Y
    (concatenated, int64) and the counts of mvgpu_split_report."""
    nv, src, dst = global_records(parts, rowptrs, edge_lists)
    X = np.concatenate([np.asarray(c, np.int64) for c in comm]) if isinstance(comm, (list, tuple)) else np.asarray(comm, np.int64)
    assert len(X) == nv and (nv == 0 or (X.min() >= 0 and X.max() < nv))
    if nv == 0:
        return {"Y": np.zeros(0, np.int64), "communities": 0, "components": 0, "disconnected": 0}
    keep = (X[src] == X[dst]) & (src != dst)
    G = sp.coo_matrix((np.ones(int(keep.sum()), np.int8), (src[keep], dst[keep])), shape=(nv, nv)).tocsr()
    ncomp, comp = connected_components(G, directed=True, connection="weak")
    smallest = np.full(ncomp, nv, np.int64)
    np.minimum.at(smallest, comp, np.arange(nv, dtype=np.int64))
    pieces = np.unique(np.stack([X, comp]), axis=1)[0]            # one entry per (community, component) pair
    per_comm = np.bincount(pieces, minlength=nv)
    return {"Y": smallest[comp], "communities": int((per_comm > 0).sum()), "components": int(ncomp),
            "disconnected": int((per_comm > 1).sum())}
