"""NumPy restatement of mvgpu_update_shard (DESIGN.md §3.11) and the plain per-row loop it is checked against.

A batch is deletions (src, dst) and insertions (src, dst, w), directed records in global ids whose src lies in the
shard's rows [base, base + lnv).  Per row v:
  1. every old record of v whose tail is the dst of some deletion (v, dst) goes; the rest keep their order;
  2. v's insertions, stably sorted by (dst, position in the batch), are merged into the survivors by "emit the next
     old record while its tail <= the next insertion's tail, otherwise the insertion";
  3. deletions match old records only.
"""
import numpy as np

EDGE_DTYPE = np.dtype([("tail", "<i8"), ("weight", "<f8")])


def _cols(batch, dtypes):
    if batch is None:
        return [np.zeros(0, d) for d in dtypes]
    return [np.asarray(a, d) for a, d in zip(batch, dtypes)]


DEL, INS = (np.int64, np.int64), (np.int64, np.int64, np.float64)


def apply_loop(base, rowptr, edges, delete=None, insert=None):
    """Rules 1-3 as a plain loop over rows and records."""
    ds, dd = _cols(delete, DEL)
    is_, id_, iw = _cols(insert, INS)
    lnv = len(rowptr) - 1
    dels = [set() for _ in range(lnv)]
    for s, d in zip(ds.tolist(), dd.tolist()):
        dels[s - base].add(d)
    ins = [[] for _ in range(lnv)]
    for k, (s, d, w) in enumerate(zip(is_.tolist(), id_.tolist(), iw.tolist())):
        ins[s - base].append((d, k, w))
    out_rp, out = [0], []
    for v in range(lnv):
        old = [(int(edges["tail"][a]), float(edges["weight"][a])) for a in range(int(rowptr[v]), int(rowptr[v + 1]))]
        old = [r for r in old if r[0] not in dels[v]]
        new = sorted(ins[v])
        a = b = 0
        while a < len(old) or b < len(new):
            if b >= len(new) or (a < len(old) and old[a][0] <= new[b][0]):
                out.append(old[a])
                a += 1
            else:
                out.append((new[b][0], new[b][2]))
                b += 1
        out_rp.append(len(out))
    e = np.zeros(len(out), EDGE_DTYPE)
    if out:
        e["tail"] = [t for t, _ in out]
        e["weight"] = [w for _, w in out]
    return np.array(out_rp, np.int64), e


def apply(base, rowptr, edges, delete=None, insert=None):
    """The same result, vectorised the way the device computes it: with M(a) the running maximum of row v's kept
    tails up to record a, kept record a lands at newrow[v] + #kept before a + #{insertions of v with tail < M(a)} and
    the j-th insertion of v (tail t) at newrow[v] + j + #{kept a of v with M(a) <= t}."""
    ds, dd = _cols(delete, DEL)
    is_, id_, iw = _cols(insert, INS)
    lnv = len(rowptr) - 1
    rowptr = np.asarray(rowptr, np.int64)
    tail = np.asarray(edges["tail"], np.int64)
    row = np.repeat(np.arange(lnv, dtype=np.int64), np.diff(rowptr))
    span = int(max(tail.max(initial=0), dd.max(initial=0), id_.max(initial=0))) + 2
    keep = ~np.isin(row * span + tail, (ds.astype(np.int64) - base) * span + dd.astype(np.int64))
    kscan = np.concatenate([[0], np.cumsum(keep)])
    # segmented running max (-1 before the row's first kept record): rows are made disjoint by an offset of row * span
    m = np.maximum.accumulate(np.where(keep, tail + 1, 0) + row * span) - row * span - 1
    order = np.lexsort((np.arange(len(is_)), id_, is_))
    irow, itail, iwt = (is_[order] - base).astype(np.int64), id_[order].astype(np.int64), iw[order]
    istart = np.searchsorted(irow, np.arange(lnv + 1))
    ikey = irow * span + itail
    deg = (kscan[rowptr[1:]] - kscan[rowptr[:-1]]) + np.diff(istart)
    nrow = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    out = np.zeros(int(nrow[-1]), EDGE_DTYPE)
    a = np.nonzero(keep)[0]
    below = np.searchsorted(ikey, row[a] * span + m[a], "left") - istart[row[a]]
    pos = nrow[row[a]] + (kscan[a] - kscan[rowptr[row[a]]]) + below
    out[pos] = edges[a]
    mkey = row * span + (m + 1)                  # non-decreasing: rows ascend and M ascends within a row
    upto = np.searchsorted(mkey, irow * span + itail + 1, "right")
    j = np.arange(len(irow)) - istart[irow]
    pos = nrow[irow] + j + (kscan[upto] - kscan[rowptr[irow]])
    out["tail"][pos] = itail
    out["weight"][pos] = iwt
    return nrow, out


def extras(small, big):
    """The records of shard `big` whose (row, tail) pair has no record in shard `small`, in big's order, as an
    insertion batch (src, dst, w) -- for big = small + `-p` random edges, which never hit an RGG pair.  Both shards'
    rows are sorted by tail, as the generator writes them."""
    lnv = len(small.rowptr) - 1
    span = small.nv + 1
    skey = np.repeat(np.arange(lnv, dtype=np.int64), np.diff(small.rowptr)) * span + small.edges["tail"]
    rb = np.repeat(np.arange(lnv, dtype=np.int64), np.diff(big.rowptr))
    bkey = rb * span + big.edges["tail"]
    assert np.all(np.diff(skey) >= 0)
    at = np.minimum(np.searchsorted(skey, bkey), max(len(skey) - 1, 0))
    new = skey[at] != bkey if len(skey) else np.ones(len(bkey), bool)
    return (rb[new] + small.base, big.edges["tail"][new].copy(), big.edges["weight"][new].copy())
