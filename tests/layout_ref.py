"""Exact host restatement of the setup decisions and of the layout the locality renumbering builds (DESIGN.md §3.3).

Everything here is an integer function of one shard (parts, rowptr, global tails, rank) and the options, so the device
arrays that mv_layout_readback returns can be compared with it element for element (tests/test_gpu_layout.py):

  compact CSR  own vertices are slots [0, lnv); a non-owned tail becomes lnv + its rank among the sorted unique
               non-owned tails; nlow of those lie below base.
  auto mode    reorder=2 samples rows 0, 64, 128, ... and renumbers when lnv >= 65536, at least one sampled edge stays
               on the rank, and (double) sum |t - v| / (double) count > lnv / 64.0 over the sampled edges with t < lnv.
  BFS key      seeds are the vertices v % stride == 0, region v / stride, level 0.  The BFS follows out-edges to own
               slots only.  key(v) = d << 22 | region, d the BFS distance to the nearest seed and region the smallest
               region among the seeds at distance d; distances above 1023 stay 0xFFFFFFFF (unreached).
  sort key     (region << 8) | min(level, 255); unreached vertices get all ones over sort_bits.
  layout       perm = stable argsort of the sort keys, inv = perm^-1, lab = base + perm; the renumbered CSR keeps each
               row's edge order, maps own tails through inv, leaves ghost slots alone and carries the weights along.
  keep order   a rank that does not renumber while another does: perm = inv = identity, lab = base + v, CSR unchanged.
  FIRST gate   simple_sorted = unit and not unordered and not has_self; iteration 1 runs the singleton reduction when
               simple_sorted, first_iter, scan_variant >= 4 and the 64-bit surface all hold.
"""
import numpy as np

REGION_BITS = 22
LEVEL_BITS = 8
MAX_LEVELS = 1023
MAX_REGIONS = (1 << REGION_BITS) - 1
UNREACHED = 0xFFFFFFFF
AUTO_MIN_LNV = 65536
SPAN_STRIDE = 64


def edge_index(rowptr, rows):
    """Concatenated edge positions of `rows` (in that order) and the row each one belongs to."""
    rowptr = np.asarray(rowptr, np.int64)
    rows = np.asarray(rows, np.int64)
    starts = rowptr[rows]
    deg = rowptr[rows + 1] - starts
    n = int(deg.sum())
    first = np.cumsum(deg) - deg
    idx = np.repeat(starts - first, deg) + np.arange(n, dtype=np.int64)
    return idx, np.repeat(rows, deg)


def compact_csr(parts, rowptr, tails, rank=0):
    """The compact CSR the device renumbers: (rowptr, slot tails, nlow, sorted unique ghost ids)."""
    base, bound = int(parts[rank]), int(parts[rank + 1])
    lnv = bound - base
    t = np.asarray(tails, np.int64)
    own = (t >= base) & (t < bound)
    ghosts = np.unique(t[~own])
    slots = np.where(own, t - base, lnv + np.searchsorted(ghosts, t))
    return (np.asarray(rowptr, np.int64).astype(np.uint32), slots.astype(np.int32), int(np.searchsorted(ghosts, base)),
            ghosts)


def span_sample(lnv, rowptr, tails, stride=SPAN_STRIDE):
    """k_span_sample: (sum |t - v|, count) over the edges with t < lnv of rows 0, stride, 2 stride, ..."""
    idx, src = edge_index(rowptr, np.arange(0, lnv, stride))
    t = np.asarray(tails, np.int64)[idx]
    keep = t < lnv
    return int(np.abs(t[keep] - src[keep]).sum()), int(keep.sum())


def auto_wants(lnv, span_sum, span_cnt):
    """The auto decision, compared in double exactly as setup_run compares it."""
    return lnv >= AUTO_MIN_LNV and span_cnt > 0 and float(span_sum) / float(span_cnt) > float(lnv) / 64.0


def effective_stride(lnv, region_size):
    """Region stride after the clamp that keeps every region id below 2^22 - 1."""
    return max(int(region_size), -(-int(lnv) // MAX_REGIONS))


def nregions_of(lnv, stride):
    return -(-int(lnv) // int(stride))


def bfs_keys(lnv, rowptr, tails, stride, max_levels=MAX_LEVELS):
    """k_msbfs's final keys, level by level: a vertex first reached from level L gets level L + 1 and the smallest region
    among its reached in-neighbours at level L (which is the smallest region among its nearest seeds)."""
    rowptr = np.asarray(rowptr, np.int64)
    tails = np.asarray(tails, np.int64)
    key = np.full(lnv, UNREACHED, np.uint32)
    region = np.zeros(lnv, np.int64)
    frontier = np.arange(0, lnv, stride, dtype=np.int64)
    region[frontier] = frontier // stride
    key[frontier] = (frontier // stride).astype(np.uint32)
    level = 0
    while level < max_levels and len(frontier):
        idx, src = edge_index(rowptr, frontier)
        w = tails[idx]
        own = w < lnv
        src, w = src[own], w[own]
        new = key[w] == UNREACHED
        src, w = src[new], w[new]
        reg = region[src]
        order = np.lexsort((reg, w))
        uw, first = np.unique(w[order], return_index=True)
        ureg = reg[order][first]
        region[uw] = ureg
        key[uw] = (((level + 1) << REGION_BITS) | ureg).astype(np.uint32)
        frontier = uw
        level += 1
    return key


def sort_bits_of(nregions):
    """setup_run's radix width: the level bits plus enough region bits to hold nregions (so all ones is above every key)."""
    b = LEVEL_BITS
    while (1 << (b - LEVEL_BITS)) <= nregions and b < 32:
        b += 1
    return b


def sort_keys(key, nregions):
    """k_bfs_sortkeys: region major, level minor (clamped to 8 bits), unreached = all ones over sort_bits."""
    key = np.asarray(key, np.uint32).astype(np.int64)
    sb = sort_bits_of(nregions)
    region = key & ((1 << REGION_BITS) - 1)
    level = np.minimum(key >> REGION_BITS, (1 << LEVEL_BITS) - 1)
    sk = (region << LEVEL_BITS) | level
    sk[key == UNREACHED] = (1 << sb) - 1
    return sk.astype(np.uint32)


def permute_csr(perm, inv, rowptr, tails, weights=None):
    """k_permute_adj: row i of the new CSR is row perm[i] of the old one, own tails mapped through inv."""
    lnv = len(perm)
    rowptr = np.asarray(rowptr, np.int64)
    idx, _ = edge_index(rowptr, perm)
    deg = (rowptr[1:] - rowptr[:-1])[perm]
    rowptr2 = np.concatenate([[0], np.cumsum(deg)]).astype(np.uint32)
    t = np.asarray(tails, np.int64)[idx]
    own = t < lnv
    t2 = t.copy()
    t2[own] = inv[t[own]]
    w2 = None if weights is None else np.asarray(weights, np.float64)[idx]
    return rowptr2, t2.astype(np.int32), w2


def out_of_order(rowptr, tails, lnv, nlow):
    """Some row is not strictly increasing in tails_ascend order (lower ghosts, own slots, upper ghosts)."""
    rowptr = np.asarray(rowptr, np.int64)
    t = np.asarray(tails, np.int64)
    cls = np.where(t < lnv, 1, np.where(t < lnv + nlow, 0, 2))
    k = (cls << 32) | t
    if len(k) < 2:
        return False
    step_ok = k[1:] > k[:-1]
    row_start = np.zeros(len(k), bool)
    row_start[rowptr[:-1][rowptr[:-1] < len(k)]] = True
    return bool(np.any(~step_ok & ~row_start[1:]))


def has_self_loop(rowptr, tails, weights=None):
    """k_vertex_init's has_self: a self loop (unit path) or a nonzero self-loop weight sum (weighted path)."""
    rowptr = np.asarray(rowptr, np.int64)
    src = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
    loop = np.asarray(tails, np.int64) == src
    if weights is None:
        return bool(loop.any())
    sums = np.zeros(len(rowptr) - 1)
    np.add.at(sums, src[loop], np.asarray(weights, np.float64)[loop])
    return bool(np.any(sums != 0.0))


def rank_want(parts, rowptr, tails, rank=0, reorder=2):
    """This rank's own decision (want) and the span sample, (-1, -1) where the sample does not run."""
    lnv = int(parts[rank + 1] - parts[rank])
    rp, slots, _, _ = compact_csr(parts, rowptr, tails, rank)
    span = (-1, -1)
    if reorder == 2 and lnv >= AUTO_MIN_LNV:
        span = span_sample(lnv, rp, slots)
    want = reorder == 1 or (reorder == 2 and auto_wants(lnv, *span))
    return bool(want), span


def layout(parts, rowptr, tails, rank=0, weights=None, reorder=2, region_size=512, relabel=None, unit=True,
           first_iter=1, scan_variant=6, f32=False):
    """Everything mv_layout_readback reports for one rank.  relabel: whether ANY rank renumbers (default: this one's
    decision, i.e. a single rank).  weights: the weighted path's edge weights (None: unit path)."""
    base = int(parts[rank])
    lnv = int(parts[rank + 1]) - base
    rp, slots, nlow, ghosts = compact_csr(parts, rowptr, tails, rank)
    want, span = rank_want(parts, rowptr, tails, rank, reorder)
    if relabel is None:
        relabel = want
    stride = effective_stride(lnv, region_size)
    out = {"lnv": lnv, "lne": len(slots), "nlow": nlow, "nghost": len(ghosts), "rowptr": rp, "tails": slots,
           "want": int(want), "relabel": int(bool(relabel)), "span": span, "stride": stride, "nregions": 0,
           "reordered": int(bool(want and lnv > 0))}
    if relabel and lnv > 0:
        if want:
            nreg = nregions_of(lnv, stride)
            key = bfs_keys(lnv, rp, slots, stride)
            perm = np.argsort(sort_keys(key, nreg), kind="stable").astype(np.int32)
            inv = np.empty(lnv, np.int32)
            inv[perm] = np.arange(lnv, dtype=np.int32)
            out.update(nregions=nreg, bfs_key=key)
            out["rowptr2"], out["tails2"], out["weights2"] = permute_csr(perm, inv, rp, slots, weights)
        else:
            perm = inv = np.arange(lnv, dtype=np.int32)
        out.update(perm=perm, inv=inv, lab=(base + perm.astype(np.int64)).astype(np.int32))
    unordered = out_of_order(rp, slots, lnv, nlow) if (out["reordered"] or unit) else False
    has_self = has_self_loop(rp, slots, None if unit else weights)
    simple = unit and not unordered and not has_self
    out.update(unordered=int(unordered), has_self=int(has_self), simple_sorted=int(simple),
               first_ran=int(simple and bool(first_iter) and scan_variant >= 4 and not f32 and lnv > 0))
    return out


def shard_layouts(parts, rowptrs, tails_list, weights_list=None, **opts):
    """Layouts of every rank of a run: relabel is the OR of the ranks' own decisions, as the all-reduce makes it."""
    n = len(rowptrs)
    wants = [rank_want(parts, rowptrs[r], tails_list[r], r, opts.get("reorder", 2))[0] for r in range(n)]
    return [layout(parts, rowptrs[r], tails_list[r], r, None if weights_list is None else weights_list[r],
                   relabel=any(wants), **opts) for r in range(n)]
