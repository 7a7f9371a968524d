"""Engineered shards for the persistent scan kernels (test infrastructure; tests/scan_schedule.py restates the kernels).

A layout is a list of 32-vertex groups, each of one "kind", with every vertex's degree chosen so that the group lands
on a boundary of the group schedule: an empty edge block, a block that widens to exactly one staging buffer or to one
to three edges more, a sub-range that stops at a given lane, vertices of degree heavy_deg / heavy_deg + 1 at every
alignment, heavy vertices at the edges of a group.  Group g goes to warp g mod (8 k) on a grid of k CTAs; the kinds
follow a de Bruijn order, so that with one CTA every warp meets every ordered pair of kinds.  The degree sequence is
then realised as a simple graph (no loops, no parallel edges, sorted adjacency: iteration 1 can take the singleton
reduction), unit weights or dyadic k/4.  The tests check through the restatement that every boundary is actually hit.
"""
import numpy as np

EDGE_DTYPE = np.dtype([("tail", "<i8"), ("weight", "<f8")])
GROUP_KINDS = ("empty", "whole_cap", "over", "split", "boundary", "heavy")


def de_bruijn(k):
    """Cyclic de Bruijn sequence B(k, 2) plus its first symbol: every ordered pair (a, b) of 0..k-1 is adjacent once."""
    a = [0] * (2 * k)
    seq = []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq + seq[:1]


def _spread(total, n):
    """n non-negative degrees summing to total, as equal as possible."""
    q, r = divmod(total, n)
    return [q + (1 if i < r else 0) for i in range(n)]


class _Builder:
    def __init__(self, cap, heavy_deg):
        self.cap, self.hd = cap, heavy_deg
        self.deg, self.kinds, self.notes = [], [], []
        self.count = {}

    @property
    def e0(self):
        return sum(self.deg)

    def _n(self, kind):
        i = self.count.get(kind, 0)
        self.count[kind] = i + 1
        return i

    def add(self, kind, degs, note=None, trim_lane=None, next_r=None):
        """Append one group; trim_lane: a lane whose degree may grow by 0..3 so that the next group starts at an edge
        offset congruent to next_r mod 4."""
        degs = list(degs)
        if trim_lane is not None and next_r is not None:
            degs[trim_lane] += (next_r - (self.e0 + sum(degs))) % 4
        self.deg.extend(degs)
        self.kinds.append(kind)
        self.notes.append(note)

    def group(self, kind, next_r):
        cap, hd = self.cap, self.hd
        r = self.e0 % 4
        i = self._n(kind)
        if kind == "empty":
            self.add(kind, [0] * 32)
        elif kind == "whole_cap":                  # e1 - lo4 == CAP exactly
            self.add(kind, _spread(cap - r, 32), note=r)
        elif kind == "over":                       # e1 - lo4 == CAP + 1..3
            j = 1 + i % 3
            self.add(kind, _spread(cap + j - r, 32), note=j)
        elif kind == "split":                      # the first sub-range stops at lane k (capacity), zero degrees inside
            k = 1 + i % 31
            head = cap - r - 20
            lanes = [0] * 32
            inner = [l for l in range(k) if not (k >= 3 and l == k // 2)]
            for l, d in zip(inner, _spread(head, len(inner))):
                lanes[l] = d
            lanes[k] = 40
            for l in range(k + 1, 32):
                lanes[l] = 0 if l % 3 == 0 else 2
            self.add(kind, lanes, note=k, trim_lane=31, next_r=next_r)
        elif kind == "boundary":                   # degree heavy_deg at ra mod 4 = r and r + 1, then heavy_deg + 1
            lanes = [hd, 1, hd] + [0 if l % 4 == 0 else 12 for l in range(3, 32)]
            if self.with_heavy:
                lanes[3] = hd + 1
            self.add(kind, lanes, trim_lane=31, next_r=next_r)
        elif kind == "heavy":
            v = i % 8
            lanes = [12] * 32
            if v in (0, 4):                        # lane 0, table just above heavy_deg
                lanes[0] = hd + 1
            elif v in (1, 5):                      # lane 31, degree just above a power of two
                lanes[31] = 513
            elif v == 2:                           # two adjacent heavies at k_scan_ws's kECap boundary (2048 / 2049)
                lanes[10], lanes[11] = 2048, 2049
                lanes[20] = 1025
            elif v == 6:                           # two adjacent heavies just above heavy_deg
                lanes[10], lanes[11] = hd + 1, hd + 2
            elif v == 3 and i < 8:                 # a group of 32 heavy vertices
                lanes = [hd + 1 + l for l in range(32)]
            else:                                  # lanes 0 and 31
                lanes[0], lanes[31] = hd + 1, hd + 3
            self.add(kind, lanes, note=v, trim_lane=30 if v in (1, 5) else 29, next_r=next_r)
        else:
            raise ValueError(kind)


def layout(cap, heavy_deg, kinds, warps=8, ragged=1, seed=0):
    """Degree sequence of a de Bruijn layout over `kinds` for `warps` warps, plus one ragged group of `ragged`
    vertices.  Returns (deg, kind_of_group, notes)."""
    seq = de_bruijn(len(kinds))
    b = _Builder(cap, heavy_deg)
    b.with_heavy = "heavy" in kinds
    order = [kinds[s] for s in seq for _w in range(warps)]
    steer = {}
    for i, kind in enumerate(order):
        nxt = order[i + 1] if i + 1 < len(order) else None
        if kind in ("split", "boundary", "heavy"):      # the kinds with a trim lane: cycle the next group's offset mod 4
            steer[nxt] = steer.get(nxt, seed) + 1
        b.group(kind, next_r=steer.get(nxt, seed) % 4)
    b.deg.extend([1] + [2] * (ragged - 1))
    b.kinds.append("ragged")
    b.notes.append(ragged)
    if sum(b.deg) % 2:
        b.deg[-1] += 1
    return np.array(b.deg, np.int64), b.kinds, b.notes


def realize(deg, seed=0):
    """A simple graph with exactly these degrees.  Kleitman-Wang: the vertices are laid off in index order, each to
    the others of largest remaining degree (ties broken at random), which succeeds on every graphical sequence.
    Returns (rowptr, tails) with sorted adjacency."""
    deg = np.asarray(deg, np.int64)
    n = len(deg)
    assert deg.sum() % 2 == 0
    rng = np.random.default_rng(seed)
    rem = deg.copy()
    us, vs = [], []
    for v in range(n):
        k = int(rem[v])
        if k == 0:
            continue
        rem[v] = 0
        key = rem + rng.random(n) * 0.5
        idx = np.argpartition(-key, k - 1)[:k]
        assert np.all(rem[idx] > 0), "degree sequence is not graphical"
        rem[idx] -= 1
        us.append(np.full(k, v, np.int64))
        vs.append(idx.astype(np.int64))
    u, v = np.concatenate(us), np.concatenate(vs)
    src = np.concatenate([u, v])
    dst = np.concatenate([v, u])
    order = np.lexsort((dst, src))
    src, dst = src[order], dst[order]
    rowptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=rowptr[1:])
    assert np.array_equal(np.diff(rowptr), deg)
    return rowptr, dst


def edges_of(rowptr, tails, dyadic=False, seed=0):
    """{tail, weight} records: unit weights, or k/4 (k in 1..8) per undirected edge, equal in both directions."""
    tails = np.asarray(tails, np.int64)
    n = len(rowptr) - 1
    e = np.zeros(len(tails), EDGE_DTYPE)
    e["tail"] = tails
    if not dyadic:
        e["weight"] = 1.0
        return e
    src = np.repeat(np.arange(n, dtype=np.int64), np.diff(rowptr))
    a, b = np.minimum(src, tails), np.maximum(src, tails)
    e["weight"] = ((a * 7 + b * 13 + seed) % 8 + 1).astype(np.float64) / 4.0
    return e


def split_at(rowptr, edges, parts):
    """Shards of a global CSR at the given vertex offsets (any offsets, not only the reference's even split)."""
    rps, eds = [], []
    for r in range(len(parts) - 1):
        a, b = int(parts[r]), int(parts[r + 1])
        rp = rowptr[a:b + 1] - rowptr[a]
        rps.append(rp.astype(np.int64))
        eds.append(edges[rowptr[a]:rowptr[b]].copy())
    return rps, eds


def claims(rowptr, kinds, cap, heavy_deg, layout_kinds, with_heavy, whole_path):
    """What a de Bruijn layout claims to cover, counted from the schedule restatement (tests/scan_schedule.py) rather
    than from the builder's intent.  Returns (counts, required keys)."""
    import scan_schedule as SS
    from collections import Counter
    warps, plans = SS.schedule(rowptr, cap, heavy_deg, 1)
    c = Counter()
    req = []
    for p, kind in zip(plans, kinds):
        span, r = p["e1"] - p["lo4"], p["e0"] % 4
        c[f"kind_{kind}"] += 1
        if kind == "empty" and p["e1"] == p["e0"]:
            c["empty"] += 1
            c["empty_unaligned_block"] += r != 0 and p["n4"] == 4
        if kind == "whole_cap" and span == cap and p["n4"] == cap:
            c[f"whole_cap_r{r}"] += 1
            c["whole_path_at_cap"] += p["whole"]
        if kind == "over" and cap < span <= cap + 3:
            c[f"over_by_{span - cap}"] += 1
            c["over_split"] += len(p["subs"]) == 2 and p["subs"][1]["sync"]
        if kind == "split" and p["subs"] and p["subs"][0]["stop"] == "cap":
            c[f"stop_lane_{p['subs'][0]['end']}"] += 1
            for s in p["subs"]:
                c["zero_deg_in_sub"] += any(p["deg"][l] == 0 for l in range(s["start"] + 1, s["end"] - 1))
        for l in range(p["nvalid"]):
            if p["deg"][l] == heavy_deg and l not in p["heavy"]:
                c[f"deg_hd_ra{p['ra'][l] % 4}"] += 1
            if p["deg"][l] == heavy_deg + 1 and l in p["heavy"]:
                c[f"deg_hd1_ra{p['ra'][l] % 4}"] += 1
        h = p["heavy"]
        if h:
            c["heavy_lane0"] += 0 in h
            c["heavy_lane31"] += 31 in h
            c["heavy_adjacent"] += any(b == a + 1 for a, b in zip(h, h[1:]))
            c["heavy_all32"] += len(h) == 32
            for l in h:
                d = p["deg"][l]
                c["table_just_above_hd"] += d == heavy_deg + 1
                c["table_just_above_pow2"] += d > 64 and (d - 1) & (d - 2) == 0
    last = plans[-1]
    c[f"ragged_{last['nvalid']}"] += last["nvalid"] < 32
    pairs = SS.pair_coverage(kinds, len(kinds), 1)
    for a in layout_kinds:
        for b in layout_kinds:
            c[f"pair_{a}_{b}"] = pairs.get((a, b), 0)
            req.append(f"pair_{a}_{b}")
    req += ["empty", "empty_unaligned_block"] + [f"whole_cap_r{r}" for r in range(4)] + \
        [f"over_by_{j}" for j in (1, 2, 3)] + ["over_split"] + [f"stop_lane_{k}" for k in range(1, 32)] + \
        ["zero_deg_in_sub"] + [f"deg_hd_ra{q}" for q in range(4)] + [f"ragged_{last['nvalid']}"]
    if whole_path:
        req.append("whole_path_at_cap")
    if with_heavy:
        req += [f"deg_hd1_ra{q}" for q in range(4)] + ["heavy_lane0", "heavy_lane31", "heavy_adjacent", "heavy_all32",
                                                       "table_just_above_hd", "table_just_above_pow2"]
    return c, req


# ---- the layouts the tests run --------------------------------------------------------------------------------------
UNIT_CAP, UNIT_HD = 512, 508
W_CAP, W_HD = 320, 316
LIGHT_KINDS = ("empty", "whole_cap", "over", "split", "boundary")


def unit_heavy():
    """Every kind, heavy vertices included (has_heavy: no group takes the whole-block path); last group 1 vertex."""
    deg, kinds, notes = layout(UNIT_CAP, UNIT_HD, GROUP_KINDS, ragged=1, seed=1)
    rowptr, tails = realize(deg, seed=1)
    return rowptr, tails, kinds, notes


def unit_light():
    """No heavy vertex (the whole-block path is live); last group 31 vertices."""
    deg, kinds, notes = layout(UNIT_CAP, UNIT_HD, LIGHT_KINDS, ragged=31, seed=1)
    rowptr, tails = realize(deg, seed=2)
    return rowptr, tails, kinds, notes


def weighted_heavy():
    """The heavy layout at the weighted path's buffer (CAP 320, heavy_deg 316); weights k/4."""
    deg, kinds, notes = layout(W_CAP, W_HD, GROUP_KINDS, ragged=31, seed=0)
    rowptr, tails = realize(deg, seed=3)
    return rowptr, tails, kinds, notes


# k_scan_pq under X = identity: every vertex with edges is hard with m = its degree, so the ring follows the degrees.
PQ_CTAS = 4                                   # 32 warps: one final-drain residue per warp
PQ_STREAM = ("p12", "p31", "p12", "m13", "split_pq", "p12", "residue")


def pq_layout():
    """Groups for k_scan_pq with PQ_CTAS CTAs (group 32 i + w is warp w's i-th), padded by one group of heavy vertices
    so that 2m is a power of two (c = 1/2m exact).  Returns (rowptr, tails, kind_of_group)."""
    nw = PQ_CTAS * 8
    deg, kinds = [], []
    for i, kind in enumerate(PQ_STREAM):
        for w in range(nw):
            if kind == "p12":                                  # 32 hard vertices with m = 12: parked, drained
                lanes = [12] * 32
            elif kind == "p31":                                # 31 parked, one isolated vertex
                lanes = [1 + (l + w) % 12 for l in range(32)]
                lanes[w % 32] = 0
            elif kind == "m13":                                # one vertex with m = 13: the group runs in place
                lanes = [(l + w) % 13 for l in range(32)]
                lanes[(w * 7) % 32] = 13
            elif kind == "split_pq":                           # sub-range 1 in place (300 edges), sub-range 2 parks
                lanes = [300] + [12] * 31
            else:                                              # final residue t = w mod 31 + 1 after 13 waiting
                t = w % 31 + 1
                f = t - 13 if t >= 13 else t + 19
                lanes = [1 + l % 12 if l < f else 0 for l in range(32)]
            deg.extend(lanes)
            kinds.append(kind)
    total = sum(deg)
    target = 1 << int(np.ceil(np.log2(total + 32 * (UNIT_HD + 1))))
    pad = _spread(target - total, 32)
    assert min(pad) > UNIT_HD
    deg.extend(pad)
    kinds.append("pad_heavy")
    rowptr, tails = realize(np.array(deg, np.int64), seed=5)
    assert rowptr[-1] == target
    return rowptr, tails, kinds


def pq_bound_assignment(rowptr, tails):
    """X for the exact-bound cases of k_scan_pq on pq_layout() (2m = 2^k, so c and the bounds are exact): identity
    except (a) a degree-8 vertex v whose community C holds 5 of its neighbours and other vertices up to
    vol(C) - 8 = 2m / 4, so that its bound 2 (3 - 5) + fl(fl(16 (2m / 4)) c) is exactly 0.0, and (b) a vertex joined to
    the neighbour u of smallest degree while another neighbour has that degree too: its bound is positive and its best
    gain is exactly 0.0.  Returns (X, v_zero_bound, v_zero_gain)."""
    import scan_schedule as SS
    rowptr = np.asarray(rowptr, np.int64)
    deg = np.diff(rowptr)
    n = len(deg)
    two_m = int(rowptr[-1])
    assert two_m & (two_m - 1) == 0
    X = np.arange(n, dtype=np.int64)
    v = int(np.nonzero(deg == 8)[0][0])
    nb = [int(t) for t in tails[rowptr[v]:rowptr[v + 1]]]
    inside, need = nb[:5], two_m // 4 - int(deg[nb[:5]].sum())
    banned = set(nb) | {v}
    members = list(inside)
    for x in np.argsort(-deg, kind="stable").tolist():
        if need == 0:
            break
        if x not in banned and 0 < deg[x] <= need:
            members.append(x)
            banned.add(x)
            need -= int(deg[x])
    assert need == 0
    X[members] = v
    c = 1.0 / float(two_m)
    for v2 in range(n):
        if v2 in banned or deg[v2] < 2 or deg[v2] > 12:
            continue
        nb2 = tails[rowptr[v2]:rowptr[v2 + 1]]
        if any(int(y) in banned for y in nb2):
            continue
        dn = deg[nb2]
        if np.count_nonzero(dn == dn.min()) < 2:
            continue
        u = int(nb2[np.argmin(dn)])
        Y = X.copy()
        Y[v2] = u
        cdeg, csize = SS.community_state(rowptr, tails, Y)
        r = SS.vertex_pq(v2, rowptr, tails, Y, cdeg, csize, c)
        if r["hard"] and r["best_gain"] == 0.0 and r["bound"] > 0.0:
            return Y, v, v2
    raise AssertionError("no vertex with a zero best gain")


def default_grid_layout(groups, seed=0):
    """A large, cheap shard for the default grid: `groups` groups, each empty, a perfect matching inside the group
    (degree 1), or a clique on lanes 0..k-1 with k in 22..26 (506..650 edges: the whole block or sub-ranges).  Returns
    (rowptr, tails, kind_of_group)."""
    rng = np.random.default_rng(seed)
    kinds = [("empty", "pairs", "clique")[i] for i in rng.integers(0, 3, groups)]
    src, dst = [], []
    for g, kind in enumerate(kinds):
        b = 32 * g
        if kind == "pairs":
            a = np.arange(b, b + 32, 2)
            src += [a, a + 1]
            dst += [a + 1, a]
        elif kind == "clique":
            k = 22 + g % 5
            i, j = np.meshgrid(np.arange(k), np.arange(k), indexing="ij")
            off = i != j
            src.append(b + i[off])
            dst.append(b + j[off])
    src, dst = np.concatenate(src), np.concatenate(dst)
    order = np.lexsort((dst, src))
    src, dst = src[order], dst[order]
    n = 32 * groups
    rowptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=rowptr[1:])
    return rowptr, dst.astype(np.int64), kinds
