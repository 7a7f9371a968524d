/* oracle/louvain_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of miniVite's single-phase distributed Louvain loop
 * (reference dspl.hpp:82-486, 488-952, 978-1103, 1106-1272, 1280-1441) used as
 * the CPU checker for the CUDA path.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline leg may call into this file; the product never does.
 *
 * Parity status: PINNED.  tests/test_oracle.py checks this restatement against
 * golden per-iteration traces (modularity %.17g, moved count, community hash)
 * captured from the UNMODIFIED reference built by oracle/build_ref.py
 * (tests/golden/, generator script tests/golden/make_golden.py), for 1, 2, 4 and
 * 8 ranks, and -- where /root/reference is present -- against live runs of
 * oracle/_ref/miniVite_ref.
 *
 * The `nranks` shards are executed in lock step inside one process; "messages"
 * are reads of the owner's arrays at the points where the reference exchanges
 * them, so every rank sees exactly the snapshot the MPI code would deliver:
 *   fillRemoteCommunities   dspl.hpp:488-952   ghost community + {size,degree} of remote communities
 *   scan                    dspl.hpp:276-405   (with 230-274 and 174-228)
 *   distUpdateLocalCinfo    dspl.hpp:458-471
 *   updateRemoteCommunities dspl.hpp:978-1103  remote deltas added at the owner, in source-rank order
 *   distComputeModularity   dspl.hpp:407-456   partial sums combined in rank order
 * Vertices are scanned in index order and edges in CSR order, i.e. the floating
 * point summation order of the reference run with one OpenMP thread per rank.
 * None of the reference's quirks are "fixed": selfLoop is truncated to an
 * integer (dspl.hpp:285), clusterWeight is measured before the moves and the
 * degree term after them (407-456), the returned modularity is that of the last
 * ACCEPTED iteration while `iters` counts the rejected one too (1401-1440).
 *
 * Three extensions, each off by default (init_comm = NULL, stop_after = 0, movable = NULL gives the pinned loop above,
 * operation for operation); tests/test_oracle.py and tests/test_movable_oracle.py hold them to the pinned path:
 *   init_comm   (warm start, DESIGN.md §3.9) every shard's starting currComm, global community ids in [0, nv).
 *               localCinfo is then the aggregate of that assignment: sizes counted and degrees summed in global vertex
 *               order.
 *   stop_after  > 0: end the run after that many ACCEPTED iterations; currComm is then the assignment after the last one
 *               and the return value its clamped prevMod (the `lower` to resume with).  *converged_out (may be NULL)
 *               is 0 then, and 1 when the reference's exit test ended the run.
 *   movable     (movable set, DESIGN.md §3.14) per shard, one byte per vertex, nonzero = movable.  A vertex outside M_k
 *               keeps its community in iteration k (targetComm = currComm, no Comm deltas); its counter[0] still enters
 *               clusterWeight, so the modularity keeps its definition.
 *   frontier    1: M_{k+1} = M_k + { u : a vertex v != u with a record v->u has targetComm != currComm in iteration k },
 *               taken over only when iteration k is accepted; 0: M_k = M.  Without a movable set it changes nothing.
 *   movable_out (may be NULL) per shard: the set the next iteration would use when the run ends (all ones without a
 *               movable set).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef int64_t GraphElem;   /* utils.hpp:78 */
typedef double GraphWeight;  /* utils.hpp:79 */

typedef struct { GraphElem tail; GraphWeight weight; } Edge;        /* graph.hpp:60-66 */
typedef struct { GraphElem size; GraphWeight degree; } Comm;        /* dspl.hpp:61-66 */

typedef struct {
  double modularity;     /* currMod of this iteration */
  int64_t moved;         /* #{i : targetComm[i] != currComm[i]} over all ranks */
  uint64_t chash;        /* shard-combinable hash of targetComm (SURVEY.md 8(c)) */
} MvoIterTrace;

/* ---- small int64 -> slot hash map (stands in for std::unordered_map / std::map) ---- */
typedef struct { GraphElem *keys; int64_t *vals; int64_t cap, n; } Map;

static uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
static uint64_t vhash(GraphElem gid, GraphElem val) {
  return mix64(((uint64_t)gid) * 0x9E3779B97F4A7C15ULL ^ (uint64_t)val);
}
static void map_init(Map *m, int64_t expect) {
  int64_t cap = 16;
  while (cap < 2 * expect + 2) cap <<= 1;
  m->cap = cap; m->n = 0;
  m->keys = (GraphElem *)malloc(sizeof(GraphElem) * cap);
  m->vals = (int64_t *)malloc(sizeof(int64_t) * cap);
  for (int64_t i = 0; i < cap; i++) m->keys[i] = -1;
}
static void map_free(Map *m) { free(m->keys); free(m->vals); m->keys = NULL; m->vals = NULL; m->cap = m->n = 0; }
static void map_clear(Map *m) { for (int64_t i = 0; i < m->cap; i++) m->keys[i] = -1; m->n = 0; }
static int64_t map_find(const Map *m, GraphElem k) {
  uint64_t h = mix64((uint64_t)k) & (uint64_t)(m->cap - 1);
  while (m->keys[h] != -1) { if (m->keys[h] == k) return m->vals[h]; h = (h + 1) & (uint64_t)(m->cap - 1); }
  return -1;
}
static void map_grow(Map *m);
/* insert if absent; returns the stored value; *where (optional) receives the table position */
static int64_t map_put_at(Map *m, GraphElem k, int64_t v, int64_t *where) {
  if (2 * (m->n + 1) > m->cap) map_grow(m);
  uint64_t h = mix64((uint64_t)k) & (uint64_t)(m->cap - 1);
  while (m->keys[h] != -1) { if (m->keys[h] == k) return m->vals[h]; h = (h + 1) & (uint64_t)(m->cap - 1); }
  m->keys[h] = k; m->vals[h] = v; m->n++;
  if (where) *where = (int64_t)h;
  return v;
}
static int64_t map_put(Map *m, GraphElem k, int64_t v) { return map_put_at(m, k, v, NULL); }
static void map_grow(Map *m) {
  Map o = *m;
  map_init(m, o.cap);
  for (int64_t i = 0; i < o.cap; i++) if (o.keys[i] != -1) map_put(m, o.keys[i], o.vals[i]);
  free(o.keys); free(o.vals);
}

/* ---- per-rank state: the locals of distLouvainMethod (dspl.hpp:1286-1292) ---- */
typedef struct {
  GraphElem base, bound, nv;
  const GraphElem *rowptr;
  const Edge *edges;
  GraphElem *pastComm, *currComm, *targetComm;
  GraphWeight *vDegree, *clusterWeight;
  Comm *localCinfo, *localCupdate;
  /* ghost lists (exchangeVertexReqs, dspl.hpp:1106-1272): unique non-owned tails */
  GraphElem *rvdata; int64_t rsz;
  Map remoteComm;            /* ghost vertex -> index into rcomm_val */
  GraphElem *rcomm_val;
  Map remoteC;               /* remote community -> index into remoteCinfo/remoteCupdate */
  GraphElem *remoteCkey; Comm *remoteCinfo, *remoteCupdate; int64_t nremoteC, capremoteC;
} Rank;

static int get_owner(const GraphElem *parts, int nranks, GraphElem v) {   /* graph.hpp:167-173 (upper_bound - 1) */
  int lo = 0, hi = nranks + 1;
  while (lo < hi) { int mid = (lo + hi) / 2; if (parts[mid] <= v) lo = mid + 1; else hi = mid; }
  return lo - 1;
}

static int cmp_elem(const void *a, const void *b) {
  GraphElem x = *(const GraphElem *)a, y = *(const GraphElem *)b;
  return (x > y) - (x < y);
}

static int64_t remoteC_slot(Rank *R, GraphElem c) {
  int64_t s = map_find(&R->remoteC, c);
  if (s >= 0) return s;
  if (R->nremoteC == R->capremoteC) {
    R->capremoteC = R->capremoteC ? 2 * R->capremoteC : 1024;
    R->remoteCkey = (GraphElem *)realloc(R->remoteCkey, sizeof(GraphElem) * R->capremoteC);
    R->remoteCinfo = (Comm *)realloc(R->remoteCinfo, sizeof(Comm) * R->capremoteC);
    R->remoteCupdate = (Comm *)realloc(R->remoteCupdate, sizeof(Comm) * R->capremoteC);
  }
  s = R->nremoteC++;
  R->remoteCkey[s] = c;
  map_put(&R->remoteC, c, s);
  return s;
}

/* dspl.hpp:174-228 -- candidate order is irrelevant: the rule selects the largest positive gain and, among
 * equal gains, the smallest community id. */
static GraphElem get_max_index(const GraphElem *clkeys, const GraphWeight *counter, int64_t nclus,
                               GraphWeight selfLoop, const Rank *R, GraphWeight vDegree, GraphElem currSize,
                               GraphWeight currDegree, GraphElem currComm, GraphWeight constant) {
  GraphElem maxIndex = currComm;
  GraphWeight curGain = 0.0, maxGain = 0.0;
  GraphWeight eix = counter[0] - selfLoop;
  GraphWeight ax = currDegree - vDegree;
  GraphWeight eiy = 0.0, ay = 0.0;
  GraphElem maxSize = currSize, size = 0;
  for (int64_t k = 0; k < nclus; k++) {
    const GraphElem y = clkeys[k];
    if (currComm != y) {
      if (y >= R->base && y < R->bound) { ay = R->localCinfo[y - R->base].degree; size = R->localCinfo[y - R->base].size; }
      else { int64_t s = map_find(&R->remoteC, y); ay = R->remoteCinfo[s].degree; size = R->remoteCinfo[s].size; }
      eiy = counter[k];
      curGain = 2.0 * (eiy - eix) - 2.0 * vDegree * (ay - ax) * constant;          /* dspl.hpp:212 */
      if ((curGain > maxGain) || ((curGain == maxGain) && (curGain != 0.0) && (y < maxIndex))) {
        maxGain = curGain; maxIndex = y; maxSize = size;
      }
    }
  }
  if ((maxSize == 1) && (currSize == 1) && (maxIndex > currComm)) maxIndex = currComm;   /* dspl.hpp:224-225 */
  return maxIndex;
}

/* Runs the whole phase.  Shard r owns vertices [parts[r], parts[r+1]); rowptr[r] are LOCAL offsets
 * (lnv+1 entries), edges[r] carry GLOBAL tails, exactly the arrays of a reference Graph.
 * Outputs: *iters_out (dspl.hpp:1430), returns prevMod (dspl.hpp:1440); comm_out[r] (may be NULL)
 * receives currComm of shard r at exit; trace[0..min(iters,max_trace)) the per-iteration records;
 * *constant_out = 1/(2m).  Returns NaN on allocation failure.  init_comm, stop_after, converged_out, movable,
 * frontier and movable_out are the extensions of the header. */
double mvo_louvain(int nranks, const int64_t *parts, const int64_t *const *rowptr, const void *const *edges,
                   double lower, double thresh, int *iters_out, int64_t *const *comm_out,
                   MvoIterTrace *trace, int max_trace, double *constant_out,
                   const int64_t *const *init_comm, int stop_after, int *converged_out,
                   const uint8_t *const *movable, int frontier, uint8_t *const *movable_out) {
  Rank *RK = (Rank *)calloc((size_t)nranks, sizeof(Rank));
  GraphElem nv_global = parts[nranks];
  GraphElem maxdeg = 0;
  uint8_t **M = NULL, **Mn = NULL;   /* M_k, and M_{k+1} while iteration k runs; NULL = every vertex movable */
  if (movable) {
    M = (uint8_t **)calloc((size_t)nranks, sizeof(uint8_t *));
    Mn = (uint8_t **)calloc((size_t)nranks, sizeof(uint8_t *));
    for (int r = 0; r < nranks; r++) {
      const GraphElem nv = parts[r + 1] - parts[r];
      M[r] = (uint8_t *)malloc((size_t)nv + 1); Mn[r] = (uint8_t *)malloc((size_t)nv + 1);
      for (GraphElem i = 0; i < nv; i++) M[r][i] = (movable[r][i] != 0);
    }
  }

  /* ---- distInitLouvain, dspl.hpp:151-172 ---- */
  GraphWeight totalEdgeWeightTwice = 0.0;
  for (int r = 0; r < nranks; r++) {
    Rank *R = &RK[r];
    R->base = parts[r]; R->bound = parts[r + 1]; R->nv = R->bound - R->base;
    R->rowptr = rowptr[r]; R->edges = (const Edge *)edges[r];
    const GraphElem nv = R->nv;
    R->pastComm = (GraphElem *)malloc(sizeof(GraphElem) * (nv + 1));
    R->currComm = (GraphElem *)malloc(sizeof(GraphElem) * (nv + 1));
    R->targetComm = (GraphElem *)malloc(sizeof(GraphElem) * (nv + 1));
    R->vDegree = (GraphWeight *)malloc(sizeof(GraphWeight) * (nv + 1));
    R->clusterWeight = (GraphWeight *)malloc(sizeof(GraphWeight) * (nv + 1));
    R->localCinfo = (Comm *)malloc(sizeof(Comm) * (nv + 1));
    R->localCupdate = (Comm *)malloc(sizeof(Comm) * (nv + 1));
    GraphWeight localWeight = 0.0;
    for (GraphElem i = 0; i < nv; i++) {                 /* distSumVertexDegree, dspl.hpp:82-107 */
      GraphWeight tw = 0.0;
      for (GraphElem k = R->rowptr[i]; k < R->rowptr[i + 1]; k++) tw += R->edges[k].weight;
      R->vDegree[i] = tw;
      R->localCinfo[i].degree = tw;
      R->localCinfo[i].size = 1;
      if (R->rowptr[i + 1] - R->rowptr[i] > maxdeg) maxdeg = R->rowptr[i + 1] - R->rowptr[i];
    }
    for (GraphElem i = 0; i < nv; i++) localWeight += R->vDegree[i];   /* dspl.hpp:122-123 */
    totalEdgeWeightTwice += localWeight;                                  /* Allreduce, rank order */
    for (GraphElem i = 0; i < nv; i++) { R->pastComm[i] = i + R->base; R->currComm[i] = i + R->base; }  /* 132-149 */
  }
  if (init_comm) {                                         /* warm start: the aggregate of the given assignment */
    for (int r = 0; r < nranks; r++)
      for (GraphElem i = 0; i < RK[r].nv; i++) { RK[r].localCinfo[i].size = 0; RK[r].localCinfo[i].degree = 0.0; }
    for (int r = 0; r < nranks; r++) {
      Rank *R = &RK[r];
      for (GraphElem i = 0; i < R->nv; i++) {
        const GraphElem c = init_comm[r][i];
        const int o = get_owner(parts, nranks, c);
        R->pastComm[i] = c; R->currComm[i] = c;
        RK[o].localCinfo[c - RK[o].base].size++;
        RK[o].localCinfo[c - RK[o].base].degree += R->vDegree[i];
      }
    }
  }
  const GraphWeight constantForSecondTerm = 1.0 / totalEdgeWeightTwice;    /* dspl.hpp:129 */
  if (constant_out) *constant_out = constantForSecondTerm;

  /* ---- exchangeVertexReqs, dspl.hpp:1106-1272: unique non-owned tails (order inside the list is
   * irrelevant to the results; we keep them sorted) ---- */
  for (int r = 0; r < nranks; r++) {
    Rank *R = &RK[r];
    const GraphElem lne = R->rowptr[R->nv];
    int64_t cnt = 0;
    for (GraphElem e = 0; e < lne; e++) { GraphElem t = R->edges[e].tail; if (t < R->base || t >= R->bound) cnt++; }
    GraphElem *tmp = (GraphElem *)malloc(sizeof(GraphElem) * (cnt + 1));
    cnt = 0;
    for (GraphElem e = 0; e < lne; e++) { GraphElem t = R->edges[e].tail; if (t < R->base || t >= R->bound) tmp[cnt++] = t; }
    qsort(tmp, (size_t)cnt, sizeof(GraphElem), cmp_elem);
    int64_t u = 0;
    for (int64_t i = 0; i < cnt; i++) if (i == 0 || tmp[i] != tmp[i - 1]) tmp[u++] = tmp[i];
    R->rvdata = tmp; R->rsz = u;
    R->rcomm_val = (GraphElem *)malloc(sizeof(GraphElem) * (u + 1));
    map_init(&R->remoteComm, u);
    for (int64_t i = 0; i < u; i++) map_put(&R->remoteComm, tmp[i], i);
    map_init(&R->remoteC, 1024);
  }

  /* per-vertex scratch standing in for clmap/counter (dspl.hpp:286-287) */
  GraphElem *clkeys = (GraphElem *)malloc(sizeof(GraphElem) * (maxdeg + 2));
  GraphWeight *counter = (GraphWeight *)malloc(sizeof(GraphWeight) * (maxdeg + 2));
  int64_t *clpos = (int64_t *)malloc(sizeof(int64_t) * (maxdeg + 2));
  Map clmap; map_init(&clmap, maxdeg + 2);   /* never grows: at most maxdeg+1 keys per vertex */

  GraphWeight prevMod = lower, currMod = -1.0;
  int numIters = 0, converged = 1;

  for (;;) {                                               /* dspl.hpp:1338 */
    numIters++;
    /* ---- fillRemoteCommunities, dspl.hpp:488-952 ---- */
    for (int r = 0; r < nranks; r++) {
      Rank *R = &RK[r];
      map_clear(&R->remoteC); R->nremoteC = 0;
      for (int64_t i = 0; i < R->rsz; i++) {               /* 559-571 gather at the owner + 670-688 */
        const GraphElem v = R->rvdata[i];
        const int o = get_owner(parts, nranks, v);
        const GraphElem comm = RK[o].currComm[v - RK[o].base];
        R->rcomm_val[i] = comm;
        if (get_owner(parts, nranks, comm) != r) remoteC_slot(R, comm);
      }
      for (GraphElem i = 0; i < R->nv; i++) {              /* 690-700 */
        const GraphElem comm = R->currComm[i];
        if (get_owner(parts, nranks, comm) != r) remoteC_slot(R, comm);
      }
      for (int64_t s = 0; s < R->nremoteC; s++) {          /* 858-951: owner's localCinfo, zeroed update */
        const GraphElem c = R->remoteCkey[s];
        const int o = get_owner(parts, nranks, c);
        R->remoteCinfo[s] = RK[o].localCinfo[c - RK[o].base];
        R->remoteCupdate[s].size = 0; R->remoteCupdate[s].degree = 0.0;
      }
    }
    /* ---- clean + scan + local fold, dspl.hpp:1371-1392 ---- */
    for (int r = 0; r < nranks; r++) {
      Rank *R = &RK[r];
      const GraphElem nv = R->nv, base = R->base, bound = R->bound;
      for (GraphElem i = 0; i < nv; i++) {                 /* distCleanCWandCU, 473-486 */
        R->clusterWeight[i] = 0; R->localCupdate[i].degree = 0; R->localCupdate[i].size = 0;
      }
      for (GraphElem i = 0; i < nv; i++) {                 /* distExecuteLouvainIteration, 276-405 */
        GraphElem localTarget = -1;
        GraphElem selfLoop = 0;                            /* integer on purpose: dspl.hpp:285 */
        const GraphElem cc = R->currComm[i];
        GraphWeight ccDegree; GraphElem ccSize; int currCommIsLocal, targetCommIsLocal = 0;
        int64_t ccSlot = -1;
        if (cc >= base && cc < bound) { ccDegree = R->localCinfo[cc - base].degree; ccSize = R->localCinfo[cc - base].size; currCommIsLocal = 1; }
        else { ccSlot = map_find(&R->remoteC, cc); ccDegree = R->remoteCinfo[ccSlot].degree; ccSize = R->remoteCinfo[ccSlot].size; currCommIsLocal = 0; }
        const GraphElem e0 = R->rowptr[i], e1 = R->rowptr[i + 1];
        if (e0 != e1) {
          int64_t nclus = 1;
          map_put_at(&clmap, cc, 0, &clpos[0]); clkeys[0] = cc; counter[0] = 0.0;       /* 312-313 */
          GraphWeight sl = 0;                              /* distBuildLocalMapCounter, 230-274 */
          for (GraphElem j = e0; j < e1; j++) {
            const GraphElem tail = R->edges[j].tail; const GraphWeight w = R->edges[j].weight;
            GraphElem tcomm;
            if (tail == i + base) sl += w;
            if (tail >= base && tail < bound) tcomm = R->currComm[tail - base];
            else tcomm = R->rcomm_val[map_find(&R->remoteComm, tail)];
            int64_t s = map_find(&clmap, tcomm);
            if (s >= 0) counter[s] += w;
            else { map_put_at(&clmap, tcomm, nclus, &clpos[nclus]); clkeys[nclus] = tcomm; counter[nclus] = w; nclus++; }
          }
          selfLoop = (GraphElem)sl;                        /* GraphWeight -> GraphElem truncation, 315 */
          R->clusterWeight[i] += counter[0];               /* 318 */
          localTarget = get_max_index(clkeys, counter, nclus, (GraphWeight)selfLoop, R, R->vDegree[i], ccSize,
                                      ccDegree, cc, constantForSecondTerm);
          for (int64_t k = 0; k < nclus; k++) clmap.keys[clpos[k]] = -1;   /* reset scratch map */
          clmap.n = 0;
        } else localTarget = cc;
        if (M && !M[r][i]) localTarget = cc;               /* held in place: counter[0] above still counted */
        if (localTarget >= base && localTarget < bound) targetCommIsLocal = 1;
        if (localTarget != cc && localTarget != -1) {      /* the four cases of 331-399 */
          if (targetCommIsLocal) { R->localCupdate[localTarget - base].degree += R->vDegree[i]; R->localCupdate[localTarget - base].size++; }
          else { int64_t s = map_find(&R->remoteC, localTarget); R->remoteCupdate[s].degree += R->vDegree[i]; R->remoteCupdate[s].size++; }
          if (currCommIsLocal) { R->localCupdate[cc - base].degree -= R->vDegree[i]; R->localCupdate[cc - base].size--; }
          else { R->remoteCupdate[ccSlot].degree -= R->vDegree[i]; R->remoteCupdate[ccSlot].size--; }
        }
        R->targetComm[i] = localTarget;                    /* 404 */
      }
      for (GraphElem i = 0; i < nv; i++) {                 /* distUpdateLocalCinfo, 458-471 */
        R->localCinfo[i].size += R->localCupdate[i].size;
        R->localCinfo[i].degree += R->localCupdate[i].degree;
      }
    }
    /* ---- frontier: M_{k+1} = M_k + the tails of the movers' records (own or remote, self loops excluded) ---- */
    if (M) {
      for (int r = 0; r < nranks; r++) memcpy(Mn[r], M[r], (size_t)RK[r].nv);
      for (int r = 0; r < nranks && frontier; r++) {
        Rank *R = &RK[r];
        for (GraphElem i = 0; i < R->nv; i++) {
          if (R->targetComm[i] == R->currComm[i]) continue;
          for (GraphElem j = R->rowptr[i]; j < R->rowptr[i + 1]; j++) {
            const GraphElem u = R->edges[j].tail;
            if (u == i + R->base) continue;
            const int o = get_owner(parts, nranks, u);
            Mn[o][u - RK[o].base] = 1;
          }
        }
      }
    }
    /* ---- updateRemoteCommunities, dspl.hpp:978-1103: owner adds deltas in source-rank order,
     * each source's list in ascending community id (std::map order, 988-1004) ---- */
    for (int o = 0; o < nranks && nranks > 1; o++) {
      for (int s = 0; s < nranks; s++) {
        if (s == o) continue;
        Rank *S = &RK[s];
        /* collect S's entries owned by o, ascending */
        int64_t cnt = 0;
        for (int64_t k = 0; k < S->nremoteC; k++) if (get_owner(parts, nranks, S->remoteCkey[k]) == o) cnt++;
        if (!cnt) continue;
        GraphElem *ids = (GraphElem *)malloc(sizeof(GraphElem) * cnt);
        cnt = 0;
        for (int64_t k = 0; k < S->nremoteC; k++) if (get_owner(parts, nranks, S->remoteCkey[k]) == o) ids[cnt++] = S->remoteCkey[k];
        qsort(ids, (size_t)cnt, sizeof(GraphElem), cmp_elem);
        for (int64_t k = 0; k < cnt; k++) {
          const int64_t slot = map_find(&S->remoteC, ids[k]);
          RK[o].localCinfo[ids[k] - RK[o].base].size += S->remoteCupdate[slot].size;       /* 1100-1101 */
          RK[o].localCinfo[ids[k] - RK[o].base].degree += S->remoteCupdate[slot].degree;
        }
        free(ids);
      }
    }
    /* ---- distComputeModularity, dspl.hpp:407-456 ---- */
    GraphWeight e_xx = 0.0, a2_x = 0.0;
    for (int r = 0; r < nranks; r++) {
      Rank *R = &RK[r];
      GraphWeight le_xx = 0.0, la2_x = 0.0;
      for (GraphElem i = 0; i < R->nv; i++) {
        le_xx += R->clusterWeight[i];
        la2_x += R->localCinfo[i].degree * R->localCinfo[i].degree;
      }
      if (r == 0) { e_xx = le_xx; a2_x = la2_x; } else { e_xx += le_xx; a2_x += la2_x; }
    }
    currMod = fabs((e_xx * constantForSecondTerm) - (a2_x * constantForSecondTerm * constantForSecondTerm));

    if (trace && numIters <= max_trace) {
      MvoIterTrace *T = &trace[numIters - 1];
      T->modularity = currMod; T->moved = 0; T->chash = 0;
      for (int r = 0; r < nranks; r++) {
        Rank *R = &RK[r];
        for (GraphElem i = 0; i < R->nv; i++) {
          T->chash += vhash(i + R->base, R->targetComm[i]);
          T->moved += (R->targetComm[i] != R->currComm[i]);
        }
      }
    }

    if (currMod - prevMod < thresh) break;                 /* dspl.hpp:1401-1402 */
    prevMod = currMod;
    if (prevMod < lower) prevMod = lower;                  /* 1404-1406 */
    for (int r = 0; r < nranks; r++) {                     /* rotate, 1408-1422 */
      Rank *R = &RK[r];
      GraphElem *tmp = R->pastComm; R->pastComm = R->currComm; R->currComm = R->targetComm; R->targetComm = tmp;
    }
    if (M)                                                 /* accepted: M_{k+1} */
      for (int r = 0; r < nranks; r++) { uint8_t *t = M[r]; M[r] = Mn[r]; Mn[r] = t; }
    if (stop_after > 0 && numIters == stop_after) { converged = 0; break; }
  }
  if (converged_out) *converged_out = converged;

  *iters_out = numIters;
  for (int r = 0; r < nranks; r++) {
    Rank *R = &RK[r];
    if (comm_out && comm_out[r]) memcpy(comm_out[r], R->currComm, sizeof(GraphElem) * (size_t)R->nv);
    if (movable_out && movable_out[r]) {
      if (M) memcpy(movable_out[r], M[r], (size_t)R->nv);
      else memset(movable_out[r], 1, (size_t)R->nv);
    }
    if (M) { free(M[r]); free(Mn[r]); }
    free(R->pastComm); free(R->currComm); free(R->targetComm); free(R->vDegree); free(R->clusterWeight);
    free(R->localCinfo); free(R->localCupdate); free(R->rvdata); free(R->rcomm_val);
    map_free(&R->remoteComm); map_free(&R->remoteC);
    free(R->remoteCkey); free(R->remoteCinfo); free(R->remoteCupdate);
  }
  map_free(&clmap); free(clkeys); free(clpos); free(counter); free(RK); free(M); free(Mn);
  (void)nv_global;
  return prevMod;                                          /* dspl.hpp:1440 */
}

/* FNV-free helper for tests: the shard-combinable hash of an assignment slice. */
uint64_t mvo_comm_hash(int64_t base, int64_t n, const int64_t *comm) {
  uint64_t h = 0;
  for (int64_t i = 0; i < n; i++) h += vhash(base + i, comm[i]);
  return h;
}
