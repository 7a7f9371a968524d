/* mvgpu.h -- C ABI of the H100-native Louvain phase (drop-in for miniVite's distLouvainMethod).
 *
 * The reference has no FFI; its seam is one C++ call, main.cpp:168-169:
 *
 *     currMod = distLouvainMethod(me, nprocs, *g, ssz, rsz, ssizes, rsizes, svdata, rvdata,
 *                                 currMod, threshold, iters);            // dspl.hpp:1280-1283
 *
 * whose inputs are the arrays of `class Graph` (graph.hpp:85-296): `edge_indices_` (int64 local
 * offsets, lnv+1 entries), `edge_list_` ({int64 tail_; double weight_} = 16 B records with GLOBAL
 * tails), the partition `parts_` (nprocs+1 entries) and the scalars nv / lnv / lne.  The entry points
 * below take exactly those plain arrays -- no C++ or torch types cross the boundary -- and return
 * what the reference returns (modularity of the last accepted iteration, iteration count) plus the
 * final assignment, which the reference computes but never exports (dspl.hpp:1432-1438).
 *
 * One context == one rank == one GPU.  All functions return 0 on success; on failure they return a
 * non-zero code and mvgpu_last_error() describes it (no exceptions cross the boundary; the host
 * wrapper turns a failure into the reference's MPI_Abort(-99) behaviour).  A context must be driven
 * by one host thread at a time.  The library never falls back to a CPU implementation: without a
 * usable CUDA device every compute entry point fails.
 *
 * Per-vertex and per-community arrays in host or device memory (DESIGN.md §3.16).  Every array pointer of
 * mvgpu_set_initial_communities, mvgpu_evaluate_communities, mvgpu_split_communities, mvgpu_probe_communities,
 * mvgpu_compare_communities, mvgpu_set_movable, mvgpu_get_movable, mvgpu_update_shard, mvgpu_get_communities,
 * mvgpu_get_compact_communities, mvgpu_get_community_stats and mvgpu_get_community_matches may be pageable or pinned host
 * memory, or device (or managed) memory of the context's device; each pointer is classified on its own with
 * cudaPointerGetAttributes, so ranks, and the two arrays of a compare, may differ in kind.  Device memory of another
 * device is refused with a message naming both devices; in a collective call that refusal fails every rank, like a bad
 * id.  Inputs are read on the library's stream after the call begins (the caller must have finished writing them) and
 * are copied or consumed before it returns, never retained.  Outputs are complete when the call returns.  Every other
 * message, and the meaning of NULL, is the same in both forms.  The 32-bit surface, mvgpu_upload_shard and
 * mvgpu_download_shard take host arrays only.
 */
#ifndef MVGPU_H
#define MVGPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mvgpu_ctx mvgpu_ctx;

#define MVGPU_UNIQUE_ID_BYTES 128

/* Per-iteration record; mirrors the trace hook injected into the reference at dspl.hpp:1400. */
typedef struct {
  double modularity;   /* currMod of the iteration (dspl.hpp:447-448) */
  int64_t moved;       /* #{i : targetComm[i] != currComm[i]}, all ranks */
  uint64_t chash;      /* sum over vertices of mix64(gid*0x9E3779B97F4A7C15 ^ targetComm), mod 2^64, all ranks */
} mvgpu_iter_trace;

/* Device-side timing of the last mvgpu_louvain call (CUDA events on the context's stream). */
typedef struct {
  double total_s;        /* the reference's main.cpp:162-173 scope: setup + all iterations */
  double setup_s;        /* format conversion + ghost discovery (exchangeVertexReqs, dspl.hpp:1106-1272) + init (151-172) */
  double scan_s;         /* sum over iterations of the neighbour-scan kernel(s) (dspl.hpp:276-405) */
  double fold_s;         /* sum of fold + modularity partial kernels (dspl.hpp:458-471, 407-456) */
  double exchange_s;     /* sum of ghost exchange + collectives (dspl.hpp:488-952, 978-1103, 441) */
  double h2d_s;          /* host->device copy of the shard (mvgpu_upload_shard), not part of total_s */
  int64_t scan_launches; /* neighbour-scan kernel launches in the call */
  int64_t kernel_launches; /* all kernels of this library launched inside total_s */
  int32_t iters;
  int32_t unit_weight;   /* 1 if the integer fast path ran (all weights 1.0, 2m < 2^31) */
  double reorder_s;      /* part of setup_s spent on the locality renumbering (0 when it did not run) */
  int32_t reordered;     /* 1 if this rank's vertices were renumbered for locality */
  int32_t scan_kernel_chosen; /* scan_variant 6: the persistent kernel the run settled on (4 = k_scan_pw, 5 = k_scan_pq; 0: run too short) */
  int64_t h2d_bytes;     /* bytes mvgpu_upload_shard copied host->device for the current shard (0 for attached arrays) */
} mvgpu_timings;

const char *mvgpu_last_error(void);
/* Number of CUDA devices visible, or -1 (and an error string) when CUDA is unusable. */
int mvgpu_device_count(void);

/* ---- lifetime ------------------------------------------------------------------------------- */
/* Replaces the rank identity the reference takes from MPI_Comm_rank/size (main.cpp:97-98). */
int mvgpu_create(mvgpu_ctx **ctx, int device, int rank, int nranks);
int mvgpu_destroy(mvgpu_ctx *ctx);

/* ---- multi-GPU plumbing (nranks > 1 only) ---------------------------------------------------- */
/* Rank 0 creates the id and ships the 128 bytes to every rank by any means (torch.distributed
 * broadcast, a pipe, a file); every rank then calls mvgpu_comm_init.  Stands in for MPI_Init +
 * createCommunityMPIType (main.cpp:78-102). */
int mvgpu_get_unique_id(void *id128);
int mvgpu_comm_init(mvgpu_ctx *ctx, const void *id128);

/* ---- graph hand-off -------------------------------------------------------------------------- */
/* Shard replacement (mvgpu_upload_shard, mvgpu_upload_shard32, mvgpu_attach_shard_device, mvgpu_generate_rgg_shard[_ex]):
 * every check runs before anything changes, so a refused call changes nothing -- the current shard, its initial
 * assignment, movable set, last run, evaluation and comparison stay as they were (a generated shard is built in arrays
 * of its own and takes the current one's place only at the end).  After success the context holds the new shard and
 * nothing of the old one's: the initial assignment, the movable set, the NULL forms of evaluate / split / compare, the
 * per-community getters and the per-vertex result getters (mvgpu_get_communities, mvgpu_get_communities32,
 * mvgpu_get_communities_device) all wait for the new shard's first run or call, and mvgpu_get_shard_info reports 0 in
 * info[2..5] until its first run.  A failure after the checks (a device allocation or copy) leaves the context with no
 * shard: every compute entry point then refuses until the next successful upload / attach / generate.  With several
 * ranks that refusal is local (it comes before the first collective), so the peers of a rank without a shard wait in
 * their first collective: every rank must hold a shard before a collective call. 
 * In a multi-rank run every rank must hold a shard of the same partition (nv_global and parts): mvgpu_louvain,
 * mvgpu_evaluate_communities, mvgpu_split_communities and mvgpu_compare_communities compare the ranks' partitions in
 * their first all-reduce and fail on every rank with "ranks disagree on the partition" otherwise. */
/* Host arrays of a reference Graph shard (graph.hpp:289-293): copies them to HBM.
 * parts: nranks+1 global vertex offsets (graph.hpp:109-113 or the -b bins, graph.hpp:511);
 * edge_indices: lnv+1 LOCAL offsets; edge_list: lne records {int64 tail; double weight}. */
int mvgpu_upload_shard(mvgpu_ctx *ctx, int64_t nv_global, const int64_t *parts, int64_t lnv, int64_t lne,
                       const int64_t *edge_indices, const void *edge_list);
/* Same, for arrays that already live in this context's device memory (not copied, not freed). */
int mvgpu_attach_shard_device(mvgpu_ctx *ctx, int64_t nv_global, const int64_t *parts, int64_t lnv, int64_t lne,
                              const int64_t *d_edge_indices, const void *d_edge_list);

/* Device-side GenerateRGG (graph.hpp:584-1213): builds this rank's strip of the graph
 * `miniVite -n nv_global` creates on nranks ranks directly in HBM, bit-identical to the reference generator, and
 * attaches it as the context's shard.  unit_weight = 0 gives Euclidean edge weights (-w).  *lne_out: local edges. */
int mvgpu_generate_rgg_shard(mvgpu_ctx *ctx, int64_t nv_global, int unit_weight, int64_t *lne_out);
/* Same with the remaining generator switches: lcg = 1 draws the coordinates from the reference's LCG class like
 * `miniVite -n nv_global -l` (utils.hpp:118-303, graph.hpp:703-729), lcg = 0 is the default engine;
 * random_edge_percent > 0 adds that percentage of random long edges like `-p` (graph.hpp:939-1122; the reference
 * seeds them from time and pid, graph.hpp:990, this library from a fixed seed -- the same one its host generator
 * uses, so both build the same graph).  With nranks > 1 and random_edge_percent > 0 the call is collective and needs
 * mvgpu_comm_init first (one count is summed over the ranks, graph.hpp:941-943). */
int mvgpu_generate_rgg_shard_ex(mvgpu_ctx *ctx, int64_t nv_global, int unit_weight, int lcg, double random_edge_percent,
                                int64_t *lne_out);
/* Copy the shard's reference-format arrays (lnv+1 offsets, lne 16-byte records) back to the host. */
int mvgpu_download_shard(mvgpu_ctx *ctx, int64_t *edge_indices, void *edge_list);
/* Change the shard in place on the device (DESIGN.md §3.11): n_del deletions (del_src[i], del_dst[i]) and n_ins
 * insertions (ins_src[i], ins_dst[i], ins_weight[i]), arrays in global ids, src owned by this rank.  Per row:
 * every old record whose tail is the dst of a deletion of that row is dropped (parallel records included; deletions
 * match old records only, so delete + insert of one pair replaces its weight); the insertions, stably sorted by dst,
 * are merged into the surviving records by "next old record while its tail <= the next insertion's dst, else the
 * insertion" (std::stable_sort of the concatenation for rows sorted by tail).  Both directions of an undirected edge
 * are the caller's to give.  Validated before anything changes: src in [base, bound), dst in [0, nv), the new lne
 * < 2^32, and the shard's edge_indices (0 first, lne last, never decreasing); refused for a compact-format or 32-bit
 * shard.  Synchronous; collective when nranks > 1 (every rank calls
 * it, with an empty batch if it has none), and one rank's failure fails every rank with all shards unchanged.
 * After success: *lne_out (may be NULL) = the new lne; the shard lives in library memory (an attached shard's arrays
 * are never written); the initial assignment is kept, mvgpu_get_communities still returns the last run's result, a
 * NULL evaluation and the per-community getters wait for the next run or evaluation; h2d figures are 0. */
int mvgpu_update_shard(mvgpu_ctx *ctx, int64_t n_del, const int64_t *del_src, const int64_t *del_dst, int64_t n_ins,
                       const int64_t *ins_src, const int64_t *ins_dst, const double *ins_weight, int64_t *lne_out);

/* ---- the Louvain phase (dspl.hpp:1280-1441) --------------------------------------------------- */
/* lower/thresh as in the reference (main.cpp:149,70); *iters counts the rejected last iteration
 * (dspl.hpp:1430); *modularity is prevMod (dspl.hpp:1440).  Collective over all ranks. */
int mvgpu_louvain(mvgpu_ctx *ctx, double lower, double thresh, int *iters, double *modularity);

/* Warm start (a refused call changes nothing): the next runs on this shard start from `comm` (lnv global community ids in the caller's vertex numbering,
 * the form mvgpu_get_communities returns) instead of singletons.  Every id must lie in [0, nv); id c names the vertex
 * whose owner keeps the community's Comm record, as in the reference -- the community need not contain vertex c, need
 * not be contiguous and may be owned by another rank.  The array is copied and validated at call time (errors are
 * local: no collective).  It stays in effect for every later mvgpu_louvain on this shard until NULL clears it or the next
 * upload / attach / generate replaces the shard.  In a multi-rank run every rank or none must set one (checked at the
 * start of mvgpu_louvain, which then fails on every rank).  Resuming a run stopped by the "stop_after" option from its
 * assignment with lower = its returned modularity continues it exactly (DESIGN.md §3.9).  Not for mvgpu_louvain32. */
int mvgpu_set_initial_communities(mvgpu_ctx *ctx, const int64_t *comm);
/* 1 if the last mvgpu_louvain ended on the reference's exit test, 0 if "stop_after" ended it first. */
int mvgpu_get_converged(mvgpu_ctx *ctx, int *converged);

/* ---- holding vertices in place (DESIGN.md §3.14) ----------------------------------------------------------------------
 * Movable set M: one byte per vertex, lnv entries in the caller's vertex numbering, nonzero = movable.  In iteration k
 * with set M_k a vertex outside M_k keeps its community (target = current, no Comm deltas); its counter[0] still counts
 * toward the iteration's modularity, so the reported modularity, the exit test and the trace keep their definitions.  A
 * vertex in M_k decides exactly as without a set (same gain, tie order and singleton veto).  Option "frontier": 0
 * (default) M_k = M in every iteration; 1: M_{k+1} = M_k + { u : a vertex v != u with a stored record v->u has target !=
 * current in iteration k } (own and ghost tails; u may be owned by another rank); a rejected last iteration does not grow
 * it.  An all-ones set gives the same bits as no set.
 * mvgpu_set_movable copies the array at call time (errors are local; a refused call changes nothing); it stays in effect for every later mvgpu_louvain on
 * this shard until NULL clears it (= everything movable) or the next upload / attach / generate; mvgpu_update_shard keeps
 * it.  In a multi-rank run every rank or none must set one (checked at the start of mvgpu_louvain, which then fails on
 * every rank).  Not for mvgpu_louvain32. */
int mvgpu_set_movable(mvgpu_ctx *ctx, const uint8_t *mask);
/* lnv bytes (0 / 1, caller numbering): the set the next iteration would use -- M_{k+1} after the last accepted iteration k
 * of the last mvgpu_louvain that ran with a set; before such a run (or after mvgpu_set_movable or mvgpu_update_shard) the
 * set as given; all ones without a set.  Resuming a run stopped by "stop_after" from (its assignment, this set, lower = its
 * modularity) with the same "frontier" continues it exactly. */
int mvgpu_get_movable(mvgpu_ctx *ctx, uint8_t *out);

/* ---- quality of an assignment (DESIGN.md §3.10) ---------------------------------------------------------------------
 * The modularity mvgpu_louvain returns is the reference's mixed quantity: in iteration k the intra-community weight is
 * measured on the assignment the scan read and sum(a_c^2) on the one it wrote.  mvgpu_evaluate_communities gives the
 * modularity Q of one assignment X.  Every field is global (all ranks) and identical on every rank. */
typedef struct {
  double modularity;   /* Q(X) = e_in*c - (a2*c)*c, rounded like the run's currMod, signed (no fabs) */
  double e_in;         /* sum over vertices i, edges (i,j) with X(j) = X(i) of w_ij (self-loop records count once each) */
  double a2;           /* sum over communities of a_c^2, a_c = sum of the degrees of c's members */
  double constant;     /* c = 1/(2m), as a run computes it */
  int64_t communities; /* non-empty communities */
  int64_t singletons;  /* communities of exactly one vertex */
  int64_t max_size;    /* vertices in the largest community */
  double eval_s;       /* device time of the evaluation (CUDA events on the context's stream) */
} mvgpu_quality;
/* Collective.  comm: lnv community ids in [0, nv) in the caller's vertex numbering, the form
 * mvgpu_set_initial_communities takes; NULL evaluates the assignment the last mvgpu_louvain on this shard returned (an
 * error if there is none).  A bad id on any rank, or ranks that disagree on NULL, fail the call on every rank.  Leaves
 * everything the last run reports (communities, trace, timings, constant, converged) and the initial assignment as they
 * were.  Not for shards uploaded with mvgpu_upload_shard32. */
int mvgpu_evaluate_communities(mvgpu_ctx *ctx, const int64_t *comm, mvgpu_quality *out);
/* Per community of the last evaluation, lnv entries each (any may be NULL): entry s describes community
 * parts[rank] + s (caller numbering): its number of vertices, its volume a_c and its share of e_in.  Empty: zeros. */
int mvgpu_get_community_stats(mvgpu_ctx *ctx, int64_t *size, double *volume, double *internal);
/* Per vertex of the last evaluation, lnv entries: the rank of its community among the non-empty community ids in
 * ascending caller id, in [0, communities); independent of the rank count and of the locality renumbering. */
int mvgpu_get_compact_communities(mvgpu_ctx *ctx, int64_t *out);

/* ---- splitting disconnected communities (DESIGN.md §3.12) ------------------------------------------------------------
 * A Louvain phase can leave a community in several pieces: a vertex that joined through a bridge vertex stays after the
 * bridge leaves.  Two vertices i, j are joined when X(i) = X(j) and the shard stores a record i->j or j->i (any weight,
 * zero included; self loops join nothing; a record stored in one direction only joins too).  Y gives every vertex the
 * smallest caller global id of its component under that relation: canonical (independent of the rank count, the
 * renumbering and the device's order), a member of the community, so a valid input to mvgpu_set_initial_communities and
 * mvgpu_evaluate_communities.  Splitting never lowers the modularity.  Every count is global and identical on every rank. */
typedef struct {
  int64_t communities;  /* non-empty communities of X */
  int64_t components;   /* components, = the communities of Y */
  int64_t disconnected; /* communities of X with more than one component */
  int32_t rounds;       /* hook + pointer-jump rounds the device took */
  double split_s;       /* device time of the call (CUDA events on the context's stream) */
} mvgpu_split_report;
/* Collective.  comm: lnv community ids in [0, nv) in the caller's vertex numbering; NULL splits the assignment the last
 * mvgpu_louvain on this shard returned.  out: lnv entries of Y.  Errors as in mvgpu_evaluate_communities (a bad id on
 * any rank, NULL without a run, ranks that disagree on NULL, a shard from mvgpu_upload_shard32) fail the call on every
 * rank, and then nothing is written to out.  Leaves everything the last run reports and the initial assignment as they
 * were; the per-community arrays of the last evaluation are gone (their getters fail until the next evaluation). */
int mvgpu_split_communities(mvgpu_ctx *ctx, const int64_t *comm, int64_t *out, mvgpu_split_report *rep);

/* ---- comparing two assignments (DESIGN.md §3.13) ---------------------------------------------------------------------
 * X and Y give every vertex a community id in [0, nv).  n_xy = #{v : X(v) = x, Y(v) = y} (a cell), a_x = |x|, b_y = |y|.
 * The counts are exact: pairs_xy = sum C(n_xy, 2), pairs_x = sum C(a_x, 2), pairs_y = sum C(b_y, 2), pairs_all = C(N, 2)
 * with N = nv; cells = the non-zero n_xy.  The doubles follow from them on the host in a fixed order, so every field is
 * the same bit for bit on every rank count:
 *   ari  = den == 0 ? 1 : num / den, num = 2 (pairs_all pairs_xy - pairs_x pairs_y),
 *          den = pairs_all (pairs_x + pairs_y) - 2 pairs_x pairs_y (exact 128-bit integers, one rounding each)
 *   rand = (pairs_all + 2 pairs_xy - pairs_x - pairs_y) / pairs_all (1 when pairs_all = 0)
 *   S(h) = sum over the values k > 1 of a histogram, ascending, of m_k (k log k); h_x = log N - S(a) / N (0 for at most
 *          one community), h_y likewise, mi = log N + (S(n) - (S(a) + S(b))) / N (0 when X or Y has at most one
 *          community), nmi = 2 mi / (h_x + h_y) (1 when h_x + h_y = 0; the arithmetic normalisation), vi = h_x + h_y - 2 mi */
typedef struct {
  int64_t vertices, communities_x, communities_y, cells;
  uint64_t pairs_xy, pairs_x, pairs_y, pairs_all;
  double ari, rand, nmi, vi, mi, h_x, h_y;
  double compare_s; /* device time of the call once both arrays are on the device (CUDA events on the context's stream) */
} mvgpu_compare_report;
/* Collective.  x, y: lnv community ids each in the caller's vertex numbering (the form mvgpu_evaluate_communities
 * takes); x = NULL compares the assignment the last mvgpu_louvain on this shard returned; y must not be NULL.  A bad id
 * in either array, NULL x without a run, ranks that disagree on NULL or a shard from mvgpu_upload_shard32 fail the call
 * on every rank, and then nothing is written.  Reads none of the shard's edges, and leaves everything the last run
 * reports, the initial assignment and the last evaluation's per-community arrays as they were. */
int mvgpu_compare_communities(mvgpu_ctx *ctx, const int64_t *x, const int64_t *y, mvgpu_compare_report *rep);
/* Per community x of the last successful compare: entry s describes community parts[rank] + s (the layout of
 * mvgpu_get_community_stats).  size = a_x; best = the y with the largest n_xy, ties to the smallest y; overlap = n_x,best;
 * best_size = b_best (Jaccard = overlap / (size + best_size - overlap)).  An empty x has size 0, best -1, overlap 0,
 * best_size 0.  The reverse direction is the compare with x and y swapped.  Fails before the first compare, after a
 * failed one, and after the next upload, attach or generate.  Any of the four arrays may be NULL (not written). */
int mvgpu_get_community_matches(mvgpu_ctx *ctx, int64_t *size, int64_t *best, int64_t *overlap, int64_t *best_size);

/* ---- probing an assignment (DESIGN.md §3.15) ------------------------------------------------------------------------
 * What every vertex would do under the Louvain rule from assignment X, with the quantities iteration 1 of a warm run from
 * X reads: counter[0], the self-loop weight, vDegree, a_x / size_x and a_y / size_y of every community under X over all
 * ranks, and c = 1/(2m) as a run computes it.  For vertex i with x = X(i):
 *   candidates  the communities y != x of the tails of i's records;
 *   gain(i, y)  dspl.hpp:212 with the reference's association (2.0*(e_iy - e_ix) - ((2.0*k_i)*(a_y - a_x))*c);
 *   best(i)     the candidate with the largest gain, equal gains to the smallest id; -1 without a candidate (no records,
 *               only self loops, or every neighbour in x);
 *   gain(i)     gain(i, best(i)), which may be negative or zero; -inf when best = -1 (the stability margin);
 *   target(i)   the reference's decision (dspl.hpp:174-228, 309-324): best(i) if gain(i) > 0 and the singleton veto
 *               (size_x = size_best = 1 and best > x) does not fire, else x.
 * A movable set does not restrict the probe: it says what each vertex would do if it were movable.  Unit and dyadic
 * weights give the same bits on every rank count and every option (reorder, force_heavy_deg, force_weighted, upload mode). */
typedef struct {
  int64_t vertices;   /* nv */
  int64_t moves;      /* #{i : target(i) != X(i)}: 0 iff X is a fixed point of the rule */
  int64_t vetoed;     /* #{i : gain(i) > 0, kept in place by the singleton veto} */
  int64_t interior;   /* #{i : i has records and best(i) = -1} */
  double max_gain;    /* max over i of gain(i); -inf when no vertex has a candidate */
  double constant;    /* c = 1/(2m) used */
  double probe_s;     /* device time of the call (CUDA events on the context's stream) */
} mvgpu_probe_report;
/* Collective.  comm: lnv community ids in [0, nv) in the caller's vertex numbering (the form mvgpu_evaluate_communities
 * takes); NULL probes the assignment the last mvgpu_louvain on this shard returned.  target, best (caller ids) and gain
 * hold lnv entries each; any of them may be NULL (not written).  Errors as in mvgpu_evaluate_communities (a bad id on any
 * rank, NULL without a run, ranks that disagree on NULL, a shard from mvgpu_upload_shard32) fail the call on every rank,
 * and then nothing is written.  Changes nothing else: everything the last run reports, the initial assignment, the
 * movable set and the arrays of the last evaluation and the last comparison stay as they were. */
int mvgpu_probe_communities(mvgpu_ctx *ctx, const int64_t *comm, int64_t *target, int64_t *best, double *gain,
                            mvgpu_probe_report *rep);

/* currComm of this rank's vertices at exit (global community ids), lnv entries, of the last mvgpu_louvain on the current
 * shard: it fails with "no run on this shard" after an upload / attach / generate until the new shard's first run;
 * mvgpu_update_shard keeps serving the last run's result. */
int mvgpu_get_communities(mvgpu_ctx *ctx, int64_t *out);
/* Same values left in device memory (int32 global ids), same contract; valid until the next mvgpu_louvain. */
int mvgpu_get_communities_device(mvgpu_ctx *ctx, const int32_t **d_out);

/* Options: "trace" (0/1: record moved/chash per iteration, default 0), "max_iters" (safety cap,
 * default 10000), "force_weighted" (0/1: use the fp64 path even for unit weights, default 0),
 * "force_heavy_deg" (test hook: treat vertices with degree > value as high-degree, default 0 = off),
 * "scan_ctas" (test hook: k > 0 caps the grids of the persistent scan kernels k_scan_pw and k_scan_pq at k CTAs, so
 * every warp strides over many 32-vertex groups even on a small shard, as a large shard or a part with fewer SMs does;
 * default 0 = resident CTAs per SM x SMs; negative values are refused; identical results),
 * "scan_variant" (6 (default): iterations 2 and 4 run k_scan_pw, iteration 3 k_scan_pq, and from iteration 5 on
 * k_scan_pq runs if it beat the geometric mean of its neighbours, else k_scan_pw; 5 = k_scan_pq: persistent warps fed by TMA bulk copies, boundary vertices reduced from a
 * per-warp ring -- unit weights; iteration 1 and weighted graphs run k_scan_pw; 4 = k_scan_pw throughout; 3 =
 * k_scan_ws: one CTA per 128-vertex tile, the default of round 1; identical results), "first_iter" (1 (default):
 * iteration 1 of a simple unit-weight graph uses the singleton-community reduction of k_scan_pw; 0: the general
 * reduction; identical results), "upload_chunk" (edges per chunk of the compact upload, default 4 Mi; test hook),
 * "cache_policy" (bit2 = L2 evict_first hint on the streamed arrays of k_scan_ws; other bits are accepted and
 * ignored; default 5), "reorder" (0 never, 1 always, 2 auto (default): renumber vertices for memory
 * locality when the given numbering has none -- layout only, results are identical), "region_size" (target
 * vertices per BFS region of the renumbering, default 512), "comm_mode" (multi-GPU per-iteration exchanges: 1 = stores /
 * flags in peer memory over NVLink (default), 0 = NCCL all-to-all-v + all-reduce), "host_transport" (set before
 * mvgpu_comm_init; 1: the setup-time exchanges go through a shared-memory segment of the host instead of NCCL --
 * required when several ranks share one device, which NCCL refuses; needs comm_mode 1; default 0), "compact_upload" (1:
 * mvgpu_upload_shard sends unit-weight shards as 4-byte tails narrowed on the host; 2: the copy engine additionally
 * takes raw chunks from the far end of the array whenever no narrowed chunk is ready (narrowed on the device);
 * 0 (default) = the 16-byte records as they are), "host_threads" (threads of that host pass, default 8), "stop_after"
 * (0 = off (default); k > 0: end the run successfully after k ACCEPTED iterations: *iters = k, *modularity = prevMod
 * after iteration k -- the `lower` to resume with --, k trace records, mvgpu_get_communities returns the assignment
 * after iteration k; if the exit test fires first the run ends as without it, see mvgpu_get_converged), "frontier" (0
 * (default) / 1: grow the movable set from the vertices that move, see mvgpu_set_movable; no effect without a set).
 * The environment variable MVGPU_OPTIONS="name=value,name=value" presets options for every context of the process. */
/* In a multi-rank run every rank must set the same options (they change which collectives a run issues).  A refused
 * value or an unknown name changes nothing. */
int mvgpu_set_option(mvgpu_ctx *ctx, const char *name, int64_t value);
/* mvgpu_get_trace, mvgpu_get_timings, mvgpu_get_scan_times, mvgpu_get_constant and mvgpu_get_converged describe the last
 * mvgpu_louvain call, whatever shard the context holds now. */
int mvgpu_get_trace(mvgpu_ctx *ctx, int max_entries, mvgpu_iter_trace *out, int *n);
int mvgpu_get_timings(mvgpu_ctx *ctx, mvgpu_timings *out);
/* Device time (seconds) of the neighbour-scan launch(es) of each iteration of the last run; *n = #iterations. */
int mvgpu_get_scan_times(mvgpu_ctx *ctx, int max_entries, double *out, int *n);
/* 1/(2m), the reference's constantForSecondTerm (dspl.hpp:129), of the last run. */
int mvgpu_get_constant(mvgpu_ctx *ctx, double *out);
/* Shard statistics: info[0]=lnv, [1]=lne of the current shard; from the setup of the last run on it (0 until its first
 * run): [2]=nghost, [3]=send list length, [4]=#high-degree vertices, [5]=max degree. */
int mvgpu_get_shard_info(mvgpu_ctx *ctx, int64_t *info6);

/* ---- one-call form of the reference seam ------------------------------------------------------ */
/* ---- the reference's USE_32_BIT_GRAPH build (utils.hpp:72-82: GraphElem = int32_t, GraphWeight = float) ------------
 * A miniVite compiled with -DUSE_32_BIT_GRAPH holds int32 offsets and 8-byte {int32 tail_; float weight_} records
 * (graph.hpp:60-66 with those types) and computes gains, 1/(2m) and the modularity in float.  These entry points take
 * that build's arrays and reproduce that build's arithmetic: the gain is rounded where the float build rounds it
 * (see gain_of in kernels.cuh), 1/(2m), the modularity and the exit test are evaluated in float (dspl.hpp:129,
 * 447-448, 1401).  For unit-weight graphs whose integer sums stay below 2^24 every float sum of the reference is
 * exact, and the results -- assignment, iteration count, modularity -- are bit-identical to the float build's;
 * beyond that the float build is not reproducible against itself (its OpenMP reductions round in arbitrary order)
 * and the comparison is by tolerance.  parts / edge_indices are int32 here, like every GraphElem of that build. */
int mvgpu_upload_shard32(mvgpu_ctx *ctx, int32_t nv_global, const int32_t *parts, int32_t lnv, int32_t lne,
                         const int32_t *edge_indices, const void *edge_list8);
/* Fails while an initial assignment or "stop_after" is set (warm start is a 64-bit surface feature). */
int mvgpu_louvain32(mvgpu_ctx *ctx, float lower, float thresh, int *iters, float *modularity);
/* The contract of mvgpu_get_communities. */
int mvgpu_get_communities32(mvgpu_ctx *ctx, int32_t *out);

/* distLouvainMethod(me, nprocs, g, ..., lower, thresh, iters) for a single-GPU run with HOST arrays:
 * create + upload + louvain (+ optional assignment download into comm_out, may be NULL) + destroy. */
int mvgpu_dist_louvain_method(int device, int64_t nv, int64_t ne_local, const int64_t *edge_indices,
                              const void *edge_list, double lower, double thresh, int *iters,
                              double *modularity, int64_t *comm_out);

#ifdef __cplusplus
}
#endif
#endif /* MVGPU_H */
