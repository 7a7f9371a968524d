// libmvgpu.so: the H100 (sm_90a) implementation behind include/mvgpu.h.
//
// Replaces miniVite's distLouvainMethod (reference dspl.hpp:1280-1441) for one rank == one GPU:
//   setup      format conversion + ghost discovery + init   (dspl.hpp:1106-1272, 151-172)
//   iteration  scan kernel -> [ghost exchange, barrier] -> fold kernel -> [all-reduce] -> host test
// Multi-GPU: vertex-range shards, one rank per GPU.  Comm{size,degree} of remotely owned communities is read, and
// their deltas are pushed, directly in the owner's HBM over NVLink (peer pointers obtained through CUDA IPC), which
// removes the reference's request/reply and delta-push message rounds (dspl.hpp:719-929, 1022-1102).  The
// per-iteration ghost vertex->community map and the modularity reduction (dspl.hpp:559-646, 441) run, by default
// (comm_mode 1), as this library's own kernels over the same peer memory: k_push_ghosts stores every send segment
// straight into the ghost tail of the peer's community array, k_p2p_barrier / k_p2p_allreduce are flag-based
// collectives.  comm_mode 0 keeps them as one grouped ncclSend/ncclRecv all-to-all-v with run-constant counts plus
// one ncclAllReduce of two doubles.  The setup exchanges (ghost lists, counts, IPC handles) go through NCCL, or through
// the host transport (option host_transport=1, a shared-memory segment) that also lets ranks share one device.
#include <cuda_runtime.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cub/cub.cuh>
#include <map>
#include <random>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/mvgpu.h"
#include "host_comm.hpp"
#include "kernels.cuh"
#include "scan_pipe.cuh"
#include "scan_queue.cuh"
#include "nccl_dyn.h"
#include "rgg_gpu.cuh"
#include "merge_gpu.cuh"
#include "compare_gpu.cuh"
#include "probe_gpu.cuh"

// host-only helper of the compact upload (narrow.cpp): 16-byte edge records -> 4-byte tails + validation
extern "C" void mv_narrow_edges(const void *edge_records, long long n, long long nv, long long base, long long bound,
                                int32_t *dst, long long *nremote, int *bad);

namespace {

thread_local std::string g_err;
mvnccl::Api g_nccl;

int fail(const std::string &msg) { g_err = msg; return 1; }

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      return fail(std::string(#call) + ": " + cudaGetErrorString(e_) + " (" __FILE__ ":" + std::to_string(__LINE__) + ")"); \
  } while (0)
#define NK(call)                                                                                   \
  do {                                                                                             \
    ncclResult_t r_ = (call);                                                                      \
    if (r_ != ncclSuccess)                                                                         \
      return fail(std::string(#call) + ": " + g_nccl.GetErrorString(r_) + " (" __FILE__ ":" + std::to_string(__LINE__) + ")"); \
  } while (0)
#define TRY(expr)            \
  do {                       \
    int rc_ = (expr);        \
    if (rc_) return rc_;     \
  } while (0)

template <typename T>
struct DevBuf {              // grow-only device buffer (allocations are cached across runs); frees itself
  T *p = nullptr;
  size_t cap = 0;
  unsigned gen = 0;          // bumped by every (re)allocation: cudaMalloc may hand the old address back for a new block
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() { release(); }
  void swap(DevBuf &o) { std::swap(p, o.p); std::swap(cap, o.cap); gen++; o.gen++; }
  int ensure(size_t n) {
    if (n <= cap && p) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    if (n == 0) n = 1;
    CK(cudaMalloc(&p, n * sizeof(T)));
    cap = n;
    gen++;
    return 0;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// The arrays every rank exports to its peers (CUDA IPC, or plain pointers between threads of one process), listed here
// only: X(buffer, exported by this run, the size a run ensures it at (0: not allocated by this run), where rank r's
// copy is bound).  need_v = lnv, need_s = lnv + the non-owned edge tails.
#define MV_EXPORTS(X)                                               \
  X(cdeg, c->unit, need_v, c->pt.cdeg[r])                           \
  X(csize, c->unit, need_v, c->pt.csize[r])                         \
  X(upd, c->unit, need_v, c->pt.upd[r])                             \
  X(cinfo_w, !c->unit, need_v, c->pt.cinfo_w[r])                    \
  X(usize, !c->unit, need_v, c->pt.usize[r])                        \
  X(udeg, !c->unit, need_v, c->pt.udeg[r])                          \
  X(lab, c->relabel, need_v, c->pt.lab[r])                          \
  X(comm_a, true, need_s, c->peer_comm[0][r])                       \
  X(comm_b, true, need_s, c->peer_comm[1][r])                       \
  X(p2p, true, 1, c->pp.st[r])                                      \
  X(inv, c->relabel, need_v, c->peer_inv[r])                        \
  X(q_internal, true, ev ? need_v : 0, c->qp.internal[r])           \
  X(q_rank, true, ev ? need_v + 1 : 0, c->qp.rank[r])                \
  X(split_lab, true, split ? need_v : 0, c->spp.lab[r])             \
  X(mov_a, c->mov_run && c->opt_frontier, c->mov_run && c->opt_frontier ? need_v : 0, c->peer_mov[0][r]) \
  X(mov_b, c->mov_run && c->opt_frontier, c->mov_run && c->opt_frontier ? need_v : 0, c->peer_mov[1][r])
#define MV_COUNT(...) +1
constexpr int kPeerArrays = 0 MV_EXPORTS(MV_COUNT);
#undef MV_COUNT

struct Export {
  void *p;                             // NULL: this run does not export the array
  unsigned gen;                        // its DevBuf generation
  size_t cap, need;                    // its capacity (0: not allocated) and the size this run ensures (0: none)
};

struct PeerBlob {            // what every rank publishes about its community arrays
  cudaIpcMemHandle_t h[kPeerArrays];
  unsigned long long raw[kPeerArrays];
  int pid, device, unit, pad;
};

// what the last setup decided about the layout, kept on the host for mv_layout_readback (a test hook, not in mvgpu.h);
// every value is one that setup_run or run_louvain already had on the host
struct LayoutReport {
  int want = 0, stride = 0, unordered = 0, has_self = 0;
  long long nregions = 0;
  long long span[2] = {-1, -1};       // k_span_sample's sum and count; -1: the sample did not run
  bool first_ran = false;             // iteration 1 launched k_scan_pw's FIRST instantiation
  const int32_t *tails = nullptr;     // the compact tails before renumbering (c->tails or the uploaded compact array)
};

}  // namespace

using namespace mv;

struct mvgpu_ctx {
  int device = 0, rank = 0, nranks = 1;
  cudaStream_t stream = nullptr;
  int num_sms = 132;
  // communicator: NCCL, or the host transport (option host_transport=1) for the setup-time exchanges
  ncclComm_t comm = nullptr;
  mvhost::HostComm hc;
  // input (reference format, device)
  long long nv_global = 0, lnv = 0, lne = 0, base = 0, bound = 0;
  std::vector<long long> parts;
  const long long *d_rowptr64 = nullptr;
  const Edge16 *d_edges = nullptr;
  DevBuf<long long> in_rowptr;
  DevBuf<Edge16> in_edges;
  DevBuf<long long> gen_rowptr;       // device-generated RGG shard (mvgpu_generate_rgg_shard)
  DevBuf<Edge16> gen_edges;
  // compact upload format (unit-weight shards): int32 global tails, staged through pinned chunks
  DevBuf<int32_t> in_tails32;
  DevBuf<Edge16> raw_ring;             // compact upload: raw chunks narrowed on the device (two slots)
  long long raw_chunks = 0;
  DevBuf<long long> wide;              // int64 per-vertex arrays on their way to or from host memory
  void *h_bounce[2] = {nullptr, nullptr};   // pinned chunks between the device and pageable host arrays, both ways
  cudaEvent_t bounce_ev[2] = {nullptr, nullptr};   // the last copy in or out of h_bounce[b]
  DevBuf<unsigned long long> take_bad; // k_take_ids: the smallest local index of a bad id
  const int32_t *d_tails32 = nullptr;
  long long in_nremote = 0;
  void *h_stage = nullptr;
  size_t h_stage_cap = 0;
  // compact CSR the iterations run on (original numbering or renumbered)
  const uint32_t *a_rowptr = nullptr;
  const int32_t *a_tails = nullptr;
  const double *a_weights = nullptr;
  bool have_graph = false;
  // compact graph
  DevBuf<uint32_t> rowptr;
  DevBuf<int32_t> tails;
  DevBuf<double> weights;
  DevBuf<int32_t> self_i;
  // locality renumbering
  DevBuf<uint32_t> bfs_key, sortkey, sortkey2, deg_new, rowptr2;
  DevBuf<int32_t> ids, perm, inv, lab, tails2, final_orig;
  DevBuf<double> weights2;
  DevBuf<unsigned int> bfs_level_count;
  bool reordered = false;
  int relabel = 0;
  double reorder_s = 0.0;
  LayoutReport lay;
  DevBuf<double> self_d, vdeg;
  // state
  DevBuf<int32_t> comm_a, comm_b;
  DevBuf<uint32_t> cdeg;
  DevBuf<int32_t> csize;
  DevBuf<unsigned long long> upd;
  DevBuf<CommW> cinfo_w;
  DevBuf<long long> usize;
  DevBuf<double> udeg;
  DevBuf<Acc> acc;
  DevBuf<unsigned char> scratch;       // small device scalars
  DevBuf<unsigned char> cub_tmp, coll_tmp;
  DevBuf<long long> sorted_tmp;
  // ghosts
  DevBuf<long long> remote_list, ghost_gid, send_gid;
  DevBuf<uint32_t> remote_pos;
  DevBuf<int32_t> send_lid, send_buf;
  long long nghost = 0, nsend = 0;
  std::vector<long long> rcount, scount, roff, soff;   // per peer
  // heavy vertices
  DevBuf<int32_t> heavy_list, hkeys, hvals_i;
  DevBuf<double> hvals_d;
  DevBuf<unsigned long long> heavy_off;
  long long nheavy = 0, maxdeg = 0;
  int scan_has_self = 0, scan_heavy_deg = kECap;
  int scan_kernel = 4;                 // the persistent kernel this iteration runs: 4 = k_scan_pw, 5 = k_scan_pq (see run_louvain)
  bool simple_sorted = false;          // unit graph, adjacency lists strictly increasing (no parallel edges), no self loops
  // peers
  DevBuf<P2PState> p2p;
  P2PPeers pp;
  PushTable push[2];
  unsigned long long p2p_epoch = 0;
  bool p2p_zeroed = false;
  int32_t *peer_comm[2][kMaxRanks];
  PeerTable pt;
  std::vector<void *> ipc_opened;
  bool peers_ready = false, ipc_valid = false;
  const int32_t *peer_inv[kMaxRanks];  // every rank's inv (old -> new local index) while some rank renumbers: warm-start init only
  Export last_export[kPeerArrays] = {};   // what the last IPC exchange published
  // options
  int opt_trace = 0, opt_force_weighted = 0, opt_scan_variant = 6, opt_cache_policy = 5, opt_reorder = 2, opt_region = 512, opt_comm_mode = 1, opt_compact_upload = 0, opt_host_threads = 8, opt_first_iter = 1, opt_host_transport = 0, opt_frontier = 0;
  long long opt_upload_chunk = 4LL << 20;
  long long opt_max_iters = 10000, opt_force_heavy_deg = 0, opt_stop_after = 0;
  int opt_scan_ctas = 0;               // test hook: > 0 caps the persistent scan grids at that many CTAs (0 = occupancy x SMs)
  // warm start (mvgpu_set_initial_communities): caller-numbered community ids of this shard, until the next graph
  DevBuf<int32_t> init_comm;
  bool have_init = false;
  bool warm_run = false;               // the current / last run started from init_comm
  int converged = 1;                   // the last run ended on the exit test (0: stopped by stop_after)
  // movable set (mvgpu_set_movable, DESIGN.md §3.14): mov_in holds the caller's bytes (caller numbering) until the next
  // graph; a run keeps M_k in internal numbering in mov_a / mov_b (double-buffered and peer-exported with the frontier
  // option) and leaves M_{k+1} of its last accepted iteration in mov_out (caller numbering)
  DevBuf<uint8_t> mov_in, mov_a, mov_b, mov_out;
  bool have_mov = false;
  bool mov_run = false;                // the current / last run reads a movable set (the MASKED scan instantiations)
  bool mov_out_valid = false;          // mov_out describes the last run on this shard
  uint8_t *peer_mov[2][kMaxRanks];
  // evaluation (mvgpu_evaluate_communities): q_internal and q_rank are peer-exported, the rest stays local
  DevBuf<int32_t> eval_comm;           // the caller's assignment to evaluate (int32 caller ids)
  DevBuf<double> q_internal, q_vol;
  DevBuf<int32_t> q_rank, q_flag, q_lab;
  DevBuf<long long> q_size;
  QualPeers qp;
  // splitting (mvgpu_split_communities): labels, peer-exported; the counters reuse q_internal
  DevBuf<int32_t> split_lab;
  SplitPeers spp;
  // comparing (mvgpu_compare_communities): nothing is peer-exported, every exchange is a collective.  The two
  // assignments (int32 caller ids), the owned cells and Y-counts, work arrays, and the matches [size|best|overlap|best_size]
  DevBuf<int32_t> cmp_x, cmp_y, cmp_i0, cmp_i1;
  DevBuf<unsigned long long> cmp_k0, cmp_k1, cmp_k2, cmp_cell_k, cmp_y_k;
  DevBuf<uint32_t> cmp_c0, cmp_c1, cmp_c2, cmp_cell_c, cmp_y_c, cmp_b, cmp_hv, cmp_hm;
  DevBuf<CmpRow> cmp_row0, cmp_row1;
  DevBuf<long long> cmp_match, cmp_off;
  DevBuf<int> cmp_n;
  // probing (mvgpu_probe_communities): target, best (int32 caller ids) and gain per own vertex; nothing is peer-exported
  DevBuf<int32_t> probe_tgt, probe_best;
  DevBuf<double> probe_gain;
  bool run_on_shard = false;           // final_orig holds a run's assignment of the current shard
  bool eval_on_shard = false;          // the q_* arrays describe an evaluation of the current shard
  bool cmp_on_shard = false;           // cmp_match describes a successful comparison on the current shard's vertices
  // results
  bool unit = true;
  bool f32 = false;                    // shard came through mvgpu_upload_shard32: float-build arithmetic (see mvgpu.h)
  double constant = 0.0;
  int32_t *d_final = nullptr;          // currComm at exit (points into comm_a/comm_b)
  bool final_ready = false;            // final_orig holds the assignment of the last run in the caller's numbering
  bool final_on_shard = false;         // d_final / final_orig describe the current shard's vertices (update_shard keeps it,
                                       // a shard replacement clears it): what the per-vertex result getters serve
  std::vector<mvgpu_iter_trace> trace;
  std::vector<double> scan_times;
  mvgpu_timings tm;
  double h2d_s = 0.0;
  long long h2d_bytes = 0;
  // pinned host mailbox
  void *h_pin = nullptr;
  // events
  std::vector<cudaEvent_t> events;
  ScanParams last_sp;
};

namespace {

int grid_for(long long n, int threads, int num_sms, int per_sm = 8) {
  long long b = (n + threads - 1) / threads;
  long long cap = (long long)num_sms * per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

cudaEvent_t get_event(mvgpu_ctx *c, size_t i) {
  while (c->events.size() <= i) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    c->events.push_back(e);
  }
  return c->events[i];
}

// device scalar slots inside c->scratch
struct Scalars {
  EdgeStats st;
  unsigned long long remote_cursor;
  unsigned int maxdeg, bad_rowptr, has_self, heavy_count;
  int nunique;
  unsigned int unordered;              // some adjacency list is not strictly increasing by global tail id
  double total_weight;
  double red2[2];
  unsigned long long tr2[2];
  long long counts[2 * kMaxRanks];
  unsigned long long span_sum, span_cnt;
  unsigned long long q_agg[2];         // evaluation: singletons, largest community
  unsigned long long split_agg[3];     // splitting: non-empty communities, components, disconnected communities
  unsigned long long probe_agg[4];     // probing: moves, vetoed, interior, largest gain as probe_key (ProbeOut::agg)
};
Scalars *dev_scalars(mvgpu_ctx *c) { return reinterpret_cast<Scalars *>(c->scratch.p); }

// ---- setup-time collectives (a handful per run): NCCL on the library's stream, or the host transport ----------------
int coll_sync(mvgpu_ctx *c) { CK(cudaStreamSynchronize(c->stream)); return 0; }

// element-wise sum / max of n <= 2*kMaxRanks int64 values held on the host, result on every rank
int coll_allreduce_i64(mvgpu_ctx *c, long long *v, int n, bool is_max) {
  if (c->nranks == 1) return 0;
  if (c->hc.is_open()) {
    if (is_max) c->hc.allreduce(v, n, [](long long a, long long b) { return a > b ? a : b; });
    else c->hc.allreduce(v, n, [](long long a, long long b) { return a + b; });
    return 0;
  }
  long long *d = dev_scalars(c)->counts;
  CK(cudaMemcpyAsync(d, v, sizeof(long long) * n, cudaMemcpyHostToDevice, c->stream));
  NK(g_nccl.AllReduce(d, d, n, ncclInt64, is_max ? ncclMax : ncclSum, c->comm, c->stream));
  CK(cudaMemcpyAsync(v, d, sizeof(long long) * n, cudaMemcpyDeviceToHost, c->stream));
  return coll_sync(c);
}
// every rank contributes `bytes` from host memory; all[r * bytes ..] = rank r's contribution
int coll_allgather(mvgpu_ctx *c, const void *mine, void *all, size_t bytes) {
  if (c->hc.is_open()) { c->hc.allgather(mine, all, bytes); return 0; }
  DevBuf<unsigned char> &d = c->coll_tmp;        // grow-only staging buffer: no allocation inside the timed setup after the first run
  TRY(d.ensure(bytes * (c->nranks + 1)));
  unsigned char *dm = d.p + bytes * c->nranks;
  CK(cudaMemcpyAsync(dm, mine, bytes, cudaMemcpyHostToDevice, c->stream));
  NK(g_nccl.AllGather(dm, d.p, bytes, ncclChar, c->comm, c->stream));
  CK(cudaMemcpyAsync(all, d.p, bytes * c->nranks, cudaMemcpyDeviceToHost, c->stream));
  return coll_sync(c);
}
// all-to-all-v between device buffers with counts known on both sides (elements of `elem` bytes, 4 or 8).  NCCL: one
// grouped send/recv round, left on the stream.  Host transport: staged through the shared segment (synchronous).
int coll_alltoallv_dev(mvgpu_ctx *c, const void *d_send, const std::vector<long long> &scount, const std::vector<long long> &soff,
                       void *d_recv, const std::vector<long long> &rcount, const std::vector<long long> &roff, size_t elem) {
  const int n = c->nranks;
  if (c->hc.is_open()) {
    std::vector<size_t> sc(n), so(n), rc(n), ro(n);
    for (int r = 0; r < n; r++) { sc[r] = (r == c->rank ? 0 : scount[r]) * elem; so[r] = soff[r] * elem; rc[r] = (r == c->rank ? 0 : rcount[r]) * elem; ro[r] = roff[r] * elem; }
    const size_t sbytes = (size_t)soff[n] * elem, rbytes = (size_t)roff[n] * elem;
    std::vector<unsigned char> hs(sbytes + 1), hr(rbytes + 1);
    if (sbytes) CK(cudaMemcpyAsync(hs.data(), d_send, sbytes, cudaMemcpyDeviceToHost, c->stream));
    TRY(coll_sync(c));
    c->hc.alltoallv(hs.data(), sc.data(), so.data(), hr.data(), rc.data(), ro.data());
    for (int r = 0; r < n; r++)
      if (rc[r]) CK(cudaMemcpyAsync((unsigned char *)d_recv + ro[r], hr.data() + ro[r], rc[r], cudaMemcpyHostToDevice, c->stream));
    return coll_sync(c);
  }
  const ncclDataType_t ty = elem == 8 ? ncclInt64 : ncclInt32;
  NK(g_nccl.GroupStart());
  for (int r = 0; r < n; r++) {
    if (r == c->rank) continue;
    if (scount[r]) NK(g_nccl.Send((const unsigned char *)d_send + soff[r] * elem, scount[r], ty, r, c->comm, c->stream));
    if (rcount[r]) NK(g_nccl.Recv((unsigned char *)d_recv + roff[r] * elem, rcount[r], ty, r, c->comm, c->stream));
  }
  NK(g_nccl.GroupEnd());
  return 0;
}
// everything enqueued on every rank's stream so far has completed when this returns
int coll_barrier(mvgpu_ctx *c) {
  if (c->nranks == 1) return coll_sync(c);
  if (c->hc.is_open()) { TRY(coll_sync(c)); c->hc.barrier(); return 0; }
  long long *d = dev_scalars(c)->counts;
  NK(g_nccl.AllReduce(d, d, 1, ncclInt64, ncclSum, c->comm, c->stream));
  return coll_sync(c);
}

// what is wrong with a shard description ("" if nothing); reads nothing of the context but its rank identity
std::string check_graph(const mvgpu_ctx *c, long long nv_global, const int64_t *parts, long long lnv, long long lne) {
  if (c->nranks > kMaxRanks) return "too many ranks";
  if (nv_global < 0 || lnv < 0 || lne < 0) return "negative graph size";
  if (nv_global >= (1LL << 31)) return "nv_global >= 2^31: 32-bit community ids would overflow (not supported)";
  if (lne >= (1LL << 32)) return "lne >= 2^32 per shard: 32-bit edge offsets would overflow (not supported)";
  if (parts[0] != 0 || parts[c->nranks] != nv_global) return "parts[] must run from 0 to nv_global";
  for (int r = 0; r < c->nranks; r++) if (parts[r + 1] < parts[r]) return "parts[] not monotone";
  if (parts[c->rank + 1] - parts[c->rank] != lnv) return "lnv does not match parts[rank+1]-parts[rank]";
  return "";
}

// The shard is replaced: validated first, so that a refusal changes nothing.  From here on the context has no shard
// until set_source names the new arrays -- a failure in between leaves it without one, and every compute entry point
// refuses (check_ready).
int set_graph(mvgpu_ctx *c, long long nv_global, const int64_t *parts, long long lnv, long long lne) {
  const std::string err = check_graph(c, nv_global, parts, lnv, lne);
  if (!err.empty()) return fail(err);
  c->have_init = false;                     // an initial assignment belongs to the shard it was given for
  c->have_mov = c->mov_out_valid = false;   // and so does a movable set
  c->run_on_shard = c->eval_on_shard = false;   // so do a run's assignment and an evaluation
  c->cmp_on_shard = false;                      // and a comparison's matches
  c->final_on_shard = c->final_ready = false;   // and the result the per-vertex getters serve
  c->parts.assign(parts, parts + c->nranks + 1);
  c->base = c->parts[c->rank];
  c->bound = c->parts[c->rank + 1];
  c->nv_global = nv_global; c->lnv = lnv; c->lne = lne;
  c->have_graph = false;
  c->peers_ready = false;
  c->d_rowptr64 = nullptr; c->d_edges = nullptr; c->d_tails32 = nullptr;   // set_source names the new shard's arrays
  return 0;
}

// where setup_run reads the shard set_graph described (full records or compact tails) and what uploading it cost; the
// context has a shard from here on
void set_source(mvgpu_ctx *c, const long long *rowptr64, const Edge16 *edges, const int32_t *tails32, bool f32, double h2d_s,
                long long h2d_bytes) {
  c->d_rowptr64 = rowptr64; c->d_edges = edges; c->d_tails32 = tails32; c->f32 = f32;
  c->h2d_s = h2d_s; c->h2d_bytes = h2d_bytes;
  c->have_graph = true;
}

// CUB's two-phase protocol for one or more calls that share c->cub_tmp: every size query, one (grow-only) ensure of the
// largest, then the calls in order.  Each f(temp, bytes) is one CUB call.
template <typename... F>
int cub_run(mvgpu_ctx *c, F &&...f) {
  size_t need = 0;
  auto query = [&](auto &g) { size_t tb = 0; g(nullptr, tb); need = std::max(need, tb); };
  (query(f), ...);
  TRY(c->cub_tmp.ensure(need));
  cudaError_t e = cudaSuccess;
  auto call = [&](auto &g) { size_t tb = c->cub_tmp.cap; if (e == cudaSuccess) e = g(c->cub_tmp.p, tb); };
  (call(f), ...);
  CK(e);
  return 0;
}

// ---- multi-GPU: publish/obtain peer pointers for the exported arrays (MV_EXPORTS) ------------------------------------
// this rank's exported arrays, in MV_EXPORTS order (the sizes matter to the grow test of setup_agree only)
void exports(const mvgpu_ctx *c, Export (&x)[kPeerArrays], size_t need_v = 0, size_t need_s = 0, bool ev = false,
             bool split = false) {
  int k = 0;
#define MV_EXPORT(buf, on, need, dst) x[k++] = {(on) ? (void *)c->buf.p : nullptr, c->buf.gen, c->buf.cap, (size_t)(need)};
  MV_EXPORTS(MV_EXPORT)
#undef MV_EXPORT
}

// rank r's copies of the exported arrays (q in MV_EXPORTS order) -> the peer tables
void bind_peer(mvgpu_ctx *c, int r, void *const *q) {
  int k = 0;
#define MV_BIND(buf, on, need, dst) dst = static_cast<std::remove_reference_t<decltype(dst)>>(q[k++]);
  MV_EXPORTS(MV_BIND)
#undef MV_BIND
}

void close_ipc(mvgpu_ctx *c) {
  for (void *p : c->ipc_opened) cudaIpcCloseMemHandle(p);
  c->ipc_opened.clear();
  c->ipc_valid = false;
}

int setup_peers(mvgpu_ctx *c) {
  PeerTable &pt = c->pt;
  pt.nranks = c->nranks; pt.rank = c->rank;
  for (int r = 0; r <= c->nranks; r++) pt.parts[r] = c->parts[r];
  Export x[kPeerArrays];
  exports(c, x);
  void *ptrs[kPeerArrays];
  for (int k = 0; k < kPeerArrays; k++) ptrs[k] = x[k].p;
  if (c->nranks == 1) { bind_peer(c, 0, ptrs); return 0; }
  if (c->peers_ready) return 0;            // same graph, same buffers: tables are still valid
  // IPC handles are expensive to (re)open: skip the exchange when no rank's buffers moved since the last one.  The
  // evaluation arrays are exported whenever they exist, so alternating runs and evaluations reopen no mapping for them;
  // lab / inv are exported by a renumbering run and never by an evaluation, so switching between those two does.
  long long changed = c->ipc_valid ? 0 : 1;
  for (int k = 0; k < kPeerArrays; k++) if (ptrs[k] != c->last_export[k].p || (ptrs[k] && x[k].gen != c->last_export[k].gen)) changed = 1;
  TRY(coll_allreduce_i64(c, &changed, 1, true));
  if (changed) {
    close_ipc(c);
    PeerBlob mine;
    memset(&mine, 0, sizeof mine);
    for (int k = 0; k < kPeerArrays; k++) {
      mine.raw[k] = (unsigned long long)ptrs[k];
      if (ptrs[k]) CK(cudaIpcGetMemHandle(&mine.h[k], ptrs[k]));
    }
    mine.pid = (int)getpid(); mine.device = c->device; mine.unit = c->unit ? 1 : 0;
    std::vector<PeerBlob> all(c->nranks);
    TRY(coll_allgather(c, &mine, all.data(), sizeof(PeerBlob)));
    for (int r = 0; r < c->nranks; r++) {
      void *q[kPeerArrays] = {};
      if (all[r].unit != mine.unit) return fail("ranks disagree on the unit-weight path");
      if (r == c->rank) { for (int k = 0; k < kPeerArrays; k++) q[k] = ptrs[k]; }
      else if (all[r].pid == mine.pid) {           // same process (threads): plain UVA pointers + peer access
        if (all[r].device != c->device) {          // ranks sharing one device need no peer mapping at all
          int can = 0;
          CK(cudaDeviceCanAccessPeer(&can, c->device, all[r].device));
          if (!can) return fail("GPU " + std::to_string(c->device) + " cannot access peer GPU " + std::to_string(all[r].device));
          cudaError_t e = cudaDeviceEnablePeerAccess(all[r].device, 0);
          if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e);
          cudaGetLastError();
        }
        for (int k = 0; k < kPeerArrays; k++) q[k] = (void *)all[r].raw[k];
      } else {
        for (int k = 0; k < kPeerArrays; k++)
          if (all[r].raw[k]) {
            CK(cudaIpcOpenMemHandle(&q[k], all[r].h[k], cudaIpcMemLazyEnablePeerAccess));
            c->ipc_opened.push_back(q[k]);
          }
      }
      bind_peer(c, r, q);
    }
    std::copy(x, x + kPeerArrays, c->last_export);
    c->ipc_valid = true;
  }
  // where my send segments land in each peer's community array: its lnv + its receive offset for me
  std::vector<long long> gb(c->nranks), allgb((size_t)c->nranks * c->nranks);
  for (int r = 0; r < c->nranks; r++) gb[r] = c->lnv + c->roff[r];
  TRY(coll_allgather(c, gb.data(), allgb.data(), sizeof(long long) * c->nranks));
  for (int b = 0; b < 2; b++) {
    PushTable &t = c->push[b];
    t.nranks = c->nranks;
    for (int r = 0; r <= c->nranks; r++) t.soff[r] = c->soff[r];
    for (int r = 0; r < c->nranks; r++) t.dst[r] = c->peer_comm[b][r] + allgb[(size_t)r * c->nranks + c->rank];
  }
  c->pp.rank = c->rank; c->pp.nranks = c->nranks;
  c->peers_ready = true;
  return 0;
}

// MASKED: the run reads a movable set (mov, internal numbering); iteration 1 never takes FIRST then (run_louvain)
template <bool UNIT, bool MULTI, bool TRACE, bool MASKED>
int launch_scan_t(mvgpu_ctx *c, const ScanParams &sp, bool first, const uint8_t *mov) {
  const size_t smem = UNIT ? sizeof(int32_t) * 2 * kECap : sizeof(int32_t) * kECap + sizeof(double) * kECap;
  static bool attr_done = false;
  if (!attr_done) {
    CK(cudaFuncSetAttribute(k_scan_ws<UNIT, MULTI, TRACE, MASKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  const int tiles = (int)((c->lnv + kTileV - 1) / kTileV);
  if (tiles > 0 && c->opt_scan_variant >= 5 && c->scan_kernel == 5 && UNIT && !first) {
    // k_scan_pw's pipeline with a per-warp ring of hard vertices (scan_queue.cuh); iteration 1 and the weighted path
    // stay with k_scan_pw
    static int pq_ctas_per_sm = 0;
    if (!pq_ctas_per_sm) {
      CK(cudaFuncSetAttribute(k_scan_pq<MULTI, TRACE, MASKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pq_smem_bytes()));
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pq_ctas_per_sm, k_scan_pq<MULTI, TRACE, MASKED>, kPwWarps * 32, pq_smem_bytes()));
      if (pq_ctas_per_sm < 1) return fail("k_scan_pq cannot be made resident");
    }
    const int ngroups = (int)((c->lnv + 31) / 32);
    const int grid = std::min((ngroups + kPwWarps - 1) / kPwWarps, c->opt_scan_ctas > 0 ? c->opt_scan_ctas : pq_ctas_per_sm * c->num_sms);
    k_scan_pq<MULTI, TRACE, MASKED><<<grid, kPwWarps * 32, pq_smem_bytes(), c->stream>>>(sp, ngroups, mov);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  } else if (tiles > 0 && c->opt_scan_variant >= 4) {
    // persistent warps, TMA-fed double buffer (scan_pipe.cuh): one CTA slot per resident block, warps stride over groups
    static int pw_ctas_per_sm = 0;
    if (!pw_ctas_per_sm) {
      CK(cudaFuncSetAttribute(k_scan_pw<UNIT, MULTI, TRACE, false, MASKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pw_smem_bytes<UNIT>()));
      CK(cudaFuncSetAttribute(k_scan_pw<UNIT, MULTI, TRACE, UNIT && !MASKED, MASKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pw_smem_bytes<UNIT>()));
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pw_ctas_per_sm, k_scan_pw<UNIT, MULTI, TRACE, false, MASKED>, kPwWarps * 32, pw_smem_bytes<UNIT>()));
      if (pw_ctas_per_sm < 1) return fail("k_scan_pw cannot be made resident");
    }
    const int ngroups = (int)((c->lnv + 31) / 32);
    const int grid = std::min((ngroups + kPwWarps - 1) / kPwWarps, c->opt_scan_ctas > 0 ? c->opt_scan_ctas : pw_ctas_per_sm * c->num_sms);
    if (UNIT && first) {
      k_scan_pw<UNIT, MULTI, TRACE, UNIT && !MASKED, MASKED><<<grid, kPwWarps * 32, pw_smem_bytes<UNIT>(), c->stream>>>(sp, ngroups, mov);
      c->lay.first_ran = true;
    } else k_scan_pw<UNIT, MULTI, TRACE, false, MASKED><<<grid, kPwWarps * 32, pw_smem_bytes<UNIT>(), c->stream>>>(sp, ngroups, mov);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  } else if (tiles > 0) {
    k_scan_ws<UNIT, MULTI, TRACE, MASKED><<<tiles, kTileV, UNIT ? sizeof(int32_t) * kECap : smem, c->stream>>>(sp, mov);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  }
  if (c->nheavy > 0) {
    k_scan_heavy<UNIT, MULTI, TRACE, MASKED><<<(int)c->nheavy, 256, 0, c->stream>>>(sp, mov);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  }
  CK(cudaGetLastError());
  return 0;
}

int launch_scan(mvgpu_ctx *c, const ScanParams &sp, bool first, const uint8_t *mov) {
  const bool multi = c->nranks > 1, tr = c->opt_trace != 0;
#define MV_CASE(U, M, T)                                                                                             \
  if (c->unit == U && multi == M && tr == T)                                                                         \
    return c->mov_run ? launch_scan_t<U, M, T, true>(c, sp, first, mov) : launch_scan_t<U, M, T, false>(c, sp, first, mov);
  MV_CASE(true, false, false) MV_CASE(true, false, true) MV_CASE(true, true, false) MV_CASE(true, true, true)
  MV_CASE(false, false, false) MV_CASE(false, false, true) MV_CASE(false, true, false) MV_CASE(false, true, true)
#undef MV_CASE
  return fail("unreachable");
}

int exchange_ghosts(mvgpu_ctx *c, int32_t *comm);
int final_in_caller_order(mvgpu_ctx *c);

// "every rank's stream has reached this point" on the run's data plane (comm_mode): one-rank runs are stream ordered
int run_barrier(mvgpu_ctx *c) {
  if (c->nranks == 1) return 0;
  if (c->opt_comm_mode == 1) {
    k_p2p_barrier<<<1, 32, 0, c->stream>>>(c->pp, ++c->p2p_epoch);
    c->tm.kernel_launches++;
    CK(cudaGetLastError());
    return 0;
  }
  return coll_barrier(c);
}

// Warm start: comm_a := the initial assignment `init` (caller ids) in internal ids (ghost slots by the usual exchange),
// Comm records := its aggregates.  Runs after setup_peers, over k_vertex_init's singleton state (degrees, self loops,
// 1/(2m) stay).
int warm_init(mvgpu_ctx *c, const int32_t *init) {
  cudaStream_t s = c->stream;
  const int lnv = (int)c->lnv, nsm = c->num_sms;
  // every rank's inv is written and its update arrays are zeroed (k_vertex_init) before a peer reads or adds to them
  if (c->nranks > 1) TRY(coll_barrier(c));
  WarmInv m;
  memset(&m, 0, sizeof m);
  for (int r = 0; r < c->nranks; r++) m.inv[r] = c->relabel ? c->peer_inv[r] : nullptr;
  k_warm_map<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, init, c->relabel ? c->inv.p : nullptr, c->pt, m, c->comm_a.p);
  c->tm.kernel_launches++;
  if (c->nranks > 1) TRY(exchange_ghosts(c, c->comm_a.p));
  if (c->unit) k_warm_comm_unit<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->comm_a.p, c->a_rowptr, c->pt);
  else k_warm_comm_w<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->comm_a.p, c->vdeg.p, c->pt);
  c->tm.kernel_launches++;
  TRY(run_barrier(c));                        // all deltas have landed
  CK(cudaMemsetAsync(c->acc.p, 0, sizeof(Acc), s));
  if (c->unit) k_warm_fold_unit<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->cdeg.p, c->csize.p, c->upd.p, c->acc.p);
  else k_warm_fold_w<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->cinfo_w.p, c->usize.p, c->udeg.p);
  c->tm.kernel_launches++;
  TRY(run_barrier(c));                        // no scan reads or updates a record before its owner has folded it
  CK(cudaGetLastError());
  return 0;
}

// What an evaluation hands to setup_run: the assignment (caller ids, device) and what the caller side found wrong with
// it, which joins the input agreement so that every rank fails together.
struct EvalSetup {
  const int32_t *X = nullptr;
  bool given = false;                  // the caller passed an array (not NULL)
  bool split = false;                  // for mvgpu_split_communities: the labels are allocated and exported too
  bool probe = false;                  // for mvgpu_probe_communities: the evaluation's arrays are left alone
  std::string err;
};

// the compact CSR the iterations run on: the converted shard, then possibly its renumbered copy
struct Csr { const uint32_t *rowptr = nullptr; const int32_t *tails = nullptr; const double *weights = nullptr; };

// ---- setup: reference-format arrays -> compact graph, ghosts, init, as the stages of setup_run ------------------------
// Pass 1 over the edges: unit weights? how many non-owned tails? (+ input validation).  The compact upload format has
// answered all of that on the host already.  h: the device scalars after the pass; err: what this rank finds wrong.
int input_pass(mvgpu_ctx *c, const EvalSetup *ev, Scalars &h, int &unit, std::string &err) {
  cudaStream_t s = c->stream; const int nsm = c->num_sms; Scalars *d_sc = dev_scalars(c);
  const long long lnv = c->lnv, lne = c->lne;
  const bool compact_in = c->d_tails32 != nullptr;
  if (!compact_in && c->nranks == 1) {      // single rank: statistics ride on the conversion pass
    TRY(c->tails.ensure(lne + 4));
    k_convert_edges<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->d_edges, lne, c->base, c->bound, c->nv_global, c->tails.p,
                                                              nullptr, nullptr, nullptr, nullptr, &d_sc->st);
    c->tm.kernel_launches++;
  } else if (!compact_in) {
    k_edge_stats<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->d_edges, lne, c->base, c->bound, c->nv_global, &d_sc->st);
    c->tm.kernel_launches++;
  }
  TRY(c->rowptr.ensure(lnv + 1 + 40));        // + slack: the scan's row-offset bulk copies read 36 entries per group
  k_rowptr32<<<grid_for(lnv + 1, 256, nsm), 256, 0, s>>>(c->d_rowptr64, (int)lnv, lne, c->rowptr.p, &d_sc->maxdeg, &d_sc->bad_rowptr);
  c->tm.kernel_launches++;
  CK(cudaMemcpyAsync(&h, d_sc, sizeof h, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (compact_in) { h.st.nremote = (unsigned long long)c->in_nremote; h.st.nonunit = 0; h.st.bad_tail = 0; }
  if (h.st.bad_tail) err = "edge tail outside [0, nv)";
  else if (h.bad_rowptr) err = "edge_indices malformed (must start at 0, end at lne and never decrease)";
  else if (c->nranks == 1 && h.st.nremote) err = "non-local tail in a single-rank graph";
  c->maxdeg = h.maxdeg;
  unit = (!h.st.nonunit && !c->opt_force_weighted) ? 1 : 0;
  if (err.empty() && compact_in && !unit) err = "force_weighted needs the full edge records: set compact_upload=0";
  if (err.empty() && ev) err = ev->err;
  return 0;
}

// The partition agreement rides on a sum all-reduce: slot r carries rank r's fingerprint of (nv_global, parts) and every
// other rank contributes 0 there, so after the sum every rank holds every rank's fingerprint and reaches the same verdict.
const char *const kPartitionDisagree = "ranks disagree on the partition: every rank must hold a shard of the same nv_global and parts";
void partition_slots(const mvgpu_ctx *c, long long *slots) {
  unsigned long long h = 0xcbf29ce484222325ULL ^ (unsigned long long)c->nv_global;
  for (long long p : c->parts) h = (h ^ (unsigned long long)p) * 0x100000001b3ULL;   // FNV-1a over the offsets
  h ^= h >> 29;
  for (int r = 0; r < c->nranks; r++) slots[r] = 0;
  slots[c->rank] = (long long)(h >> 1);                  // non-negative: a sum of one of them and zeros cannot overflow
}
bool partition_agrees(const mvgpu_ctx *c, const long long *slots) {
  for (int r = 1; r < c->nranks; r++) if (slots[r] != slots[0]) return false;
  return true;
}

// The one setup agreement (one all-reduce): path, edge total, input errors, "must grow an exported array", "was given
// an assignment", the partition.  Errors are agreed on before anybody returns: a rank that left alone would leave its
// peers blocked in the next collective.  Sets c->unit (2m < 2^31 settles from the edge total; the weight total comes later).
int setup_agree(mvgpu_ctx *c, const EvalSetup *ev, long long nremote, int unit, std::string err) {
  long long ne_global = c->lne;
  if (c->nranks > 1) {
    // CUDA IPC requires every peer to close its mapping before the owner frees the block, so growing an exported array
    // is agreed on here and done collectively (need_s: init_state's bound lnv + #non-owned edge tails >= lnv + nghost)
    Export x[kPeerArrays];
    exports(c, x, (size_t)c->lnv, (size_t)(c->lnv + nremote), ev && !ev->probe, ev && ev->split);
    bool grow = false;
    for (const Export &e : x) grow = grow || (c->ipc_valid && e.cap && e.cap < e.need);
    const bool assigned = ev ? ev->given : c->warm_run;
    // [5], [6]: a movable set, and its frontier option (a rank would store into a peer's unexported next set);
    // [7 + r]: rank r's partition fingerprint
    long long hv[7 + kMaxRanks] = {unit ? 0 : 1, c->lne, err.empty() ? 0 : 1, grow ? 1 : 0, assigned ? 1 : 0, c->mov_run ? 1 : 0,
                                   c->mov_run && c->opt_frontier ? 1 : 0};
    partition_slots(c, hv + 7);
    TRY(coll_allreduce_i64(c, hv, 7 + c->nranks, false));
    unit = hv[0] == 0;
    ne_global = hv[1];
    if (err.empty() && !partition_agrees(c, hv + 7)) err = kPartitionDisagree;
    if (hv[2] && err.empty()) err = ev ? "another rank rejected its shard or its assignment" : "another rank rejected its shard";
    if (err.empty() && hv[4] != 0 && hv[4] != c->nranks)
      err = ev ? std::string("ranks disagree on the assignment to ") + (ev->split ? "split" : ev->probe ? "probe" : "evaluate") +
                     ": every rank or none must pass NULL"
               : "ranks disagree on the initial assignment: every rank or none must set one";
    if (err.empty() && hv[5] != 0 && hv[5] != c->nranks)
      err = "ranks disagree on the movable set: every rank or none must set one (mvgpu_set_movable)";
    if (err.empty() && hv[6] != 0 && hv[6] != c->nranks)
      err = "ranks disagree on the frontier option of the movable set: every rank must set the same value";
    if (hv[3]) {
      close_ipc(c);
      c->peers_ready = false;
      TRY(coll_barrier(c));                       // all mappings are closed before any owner reallocates
    }
  }
  if (!err.empty()) return fail(err);
  if (unit && ne_global >= (1LL << 31)) unit = 0;   // packed 32-bit degree deltas need 2m < 2^31
  c->unit = unit != 0;
  return 0;
}

// pass 2: tails -> slots, weights split off, remote tails listed
int compact_edges(mvgpu_ctx *c, long long nremote, Csr &g) {
  cudaStream_t s = c->stream; const int nsm = c->num_sms; Scalars *d_sc = dev_scalars(c);
  const long long lne = c->lne;
  const bool compact_in = c->d_tails32 != nullptr;
  if (nremote) { TRY(c->remote_list.ensure(nremote)); TRY(c->remote_pos.ensure(nremote)); }
  g.rowptr = c->rowptr.p;
  if (compact_in && c->nranks == 1) {
    g.tails = c->d_tails32;                       // global id == local slot: the uploaded array is used as is (read-only)
    if (!c->unit) {                               // 2m >= 2^31: fp64 path on a shard that arrived without weights
      TRY(c->weights.ensure(lne + 4));
      k_fill_ones<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->weights.p, lne);
      c->tm.kernel_launches++;
      g.weights = c->weights.p;
    }
  } else if (c->nranks == 1) {
    g.tails = c->tails.p;                         // converted by input_pass
    if (!c->unit) {
      TRY(c->weights.ensure(lne + 4));
      k_extract_weights<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->d_edges, lne, c->weights.p);
      c->tm.kernel_launches++;
      g.weights = c->weights.p;
    }
  } else {
    TRY(c->tails.ensure(lne + 4));
    if (!c->unit) TRY(c->weights.ensure(lne + 4));
    if (compact_in)
      k_convert_tails32<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->d_tails32, lne, c->base, c->bound, c->tails.p,
                                                                  nremote ? c->remote_list.p : nullptr, c->remote_pos.p, &d_sc->remote_cursor);
    else
      k_convert_edges<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->d_edges, lne, c->base, c->bound, c->nv_global, c->tails.p,
                                                                c->unit ? nullptr : c->weights.p,
                                                                nremote ? c->remote_list.p : nullptr, c->remote_pos.p, &d_sc->remote_cursor, nullptr);
    c->tm.kernel_launches++;
    if (compact_in && !c->unit) {                 // a peer's shard is weighted (or 2m >= 2^31): this one's weights are all 1.0
      k_fill_ones<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->weights.p, lne);
      c->tm.kernel_launches++;
    }
    g.tails = c->tails.p;
    g.weights = c->unit ? nullptr : c->weights.p;
  }
  return 0;
}

// ghost discovery (exchangeVertexReqs, dspl.hpp:1106-1272): sorted unique non-owned tails, per-peer counts both ways,
// and the send lists
int discover_ghosts(mvgpu_ctx *c, long long nremote) {
  cudaStream_t s = c->stream; const int nsm = c->num_sms; Scalars *d_sc = dev_scalars(c);
  const long long lnv = c->lnv;
  c->nghost = 0; c->nsend = 0;
  c->rcount.assign(c->nranks, 0); c->scount.assign(c->nranks, 0);
  c->roff.assign(c->nranks + 1, 0); c->soff.assign(c->nranks + 1, 0);
  if (c->nranks == 1) return 0;
  if (nremote) {
    DevBuf<long long> &sorted = c->sorted_tmp;   // grow-only: no cudaMalloc/cudaFree inside the timed setup after the first run
    TRY(sorted.ensure(nremote));
    TRY(c->ghost_gid.ensure(nremote));
    int bits = 1;
    while ((1LL << bits) < c->nv_global && bits < 63) bits++;
    TRY(cub_run(c,
                [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortKeys(t, tb, c->remote_list.p, sorted.p, nremote, 0, bits, s); },
                [&](void *t, size_t &tb) { return cub::DeviceSelect::Unique(t, tb, sorted.p, c->ghost_gid.p, &d_sc->nunique, nremote, s); }));
    c->tm.kernel_launches += 2;
    int nu = 0;
    CK(cudaMemcpyAsync(&nu, &d_sc->nunique, sizeof nu, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    c->nghost = nu;
    if (lnv + c->nghost >= (1LL << 31)) return fail("lnv + nghost >= 2^31");
    k_remap_ghost_tails<<<grid_for(nremote, 256, nsm, 16), 256, 0, s>>>(c->remote_list.p, c->remote_pos.p, nremote, c->tails.p, c->ghost_gid.p, (int)c->nghost, (int)lnv);
    c->tm.kernel_launches++;
    // per-owner counts of my ghosts (the list is sorted, owners are contiguous ranges)
    std::vector<long long> hg(c->nghost);
    CK(cudaMemcpyAsync(hg.data(), c->ghost_gid.p, sizeof(long long) * c->nghost, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int r = 0; r < c->nranks; r++) {
      const long long lo = std::lower_bound(hg.begin(), hg.end(), c->parts[r]) - hg.begin();
      const long long hi = std::lower_bound(hg.begin(), hg.end(), c->parts[r + 1]) - hg.begin();
      c->rcount[r] = hi - lo;
    }
  }
  for (int r = 0; r < c->nranks; r++) c->roff[r + 1] = c->roff[r] + c->rcount[r];
  // tell every owner how many of its vertices I ghost (MPI_Alltoall of sizes, dspl.hpp:1184)
  std::vector<long long> allc((size_t)c->nranks * c->nranks);
  TRY(coll_allgather(c, c->rcount.data(), allc.data(), sizeof(long long) * c->nranks));
  for (int r = 0; r < c->nranks; r++) c->scount[r] = allc[(size_t)r * c->nranks + c->rank];
  for (int r = 0; r < c->nranks; r++) c->soff[r + 1] = c->soff[r] + c->scount[r];
  c->nsend = c->soff[c->nranks];
  // ship the ghost id lists to their owners (dspl.hpp:1228-1252); they become the owners' send lists
  TRY(c->send_gid.ensure(c->nsend));
  TRY(c->send_lid.ensure(c->nsend));
  TRY(c->send_buf.ensure(c->nsend));
  TRY(c->ghost_gid.ensure(c->nghost));
  TRY(coll_alltoallv_dev(c, c->ghost_gid.p, c->rcount, c->roff, c->send_gid.p, c->scount, c->soff, sizeof(long long)));
  if (c->nsend) {
    k_gid_to_lid<<<grid_for(c->nsend, 256, nsm), 256, 0, s>>>(c->send_gid.p, (int)c->nsend, c->base, c->send_lid.p);
    c->tm.kernel_launches++;
  }
  return 0;
}

// locality renumbering (see kernels.cuh): decide, then BFS regions -> sort -> permute the compact CSR g in place of the
// original numbering; fills c->lay.  An evaluation makes one pass over the edges, which does not pay for a renumbering.
int renumber(mvgpu_ctx *c, const EvalSetup *ev, Csr &g) {
  cudaStream_t s = c->stream; const int nsm = c->num_sms; Scalars *d_sc = dev_scalars(c);
  const long long lnv = c->lnv, lne = c->lne;
  c->reordered = false;
  c->relabel = 0;
  c->lay = LayoutReport();
  c->lay.tails = g.tails;
  int want = !ev && c->opt_reorder == 1 ? 1 : 0;
  if (!ev && c->opt_reorder == 2 && lnv >= 65536) {
    // auto: renumber when the given numbering has no locality (mean |tail - v| above lnv/64 on a vertex sample)
    k_span_sample<<<grid_for(lnv / 64 + 1, 256, nsm), 256, 0, s>>>((int)lnv, g.rowptr, g.tails, 64, &d_sc->span_sum, &d_sc->span_cnt);
    c->tm.kernel_launches++;
    unsigned long long sp2[2];
    CK(cudaMemcpyAsync(sp2, &d_sc->span_sum, sizeof sp2, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (sp2[1] > 0 && (double)sp2[0] / (double)sp2[1] > (double)lnv / 64.0) want = 1;
    c->lay.span[0] = (long long)sp2[0]; c->lay.span[1] = (long long)sp2[1];
  }
  // region ids have kBfsRegionBits bits: past 2^22 - 1 regions they would spill into the level field (and region
  // 2^22 - 1 at level 1023 would read as kBfsUnreached), so very large shards get proportionally larger regions
  const int stride = (int)std::max<long long>(c->opt_region, (lnv + kBfsMaxRegions - 1) / kBfsMaxRegions);
  c->lay.want = want;
  c->lay.stride = stride;
  int any = want;
  if (c->nranks > 1) {
    long long hv = want;
    TRY(coll_allreduce_i64(c, &hv, 1, true));
    any = hv != 0;
  }
  c->relabel = any;                         // labels are needed everywhere as soon as one rank renumbers
  if (any && lnv > 0) {
    cudaEvent_t r0 = get_event(c, 2), r1 = get_event(c, 3);
    CK(cudaEventRecord(r0, s));
    TRY(c->perm.ensure(lnv)); TRY(c->inv.ensure(lnv)); TRY(c->lab.ensure(lnv)); TRY(c->ids.ensure(lnv));
    TRY(c->bfs_key.ensure(lnv)); TRY(c->sortkey.ensure(lnv)); TRY(c->sortkey2.ensure(std::max(lnv, 4 * ((lnv + 31) / 32))));
    TRY(c->deg_new.ensure(lnv + 1)); TRY(c->rowptr2.ensure(lnv + 1 + 40)); TRY(c->tails2.ensure(lne + 4));
    if (!c->unit) TRY(c->weights2.ensure(lne + 4));
    const int max_levels = 1023;
    if (want) {
      TRY(c->bfs_level_count.ensure(max_levels));
      int occ = 0;
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_msbfs, 256, 0));
      if (occ < 1) return fail("k_msbfs cannot be made resident");
      int ilnv = (int)lnv, st = stride, ml = max_levels;
      const uint32_t *rp = g.rowptr; const int32_t *tl = g.tails; uint32_t *key = c->bfs_key.p;
      // the BFS queue and its level bitmaps (4 bits per vertex) live in ids and sortkey2, which k_bfs_sortkeys and the
      // sort only write after the BFS
      int32_t *q = c->ids.p; unsigned int *lc = c->bfs_level_count.p; uint32_t *lm = c->sortkey2.p;
      void *args[] = {&ilnv, &rp, &tl, &key, &st, &ml, &q, &lc, &lm};
      CK(cudaLaunchCooperativeKernel((void *)k_msbfs, dim3(occ * nsm), dim3(256), args, 0, s));
      // sort by (region, level): only the bits that can be set take part (one radix pass less than a 32-bit sort)
      const long long nregions = (lnv + stride - 1) / stride;
      c->lay.nregions = nregions;
      int sort_bits = (int)kBfsLevelBits;
      while ((1LL << (sort_bits - (int)kBfsLevelBits)) <= nregions && sort_bits < 32) sort_bits++;
      const unsigned int unreached_key = sort_bits >= 32 ? 0xFFFFFFFFu : ((1u << sort_bits) - 1u);
      k_bfs_sortkeys<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->bfs_key.p, c->sortkey.p, c->ids.p, unreached_key);
      TRY(cub_run(c, [&](void *t, size_t &tb) {
        return cub::DeviceRadixSort::SortPairs(t, tb, c->sortkey.p, c->sortkey2.p, c->ids.p, c->perm.p, (int)lnv, 0, sort_bits, s); }));
      c->tm.kernel_launches += 3;
    } else {
      // another rank renumbers, this one keeps its order: identity permutation, labels still required
      k_bfs_sortkeys<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->bfs_key.p, c->sortkey.p, c->perm.p, 0xFFFFFFFFu);
      c->tm.kernel_launches++;
    }
    k_perm_inverse<<<grid_for(lnv + 1, 256, nsm), 256, 0, s>>>((int)lnv, c->perm.p, c->base, want ? nullptr : c->inv.p, c->lab.p, g.rowptr, c->deg_new.p);
    c->tm.kernel_launches++;
    if (want) {
      // inv[old] = new as a second radix sort (keys perm, values the ids 0..lnv-1 still in c->ids): lnv random 4-byte
      // stores inv[perm[i]] = i cost more than twice as much as the sort's bucketed scatters (DESIGN.md §3.3)
      int bits = 1;
      while ((1LL << bits) < lnv && bits < 31) bits++;
      const uint32_t *pk = reinterpret_cast<const uint32_t *>(c->perm.p);
      TRY(cub_run(c, [&](void *t, size_t &tb) {
        return cub::DeviceRadixSort::SortPairs(t, tb, pk, c->sortkey2.p, c->ids.p, c->inv.p, (int)lnv, 0, bits, s); }));
      TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::ExclusiveSum(t, tb, c->deg_new.p, c->rowptr2.p, (int)lnv + 1, s); }));
      k_permute_adj<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->perm.p, c->inv.p, g.rowptr, g.tails, g.weights,
                                                             c->rowptr2.p, c->tails2.p, c->unit ? nullptr : c->weights2.p,
                                                             (int)c->roff[c->rank], &d_sc->unordered);
      c->tm.kernel_launches += 3;
      g.rowptr = c->rowptr2.p;
      g.tails = c->tails2.p;
      g.weights = c->unit ? nullptr : c->weights2.p;
      c->reordered = true;
    }
    CK(cudaEventRecord(r1, s));
  }
  // peers asked for my vertices by ORIGINAL id: the send list holds their current (internal) local index
  if (c->relabel && c->nsend) {
    k_apply_inv<<<grid_for(c->nsend, 256, nsm), 256, 0, s>>>(c->send_lid.p, (int)c->nsend, c->inv.p);
    c->tm.kernel_launches++;
  }
  return 0;
}

// state arrays and the singleton start (k_vertex_init) over the compact CSR in c->a_*
int init_state(mvgpu_ctx *c, const EvalSetup *ev, long long nremote) {
  cudaStream_t s = c->stream; const int nsm = c->num_sms; Scalars *d_sc = dev_scalars(c);
  const long long lnv = c->lnv;
  // sized for the bound the collective "does an exported array have to grow?" test can evaluate before the ghosts are
  // known (lnv + #non-owned edge tails >= lnv + nghost), so that a repeated run never looks like a growing one
  const long long nslots = lnv + c->nghost;
  TRY(c->comm_a.ensure(std::max(nslots, lnv + nremote)));
  TRY(c->comm_b.ensure(std::max(nslots, lnv + nremote)));
  if (c->unit) { TRY(c->cdeg.ensure(lnv)); TRY(c->csize.ensure(lnv)); TRY(c->upd.ensure(lnv)); TRY(c->self_i.ensure(lnv)); }
  else { TRY(c->cinfo_w.ensure(lnv)); TRY(c->usize.ensure(lnv)); TRY(c->udeg.ensure(lnv)); TRY(c->vdeg.ensure(lnv)); TRY(c->self_d.ensure(lnv)); }
  TRY(c->acc.ensure((size_t)c->opt_max_iters + 2));
  CK(cudaMemsetAsync(c->acc.p, 0, sizeof(Acc) * ((size_t)c->opt_max_iters + 2), s));
  if (ev && !ev->probe) {                     // zeroed before warm_init's last barrier: no peer adds to it earlier
    TRY(c->q_internal.ensure(lnv)); TRY(c->q_rank.ensure(lnv + 1));
    CK(cudaMemsetAsync(c->q_internal.p, 0, sizeof(double) * lnv, s));
    if (ev->split) TRY(c->split_lab.ensure(lnv));
  }
  if (c->mov_run) {                           // M_1 = M in internal numbering (both buffers: see k_frontier_mark)
    TRY(c->mov_a.ensure(lnv)); TRY(c->mov_b.ensure(lnv));
    if (lnv > 0) {
      k_movable_in<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->mov_in.p, c->relabel ? c->inv.p : nullptr, c->mov_a.p,
                                                           c->opt_frontier ? c->mov_b.p : nullptr);
      c->tm.kernel_launches++;
    }
  }
  if (c->unit)
    k_vertex_init<true><<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->base, c->a_rowptr, c->a_tails, nullptr, c->comm_a.p,
                                                              c->cdeg.p, c->csize.p, c->upd.p, nullptr, nullptr, nullptr, nullptr,
                                                              c->self_i.p, nullptr, &d_sc->total_weight, &d_sc->has_self,
                                                              (int)c->roff[c->rank], c->reordered ? nullptr : &d_sc->unordered, c->acc.p);
  else
    k_vertex_init<false><<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->base, c->a_rowptr, c->a_tails, c->a_weights, c->comm_a.p,
                                                               nullptr, nullptr, nullptr, c->cinfo_w.p, c->usize.p, c->udeg.p, c->vdeg.p,
                                                               nullptr, c->self_d.p, &d_sc->total_weight, &d_sc->has_self, 0, nullptr, nullptr);
  c->tm.kernel_launches++;
  // ghosts start in their own (internal) singleton community, which only the owner knows after renumbering:
  // fetch it with the same all-to-all-v the iterations use (a warm run fills comm_a in warm_init instead)
  if (c->nranks > 1 && !c->warm_run) TRY(exchange_ghosts(c, c->comm_a.p));
  return 0;
}

// high-degree vertices, launched here and listed by heavy_finish after the 1/(2m) read-back.  heavy_deg: the largest
// degree the tile kernels take, one staging buffer (minus the 16-byte alignment slack of the bulk copies)
int heavy_launch(mvgpu_ctx *c, long long &heavy_deg) {
  const long long tile_cap = c->opt_scan_variant >= 4 ? (c->unit ? PwCap<true>::value : PwCap<false>::value) - 4 : kECap;
  heavy_deg = (c->opt_force_heavy_deg > 0) ? std::min<long long>(c->opt_force_heavy_deg, tile_cap) : tile_cap;
  c->nheavy = 0;
  if (c->maxdeg > heavy_deg) {
    TRY(c->heavy_list.ensure(c->lnv));
    k_collect_heavy<<<grid_for(c->lnv, 256, c->num_sms), 256, 0, c->stream>>>((int)c->lnv, c->a_rowptr, (unsigned int)heavy_deg, c->heavy_list.p,
                                                                              &dev_scalars(c)->heavy_count);
    c->tm.kernel_launches++;
  }
  return 0;
}

// 1/(2m): MPI_Allreduce of the local degree sums (dspl.hpp:109-130), read back with the flags of k_vertex_init into h
int total_weight(mvgpu_ctx *c, Scalars &h) {
  cudaStream_t s = c->stream; Scalars *d_sc = dev_scalars(c);
  if (c->nranks > 1 && !c->hc.is_open()) NK(g_nccl.AllReduce(&d_sc->total_weight, &d_sc->total_weight, 1, ncclDouble, ncclSum, c->comm, s));
  CK(cudaMemcpyAsync(&h, d_sc, sizeof h, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (c->nranks > 1 && c->hc.is_open()) c->hc.allreduce(&h.total_weight, 1, [](double a, double b) { return a + b; });
  c->constant = 1.0 / h.total_weight;
  if (c->f32) c->constant = (double)(float)(1.0 / (double)(float)h.total_weight);   // dspl.hpp:129 with GraphWeight = float
  c->lay.has_self = h.has_self ? 1 : 0;
  c->lay.unordered = h.unordered ? 1 : 0;
  c->simple_sorted = c->unit && !h.unordered && !h.has_self;
  return 0;
}

// high-degree vertices, second half: the sorted list and each one's hash-table offset
int heavy_finish(mvgpu_ctx *c, long long heavy_deg, unsigned int heavy_count) {
  if (c->maxdeg <= heavy_deg) return 0;
  c->nheavy = heavy_count;
  std::vector<int32_t> hl(c->nheavy);
  CK(cudaMemcpy(hl.data(), c->heavy_list.p, sizeof(int32_t) * c->nheavy, cudaMemcpyDeviceToHost));
  std::sort(hl.begin(), hl.end());
  CK(cudaMemcpy(c->heavy_list.p, hl.data(), sizeof(int32_t) * c->nheavy, cudaMemcpyHostToDevice));
  std::vector<unsigned long long> off(c->nheavy + 1, 0);
  for (long long i = 0; i < c->nheavy; i++) {
    uint32_t r2[2];
    CK(cudaMemcpy(r2, c->a_rowptr + hl[i], sizeof r2, cudaMemcpyDeviceToHost));
    unsigned long long T = 64;
    while (T < 2ULL * (r2[1] - r2[0])) T <<= 1;
    off[i + 1] = off[i] + T;
  }
  TRY(c->heavy_off.ensure(c->nheavy + 1));
  CK(cudaMemcpy(c->heavy_off.p, off.data(), sizeof(unsigned long long) * (c->nheavy + 1), cudaMemcpyHostToDevice));
  TRY(c->hkeys.ensure(off[c->nheavy]));
  if (c->unit) TRY(c->hvals_i.ensure(off[c->nheavy])); else TRY(c->hvals_d.ensure(off[c->nheavy]));
  return 0;
}

// ev != nullptr: setup for an evaluation -- warm init from ev->X, no locality renumbering, evaluation arrays allocated
int setup_run(mvgpu_ctx *c, const EvalSetup *ev = nullptr) {
  TRY(c->scratch.ensure(sizeof(Scalars)));
  CK(cudaMemsetAsync(c->scratch.p, 0, sizeof(Scalars), c->stream));
  c->warm_run = ev ? true : c->have_init;
  c->mov_run = !ev && c->have_mov;
  Scalars h;                                 // the device scalars after the input pass, then after the 1/(2m) read-back
  int unit = 0;
  std::string err;
  TRY(input_pass(c, ev, h, unit, err));
  const long long nremote = (long long)h.st.nremote;
  TRY(setup_agree(c, ev, nremote, unit, err));
  Csr g;
  TRY(compact_edges(c, nremote, g));
  TRY(discover_ghosts(c, nremote));
  TRY(renumber(c, ev, g));
  c->a_rowptr = g.rowptr; c->a_tails = g.tails; c->a_weights = g.weights;
  TRY(init_state(c, ev, nremote));
  if (!ev) {
    // The arrays the run writes after its last iteration are sized here, before the first peer-memory collective: a
    // grow there frees the old block, and cudaFree waits for the whole device -- including a peer rank's barrier kernel
    // that spins until this rank's barrier arrives (ranks sharing a device would wait on each other until the watchdog).
    TRY(c->final_orig.ensure(c->lnv));
    if (c->mov_run) TRY(c->mov_out.ensure(c->lnv));
  }
  long long heavy_deg = 0;
  TRY(heavy_launch(c, heavy_deg));
  TRY(total_weight(c, h));
  TRY(heavy_finish(c, heavy_deg, h.heavy_count));
  if (c->nranks > 1) {
    TRY(c->p2p.ensure(1));
    if (!c->p2p_zeroed) { CK(cudaMemsetAsync(c->p2p.p, 0, sizeof(P2PState), c->stream)); CK(cudaStreamSynchronize(c->stream)); c->p2p_zeroed = true; }
  }
  TRY(setup_peers(c));
  if (c->warm_run) TRY(warm_init(c, ev ? ev->X : c->init_comm.p));
  c->tm.unit_weight = c->unit ? 1 : 0;
  c->scan_has_self = c->lay.has_self;
  c->scan_heavy_deg = (int)heavy_deg;
  return 0;
}

// ---- ghost exchange: targetComm of the vertices peers ghost -> ghost tail of their community array.
// The reference's gather + Isend/Irecv/Waitall (dspl.hpp:559-646) as one grouped NCCL all-to-all-v with
// the run-constant counts from setup; the payload lands in place (no unpack, no remoteComm map).
int exchange_ghosts(mvgpu_ctx *c, int32_t *comm) {
  cudaStream_t s = c->stream;
  if (c->nsend) {
    k_pack_send<<<grid_for(c->nsend, 256, c->num_sms), 256, 0, s>>>(comm, c->send_lid.p, (int)c->nsend, c->send_buf.p);
    c->tm.kernel_launches++;
  }
  std::vector<long long> roff_slots(c->roff);
  return coll_alltoallv_dev(c, c->send_buf.p, c->scount, c->soff, comm + c->lnv, c->rcount, roff_slots, sizeof(int32_t));
}

// a graph and, with several ranks, a communicator that carries the run's data plane
int check_ready(mvgpu_ctx *c) {
  if (!c->have_graph || !c->d_rowptr64) return fail("no graph uploaded");
  if (c->nranks > 1 && !c->comm && !c->hc.is_open()) return fail("mvgpu_comm_init has not been called");
  if (c->nranks > 1 && !c->comm && c->opt_comm_mode != 1) return fail("comm_mode=0 (NCCL data plane) needs the NCCL communicator: host_transport=1 supports comm_mode=1 only");
  return 0;
}

// ---- the cross-rank sum of an Acc record (dspl.hpp:441): e and a2 in rank order, plus the trace counters.
// acc_sum_enqueue puts it on the stream, into the pinned mailbox; acc_sum_read reads it after the caller's synchronise.
struct HostMail { Acc acc; double red2[2]; unsigned long long tr2[2]; unsigned int p2p_error; };
struct AccSum { double e, a2; unsigned long long moved, hash; };

int acc_sum_enqueue(mvgpu_ctx *c, Acc *acc, bool trace) {
  cudaStream_t s = c->stream; Scalars *d_sc = dev_scalars(c);
  HostMail *mail = reinterpret_cast<HostMail *>(c->h_pin);
  if (c->nranks == 1) CK(cudaMemcpyAsync(&mail->acc, acc, sizeof(Acc), cudaMemcpyDeviceToHost, s));
  else if (c->opt_comm_mode == 1) {
    k_p2p_allreduce<<<1, 32, 0, s>>>(c->pp, ++c->p2p_epoch, acc, c->unit ? 1 : 0, d_sc->red2, d_sc->tr2);
    c->tm.kernel_launches++;
    CK(cudaMemcpyAsync(mail->red2, d_sc->red2, sizeof mail->red2 + sizeof mail->tr2, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&mail->p2p_error, &c->p2p.p->error, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
  } else {
    k_acc_to_double<<<1, 32, 0, s>>>(acc, c->unit ? 1 : 0, d_sc->red2);
    c->tm.kernel_launches++;
    NK(g_nccl.AllReduce(d_sc->red2, d_sc->red2, 2, ncclDouble, ncclSum, c->comm, s));
    CK(cudaMemcpyAsync(mail->red2, d_sc->red2, sizeof mail->red2, cudaMemcpyDeviceToHost, s));
    if (trace) {
      k_trace_to_u64<<<1, 32, 0, s>>>(acc, d_sc->tr2);
      c->tm.kernel_launches++;
      NK(g_nccl.AllReduce(d_sc->tr2, d_sc->tr2, 2, ncclUint64, ncclSum, c->comm, s));
      CK(cudaMemcpyAsync(mail->tr2, d_sc->tr2, sizeof mail->tr2, cudaMemcpyDeviceToHost, s));
    }
  }
  return 0;
}

// moved / hash are only summed over several NCCL ranks when acc_sum_enqueue was asked for the trace
int acc_sum_read(mvgpu_ctx *c, AccSum &r) {
  const HostMail *mail = reinterpret_cast<const HostMail *>(c->h_pin);
  const Acc &a = mail->acc;
  if (c->nranks == 1) r = {c->unit ? (double)a.le_u : a.le_d, c->unit ? (double)a.la2_u : a.la2_d, a.moved, a.hash};
  else if (c->opt_comm_mode == 1 && mail->p2p_error) return fail("peer-memory collective timed out (a peer rank is gone)");
  else r = {mail->red2[0], mail->red2[1], mail->tr2[0], mail->tr2[1]};
  return 0;
}

// Q = e * constant - a2 * constant * constant with every product rounded on its own (dspl.hpp:447-448)
double modularity(double e, double a2, double cst) {
  volatile double term1 = e * cst;
  volatile double term2a = a2 * cst;
  volatile double term2 = term2a * cst;
  return term1 - term2;
}

// what the scan kernels read of the state setup_run left (cur, tgt and acc are per iteration: the caller's)
ScanParams scan_params(const mvgpu_ctx *c) {
  ScanParams sp;
  memset(&sp, 0, sizeof sp);
  sp.lnv = (int)c->lnv; sp.has_self = c->scan_has_self; sp.heavy_deg = c->scan_heavy_deg; sp.has_heavy = c->nheavy > 0; sp.base = c->base;
  sp.cache_policy = c->opt_cache_policy;
  sp.relabel = c->relabel;
  sp.rowptr = c->a_rowptr; sp.tails = c->a_tails; sp.weights = c->unit ? nullptr : c->a_weights;
  sp.self_i = c->self_i.p; sp.self_d = c->self_d.p; sp.vdeg = c->vdeg.p; sp.constant = c->constant; sp.f32 = c->f32 ? 1 : 0;
  sp.heavy_list = c->heavy_list.p; sp.heavy_off = c->heavy_off.p; sp.hkeys = c->hkeys.p; sp.hvals_d = c->hvals_d.p; sp.hvals_i = c->hvals_i.p;
  sp.pt = c->pt;
  sp.loc_cdeg = c->cdeg.p; sp.loc_csize = c->csize.p; sp.loc_upd = c->upd.p; sp.loc_cinfo_w = c->cinfo_w.p;
  sp.loc_usize = c->usize.p; sp.loc_udeg = c->udeg.p; sp.loc_lab = c->relabel ? c->lab.p : nullptr;
  return sp;
}

int run_louvain(mvgpu_ctx *c, double lower, double thresh, int *iters_out, double *mod_out) {
  TRY(check_ready(c));
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  memset(&c->tm, 0, sizeof c->tm);
  c->trace.clear();
  c->scan_times.clear();
  size_t ev = 0;
  cudaEvent_t e_begin = get_event(c, ev++), e_setup = get_event(c, ev++);
  ev = 4;                                   // events 2,3 bracket the renumbering inside setup_run
  CK(cudaEventRecord(e_begin, s));
  TRY(setup_run(c));
  CK(cudaEventRecord(e_setup, s));

  int32_t *cur = c->comm_a.p, *tgt = c->comm_b.p;
  ScanParams sp = scan_params(c);
  // movable set: M_k in mov[k_cur]; with the frontier option the scan's movers grow M_{k+1} into the other buffer,
  // every rank's (mp[b] addresses buffer b on every rank), and an accepted iteration swaps them like cur / tgt
  uint8_t *mov[2] = {c->mov_a.p, c->mov_b.p};
  int k_cur = 0;
  const bool frontier = c->mov_run && c->opt_frontier;
  MovPeers mp[2];
  memset(mp, 0, sizeof mp);
  for (int b = 0; b < 2 && frontier; b++)
    for (int r = 0; r < c->nranks; r++) { mp[b].next[r] = c->peer_mov[b][r]; mp[b].inv[r] = c->relabel ? c->peer_inv[r] : nullptr; }
  c->mov_out_valid = false;
  c->last_sp = sp;

  const size_t ev_iter0 = ev;
  double prevMod = lower, currMod = -1.0;
  int numIters = 0, auto_choice = 4;
  c->converged = 1;
  const int fold_grid = grid_for(c->lnv, 256, c->num_sms, 8);
  for (;;) {                                                   // dspl.hpp:1338
    if (numIters >= c->opt_max_iters) return fail("max_iters reached without convergence");
    numIters++;
    Acc *acc = c->acc.p + numIters;
    sp.cur = cur; sp.tgt = tgt; sp.acc = acc;
    cudaEvent_t e0 = get_event(c, ev++), e1 = get_event(c, ev++), e2 = get_event(c, ev++), e3 = get_event(c, ev++);
    CK(cudaEventRecord(e0, s));
    // iteration 1 of a simple graph: every community is a singleton (scan_pipe.cuh, FIRST)
    // Which persistent kernel?  k_scan_pq wins where the gathers hit L1 (RGG: 0.49 vs 0.60 ms per launch) and loses
    // badly where they do not (its single tail buffer exposes the bulk-copy latency: -p 2 graph, 1.40 vs 0.80 ms), and
    // that already shows in iteration 3.  scan_variant 6 (default) therefore measures: iterations 2 and 4 run
    // k_scan_pw, iteration 3 k_scan_pq, and from iteration 5 on k_scan_pq runs if its launch was faster than the
    // geometric mean of its two neighbours (scan times fall roughly geometrically there), else k_scan_pw.  Results
    // are identical either way; every rank decides for itself.
    c->scan_kernel = c->opt_scan_variant == 5 ? 5 : 4;
    if (c->opt_scan_variant == 6) {
      if (numIters == 3) c->scan_kernel = 5;
      else if (numIters >= 5) c->scan_kernel = auto_choice;
    }
    // (not on a warm run: its communities are not singletons; not with a movable set: the general reduction gives the
    // same decisions, and only it has a MASKED instantiation)
    TRY(launch_scan(c, sp, numIters == 1 && c->simple_sorted && c->opt_first_iter && c->opt_scan_variant >= 4 && !c->f32 && !c->warm_run &&
                               !c->mov_run, c->mov_run ? mov[k_cur] : nullptr));
    CK(cudaEventRecord(e1, s));
    if (frontier && c->lnv > 0) {
      // M_{k+1} from this scan's movers; the stores into peers' sets are ordered before their next scan by the barrier
      // below, like the remote Comm deltas
      k_frontier_mark<<<grid_for((c->lnv + 7) / 8, 256, c->num_sms), 256, 0, s>>>((int)c->lnv, c->a_rowptr, c->a_tails, cur, tgt, mov[k_cur],
                                                                                 mov[k_cur ^ 1], c->ghost_gid.p, c->pt, mp[k_cur ^ 1]);
      c->tm.kernel_launches++;
      CK(cudaGetLastError());
    }
    const bool p2p = c->nranks > 1 && c->opt_comm_mode == 1;
    if (c->nranks > 1) {
      // ghost values of the NEW assignment go into the ghost tail of every peer's tgt array; then "every scan has
      // finished" (its remote atomics and ghost stores included) must hold before any rank folds.
      if (p2p) {
        if (c->nsend) {
          k_push_ghosts<<<grid_for(c->nsend, 256, c->num_sms), 256, 0, s>>>(tgt, c->send_lid.p, c->nsend, c->push[tgt == c->comm_b.p ? 1 : 0]);
          c->tm.kernel_launches++;
        }
        k_p2p_barrier<<<1, 32, 0, s>>>(c->pp, ++c->p2p_epoch);
        c->tm.kernel_launches++;
      } else {
        TRY(exchange_ghosts(c, tgt));
        NK(g_nccl.AllReduce(dev_scalars(c)->counts, dev_scalars(c)->counts, 1, ncclInt64, ncclSum, c->comm, s));
      }
    }
    CK(cudaEventRecord(e2, s));
    if (c->unit) k_fold_unit<<<grid_for((c->lnv >> 2) + 1, 256, c->num_sms, 8), 256, 0, s>>>((int)c->lnv, c->cdeg.p, c->csize.p, c->upd.p, acc, acc - 1);
    else k_fold_w<<<fold_grid, 256, 0, s>>>((int)c->lnv, c->cinfo_w.p, c->usize.p, c->udeg.p, acc);
    c->tm.kernel_launches++;
    CK(cudaEventRecord(e3, s));
    TRY(acc_sum_enqueue(c, acc, c->opt_trace != 0));
    CK(cudaStreamSynchronize(s));
    AccSum sum;
    TRY(acc_sum_read(c, sum));
    if (c->opt_scan_variant == 6 && numIters == 4) {           // iterations 2..4 have completed (the stream was just synchronised)
      float t2 = 0, t3 = 0, t4 = 0;
      CK(cudaEventElapsedTime(&t2, c->events[ev_iter0 + 4 * 1], c->events[ev_iter0 + 4 * 1 + 1]));
      CK(cudaEventElapsedTime(&t3, c->events[ev_iter0 + 4 * 2], c->events[ev_iter0 + 4 * 2 + 1]));
      CK(cudaEventElapsedTime(&t4, c->events[ev_iter0 + 4 * 3], c->events[ev_iter0 + 4 * 3 + 1]));
      auto_choice = ((double)t3 * t3 < (double)t2 * t4) ? 5 : 4;
      c->tm.scan_kernel_chosen = auto_choice;
    }
    if (c->f32) {                      // GraphWeight = float: every product and the difference round to float
      const float cf = (float)c->constant;
      volatile float t1f = (float)sum.e * cf;
      volatile float t2af = (float)sum.a2 * cf;
      volatile float t2f = t2af * cf;
      volatile float df = t1f - t2f;
      currMod = (double)std::fabs(df);
    } else {
      currMod = std::fabs(modularity(sum.e, sum.a2, c->constant));
    }
    if (c->opt_trace) {
      mvgpu_iter_trace t;
      t.modularity = currMod; t.moved = (int64_t)sum.moved; t.chash = sum.hash;
      c->trace.push_back(t);
    }
    if (c->f32 ? ((float)currMod - (float)prevMod < (float)thresh) : (currMod - prevMod < thresh)) break;   // dspl.hpp:1401-1402
    prevMod = currMod;
    if (prevMod < lower) prevMod = lower;                      // dspl.hpp:1404-1406
    std::swap(cur, tgt);                                       // rotation (dspl.hpp:1408-1422) is a pointer swap
    if (frontier) k_cur ^= 1;                                  // M_{k+1} only for an accepted iteration
    if (c->opt_stop_after > 0 && numIters == c->opt_stop_after) { c->converged = 0; break; }   // checkpoint: resume with lower = prevMod
  }
  cudaEvent_t e_end = get_event(c, ev++);
  CK(cudaEventRecord(e_end, s));
  c->d_final = cur;
  c->final_ready = false;
  c->run_on_shard = c->final_on_shard = true;
  if (c->mov_run) {                                            // M_{k+1} in caller numbering, outside the timed region
    if (c->lnv > 0) {                                          // mov_out was sized in setup_run
      k_movable_out<<<grid_for(c->lnv, 256, c->num_sms), 256, 0, s>>>((int)c->lnv, mov[k_cur], c->relabel ? c->inv.p : nullptr, c->mov_out.p);
      CK(cudaGetLastError());
    }
    c->mov_out_valid = true;
  }
  if (c->nranks > 1) {
    // the assignment in the caller's numbering needs the label arrays of the PEERS (a community may be owned by another
    // rank): resolve it now, while every rank is still inside this call, and leave together -- afterwards a rank may
    // free its arrays (mvgpu_destroy) without a peer still reading them.  Outside the timed region, like the
    // reference's output code is outside its timer.
    TRY(final_in_caller_order(c));
    TRY(run_barrier(c));
    CK(cudaStreamSynchronize(s));
  }
  CK(cudaEventSynchronize(e_end));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e_begin, e_end)); c->tm.total_s = ms * 1e-3;
  CK(cudaEventElapsedTime(&ms, e_begin, e_setup)); c->tm.setup_s = ms * 1e-3;
  if (c->relabel && c->lnv > 0) { CK(cudaEventElapsedTime(&ms, c->events[2], c->events[3])); c->tm.reorder_s = ms * 1e-3; }
  c->tm.reordered = c->reordered ? 1 : 0;
  for (int k = 0; k < numIters; k++) {
    cudaEvent_t e0 = c->events[ev_iter0 + 4 * k], e1 = c->events[ev_iter0 + 4 * k + 1], e2 = c->events[ev_iter0 + 4 * k + 2],
                e3 = c->events[ev_iter0 + 4 * k + 3];
    CK(cudaEventElapsedTime(&ms, e0, e1)); c->tm.scan_s += ms * 1e-3; c->scan_times.push_back(ms * 1e-3);
    CK(cudaEventElapsedTime(&ms, e1, e2)); c->tm.exchange_s += ms * 1e-3;
    CK(cudaEventElapsedTime(&ms, e2, e3)); c->tm.fold_s += ms * 1e-3;
  }
  c->tm.iters = numIters;
  c->tm.h2d_s = c->h2d_s;
  c->tm.h2d_bytes = c->h2d_bytes;
  *iters_out = numIters;                                       // dspl.hpp:1430
  *mod_out = prevMod;                                          // dspl.hpp:1440
  return 0;
}

// currComm in the caller's vertex numbering, as labels (original global ids)
int final_in_caller_order(mvgpu_ctx *c) {
  if (c->final_ready) return 0;
  CK(cudaSetDevice(c->device));
  TRY(c->final_orig.ensure(c->lnv));
  c->final_ready = true;
  if (c->lnv == 0) return 0;
  const int32_t *perm = c->reordered ? c->perm.p : nullptr;
  if (c->nranks > 1) k_final_labels<true><<<grid_for(c->lnv, 256, c->num_sms), 256, 0, c->stream>>>((int)c->lnv, c->d_final, perm, c->last_sp, c->final_orig.p);
  else k_final_labels<false><<<grid_for(c->lnv, 256, c->num_sms), 256, 0, c->stream>>>((int)c->lnv, c->d_final, perm, c->last_sp, c->final_orig.p);
  CK(cudaGetLastError());
  return 0;
}

__global__ void k_widen(const int32_t *in, long long n, long long *out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = in[i];
}

// ---- caller arrays in host or device memory (DESIGN.md §3.16) -------------------------------------------------------
// The one range check of caller community ids, for both forms: ids[i] in [0, nv) narrowed to out[i]; *bad = the smallest
// i whose id lies outside (left at its preset ~0 when every id is good).
__global__ void __launch_bounds__(256) k_take_ids(const long long *ids, long long n, long long nv, int32_t *out,
                                                  unsigned long long *bad) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long v = ids[i];
    if (v < 0 || v >= nv) atomicMin(bad, (unsigned long long)i);
    out[i] = (int32_t)v;
  }
}

// a movable set as 0 / 1 (may run in place)
__global__ void __launch_bounds__(256) k_mask01(const uint8_t *in, long long n, uint8_t *out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = in[i] != 0;
}

// Where a caller's array lives.  Each pointer is classified on its own: pageable or pinned host memory takes the host
// form, device or managed memory of the context's device the device form.
enum class Where { Pageable, Pinned, Device };

// p's class in w; device memory of another device is refused: the message ("" if none) names the array as `name`
std::string locate(const mvgpu_ctx *c, const void *p, const char *name, Where &w) {
  w = Where::Pageable;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {   // not known to CUDA: plain host memory
    cudaGetLastError();
    return "";
  }
  if (a.type == cudaMemoryTypeHost) w = Where::Pinned;
  if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
    if (a.device != c->device)
      return std::string(name) + " is memory of device " + std::to_string(a.device) + ", the context's device is " +
             std::to_string(c->device);
    w = Where::Device;
  }
  return "";
}

// The one rule for moving a caller's bytes: device memory is used in place, pinned memory takes one copy, and pageable
// memory goes through the two pinned bounce buffers in chunks (instead of the driver's staged pageable copy),
// double-buffered in both directions (DESIGN.md §3.16).  bounce_ev[b] is recorded after every copy in or out of h_bounce[b], so
// waiting on it makes the buffer free to refill, whichever routine used it last.
constexpr size_t kBounce = 32u << 20;          // bytes per pinned bounce buffer

int bounce_buffers(mvgpu_ctx *c) {
  for (int b = 0; b < 2; b++) {
    if (!c->h_bounce[b]) CK(cudaMallocHost(&c->h_bounce[b], kBounce));
    if (!c->bounce_ev[b]) CK(cudaEventCreateWithFlags(&c->bounce_ev[b], cudaEventDisableTiming));
  }
  return 0;
}

// `bytes` of the caller's array src (class w) as the device reads them: dev = src for device memory, else a copy in
// staging (grown to fit).  Asynchronous on the context's stream: pageable memory may change once this returns, pinned
// and device memory once the stream has passed the copy (every entry point synchronises before it returns).
template <typename T>
int to_device(mvgpu_ctx *c, const void *src, size_t bytes, Where w, DevBuf<T> &staging, const T *&dev) {
  dev = static_cast<const T *>(src);
  if (w == Where::Device) return 0;
  TRY(staging.ensure((bytes + sizeof(T) - 1) / sizeof(T)));
  dev = staging.p;
  char *to = reinterpret_cast<char *>(staging.p);
  if (w == Where::Pinned) {
    CK(cudaMemcpyAsync(to, src, bytes, cudaMemcpyHostToDevice, c->stream));
    return 0;
  }
  if (bytes == 0) return 0;
  TRY(bounce_buffers(c));
  for (size_t off = 0, k = 0; off < bytes; k++) {
    const int b = k & 1;
    const size_t m = std::min(kBounce, bytes - off);
    CK(cudaEventSynchronize(c->bounce_ev[b]));
    memcpy(c->h_bounce[b], static_cast<const char *>(src) + off, m);
    CK(cudaMemcpyAsync(to + off, c->h_bounce[b], m, cudaMemcpyHostToDevice, c->stream));
    CK(cudaEventRecord(c->bounce_ev[b], c->stream));
    off += m;
  }
  return 0;
}

// `bytes` of device memory src -> the caller's array dst (class w).  Synchronous.
int to_caller(mvgpu_ctx *c, const void *src, size_t bytes, Where w, void *dst) {
  if (bytes == 0) return 0;
  cudaStream_t s = c->stream;
  if (w != Where::Pageable) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s));
    CK(cudaStreamSynchronize(s));
    return 0;
  }
  TRY(bounce_buffers(c));
  size_t at[2] = {0, 0}, pend[2] = {0, 0};     // per buffer: the chunk whose copy into it is in flight
  for (size_t off = 0, k = 0; off < bytes || pend[0] || pend[1]; k++) {
    const int b = k & 1;
    if (pend[b]) {                             // drain this buffer while the other buffer's copy is in flight
      CK(cudaEventSynchronize(c->bounce_ev[b]));
      memcpy(static_cast<char *>(dst) + at[b], c->h_bounce[b], pend[b]);
      pend[b] = 0;
    }
    if (off < bytes) {
      const size_t m = std::min(kBounce, bytes - off);
      CK(cudaMemcpyAsync(c->h_bounce[b], static_cast<const char *>(src) + off, m, cudaMemcpyDeviceToHost, s));
      CK(cudaEventRecord(c->bounce_ev[b], s));
      at[b] = off; pend[b] = m;
      off += m;
    }
  }
  return 0;
}

// The caller's lnv community ids (host or device memory, named `name` in a refusal) as int32 in dst, on the device.  A
// finding goes into err ("" if none), prefixed by `who`: a refused pointer, or the smallest local index with an id
// outside [0, nv) and that id.  The return value reports CUDA failures only.  Synchronous: the ids are read before it
// returns.
int take_ids(mvgpu_ctx *c, const int64_t *ids, const char *who, const char *name, int32_t *dst, std::string &err) {
  Where w;
  err = locate(c, ids, name, w);
  if (!err.empty()) {
    err = std::string(who) + ": " + err;
    return 0;
  }
  const long long n = c->lnv;
  if (n == 0) return 0;
  cudaStream_t s = c->stream;
  const long long *src;
  TRY(to_device(c, ids, sizeof(long long) * n, w, c->wide, src));
  TRY(c->take_bad.ensure(1));
  CK(cudaMemsetAsync(c->take_bad.p, 0xff, sizeof(unsigned long long), s));
  k_take_ids<<<grid_for(n, 256, c->num_sms), 256, 0, s>>>(src, n, c->nv_global, dst, c->take_bad.p);
  CK(cudaGetLastError());
  unsigned long long bad = 0;
  CK(cudaMemcpyAsync(&bad, c->take_bad.p, sizeof bad, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad < (unsigned long long)n) {
    long long v = 0;
    CK(cudaMemcpyAsync(&v, src + bad, sizeof v, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    err = std::string(who) + ": community id " + std::to_string(v) + " of local vertex " + std::to_string(bad) +
          " outside [0, nv)";
  }
  return 0;
}

// lnv int32 ids on the device -> the caller's int64 array (class w): widened straight into device memory, or into wide
// and from there to host memory.  Synchronous.
int put_ids(mvgpu_ctx *c, const int32_t *src, int64_t *out, Where w) {
  const long long n = c->lnv;
  if (n == 0) return 0;
  long long *dst = reinterpret_cast<long long *>(out);
  if (w != Where::Device) {
    TRY(c->wide.ensure(n));
    dst = c->wide.p;
  }
  k_widen<<<grid_for(n, 256, c->num_sms), 256, 0, c->stream>>>(src, n, dst);
  CK(cudaGetLastError());
  if (w != Where::Device) return to_caller(c, dst, sizeof(long long) * n, w, out);
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

// The output arrays of a call (NULL ones skipped): the first refusal, "" if none; their classes in w
std::string locate_all(const mvgpu_ctx *c, int n, const void *const *p, const char *const *name, Where *w) {
  for (int k = 0; k < n; k++) {
    w[k] = Where::Pageable;
    if (!p[k]) continue;
    const std::string e = locate(c, p[k], name[k], w[k]);
    if (!e.empty()) return e;
  }
  return "";
}

// What the getters and mv_layout_readback report about the last run.  setup_run overwrites these, so an evaluation
// keeps a copy and puts it back.
struct RunReport {
  mvgpu_timings tm;
  LayoutReport lay;
  double constant;
  bool reordered, simple_sorted, unit, warm_run;
  int relabel;
};
RunReport save_report(const mvgpu_ctx *c) {
  return {c->tm, c->lay, c->constant, c->reordered, c->simple_sorted, c->unit, c->warm_run, c->relabel};
}
void restore_report(mvgpu_ctx *c, const RunReport &r) {
  c->tm = r.tm; c->lay = r.lay; c->constant = r.constant; c->reordered = r.reordered; c->simple_sorted = r.simple_sorted;
  c->unit = r.unit; c->warm_run = r.warm_run; c->relabel = r.relabel;
}

// ---- evaluation (DESIGN.md §3.10): after setup_run(ev), comm_a = X on every slot and the Comm records are X's -------
int evaluate_pass(mvgpu_ctx *c, const int32_t *X, mvgpu_quality *out) {
  cudaStream_t s = c->stream;
  const int lnv = (int)c->lnv, nsm = c->num_sms;
  Scalars *d_sc = dev_scalars(c);
  Acc *acc0 = c->acc.p;                        // warm_init left a2 (unit path) in record 0; e_in joins it there
  if (!c->unit) {                              // the update arrays are zero after the warm fold: this only sums a_c^2
    k_fold_w<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->cinfo_w.p, c->usize.p, c->udeg.p, acc0);
    c->tm.kernel_launches++;
  }
  if (c->unit)
    k_q_internal<true><<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->a_rowptr, c->a_tails, nullptr, c->comm_a.p, c->pt, c->qp, acc0);
  else
    k_q_internal<false><<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->a_rowptr, c->a_tails, c->a_weights, c->comm_a.p, c->pt, c->qp, acc0);
  c->tm.kernel_launches++;
  TRY(run_barrier(c));                         // every rank's internal-weight adds have landed in the owners' records
  // e_in and a2, summed over the ranks in rank order like the run's modularity partials
  TRY(acc_sum_enqueue(c, acc0, false));
  // per-community arrays, non-empty flags in owned slot order (= caller id order: no renumbering), their exclusive sum
  TRY(c->q_flag.ensure(lnv + 1)); TRY(c->q_size.ensure(lnv)); TRY(c->q_vol.ensure(lnv)); TRY(c->q_lab.ensure(lnv));
  CK(cudaMemsetAsync(d_sc->q_agg, 0, sizeof d_sc->q_agg, s));
  if (c->unit)
    k_q_stats<true><<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->cdeg.p, c->csize.p, nullptr, c->q_internal.p, c->q_size.p, c->q_vol.p,
                                                            c->q_flag.p, d_sc->q_agg);
  else
    k_q_stats<false><<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, nullptr, nullptr, c->cinfo_w.p, c->q_internal.p, c->q_size.p, c->q_vol.p,
                                                             c->q_flag.p, d_sc->q_agg);
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::ExclusiveSum(t, tb, c->q_flag.p, c->q_rank.p, lnv + 1, s); }));
  c->tm.kernel_launches += 2;
  int32_t nonempty = 0;
  unsigned long long agg[2];
  CK(cudaMemcpyAsync(&nonempty, c->q_rank.p + lnv, sizeof nonempty, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(agg, d_sc->q_agg, sizeof agg, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  AccSum sum;
  TRY(acc_sum_read(c, sum));
  // rank offsets of the compact labels: every rank's {non-empty, singletons, largest}; each rank's prefix sum is
  // complete before it contributes, so the owners' arrays are final when the gather below reads them
  std::vector<long long> all(3 * (size_t)c->nranks);
  const long long mine[3] = {nonempty, (long long)agg[0], (long long)agg[1]};
  if (c->nranks > 1) TRY(coll_allgather(c, mine, all.data(), sizeof mine));
  else std::copy(mine, mine + 3, all.begin());
  long long communities = 0, singletons = 0, max_size = 0;
  for (int r = 0; r < c->nranks; r++) {
    c->qp.off[r] = communities;
    communities += all[3 * r]; singletons += all[3 * r + 1]; max_size = std::max(max_size, all[3 * r + 2]);
  }
  if (lnv > 0) {
    k_q_labels<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, X, c->pt, c->qp, c->q_lab.p);
    c->tm.kernel_launches++;
  }
  if (c->nranks > 1) {                         // no rank leaves while a peer still reads its prefix sums
    TRY(run_barrier(c));
    CK(cudaStreamSynchronize(s));
  }
  CK(cudaGetLastError());
  out->modularity = modularity(sum.e, sum.a2, c->constant);   // run_louvain's rounding, without the fabs
  out->e_in = sum.e; out->a2 = sum.a2; out->constant = c->constant;
  out->communities = communities; out->singletons = singletons; out->max_size = max_size;
  c->eval_on_shard = true;
  return 0;
}

// The assignment an evaluation or a split reads: comm (validated and narrowed into eval_comm) or, for NULL, the last run's
// result in caller order (resolved by the caller of this).  Local findings are not returned here: they go into ev.err,
// prefixed by `who`, and join setup_run's input agreement, so that every rank fails together.  caller_err: a finding of
// the caller's own (a binding that could not build the array), which fails the call on every rank like a bad id.
int take_assignment(mvgpu_ctx *c, const int64_t *comm, const char *who, const char *verb, const char *caller_err, EvalSetup &ev) {
  const std::string w(who);
  ev.given = comm != nullptr;
  if (caller_err) ev.err = w + ": " + caller_err;
  else if (c->f32) ev.err = w + ": not for a shard uploaded with mvgpu_upload_shard32";
  else if (!comm && !c->run_on_shard) ev.err = w + ": NULL " + verb + " the last mvgpu_louvain result, and there is none on this shard";
  else if (comm) {
    TRY(c->eval_comm.ensure(c->lnv));
    TRY(take_ids(c, comm, who, "comm", c->eval_comm.p, ev.err));
    if (ev.err.empty()) ev.X = c->eval_comm.p;
  } else {
    ev.X = c->final_orig.p;
  }
  return 0;
}

// setup_run(ev), then pass(), between two events on the stream (seconds: the device time between them); leaves
// everything the last run reports as it was
template <typename F>
int assignment_pass(mvgpu_ctx *c, const EvalSetup &ev, F &&pass, double &seconds) {
  cudaStream_t s = c->stream;
  const RunReport saved = save_report(c);
  memset(&c->tm, 0, sizeof c->tm);
  c->peers_ready = false;                      // the evaluation's tables differ from the run's (no labels, q arrays)
  cudaEvent_t e0 = get_event(c, 0), e1 = get_event(c, 1);
  int rc = cudaEventRecord(e0, s) == cudaSuccess ? 0 : fail("cudaEventRecord");
  if (!rc) rc = setup_run(c, &ev);
  if (!rc) rc = pass();
  if (!rc && cudaEventRecord(e1, s) != cudaSuccess) rc = fail("cudaEventRecord");
  if (!rc && cudaEventSynchronize(e1) != cudaSuccess) rc = fail("cudaEventSynchronize");
  float ms = 0;
  if (!rc && cudaEventElapsedTime(&ms, e0, e1) != cudaSuccess) rc = fail("cudaEventElapsedTime");
  if (!rc) seconds = ms * 1e-3;
  restore_report(c, saved);
  c->peers_ready = false;                      // the next run rebuilds its own tables
  return rc;
}

// collective: every rank calls it with an array or every rank with NULL
int evaluate(mvgpu_ctx *c, const int64_t *comm, mvgpu_quality *out, const char *caller_err = nullptr) {
  TRY(check_ready(c));
  CK(cudaSetDevice(c->device));
  c->eval_on_shard = false;                    // the q_* arrays are rewritten from here on
  // The last run's assignment in caller order is resolved while comm_a / comm_b still hold it (one-rank runs leave it
  // unresolved; setup_run below overwrites comm_a), whatever is evaluated: communities(), get_communities_device and a
  // later NULL evaluation read final_orig, which an evaluation never writes.
  if (c->run_on_shard) TRY(final_in_caller_order(c));
  EvalSetup ev;
  TRY(take_assignment(c, comm, "mvgpu_evaluate_communities", "evaluates", caller_err, ev));
  return assignment_pass(c, ev, [&] { return evaluate_pass(c, ev.X, out); }, out->eval_s);
}

// ---- splitting (DESIGN.md §3.12): after setup_run(ev), comm_a = X on every slot; the labels end in split_lab ----------
// Labels only decrease, so the loop ends; the cap turns a defect into an error instead of a hang.
constexpr int kSplitMaxRounds = 1000;

int split_pass(mvgpu_ctx *c, mvgpu_split_report *rep) {
  cudaStream_t s = c->stream;
  const int lnv = (int)c->lnv, nsm = c->num_sms;
  Scalars *d_sc = dev_scalars(c);
  Acc *acc = c->acc.p + 1;                     // one record, cleared every round (record 0 holds the warm fold's a2)
  if (lnv > 0) {
    k_split_init<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->base, c->split_lab.p);
    c->tm.kernel_launches++;
  }
  TRY(run_barrier(c));                         // every rank's labels are set before a peer reads or lowers them
  int rounds = 0;
  for (;;) {
    if (rounds == kSplitMaxRounds)
      return fail("mvgpu_split_communities: labels still changing after " + std::to_string(kSplitMaxRounds) + " rounds");
    rounds++;
    CK(cudaMemsetAsync(acc, 0, sizeof(Acc), s));
    if (c->lne > 0) {
      k_split_hook<<<grid_for(c->lne, 256, nsm), 256, 0, s>>>(lnv, c->base, c->a_rowptr, c->a_tails, c->comm_a.p, c->ghost_gid.p,
                                                              c->split_lab.p, c->pt, c->spp, acc);
      c->tm.kernel_launches++;
    }
    TRY(run_barrier(c));                       // the round's hooks have landed on every rank before labels jump
    if (lnv > 0) {
      k_split_jump<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->base, c->split_lab.p, c->pt, c->spp, acc);
      c->tm.kernel_launches++;
    }
    TRY(acc_sum_enqueue(c, acc, true));        // labels lowered this round, summed over the ranks (acc->moved)
    CK(cudaStreamSynchronize(s));
    AccSum sum;
    TRY(acc_sum_read(c, sum));
    if (sum.moved == 0) break;                 // the same on every rank: every rank leaves the loop after this round
  }
  if (lnv > 0) {
    k_split_roots<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->base, c->comm_a.p, c->split_lab.p, c->pt, c->qp);
    c->tm.kernel_launches++;
  }
  // every root has been counted at its community's owner; from here on no rank touches a peer's arrays, so each may
  // leave the call when it is done
  TRY(run_barrier(c));
  CK(cudaMemsetAsync(d_sc->split_agg, 0, sizeof d_sc->split_agg, s));
  if (lnv > 0) {
    k_split_count<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, reinterpret_cast<const unsigned long long *>(c->q_internal.p),
                                                          d_sc->split_agg);
    c->tm.kernel_launches++;
  }
  unsigned long long agg[3];
  CK(cudaMemcpyAsync(agg, d_sc->split_agg, sizeof agg, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  long long tot[3] = {(long long)agg[0], (long long)agg[1], (long long)agg[2]};
  TRY(coll_allreduce_i64(c, tot, 3, false));
  rep->communities = tot[0]; rep->components = tot[1]; rep->disconnected = tot[2]; rep->rounds = rounds;
  return 0;
}

// collective like evaluate; out is written only when the call succeeds
int split(mvgpu_ctx *c, const int64_t *comm, int64_t *out, mvgpu_split_report *rep, const char *caller_err = nullptr) {
  TRY(check_ready(c));
  CK(cudaSetDevice(c->device));
  c->eval_on_shard = false;                    // the split counts components in the evaluation's q_internal
  if (c->run_on_shard) TRY(final_in_caller_order(c));   // as in evaluate: setup_run overwrites comm_a
  EvalSetup ev;
  ev.split = true;
  Where w;
  const std::string out_err = locate(c, out, "out", w);   // a refused output fails every rank, like a bad id
  TRY(take_assignment(c, comm, "mvgpu_split_communities", "splits", caller_err ? caller_err : out_err.empty() ? nullptr : out_err.c_str(), ev));
  mvgpu_split_report r;
  memset(&r, 0, sizeof r);
  TRY(assignment_pass(c, ev, [&] { return split_pass(c, &r); }, r.split_s));
  TRY(put_ids(c, c->split_lab.p, out, w));
  *rep = r;
  return 0;
}

// ---- probing (DESIGN.md §3.15, probe_gpu.cuh): after setup_run(ev), comm_a = X on every slot and the Comm records are
// X's, so the scan's per-vertex rule reads exactly what iteration 1 of a warm run from X reads
template <bool UNIT, bool MULTI>
int launch_probe_t(mvgpu_ctx *c, const ScanParams &sp, const ProbeOut &o) {
  const int tiles = (int)((c->lnv + kTileV - 1) / kTileV);
  if (tiles > 0) {
    k_probe<UNIT, MULTI><<<tiles, kTileV, UNIT ? sizeof(int32_t) * kECap : (sizeof(int32_t) + sizeof(double)) * kECap, c->stream>>>(sp, o);
    c->tm.kernel_launches++;
  }
  if (c->nheavy > 0) {
    k_probe_heavy<UNIT, MULTI><<<(int)c->nheavy, 256, 0, c->stream>>>(sp, o);
    c->tm.kernel_launches++;
  }
  CK(cudaGetLastError());
  return 0;
}

int probe_pass(mvgpu_ctx *c, mvgpu_probe_report &rep) {
  cudaStream_t s = c->stream;
  Scalars *d_sc = dev_scalars(c);               // probe_agg was zeroed with the other scalars at the start of setup_run
  TRY(c->probe_tgt.ensure(c->lnv)); TRY(c->probe_best.ensure(c->lnv)); TRY(c->probe_gain.ensure(c->lnv));
  ScanParams sp = scan_params(c);
  sp.cur = c->comm_a.p;
  const ProbeOut o = {c->probe_tgt.p, c->probe_best.p, c->probe_gain.p, d_sc->probe_agg};
  const bool multi = c->nranks > 1;
  int (*launch)(mvgpu_ctx *, const ScanParams &, const ProbeOut &) =
      c->unit ? (multi ? launch_probe_t<true, true> : launch_probe_t<true, false>)
              : (multi ? launch_probe_t<false, true> : launch_probe_t<false, false>);
  TRY(launch(c, sp, o));
  unsigned long long agg[4];
  CK(cudaMemcpyAsync(agg, d_sc->probe_agg, sizeof agg, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  // every rank's kernels have finished (and stopped reading its peers' Comm records) once these collectives return
  long long n[3] = {(long long)agg[0], (long long)agg[1], (long long)agg[2]};
  TRY(coll_allreduce_i64(c, n, 3, false));
  long long kmax = (long long)(agg[3] ^ (1ULL << 63));   // unsigned key order as signed order
  TRY(coll_allreduce_i64(c, &kmax, 1, true));
  const unsigned long long key = (unsigned long long)kmax ^ (1ULL << 63);
  const unsigned long long bits = (key >> 63) ? (key & ~(1ULL << 63)) : ~key;
  double g;
  memcpy(&g, &bits, sizeof g);
  rep.vertices = c->nv_global;
  rep.moves = n[0]; rep.vetoed = n[1]; rep.interior = n[2];
  rep.max_gain = key ? g : -INFINITY;
  rep.constant = c->constant;
  return 0;
}

// collective like evaluate; target / best / gain are written only when the call succeeds
int probe(mvgpu_ctx *c, const int64_t *comm, int64_t *target, int64_t *best, double *gain, mvgpu_probe_report *rep,
          const char *caller_err = nullptr) {
  TRY(check_ready(c));
  CK(cudaSetDevice(c->device));
  if (c->run_on_shard) TRY(final_in_caller_order(c));   // as in evaluate: setup_run overwrites comm_a
  EvalSetup ev;
  ev.probe = true;
  const void *outs[3] = {target, best, gain};
  const char *names[3] = {"target", "best", "gain"};
  Where w[3];
  const std::string out_err = locate_all(c, 3, outs, names, w);   // a refused output fails every rank, like a bad id
  TRY(take_assignment(c, comm, "mvgpu_probe_communities", "probes", caller_err ? caller_err : out_err.empty() ? nullptr : out_err.c_str(), ev));
  mvgpu_probe_report r;
  memset(&r, 0, sizeof r);
  TRY(assignment_pass(c, ev, [&] { return probe_pass(c, r); }, r.probe_s));
  if (target) TRY(put_ids(c, c->probe_tgt.p, target, w[0]));
  if (best) TRY(put_ids(c, c->probe_best.p, best, w[1]));
  if (gain) TRY(to_caller(c, c->probe_gain.p, sizeof(double) * c->lnv, w[2], gain));
  *rep = r;
  return 0;
}

// ---- comparing two assignments (DESIGN.md §3.13, compare_gpu.cuh) ---------------------------------------------------
// Values of a histogram sum to at most N < 2^31, so it has fewer than sqrt(2N) < 65536 distinct positive values: one
// rank's list (with the value 0 at most once more) always fits this many entries.
constexpr int kCmpHist = 65536;

// where the keys of a sorted array go: those whose top bits (key >> shift) rank r owns go to r.  Counts and offsets
// (nranks + 1 of them) both ways.
struct CmpRoute {
  std::vector<long long> scount, soff, rcount, roff;
};

int cmp_route(mvgpu_ctx *c, const unsigned long long *sorted, long long n, int shift, CmpRoute &rt) {
  const int nr = c->nranks;
  CmpParts parts;
  parts.n = nr;
  for (int r = 0; r <= nr; r++) parts.p[r] = c->parts[r];
  TRY(c->cmp_off.ensure(nr + 1));
  k_cmp_bounds<<<1, 32, 0, c->stream>>>(sorted, n, parts, shift, c->cmp_off.p);
  CK(cudaGetLastError());
  rt.soff.assign(nr + 1, 0);
  CK(cudaMemcpyAsync(rt.soff.data(), c->cmp_off.p, sizeof(long long) * (nr + 1), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  rt.scount.assign(nr, 0);
  for (int r = 0; r < nr; r++) rt.scount[r] = rt.soff[r + 1] - rt.soff[r];
  std::vector<long long> all(rt.scount);
  if (nr > 1) {
    all.resize((size_t)nr * nr);
    TRY(coll_allgather(c, rt.scount.data(), all.data(), sizeof(long long) * nr));
  }
  rt.rcount.assign(nr, 0);
  rt.roff.assign(nr + 1, 0);
  for (int r = 0; r < nr; r++) {
    rt.rcount[r] = all[(size_t)r * nr + c->rank];
    rt.roff[r + 1] = rt.roff[r] + rt.rcount[r];
  }
  return 0;
}

// send -> recv along rt (back: the reverse way, into an array laid out like the sending side).  The all-to-all moves
// the other ranks' segments only: this rank's own segment is copied on the device.
int cmp_move(mvgpu_ctx *c, const void *send, void *recv, const CmpRoute &rt, size_t elem, bool back) {
  const std::vector<long long> &sc = back ? rt.rcount : rt.scount, &so = back ? rt.roff : rt.soff;
  const std::vector<long long> &rc = back ? rt.scount : rt.rcount, &ro = back ? rt.soff : rt.roff;
  const int me = c->rank;
  if (sc[me])
    CK(cudaMemcpyAsync((unsigned char *)recv + ro[me] * elem, (const unsigned char *)send + so[me] * elem, sc[me] * elem,
                       cudaMemcpyDeviceToDevice, c->stream));
  if (c->nranks > 1) TRY(coll_alltoallv_dev(c, send, sc, so, recv, rc, ro, elem));
  return 0;
}

int cmp_read_n(mvgpu_ctx *c, long long &n) {
  int v = 0;
  CK(cudaMemcpyAsync(&v, c->cmp_n.p, sizeof v, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  n = v;
  return 0;
}

// The n keys in cmp_k0 (unsorted, each below 2^key_bits) -> the distinct keys whose top bits (key >> shift) this rank
// owns, ascending, in okey, with their number of occurrences over all ranks in ocnt; nout of them.  Every rank sorts and
// run-length encodes its own keys first, so a key travels to its owner at most once per rank.
int cmp_reduce(mvgpu_ctx *c, long long n, int key_bits, int shift, DevBuf<unsigned long long> &okey, DevBuf<uint32_t> &ocnt,
               long long &nout) {
  cudaStream_t s = c->stream;
  const bool one = c->nranks == 1;             // one rank owns every key: the local runs are the answer
  TRY(c->cmp_k1.ensure(n));
  DevBuf<unsigned long long> &uk = one ? okey : c->cmp_k2;
  DevBuf<uint32_t> &uc = one ? ocnt : c->cmp_c0;
  TRY(uk.ensure(n)); TRY(uc.ensure(n));
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortKeys(t, tb, c->cmp_k0.p, c->cmp_k1.p, n, 0, key_bits, s); },
              [&](void *t, size_t &tb) { return cub::DeviceRunLengthEncode::Encode(t, tb, c->cmp_k1.p, uk.p, uc.p, c->cmp_n.p, n, s); }));
  long long runs = 0;
  TRY(cmp_read_n(c, runs));
  if (one) { nout = runs; return 0; }
  CmpRoute rt;
  TRY(cmp_route(c, uk.p, runs, shift, rt));
  const long long m = rt.roff[c->nranks];
  TRY(c->cmp_k0.ensure(m)); TRY(c->cmp_k1.ensure(m)); TRY(c->cmp_c1.ensure(m)); TRY(c->cmp_c2.ensure(m));
  TRY(okey.ensure(m)); TRY(ocnt.ensure(m));
  TRY(cmp_move(c, uk.p, c->cmp_k0.p, rt, sizeof(unsigned long long), false));
  TRY(cmp_move(c, uc.p, c->cmp_c1.p, rt, sizeof(uint32_t), false));
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortPairs(t, tb, c->cmp_k0.p, c->cmp_k1.p, c->cmp_c1.p, c->cmp_c2.p, m, 0, key_bits, s); },
              [&](void *t, size_t &tb) { return cub::DeviceReduce::ReduceByKey(t, tb, c->cmp_k1.p, okey.p, c->cmp_c2.p, ocnt.p, c->cmp_n.p, CmpSum(), m, s); }));
  return cmp_read_n(c, nout);
}

// The histogram of the n values in vals (each <= nv < 2^vbits) as kCmpHist entries value << 32 | multiplicity,
// ascending value, zero-padded
int cmp_hist(mvgpu_ctx *c, const uint32_t *vals, long long n, int vbits, std::vector<unsigned long long> &h) {
  cudaStream_t s = c->stream;
  TRY(c->cmp_c1.ensure(n)); TRY(c->cmp_hv.ensure(n)); TRY(c->cmp_hm.ensure(n));
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortKeys(t, tb, vals, c->cmp_c1.p, n, 0, vbits, s); },
              [&](void *t, size_t &tb) { return cub::DeviceRunLengthEncode::Encode(t, tb, c->cmp_c1.p, c->cmp_hv.p, c->cmp_hm.p, c->cmp_n.p, n, s); }));
  long long runs = 0;
  TRY(cmp_read_n(c, runs));
  if (runs > kCmpHist) return fail("mvgpu_compare_communities: a histogram with more than 65536 distinct values (counts do not sum to N)");
  std::vector<uint32_t> v((size_t)runs), m((size_t)runs);
  if (runs) {
    CK(cudaMemcpyAsync(v.data(), c->cmp_hv.p, sizeof(uint32_t) * runs, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(m.data(), c->cmp_hm.p, sizeof(uint32_t) * runs, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  h.assign(kCmpHist, 0);
  for (long long i = 0; i < runs; i++) h[i] = (unsigned long long)v[i] << 32 | m[i];
  return 0;
}

// A histogram merged over the ranks: the number of non-zero counts, sum C(k, 2), and S = sum over k > 1, in ascending
// k, of m * (k * log k).  The merged histogram does not depend on how the vertices are sharded, so neither does S.
struct CmpHist {
  long long nonzero = 0;
  unsigned long long pairs = 0;
  double s = 0.0;
};

int cmp_merge(mvgpu_ctx *c, const std::vector<unsigned long long> &mine, CmpHist &out) {
  std::vector<unsigned long long> all(mine);
  if (c->nranks > 1) {
    all.resize((size_t)kCmpHist * c->nranks);
    TRY(coll_allgather(c, mine.data(), all.data(), sizeof(unsigned long long) * kCmpHist));
  }
  std::map<unsigned long long, unsigned long long> h;
  for (unsigned long long e : all)
    if (e >> 32) h[e >> 32] += e & 0xffffffffULL;        // value 0 (empty slots, padding) counts nothing
  out = CmpHist();
  for (const auto &[k, m] : h) {
    out.nonzero += (long long)m;
    out.pairs += m * (k * (k - 1) / 2);
    if (k > 1) out.s += (double)m * ((double)k * std::log((double)k));
  }
  return 0;
}

// X, Y: this rank's lnv caller ids on the device -> rep's counts (not compare_s) and the matches in cmp_match
int compare_pass(mvgpu_ctx *c, const int32_t *X, const int32_t *Y, mvgpu_compare_report &rep) {
  cudaStream_t s = c->stream;
  const int lnv = (int)c->lnv, nsm = c->num_sms;
  const long long nv = c->nv_global, base = c->base;
  int shift = 1, vbits = 1;
  while ((1LL << shift) < nv) shift++;         // every id < 2^shift
  while ((1LL << vbits) <= nv) vbits++;        // every count <= nv < 2^vbits
  TRY(c->cmp_n.ensure(1)); TRY(c->cmp_k0.ensure(lnv));
  // the cells n_xy of the owned x, and the sizes b_y of the owned y
  long long ncell = 0, ny = 0, nrows = 0;
  if (lnv) k_cmp_keys<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, X, Y, shift, c->cmp_k0.p);
  CK(cudaGetLastError());
  TRY(cmp_reduce(c, lnv, 2 * shift, shift, c->cmp_cell_k, c->cmp_cell_c, ncell));
  if (lnv) k_cmp_keys<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, nullptr, Y, 0, c->cmp_k0.p);
  CK(cudaGetLastError());
  TRY(cmp_reduce(c, lnv, shift, 0, c->cmp_y_k, c->cmp_y_c, ny));
  // rows: a_x and the best match of every owned non-empty x (the cells are sorted by x, so its cells are consecutive)
  TRY(c->cmp_i0.ensure(ncell)); TRY(c->cmp_i1.ensure(ncell)); TRY(c->cmp_row0.ensure(ncell)); TRY(c->cmp_row1.ensure(ncell));
  TRY(c->cmp_match.ensure(4 * (size_t)lnv));
  if (lnv) k_cmp_match_init<<<grid_for(lnv, 256, nsm), 256, 0, s>>>(lnv, c->cmp_match.p);
  if (ncell) k_cmp_cell_rows<<<grid_for(ncell, 256, nsm), 256, 0, s>>>(ncell, c->cmp_cell_k.p, c->cmp_cell_c.p, shift, base, c->cmp_i0.p,
                                                                         c->cmp_row0.p);
  CK(cudaGetLastError());
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceReduce::ReduceByKey(t, tb, c->cmp_i0.p, c->cmp_i1.p, c->cmp_row0.p, c->cmp_row1.p,
                                                                                   c->cmp_n.p, CmpRowOp(), ncell, s); }));
  TRY(cmp_read_n(c, nrows));
  TRY(c->cmp_c0.ensure(nrows)); TRY(c->cmp_k0.ensure(nrows)); TRY(c->cmp_k1.ensure(nrows)); TRY(c->cmp_c2.ensure(nrows));
  // the rows' sizes -> cmp_c0, their best-size requests (best y, asking slot) -> cmp_k0 / cmp_i0
  if (nrows) k_cmp_rows<<<grid_for(nrows, 256, nsm), 256, 0, s>>>((int)nrows, lnv, c->cmp_i1.p, c->cmp_row1.p, c->cmp_match.p, c->cmp_c0.p,
                                                                    c->cmp_k0.p, c->cmp_i0.p);
  TRY(c->cmp_b.ensure(lnv));
  CK(cudaMemsetAsync(c->cmp_b.p, 0, sizeof(uint32_t) * lnv, s));
  if (ny) k_cmp_scatter_b<<<grid_for(ny, 256, nsm), 256, 0, s>>>(ny, c->cmp_y_k.p, c->cmp_y_c.p, base, c->cmp_b.p);
  CK(cudaGetLastError());
  // best_size: requests sorted by y are grouped by owner; the owner answers b_y in request order
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortPairs(t, tb, c->cmp_k0.p, c->cmp_k1.p, c->cmp_i0.p, c->cmp_i1.p,
                                                                                    nrows, 0, shift, s); }));
  CmpRoute rt;
  TRY(cmp_route(c, c->cmp_k1.p, nrows, 0, rt));
  const long long nreq = rt.roff[c->nranks];
  TRY(c->cmp_k2.ensure(nreq)); TRY(c->cmp_c1.ensure(nreq));
  TRY(cmp_move(c, c->cmp_k1.p, c->cmp_k2.p, rt, sizeof(unsigned long long), false));
  if (nreq) k_cmp_lookup<<<grid_for(nreq, 256, nsm), 256, 0, s>>>(nreq, c->cmp_k2.p, base, c->cmp_b.p, c->cmp_c1.p);
  CK(cudaGetLastError());
  TRY(cmp_move(c, c->cmp_c1.p, c->cmp_c2.p, rt, sizeof(uint32_t), true));
  if (nrows) k_cmp_best_size<<<grid_for(nrows, 256, nsm), 256, 0, s>>>(nrows, c->cmp_i1.p, c->cmp_c2.p, lnv, c->cmp_match.p);
  CK(cudaGetLastError());
  // histograms of the cells, of a and of b, merged over the ranks
  std::vector<unsigned long long> h;
  CmpHist hxy, hx, hy;
  TRY(cmp_hist(c, c->cmp_cell_c.p, ncell, vbits, h)); TRY(cmp_merge(c, h, hxy));
  TRY(cmp_hist(c, c->cmp_c0.p, nrows, vbits, h)); TRY(cmp_merge(c, h, hx));
  TRY(cmp_hist(c, c->cmp_y_c.p, ny, vbits, h)); TRY(cmp_merge(c, h, hy));
  // the report, from the merged integers in a fixed order: the same bits on every rank count
  const unsigned long long all = (unsigned long long)nv * (unsigned long long)(nv > 0 ? nv - 1 : 0) / 2;
  rep.vertices = nv; rep.communities_x = hx.nonzero; rep.communities_y = hy.nonzero; rep.cells = hxy.nonzero;
  rep.pairs_xy = hxy.pairs; rep.pairs_x = hx.pairs; rep.pairs_y = hy.pairs; rep.pairs_all = all;
  const __int128 A = all, P = hxy.pairs, PX = hx.pairs, PY = hy.pairs;
  const __int128 num = 2 * (A * P - PX * PY), den = A * (PX + PY) - 2 * PX * PY;
  rep.ari = den == 0 ? 1.0 : (double)num / (double)den;
  rep.rand = all == 0 ? 1.0 : (double)(A + 2 * P - PX - PY) / (double)A;
  const double n = (double)nv;
  rep.h_x = rep.communities_x <= 1 ? 0.0 : std::log(n) - hx.s / n;
  rep.h_y = rep.communities_y <= 1 ? 0.0 : std::log(n) - hy.s / n;
  rep.mi = (rep.communities_x <= 1 || rep.communities_y <= 1) ? 0.0 : std::log(n) + (hxy.s - (hx.s + hy.s)) / n;
  rep.nmi = (rep.h_x + rep.h_y == 0.0) ? 1.0 : (2.0 * rep.mi) / (rep.h_x + rep.h_y);
  rep.vi = (rep.h_x + rep.h_y) - 2.0 * rep.mi;
  return 0;
}

// collective: every rank passes x or every rank NULL; y is never NULL.  rep and the matches are written only when the
// call succeeds.  Reads no edge and none of the run's or the evaluation's arrays.
int compare(mvgpu_ctx *c, const int64_t *x, const int64_t *y, mvgpu_compare_report *rep, const char *caller_err = nullptr) {
  c->cmp_on_shard = false;                     // a failed call leaves no matches behind
  TRY(check_ready(c));
  CK(cudaSetDevice(c->device));
  const std::string who = "mvgpu_compare_communities";
  std::string err;
  const long long lnv = c->lnv;
  if (caller_err) err = who + ": " + caller_err;
  else if (c->f32) err = who + ": not for a shard uploaded with mvgpu_upload_shard32";
  else if (!y) err = who + ": y must not be NULL";
  else if (!x && !c->run_on_shard) err = who + ": NULL x compares the last mvgpu_louvain result, and there is none on this shard";
  else {
    TRY(c->cmp_x.ensure(lnv)); TRY(c->cmp_y.ensure(lnv));
    if (x) TRY(take_ids(c, x, who.c_str(), "x", c->cmp_x.p, err));
    if (err.empty()) TRY(take_ids(c, y, who.c_str(), "y", c->cmp_y.p, err));
  }
  // the call's first collective: one rank's finding fails every rank before any data moves
  if (c->nranks > 1) {
    TRY(c->scratch.ensure(sizeof(Scalars)));
    long long hv[2 + kMaxRanks] = {err.empty() ? 0 : 1, x ? 1 : 0};
    partition_slots(c, hv + 2);
    TRY(coll_allreduce_i64(c, hv, 2 + c->nranks, false));
    if (err.empty() && !partition_agrees(c, hv + 2)) err = who + ": " + kPartitionDisagree;
    if (hv[0] && err.empty()) err = who + ": another rank rejected its assignment";
    if (err.empty() && hv[1] != 0 && hv[1] != c->nranks)
      err = who + ": ranks disagree on the assignment x: every rank or none must pass NULL";
  }
  if (!err.empty()) return fail(err);
  cudaStream_t s = c->stream;
  if (!x) TRY(final_in_caller_order(c));       // one-rank runs leave it unresolved
  mvgpu_compare_report r;
  memset(&r, 0, sizeof r);
  cudaEvent_t e0 = get_event(c, 0), e1 = get_event(c, 1);
  CK(cudaEventRecord(e0, s));
  TRY(compare_pass(c, x ? c->cmp_x.p : c->final_orig.p, c->cmp_y.p, r));
  CK(cudaEventRecord(e1, s));
  CK(cudaEventSynchronize(e1));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  r.compare_s = ms * 1e-3;
  if (c->nranks > 1) TRY(coll_barrier(c));     // no rank leaves while a peer may still be receiving from it
  *rep = r;
  c->cmp_on_shard = true;
  return 0;
}

// ---- shard update (DESIGN.md §3.11, merge_gpu.cuh) -------------------------------------------------------------------
// The shard (n rows, rowptr/edges, lne records) with the sorted deletion keys dkey and the stably sorted insertion keys
// ikey merged in (iidx: batch index of each sorted insertion, iw: weights in batch order) -> nrow / nedges, *lne_out.
// Reads the old shard only.  Fails (writing nothing but the outputs) when the result would hold 2^32 records or more.
int merge_records(mvgpu_ctx *c, long long n, const long long *rowptr, const Edge16 *edges, long long lne,
                  const unsigned long long *dkey, long long ndel, const unsigned long long *ikey, const unsigned int *iidx,
                  const double *iw, long long nins, DevBuf<long long> &nrow, DevBuf<Edge16> &nedges, long long *lne_out) {
  cudaStream_t s = c->stream;
  const int nsm = c->num_sms;
  DevBuf<unsigned int> dstart, istart, kept, kscan;
  DevBuf<int32_t> erow;
  DevBuf<long long> mval, mscan, deg;
  TRY(dstart.ensure(n + 1)); TRY(istart.ensure(n + 1));
  TRY(kept.ensure(lne + 1)); TRY(kscan.ensure(lne + 1));
  TRY(deg.ensure(n + 1)); TRY(nrow.ensure(n + 1));
  k_row_bounds<<<grid_for(n + 1, 256, nsm), 256, 0, s>>>(dkey, ndel, n, dstart.p);
  k_row_bounds<<<grid_for(n + 1, 256, nsm), 256, 0, s>>>(ikey, nins, n, istart.p);
  CK(cudaMemsetAsync(kept.p + lne, 0, sizeof(unsigned int), s));
  if (lne) {
    TRY(erow.ensure(lne)); TRY(mval.ensure(lne)); TRY(mscan.ensure(lne));
    k_merge_keep<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(rowptr, edges, lne, n, dkey, dstart.p, erow.p, kept.p, mval.p);
    TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::InclusiveScanByKey(t, tb, erow.p, mval.p, mscan.p, MaxLL(), lne, cub::Equality(), s); }));
  }
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::ExclusiveSum(t, tb, kept.p, kscan.p, lne + 1, s); }));
  k_merge_degree<<<grid_for(n + 1, 256, nsm), 256, 0, s>>>(rowptr, kscan.p, istart.p, n, deg.p);
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::ExclusiveSum(t, tb, deg.p, nrow.p, n + 1, s); }));
  long long lne2 = 0;
  CK(cudaMemcpyAsync(&lne2, nrow.p + n, sizeof lne2, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (lne2 >= (1LL << 32)) return fail("the updated shard would hold lne >= 2^32 records (32-bit edge offsets would overflow)");
  TRY(nedges.ensure(lne2));
  if (lne) k_merge_old<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(rowptr, edges, lne, erow.p, kscan.p, mscan.p, ikey, istart.p, nrow.p, nedges.p);
  if (nins) k_merge_ins<<<grid_for(nins, 256, nsm, 16), 256, 0, s>>>(ikey, iidx, iw, nins, istart.p, rowptr, kscan.p, mscan.p, nrow.p, nedges.p);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  *lne_out = lne2;
  return 0;
}

// This rank's part of mvgpu_update_shard before the agreement: the batch to the device (wh[k]: the class of array k, in
// the order of the arguments), validated, sorted and merged into nrow / nedges.  Leaves the shard itself as it is.
int update_prepare(mvgpu_ctx *c, long long n_del, const int64_t *del_src, const int64_t *del_dst, long long n_ins,
                   const int64_t *ins_src, const int64_t *ins_dst, const double *ins_weight, const Where *wh,
                   DevBuf<long long> &nrow, DevBuf<Edge16> &nedges, long long *lne_out) {
  cudaStream_t s = c->stream;
  const int nsm = c->num_sms;
  DevBuf<long long> dsrc, ddst, isrc, idst;
  DevBuf<double> iw;
  DevBuf<unsigned long long> dkey, dkey_s, ikey, ikey_s;
  DevBuf<unsigned int> iidx, iidx_s, bad;
  TRY(dkey.ensure(n_del)); TRY(dkey_s.ensure(n_del));
  TRY(ikey.ensure(n_ins)); TRY(ikey_s.ensure(n_ins));
  TRY(iidx.ensure(n_ins)); TRY(iidx_s.ensure(n_ins)); TRY(bad.ensure(1));
  const long long *ds, *dd, *is, *id;
  const double *w;
  TRY(to_device(c, del_src, sizeof(long long) * n_del, wh[0], dsrc, ds));
  TRY(to_device(c, del_dst, sizeof(long long) * n_del, wh[1], ddst, dd));
  TRY(to_device(c, ins_src, sizeof(long long) * n_ins, wh[2], isrc, is));
  TRY(to_device(c, ins_dst, sizeof(long long) * n_ins, wh[3], idst, id));
  TRY(to_device(c, ins_weight, sizeof(double) * n_ins, wh[4], iw, w));
  CK(cudaMemsetAsync(bad.p, 0, sizeof(unsigned int), s));
  k_rowptr_check<<<grid_for(c->lnv + 1, 256, nsm), 256, 0, s>>>(c->d_rowptr64, c->lnv, c->lne, bad.p);
  if (n_del) k_batch_keys<<<grid_for(n_del, 256, nsm), 256, 0, s>>>(ds, dd, n_del, c->base, c->bound, c->nv_global, dkey.p, nullptr, bad.p);
  if (n_ins) k_batch_keys<<<grid_for(n_ins, 256, nsm), 256, 0, s>>>(is, id, n_ins, c->base, c->bound, c->nv_global, ikey.p, iidx.p, bad.p);
  CK(cudaGetLastError());
  unsigned int hbad = 0;
  CK(cudaMemcpyAsync(&hbad, bad.p, sizeof hbad, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (hbad & kBadRowptr) return fail("mvgpu_update_shard: edge_indices malformed (must start at 0, end at lne and never decrease)");
  if (hbad & kBadBatch) return fail("mvgpu_update_shard: a batch record lies outside the shard (src must be in [base, bound), dst in [0, nv))");
  dsrc.release(); ddst.release(); isrc.release(); idst.release();
  // keys are (local row < 2^31) << 31 | (tail < 2^31): 62 bits; the radix sort is stable, so equal insertion keys keep
  // batch order
  if (n_del) TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortKeys(t, tb, dkey.p, dkey_s.p, (int)n_del, 0, 62, s); }));
  if (n_ins) TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortPairs(t, tb, ikey.p, ikey_s.p, iidx.p, iidx_s.p, (int)n_ins, 0, 62, s); }));
  return merge_records(c, c->lnv, c->d_rowptr64, c->d_edges, c->lne, dkey_s.p, n_del, ikey_s.p, iidx_s.p, w, n_ins, nrow, nedges, lne_out);
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
// `-p`: random long edges on top of the generated strip (graph.hpp:939-1122; host/rgg.hpp add_random_edges is the
// restatement this follows, including its fixed seed).  Every rank replays all p draw streams (they are cheap and
// sequential) and keeps the records that touch its strip.  rowptr / edges: the strip being built (replaced by the merge).
static int add_random_edges(mvgpu_ctx *c, const RggParams &P, int64_t nv, int unit, double pct, const double *X3, const double *Y3,
                            DevBuf<long long> &rowptr, DevBuf<Edge16> &edges, long long *lne_io) {
  const int p = c->nranks, nsm = c->num_sms;
  cudaStream_t s = c->stream;
  if (nv >= 2147483645LL) return fail("random edges: nv too large for the device generator");
  long long tot = *lne_io / 2;
  TRY(coll_allreduce_i64(c, &tot, 1, false));
  const long long nrande = ((long long)(pct * (double)tot)) / 100;
  if (nrande <= 0) return 0;
  if (nrande >= (1LL << 31)) return fail("random edges: too many draws for the device generator");
  std::vector<long long> soff(p + 1, 0);
  for (int r = 0; r < p; r++) {
    long long pn = 0;
    if (nrande < p) { if (r == p - 1) pn = nrande; }
    else { pn = nrande / p; if (r == p - 1) pn += nrande % p; }
    soff[r + 1] = soff[r] + pn;
  }
  RandeParams R;
  R.n = P.n; R.nv = nv; R.p = p; R.me = c->rank; R.seed = 20180912u;       // host/rgg.hpp kRandomEdgeSeed
  DevBuf<long long> dsoff, nrow;
  DevBuf<int> di, dgj;
  DevBuf<unsigned long long> key, skey, xkey, sxkey;
  DevBuf<unsigned int> qidx, sq, emit, epos, xidx, sxidx;
  DevBuf<double> xw;
  TRY(dsoff.ensure(p + 1)); TRY(di.ensure(nrande)); TRY(dgj.ensure(nrande));
  TRY(key.ensure(nrande)); TRY(skey.ensure(nrande)); TRY(qidx.ensure(nrande)); TRY(sq.ensure(nrande));
  TRY(emit.ensure(nrande + 1)); TRY(epos.ensure(nrande + 1));
  CK(cudaMemcpyAsync(dsoff.p, soff.data(), sizeof(long long) * (p + 1), cudaMemcpyHostToDevice, s));
  k_rande_draws<<<p, 32, 0, s>>>(R, dsoff.p, di.p, dgj.p);
  k_rande_keys<<<grid_for(nrande, 256, nsm), 256, 0, s>>>(R, dsoff.p, di.p, dgj.p, nrande, rowptr.p, edges.p, key.p, qidx.p);
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortPairs(t, tb, key.p, skey.p, qidx.p, sq.p, (int)nrande, 0, 64, s); }));
  CK(cudaMemsetAsync(emit.p + nrande, 0, sizeof(unsigned int), s));
  k_rande_first<<<grid_for(nrande, 256, nsm), 256, 0, s>>>(skey.p, sq.p, nrande, R, dsoff.p, dgj.p, emit.p);
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::ExclusiveSum(t, tb, emit.p, epos.p, (int)(nrande + 1), s); }));
  unsigned int nextra = 0;
  CK(cudaMemcpyAsync(&nextra, epos.p + nrande, sizeof nextra, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (!nextra) return 0;
  TRY(xkey.ensure(nextra)); TRY(sxkey.ensure(nextra)); TRY(xidx.ensure(nextra)); TRY(sxidx.ensure(nextra)); TRY(xw.ensure(nextra));
  k_rande_emit<<<grid_for(nrande, 256, nsm), 256, 0, s>>>(R, P, dsoff.p, di.p, dgj.p, nrande, emit.p, epos.p, unit, X3, Y3, xkey.p, xw.p,
                                                        xidx.p);
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceRadixSort::SortPairs(t, tb, xkey.p, sxkey.p, xidx.p, sxidx.p, (int)nextra, 0, 62, s); }));
  // the extras are an insert-only batch in push order: merged like an update, RGG records first among equal tails
  DevBuf<Edge16> merged;
  long long lne2 = 0;
  TRY(merge_records(c, P.n, rowptr.p, edges.p, *lne_io, nullptr, 0, sxkey.p, sxidx.p, xw.p, nextra, nrow, merged, &lne2));
  edges.swap(merged);
  rowptr.swap(nrow);
  *lne_io = lne2;
  return 0;
}

extern "C" {

const char *mvgpu_last_error(void) { return g_err.c_str(); }

int mvgpu_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) { g_err = std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e); return -1; }
  return n;
}

int mvgpu_create(mvgpu_ctx **out, int device, int rank, int nranks) {
  if (!out) return fail("null ctx pointer");
  if (nranks < 1 || nranks > kMaxRanks || rank < 0 || rank >= nranks) return fail("bad rank/nranks");
  int n = 0;
  CK(cudaGetDeviceCount(&n));
  if (n < 1) return fail("no CUDA device: this library has no CPU fallback");
  if (device < 0 || device >= n) return fail("device index out of range");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  // an arch-specific sm_90a binary loads on compute capability 9.0 only
  if (prop.major != 9 || prop.minor != 0) return fail(std::string("built for sm_90a, found ") + prop.name);
  mvgpu_ctx *c = new mvgpu_ctx;
  c->device = device; c->rank = rank; c->nranks = nranks;
  c->num_sms = prop.multiProcessorCount;
  CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  CK(cudaMallocHost(&c->h_pin, 4096));
  memset(&c->tm, 0, sizeof c->tm);
  memset(&c->pt, 0, sizeof c->pt);
  memset(&c->qp, 0, sizeof c->qp);
  // developer knob: MVGPU_OPTIONS="name=value,name=value" presets options for every context of the process
  if (const char *e = getenv("MVGPU_OPTIONS")) {
    std::string all(e);
    size_t pos = 0;
    while (pos < all.size()) {
      size_t end = all.find(',', pos);
      if (end == std::string::npos) end = all.size();
      const std::string kv = all.substr(pos, end - pos);
      pos = end + 1;
      const size_t eq = kv.find('=');
      if (kv.empty()) continue;
      if (eq == std::string::npos || mvgpu_set_option(c, kv.substr(0, eq).c_str(), atoll(kv.c_str() + eq + 1))) {
        const std::string msg = "MVGPU_OPTIONS: bad entry '" + kv + "'" + (eq == std::string::npos ? "" : ": " + g_err);
        mvgpu_destroy(c);
        return fail(msg);
      }
    }
  }
  *out = c;
  return 0;
}

int mvgpu_destroy(mvgpu_ctx *c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  close_ipc(c);
  if (c->comm) g_nccl.CommDestroy(c->comm);
  c->hc.close_comm();
  for (cudaEvent_t e : c->events) cudaEventDestroy(e);
  if (c->h_stage) cudaFreeHost(c->h_stage);
  for (int b = 0; b < 2; b++) {
    if (c->h_bounce[b]) cudaFreeHost(c->h_bounce[b]);
    if (c->bounce_ev[b]) cudaEventDestroy(c->bounce_ev[b]);
  }
  if (c->h_pin) cudaFreeHost(c->h_pin);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;                                    // the DevBufs free themselves
  return 0;
}

int mvgpu_get_unique_id(void *id128) {
  static_assert(sizeof(ncclUniqueId) == MVGPU_UNIQUE_ID_BYTES, "ncclUniqueId size");
  if (!mvnccl::load(g_nccl, g_err)) {
    // no NCCL in this process: a random id still names the host transport's rendezvous segment
    FILE *f = fopen("/dev/urandom", "rb");
    if (!f || fread(id128, 1, MVGPU_UNIQUE_ID_BYTES, f) != MVGPU_UNIQUE_ID_BYTES) { if (f) fclose(f); return 1; }
    fclose(f);
    return 0;
  }
  ncclUniqueId id;
  NK(g_nccl.GetUniqueId(&id));
  memcpy(id128, &id, sizeof id);
  return 0;
}

int mvgpu_comm_init(mvgpu_ctx *c, const void *id128) {
  if (!c) return fail("null ctx");
  if (c->nranks == 1) return 0;
  if (c->opt_host_transport) {                    // setup exchanges through shared memory; ranks may share a device
    std::string err;
    if (c->hc.open(id128, c->rank, c->nranks, err)) return fail(err);
    return 0;
  }
  if (!mvnccl::load(g_nccl, g_err)) return 1;
  CK(cudaSetDevice(c->device));
  ncclUniqueId id;
  memcpy(&id, id128, sizeof id);
  NK(g_nccl.CommInitRank(&c->comm, c->nranks, id, c->rank));
  return 0;
}

// Host side of the compact upload (opt-in): a unit-weight shard needs only its tails on the device, 4 bytes per
// edge instead of the 16-byte {tail, weight} record.  A handful of plain std::threads (they block, they never spin:
// OpenMP workers that keep spinning after a parallel region slow the CUDA submission thread down) narrow the
// records chunk by chunk into one pinned staging array while the calling thread ships every finished chunk with
// cudaMemcpyAsync, so the copy engine and the cores overlap.  Validation (weights all 1.0, tails in range) and the
// count of non-owned tails happen in the same pass.  Returns 1 when the shard does not qualify (then the full
// records are uploaded), 0 on success, <0 on CUDA errors.
static int upload_compact(mvgpu_ctx *c, int64_t nv_global, int64_t lne, const void *edge_list, long long *bytes_copied) {
  const Edge16 *E = reinterpret_cast<const Edge16 *>(edge_list);
  const long long CH = c->opt_upload_chunk;                      // edges per chunk (default 4 Mi: 64 MB read, 16 MB staged)
  const long long nchunks = (lne + CH - 1) / CH;
  if ((size_t)lne > c->h_stage_cap) {
    if (c->h_stage) cudaFreeHost(c->h_stage);
    c->h_stage = nullptr; c->h_stage_cap = 0;
    if (cudaMallocHost(&c->h_stage, sizeof(int32_t) * (size_t)lne) != cudaSuccess) { cudaGetLastError(); return 1; }
    c->h_stage_cap = (size_t)lne;
  }
  if (c->in_tails32.ensure(lne + 4)) return -1;
  if (c->raw_ring.ensure((size_t)2 * CH)) return -1;             // two raw chunks in flight on the device
  if (c->scratch.ensure(sizeof(Scalars))) return -1;
  Scalars *d_sc = dev_scalars(c);
  if (cudaMemsetAsync(&d_sc->st, 0, sizeof(EdgeStats), c->stream) != cudaSuccess) return -1;
  int32_t *stage = reinterpret_cast<int32_t *>(c->h_stage);
  const long long base = c->base, bound = c->bound;
  const int nthreads = (int)std::max<long long>(1, std::min<long long>(c->opt_host_threads > 0 ? c->opt_host_threads : 8, nchunks));
  // The chunks are consumed from both ends.  Host threads narrow chunks from the FRONT (16-byte records -> 4-byte
  // tails in the pinned staging array, shipped as soon as they are ready); whenever no narrowed chunk is ready the
  // calling thread hands the copy engine a RAW chunk from the BACK instead (64 MB of records into a two-slot device
  // ring, narrowed there by k_narrow_records).  The copy engine never idles while the cores narrow, the cores never
  // idle while the link is busy, and the meeting point adapts to whatever cores and link the box has.  Front and back
  // share one atomic word so that no chunk is claimed twice.
  std::vector<std::atomic<int>> done(nchunks);
  for (auto &d : done) d.store(0);
  std::atomic<unsigned long long> claim{0};                      // front << 32 | back
  std::atomic<long long> nremote{0};
  std::atomic<int> bad{0};
  auto claim_front = [&]() -> long long {
    unsigned long long v = claim.load();
    for (;;) {
      const unsigned long long f = v >> 32, bk = v & 0xffffffffULL;
      if ((long long)(f + bk) >= nchunks) return -1;
      if (claim.compare_exchange_weak(v, ((f + 1) << 32) | bk)) return (long long)f;
    }
  };
  auto claim_back = [&]() -> long long {
    unsigned long long v = claim.load();
    for (;;) {
      const unsigned long long f = v >> 32, bk = v & 0xffffffffULL;
      if ((long long)(f + bk) >= nchunks) return -1;
      if (claim.compare_exchange_weak(v, (f << 32) | (bk + 1))) return nchunks - 1 - (long long)bk;
    }
  };
  auto worker = [&]() {
    for (;;) {
      if (bad.load(std::memory_order_relaxed)) break;
      const long long i = claim_front();
      if (i < 0) break;
      const long long off = i * CH, n = std::min<long long>(CH, lne - off);
      long long nrem = 0;
      int b = 0;
      mv_narrow_edges(E + off, n, nv_global, base, bound, stage + off, &nrem, &b);
      if (b) bad.store(1);
      nremote.fetch_add(nrem);
      done[i].store(1, std::memory_order_release);
    }
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < nthreads; t++) pool.emplace_back(worker);
  int rc = 0;
  long long next_front = 0, raw_issued = 0, copied = 0;
  cudaEvent_t raw_ev[2] = {get_event(c, 2), get_event(c, 3)};     // completion of the raw chunk that used ring slot k
  const bool use_raw = c->opt_compact_upload >= 2;
  while (!rc && !bad.load(std::memory_order_relaxed)) {
    const unsigned long long v = claim.load();
    const long long f = (long long)(v >> 32), bk = (long long)(v & 0xffffffffULL);
    if (next_front < f && done[next_front].load(std::memory_order_acquire)) {          // a narrowed chunk is ready: ship it
      const long long off = next_front * CH, n = std::min<long long>(CH, lne - off);
      if (cudaMemcpyAsync(c->in_tails32.p + off, stage + off, sizeof(int32_t) * n, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) rc = -1;
      copied += (long long)sizeof(int32_t) * n;
      next_front++;
      continue;
    }
    if (next_front >= f && f + bk >= nchunks) break;                                    // everything claimed and shipped
    // nothing narrowed is ready: keep the link busy with a raw chunk, at most two in flight
    if (use_raw && (raw_issued < 2 || cudaEventQuery(raw_ev[raw_issued & 1]) == cudaSuccess)) {
      const long long i = claim_back();
      if (i >= 0) {
        const long long off = i * CH, n = std::min<long long>(CH, lne - off);
        Edge16 *slot = c->raw_ring.p + (raw_issued & 1) * CH;
        if (cudaMemcpyAsync(slot, E + off, sizeof(Edge16) * n, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) rc = -1;
        k_narrow_records<<<grid_for(n, 256, c->num_sms, 16), 256, 0, c->stream>>>(slot, n, nv_global, base, bound, c->in_tails32.p + off, &d_sc->st);
        if (cudaEventRecord(raw_ev[raw_issued & 1], c->stream) != cudaSuccess) rc = -1;
        copied += (long long)sizeof(Edge16) * n;
        raw_issued++;
        continue;
      }
    }
    std::this_thread::yield();
  }
  for (auto &th : pool) th.join();
  if (rc) return rc;
  if (bad.load()) { cudaStreamSynchronize(c->stream); return 1; }
  long long nrem_dev = 0;
  if (raw_issued) {
    EdgeStats hs;
    if (cudaMemcpyAsync(&hs, &d_sc->st, sizeof hs, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(c->stream) != cudaSuccess) return -1;
    if (hs.nonunit || hs.bad_tail) return 1;
    nrem_dev = (long long)hs.nremote;
  }
  c->in_nremote = nremote.load() + nrem_dev;
  c->raw_chunks = raw_issued;
  *bytes_copied = copied;
  return 0;
}

int mvgpu_upload_shard(mvgpu_ctx *c, int64_t nv_global, const int64_t *parts, int64_t lnv, int64_t lne,
                       const int64_t *edge_indices, const void *edge_list) {
  if (!c || !parts || !edge_indices || (lne && !edge_list)) return fail("null argument");
  CK(cudaSetDevice(c->device));
  TRY(set_graph(c, nv_global, parts, lnv, lne));
  TRY(c->in_rowptr.ensure(lnv + 1));
  cudaEvent_t a = get_event(c, 0), b = get_event(c, 1);
  CK(cudaEventRecord(a, c->stream));
  CK(cudaMemcpyAsync(c->in_rowptr.p, edge_indices, sizeof(long long) * (lnv + 1), cudaMemcpyHostToDevice, c->stream));
  int compact = 1;
  long long compact_bytes = 0;
  if (c->opt_compact_upload && !c->opt_force_weighted && lne > 0) {
    compact = upload_compact(c, nv_global, lne, edge_list, &compact_bytes);
    if (compact < 0) return fail(std::string("compact upload: ") + cudaGetErrorString(cudaGetLastError()));
  }
  if (compact != 0) {
    TRY(c->in_edges.ensure(lne));
    if (lne) CK(cudaMemcpyAsync(c->in_edges.p, edge_list, sizeof(Edge16) * lne, cudaMemcpyHostToDevice, c->stream));
  }
  CK(cudaEventRecord(b, c->stream));
  CK(cudaEventSynchronize(b));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, a, b));
  set_source(c, c->in_rowptr.p, compact == 0 ? nullptr : c->in_edges.p, compact == 0 ? c->in_tails32.p : nullptr, false, ms * 1e-3,
             (long long)sizeof(long long) * (lnv + 1) + (compact == 0 ? compact_bytes : (long long)sizeof(Edge16) * lne));
  return 0;
}

int mvgpu_attach_shard_device(mvgpu_ctx *c, int64_t nv_global, const int64_t *parts, int64_t lnv, int64_t lne,
                              const int64_t *d_edge_indices, const void *d_edge_list) {
  if (!c || !parts || !d_edge_indices || (lne && !d_edge_list)) return fail("null argument");
  if (((uintptr_t)d_edge_list & 15) || ((uintptr_t)d_edge_indices & 7)) return fail("device arrays must be 16/8-byte aligned");
  CK(cudaSetDevice(c->device));
  TRY(set_graph(c, nv_global, parts, lnv, lne));
  set_source(c, reinterpret_cast<const long long *>(d_edge_indices), reinterpret_cast<const Edge16 *>(d_edge_list), nullptr, false, 0.0, 0);
  return 0;
}

// ---- section 8(f) rank 1: the reference's GenerateRGG on the device (rgg_gpu.cuh) ---------------------------------
int mvgpu_generate_rgg_shard(mvgpu_ctx *c, int64_t nv_global, int unit_weight, int64_t *lne_out) {
  return mvgpu_generate_rgg_shard_ex(c, nv_global, unit_weight, 0, 0.0, lne_out);
}

int mvgpu_generate_rgg_shard_ex(mvgpu_ctx *c, int64_t nv_global, int unit_weight, int lcg, double random_edge_percent, int64_t *lne_out) {
  if (!c) return fail("null ctx");
  CK(cudaSetDevice(c->device));
  const int p = c->nranks, r = c->rank;
  if (nv_global < 1 || nv_global % p != 0) return fail("[ERROR] Number of vertices must be perfectly divisible by number of processes.");
  if (p & (p - 1)) return fail("[ERROR] Number of processes must be a power of 2.");
  if (!(random_edge_percent >= 0.0)) return fail("random_edge_percent must be >= 0");
  if (random_edge_percent > 0.0 && p > 1 && !c->comm && !c->hc.is_open())
    return fail("random edges (-p) on several ranks need the communicator: call mvgpu_comm_init first");
  RggParams P;
  memset(&P, 0, sizeof P);
  P.n = nv_global / p; P.rank = r; P.nranks = p;
  {                                                    // utils.hpp:91-98 reseeder(1)
    std::seed_seq seq({1u});
    std::vector<std::uint32_t> seeds(1);
    seq.generate(seeds.begin(), seeds.end());
    P.seed = (unsigned int)seeds[0];
  }
  const double rc = std::sqrt((double)std::log((double)nv_global) / (double)(3.14159 * nv_global));   // graph.hpp:629-631, PI of utils.hpp:44
  const double rt = std::sqrt((double)2.0736 / (double)nv_global);
  P.rn = (rc + rt) / 2.0;
  P.rec_np = (double)(1.0 / (double)p);
  if (!(P.rec_np > P.rn)) return fail("RGG radius does not fit the strip height (1/p > rn violated)");
  if (lcg) {                                           // utils.hpp:146-218 as host/rgg.hpp restates it
    P.lcg = 1;
    const int64_t M = 2147483647LL, A = 16807LL;
    const int64_t x0 = (int64_t)P.seed;
    const uint64_t len = 2ULL * (uint64_t)P.n;
    for (int k = 0; k < 3; k++) {
      const int sr = r - 1 + k;
      if (sr < 0 || sr >= p) { P.lcg_first[k] = 1; continue; }
      int64_t first;
      if (sr == 0) first = x0;
      else {
        uint64_t acc = 1, base = (uint64_t)A, e = len * (uint64_t)sr;
        while (e) { if (e & 1) acc *= base; base *= base; e >>= 1; }
        first = (int64_t)((uint64_t)x0 * acc) % M;
      }
      P.lcg_first[k] = (unsigned long long)(first < 0 ? -first : first);
    }
    P.lcg_mult = 1.0 / (double)(1.0 + (double)(M - 1));
  }
  {                                                    // divisor of std::generate_canonical<double,53>(minstd_rand0)
    const long double rr = 2147483646.0L;
    double tmp = 1.0;
    tmp *= rr;
    P.r_range = tmp;
    tmp *= rr;
    P.r_range2 = tmp;
  }
  long long ncell = (long long)std::floor(1.0 / P.rn);
  while (ncell > 1 && 1.0 / (double)ncell < P.rn * 1.000001) ncell--;
  if (ncell < 1) ncell = 1;
  P.ncell = ncell;
  P.ylo = r * P.rec_np - P.rn * 1.01;
  P.yhi = (r + 1) * P.rec_np + P.rn * 1.01;
  auto cell_of_h = [&](double v) { long long q = (long long)std::floor(v * (double)ncell); return q < 0 ? 0LL : (q >= ncell ? ncell - 1 : q); };
  const long long row0 = std::max<long long>(0, cell_of_h(P.ylo) - 1), row1 = std::min<long long>(ncell - 1, cell_of_h(P.yhi) + 1);
  P.row0 = row0; P.nrows = row1 - row0 + 1;
  const long long ncells = P.nrows * ncell;
  if (ncells + 1 >= (1LL << 31) || P.n >= (1LL << 31)) return fail("RGG too large for the device generator");
  cudaStream_t s = c->stream;
  const int nsm = c->num_sms;
  DevBuf<double> X, UY, cx, cy;                        // X, UY: coordinates of up to three strips (own + neighbours)
  DevBuf<long long> cgid, deg;
  DevBuf<unsigned int> cnt, cstart;
  // the new strip is built in its own arrays: the current shard (possibly the last generated one) stays intact until
  // everything that can refuse has passed
  DevBuf<long long> rowptr;
  DevBuf<Edge16> edges;
  TRY(X.ensure(3 * P.n)); TRY(UY.ensure(3 * P.n)); TRY(cnt.ensure(ncells + 1)); TRY(cstart.ensure(ncells + 1)); TRY(deg.ensure(P.n + 1));
  k_rgg_points<<<grid_for(P.n, 256, nsm), 256, 0, s>>>(P, X.p, UY.p);
  CK(cudaMemsetAsync(cnt.p, 0, sizeof(unsigned int) * (ncells + 1), s));
  k_rgg_bin<<<grid_for(P.n, 256, nsm), 256, 0, s>>>(P, X.p, UY.p, 0, cnt.p, nullptr, nullptr, nullptr, nullptr);
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::ExclusiveSum(t, tb, cnt.p, cstart.p, (int)(ncells + 1), s); }));
  unsigned int ncand = 0;
  CK(cudaMemcpyAsync(&ncand, cstart.p + ncells, sizeof ncand, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  TRY(cx.ensure(ncand)); TRY(cy.ensure(ncand)); TRY(cgid.ensure(ncand));
  CK(cudaMemsetAsync(cnt.p, 0, sizeof(unsigned int) * (ncells + 1), s));
  k_rgg_bin<<<grid_for(P.n, 256, nsm), 256, 0, s>>>(P, X.p, UY.p, 1, cnt.p, cstart.p, cx.p, cy.p, cgid.p);
  CK(cudaMemsetAsync(deg.p + P.n, 0, sizeof(long long), s));
  k_rgg_neighbours<false><<<grid_for(P.n, 128, nsm, 16), 128, 0, s>>>(P, X.p, UY.p, cstart.p, cx.p, cy.p, cgid.p, unit_weight, deg.p, nullptr);
  TRY(rowptr.ensure(P.n + 1));
  TRY(cub_run(c, [&](void *t, size_t &tb) { return cub::DeviceScan::ExclusiveSum(t, tb, deg.p, rowptr.p, (int)(P.n + 1), s); }));
  long long lne = 0;
  CK(cudaMemcpyAsync(&lne, rowptr.p + P.n, sizeof lne, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  TRY(edges.ensure(lne));
  k_rgg_neighbours<true><<<grid_for(P.n, 128, nsm, 16), 128, 0, s>>>(P, X.p, UY.p, cstart.p, cx.p, cy.p, cgid.p, unit_weight, rowptr.p, edges.p);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  cx.release(); cy.release(); cgid.release(); deg.release(); cnt.release(); cstart.release();
  if (random_edge_percent > 0.0) TRY(add_random_edges(c, P, nv_global, unit_weight, random_edge_percent, X.p, UY.p, rowptr, edges, &lne));
  X.release(); UY.release();
  std::vector<int64_t> parts(p + 1);
  for (int q = 0; q <= p; q++) parts[q] = (nv_global * q) / p;
  TRY(set_graph(c, nv_global, parts.data(), P.n, lne));   // validates before it changes anything
  c->gen_rowptr.swap(rowptr);                              // the old generated arrays, if any, go with the temporaries
  c->gen_edges.swap(edges);
  set_source(c, c->gen_rowptr.p, c->gen_edges.p, nullptr, false, 0.0, 0);
  if (lne_out) *lne_out = lne;
  return 0;
}

int mvgpu_download_shard(mvgpu_ctx *c, int64_t *edge_indices, void *edge_list) {
  if (!c || !c->have_graph || !c->d_rowptr64) return fail("no shard on the device");
  if (!c->d_edges) return fail("the shard was uploaded in the compact format; nothing to download");
  CK(cudaSetDevice(c->device));
  if (edge_indices) CK(cudaMemcpyAsync(edge_indices, c->d_rowptr64, sizeof(long long) * (c->lnv + 1), cudaMemcpyDeviceToHost, c->stream));
  if (edge_list && c->lne) CK(cudaMemcpyAsync(edge_list, c->d_edges, sizeof(Edge16) * c->lne, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int mvgpu_update_shard(mvgpu_ctx *c, int64_t n_del, const int64_t *del_src, const int64_t *del_dst, int64_t n_ins,
                       const int64_t *ins_src, const int64_t *ins_dst, const double *ins_weight, int64_t *lne_out) {
  if (!c) return fail("null ctx");
  CK(cudaSetDevice(c->device));
  if (c->nranks > 1 && !c->comm && !c->hc.is_open()) return fail("mvgpu_update_shard is collective on several ranks: call mvgpu_comm_init first");
  // every local finding waits for the agreement below, so that one rank's bad batch fails every rank
  std::string err;
  if (!c->have_graph || !c->d_rowptr64) err = "no shard on the device";
  else if (c->d_tails32) err = "the shard was uploaded in the compact format: it has no records to update";
  else if (c->f32) err = "a shard uploaded with mvgpu_upload_shard32 cannot be updated";
  else if (n_del < 0 || n_ins < 0) err = "negative batch size";
  else if (n_del >= (1LL << 31) || n_ins >= (1LL << 31)) err = "batch too large: fewer than 2^31 deletions and 2^31 insertions per call";
  else if ((n_del && (!del_src || !del_dst)) || (n_ins && (!ins_src || !ins_dst || !ins_weight))) err = "null batch array";
  Where w[5];
  if (err.empty()) {                            // the arrays of an empty side are not read
    const void *arr[5] = {n_del ? del_src : nullptr, n_del ? del_dst : nullptr, n_ins ? ins_src : nullptr,
                          n_ins ? ins_dst : nullptr, n_ins ? ins_weight : nullptr};
    const char *names[5] = {"del_src", "del_dst", "ins_src", "ins_dst", "ins_weight"};
    err = locate_all(c, 5, arr, names, w);
  }
  if (!err.empty()) err = "mvgpu_update_shard: " + err;
  DevBuf<long long> nrow;
  DevBuf<Edge16> nedges;
  long long lne2 = 0;
  if (err.empty() && update_prepare(c, n_del, del_src, del_dst, n_ins, ins_src, ins_dst, ins_weight, w, nrow, nedges, &lne2)) err = g_err;
  if (c->nranks > 1) {
    TRY(c->scratch.ensure(sizeof(Scalars)));
    long long any = err.empty() ? 0 : 1;
    TRY(coll_allreduce_i64(c, &any, 1, false));
    if (any && err.empty()) err = "mvgpu_update_shard: another rank rejected its batch";
  }
  if (!err.empty()) return fail(err);
  // the last run's assignment is resolved while its arrays still describe it: communities() keeps returning it
  if (c->run_on_shard) TRY(final_in_caller_order(c));
  // the result lives in library buffers from now on (never in an attached shard's arrays): the generator's, if the
  // shard came from there, the upload buffers otherwise; the old arrays go with nrow / nedges
  const bool gen = c->d_edges == c->gen_edges.p;
  DevBuf<long long> &rp = gen ? c->gen_rowptr : c->in_rowptr;
  DevBuf<Edge16> &ed = gen ? c->gen_edges : c->in_edges;
  rp.swap(nrow);
  ed.swap(nedges);
  c->lne = lne2;
  set_source(c, rp.p, ed.p, nullptr, false, 0.0, 0);
  c->run_on_shard = c->eval_on_shard = false;   // the initial assignment and the movable set stay: parts and lnv have not changed
  c->mov_out_valid = false;
  c->peers_ready = false;                       // ghost lists and receive offsets change with the records, on every rank
  if (lne_out) *lne_out = lne2;
  return 0;
}

int mvgpu_louvain(mvgpu_ctx *c, double lower, double thresh, int *iters, double *modularity) {
  if (!c || !iters || !modularity) return fail("null argument");
  return run_louvain(c, lower, thresh, iters, modularity);
}

int mvgpu_set_initial_communities(mvgpu_ctx *c, const int64_t *comm) {
  if (!c) return fail("null argument");
  if (!comm) { c->have_init = false; return 0; }
  if (!c->have_graph) return fail("mvgpu_set_initial_communities: no shard yet (upload, attach or generate one first)");
  CK(cudaSetDevice(c->device));
  // staged in eval_comm, which only lives inside one call, so that a refused array leaves the current one in place
  TRY(c->eval_comm.ensure(c->lnv));
  std::string err;
  TRY(take_ids(c, comm, "mvgpu_set_initial_communities", "comm", c->eval_comm.p, err));
  if (!err.empty()) return fail(err);
  c->init_comm.swap(c->eval_comm);
  c->have_init = true;
  return 0;
}

int mvgpu_set_movable(mvgpu_ctx *c, const uint8_t *mask) {
  if (!c) return fail("null argument");
  if (mask && !c->have_graph) return fail("mvgpu_set_movable: no shard yet (upload, attach or generate one first)");
  Where w = Where::Pageable;
  if (mask) {
    CK(cudaSetDevice(c->device));
    const std::string err = locate(c, mask, "mask", w);
    if (!err.empty()) return fail("mvgpu_set_movable: " + err);
  }
  c->mov_out_valid = false;
  c->peers_ready = false;          // a masked run with the frontier option exports two more arrays
  if (!mask) { c->have_mov = false; return 0; }
  TRY(c->mov_in.ensure(c->lnv));
  if (c->lnv) {                                // on the context's stream, behind any run still reading mov_in
    const uint8_t *src;
    TRY(to_device(c, mask, c->lnv, w, c->mov_in, src));
    // kept as 0 / 1, the form mvgpu_get_movable returns (the run's kernels read any nonzero byte as movable)
    k_mask01<<<grid_for(c->lnv, 256, c->num_sms), 256, 0, c->stream>>>(src, c->lnv, c->mov_in.p);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c->stream));
  }
  c->have_mov = true;
  return 0;
}

int mvgpu_get_movable(mvgpu_ctx *c, uint8_t *out) {
  if (!c || !out) return fail("null argument");
  if (!c->have_graph) return fail("mvgpu_get_movable: no shard yet (upload, attach or generate one first)");
  CK(cudaSetDevice(c->device));
  Where w;
  const std::string err = locate(c, out, "out", w);
  if (!err.empty()) return fail("mvgpu_get_movable: " + err);
  if (c->lnv == 0) return 0;
  // on the context's stream: the run leaves k_movable_out queued behind its end event (and c->stream does not
  // synchronise with the legacy default stream)
  if (c->mov_out_valid || c->have_mov)
    return to_caller(c, c->mov_out_valid ? c->mov_out.p : c->mov_in.p, c->lnv, w, out);
  if (w == Where::Device)
    CK(cudaMemsetAsync(out, 1, (size_t)c->lnv, c->stream));
  else
    memset(out, 1, (size_t)c->lnv);
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int mvgpu_evaluate_communities(mvgpu_ctx *c, const int64_t *comm, mvgpu_quality *out) {
  if (!c || !out) return fail("null argument");
  return evaluate(c, comm, out);
}

// Not in mvgpu.h: the Python binding's way into the collective when it cannot build the array (e.g. a wrong length), so
// that the other ranks fail with it instead of waiting in the first setup all-reduce.
int mv_evaluate_refused(mvgpu_ctx *c, const char *why, mvgpu_quality *out) {
  if (!c || !out || !why) return fail("null argument");
  return evaluate(c, nullptr, out, why);
}

int mvgpu_split_communities(mvgpu_ctx *c, const int64_t *comm, int64_t *out, mvgpu_split_report *rep) {
  if (!c || !out || !rep) return fail("null argument");
  return split(c, comm, out, rep);
}

// Not in mvgpu.h: the Python binding's way into the collective when it cannot build the array, as mv_evaluate_refused
int mv_split_refused(mvgpu_ctx *c, const char *why, mvgpu_split_report *rep) {
  if (!c || !rep || !why) return fail("null argument");
  int64_t none = 0;
  return split(c, nullptr, &none, rep, why);
}

int mvgpu_probe_communities(mvgpu_ctx *c, const int64_t *comm, int64_t *target, int64_t *best, double *gain,
                            mvgpu_probe_report *rep) {
  if (!c || !rep) return fail("null argument");
  return probe(c, comm, target, best, gain, rep);
}

// Not in mvgpu.h: the Python binding's way into the collective when it cannot build the array, as mv_evaluate_refused
int mv_probe_refused(mvgpu_ctx *c, const char *why, mvgpu_probe_report *rep) {
  if (!c || !rep || !why) return fail("null argument");
  return probe(c, nullptr, nullptr, nullptr, nullptr, rep, why);
}

int mvgpu_compare_communities(mvgpu_ctx *c, const int64_t *x, const int64_t *y, mvgpu_compare_report *rep) {
  if (!c || !rep) return fail("null argument");
  return compare(c, x, y, rep);
}

// Not in mvgpu.h: the Python binding's way into the collective when it cannot build the arrays, as mv_evaluate_refused
int mv_compare_refused(mvgpu_ctx *c, const char *why, mvgpu_compare_report *rep) {
  if (!c || !rep || !why) return fail("null argument");
  return compare(c, nullptr, nullptr, rep, why);
}

int mvgpu_get_community_matches(mvgpu_ctx *c, int64_t *size, int64_t *best, int64_t *overlap, int64_t *best_size) {
  if (!c) return fail("null argument");
  if (!c->cmp_on_shard) return fail("no comparison on this shard yet (mvgpu_compare_communities)");
  CK(cudaSetDevice(c->device));
  const size_t n = (size_t)c->lnv;
  int64_t *dst[4] = {size, best, overlap, best_size};
  const void *arr[4] = {size, best, overlap, best_size};
  const char *names[4] = {"size", "best", "overlap", "best_size"};
  Where w[4];
  const std::string err = locate_all(c, 4, arr, names, w);
  if (!err.empty()) return fail("mvgpu_get_community_matches: " + err);
  for (int k = 0; k < 4; k++)
    if (dst[k]) TRY(to_caller(c, c->cmp_match.p + k * n, sizeof(long long) * n, w[k], dst[k]));
  return 0;
}

int mvgpu_get_community_stats(mvgpu_ctx *c, int64_t *size, double *volume, double *internal) {
  if (!c) return fail("null argument");
  if (!c->eval_on_shard) return fail("no evaluation of this shard yet (mvgpu_evaluate_communities)");
  CK(cudaSetDevice(c->device));
  const size_t n = (size_t)c->lnv;
  const void *arr[3] = {size, volume, internal};
  const char *names[3] = {"size", "volume", "internal"};
  Where w[3];
  const std::string err = locate_all(c, 3, arr, names, w);
  if (!err.empty()) return fail("mvgpu_get_community_stats: " + err);
  if (size) TRY(to_caller(c, c->q_size.p, sizeof(long long) * n, w[0], size));
  if (volume) TRY(to_caller(c, c->q_vol.p, sizeof(double) * n, w[1], volume));
  if (internal) TRY(to_caller(c, c->q_internal.p, sizeof(double) * n, w[2], internal));
  return 0;
}

int mvgpu_get_compact_communities(mvgpu_ctx *c, int64_t *out) {
  if (!c || !out) return fail("null argument");
  if (!c->eval_on_shard) return fail("no evaluation of this shard yet (mvgpu_evaluate_communities)");
  CK(cudaSetDevice(c->device));
  Where w;
  const std::string err = locate(c, out, "out", w);
  if (!err.empty()) return fail("mvgpu_get_compact_communities: " + err);
  return put_ids(c, c->q_lab.p, out, w);
}

int mvgpu_get_converged(mvgpu_ctx *c, int *converged) {
  if (!c || !converged) return fail("null argument");
  if (!c->d_final) return fail("no result yet");
  *converged = c->converged;
  return 0;
}

// the per-vertex result getters serve the last run on the current shard (mvgpu_update_shard keeps it)
const char *const kNoRunOnShard = "no run on this shard yet (mvgpu_louvain after the last upload / attach / generate)";

int mvgpu_get_communities_device(mvgpu_ctx *c, const int32_t **d_out) {
  if (!c || !d_out) return fail("null argument");
  if (!c->final_on_shard) return fail(kNoRunOnShard);
  TRY(final_in_caller_order(c));
  CK(cudaStreamSynchronize(c->stream));
  *d_out = c->final_orig.p;
  return 0;
}

int mvgpu_get_communities(mvgpu_ctx *c, int64_t *out) {
  if (!c || !out) return fail("null argument");
  if (!c->final_on_shard) return fail(kNoRunOnShard);
  CK(cudaSetDevice(c->device));
  Where w;
  const std::string err = locate(c, out, "out", w);
  if (!err.empty()) return fail("mvgpu_get_communities: " + err);
  if (c->lnv == 0) return 0;
  TRY(final_in_caller_order(c));
  return put_ids(c, c->final_orig.p, out, w);
}

// one option; a refusal changes nothing
static int set_option_value(mvgpu_ctx *c, const std::string &n, int64_t value) {
  if (n == "trace") c->opt_trace = value != 0;
  else if (n == "max_iters") { if (value < 1) return fail("max_iters < 1"); c->opt_max_iters = value; }
  else if (n == "force_weighted") c->opt_force_weighted = value != 0;
  else if (n == "force_heavy_deg") c->opt_force_heavy_deg = value;
  else if (n == "scan_ctas") { if (value < 0 || value > INT32_MAX) return fail("scan_ctas must be >= 0"); c->opt_scan_ctas = (int)value; }
  else if (n == "scan_variant") { if (value < 3 || value > 6) return fail("scan_variant must be 6 (measure and choose, default), 5 (k_scan_pq), 4 (k_scan_pw) or 3 (k_scan_ws)"); c->opt_scan_variant = (int)value; }
  else if (n == "cache_policy") c->opt_cache_policy = (int)value;
  else if (n == "reorder") c->opt_reorder = (int)value;
  else if (n == "comm_mode") c->opt_comm_mode = (int)value;
  else if (n == "compact_upload") c->opt_compact_upload = (int)value;
  else if (n == "host_threads") c->opt_host_threads = (int)value;
  else if (n == "first_iter") c->opt_first_iter = value != 0;
  else if (n == "frontier") { if (value != 0 && value != 1) return fail("frontier must be 0 or 1"); c->opt_frontier = (int)value; }
  else if (n == "stop_after") { if (value < 0) return fail("stop_after < 0"); c->opt_stop_after = value; }
  else if (n == "upload_chunk") { if (value < 256 || (value & 3)) return fail("upload_chunk must be a multiple of 4, >= 256"); c->opt_upload_chunk = value; }
  else if (n == "host_transport") {
    if ((c->comm || c->hc.is_open()) && c->opt_host_transport != (value != 0)) return fail("host_transport must be set before mvgpu_comm_init");
    c->opt_host_transport = value != 0;
  }
  else if (n == "region_size") { if (value < 32) return fail("region_size < 32"); c->opt_region = (int)value; }
  else return fail("unknown option " + n);
  return 0;
}

int mvgpu_set_option(mvgpu_ctx *c, const char *name, int64_t value) {
  if (!c || !name) return fail("null argument");
  TRY(set_option_value(c, name, value));
  c->peers_ready = false;          // options may change which arrays exist: re-validate the peer tables
  return 0;
}

int mvgpu_get_trace(mvgpu_ctx *c, int max_entries, mvgpu_iter_trace *out, int *n) {
  if (!c || !n) return fail("null argument");
  const int k = std::min<int>(max_entries, (int)c->trace.size());
  if (out && k > 0) memcpy(out, c->trace.data(), sizeof(mvgpu_iter_trace) * k);
  *n = (int)c->trace.size();
  return 0;
}

int mvgpu_get_scan_times(mvgpu_ctx *c, int max_entries, double *out, int *n) {
  if (!c || !n) return fail("null argument");
  const int k = std::min<int>(max_entries, (int)c->scan_times.size());
  if (out && k > 0) memcpy(out, c->scan_times.data(), sizeof(double) * k);
  *n = (int)c->scan_times.size();
  return 0;
}

int mvgpu_get_timings(mvgpu_ctx *c, mvgpu_timings *out) {
  if (!c || !out) return fail("null argument");
  *out = c->tm;
  return 0;
}

int mvgpu_get_constant(mvgpu_ctx *c, double *out) {
  if (!c || !out) return fail("null argument");
  *out = c->constant;
  return 0;
}

int mvgpu_get_shard_info(mvgpu_ctx *c, int64_t *info6) {
  if (!c || !info6) return fail("null argument");
  const bool ran = c->final_on_shard;          // [2..5] come from a run's setup: 0 until the shard's first run
  info6[0] = c->lnv; info6[1] = c->lne; info6[2] = ran ? c->nghost : 0; info6[3] = ran ? c->nsend : 0;
  info6[4] = ran ? c->nheavy : 0; info6[5] = ran ? c->maxdeg : 0;
  return 0;
}

// Test hook, deliberately not declared in mvgpu.h: what the last mvgpu_louvain decided about the layout and which
// layout it built, valid until the next run.  info16 (may be NULL): want, relabel, reordered, region stride, regions,
// span sum, span count (-1, -1 when the sample did not run), unordered, has_self, simple_sorted, FIRST launched, unit,
// nlow, nghost, lnv, lne.  Arrays (each may be NULL): the compact CSR before renumbering (rowptr lnv+1, tails lne, in
// slot numbering), bfs_key (lnv, this rank renumbered), perm / inv / lab (lnv, some rank renumbered), the renumbered
// CSR (rowptr2 lnv+1, tails2 lne, weights2 lne on the weighted path).  Asking for an array the run did not build fails.
int mv_layout_readback(mvgpu_ctx *c, int64_t *info16, uint32_t *rowptr, int32_t *tails, uint32_t *bfs_key, int32_t *perm,
                       int32_t *inv, int32_t *lab, uint32_t *rowptr2, int32_t *tails2, double *weights2) {
  if (!c) return fail("null ctx");
  // keyed on run_on_shard, not final_on_shard: the arrays it returns are the last run's compact CSR, sized by that
  // run's lne, so it refuses after mvgpu_update_shard too (the per-vertex labels stay valid there, the CSR does not)
  if (!c->run_on_shard) return fail("no run on this shard yet: mv_layout_readback describes the last mvgpu_louvain on the current shard");
  if (info16) {
    const int64_t v[16] = {c->lay.want, c->relabel, c->reordered ? 1 : 0, c->lay.stride, c->lay.nregions, c->lay.span[0],
                           c->lay.span[1], c->lay.unordered, c->lay.has_self, c->simple_sorted ? 1 : 0,
                           c->lay.first_ran ? 1 : 0, c->unit ? 1 : 0, c->roff.empty() ? 0 : c->roff[c->rank], c->nghost,
                           c->lnv, c->lne};
    memcpy(info16, v, sizeof v);
  }
  const bool has_bfs = c->lay.want && c->relabel && c->lnv > 0, has_perm = c->relabel && c->lnv > 0;
  if ((bfs_key && !has_bfs) || ((perm || inv || lab) && !has_perm) || ((rowptr2 || tails2) && !c->reordered) ||
      (weights2 && (!c->reordered || c->unit)))
    return fail("mv_layout_readback: the last run did not build that array");
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const size_t nv = (size_t)c->lnv, ne = (size_t)c->lne;
  if (rowptr) CK(cudaMemcpyAsync(rowptr, c->rowptr.p, sizeof(uint32_t) * (nv + 1), cudaMemcpyDeviceToHost, s));
  if (tails && ne) CK(cudaMemcpyAsync(tails, c->lay.tails, sizeof(int32_t) * ne, cudaMemcpyDeviceToHost, s));
  if (bfs_key) CK(cudaMemcpyAsync(bfs_key, c->bfs_key.p, sizeof(uint32_t) * nv, cudaMemcpyDeviceToHost, s));
  if (perm) CK(cudaMemcpyAsync(perm, c->perm.p, sizeof(int32_t) * nv, cudaMemcpyDeviceToHost, s));
  if (inv) CK(cudaMemcpyAsync(inv, c->inv.p, sizeof(int32_t) * nv, cudaMemcpyDeviceToHost, s));
  if (lab) CK(cudaMemcpyAsync(lab, c->lab.p, sizeof(int32_t) * nv, cudaMemcpyDeviceToHost, s));
  if (rowptr2) CK(cudaMemcpyAsync(rowptr2, c->rowptr2.p, sizeof(uint32_t) * (nv + 1), cudaMemcpyDeviceToHost, s));
  if (tails2 && ne) CK(cudaMemcpyAsync(tails2, c->tails2.p, sizeof(int32_t) * ne, cudaMemcpyDeviceToHost, s));
  if (weights2 && ne) CK(cudaMemcpyAsync(weights2, c->weights2.p, sizeof(double) * ne, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

// ---- USE_32_BIT_GRAPH surface (utils.hpp:72-82): int32 offsets, {int32 tail; float weight} records, float results ----
int mvgpu_upload_shard32(mvgpu_ctx *c, int32_t nv_global, const int32_t *parts, int32_t lnv, int32_t lne,
                         const int32_t *edge_indices, const void *edge_list8) {
  if (!c || !parts || !edge_indices || (lne && !edge_list8)) return fail("null argument");
  CK(cudaSetDevice(c->device));
  std::vector<int64_t> parts64(parts, parts + c->nranks + 1);
  TRY(set_graph(c, nv_global, parts64.data(), lnv, lne));
  DevBuf<Edge8> e8;
  DevBuf<int32_t> rp32;
  TRY(e8.ensure((size_t)lne)); TRY(rp32.ensure((size_t)lnv + 1));
  TRY(c->in_edges.ensure(lne)); TRY(c->in_rowptr.ensure(lnv + 1));
  cudaEvent_t a = get_event(c, 0), b = get_event(c, 1);
  CK(cudaEventRecord(a, c->stream));
  CK(cudaMemcpyAsync(rp32.p, edge_indices, sizeof(int32_t) * ((size_t)lnv + 1), cudaMemcpyHostToDevice, c->stream));
  if (lne) CK(cudaMemcpyAsync(e8.p, edge_list8, sizeof(Edge8) * (size_t)lne, cudaMemcpyHostToDevice, c->stream));
  k_widen_shard32<<<grid_for(std::max<long long>(lne, lnv + 1), 256, c->num_sms, 16), 256, 0, c->stream>>>(e8.p, lne, rp32.p, lnv, c->in_edges.p,
                                                                                                      c->in_rowptr.p);
  CK(cudaEventRecord(b, c->stream));
  CK(cudaEventSynchronize(b));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, a, b));
  set_source(c, c->in_rowptr.p, c->in_edges.p, nullptr, true, ms * 1e-3,
             (long long)sizeof(int32_t) * (lnv + 1) + (long long)sizeof(Edge8) * lne);
  return 0;
}

int mvgpu_louvain32(mvgpu_ctx *c, float lower, float thresh, int *iters, float *modularity) {
  if (!c || !iters || !modularity) return fail("null argument");
  if (!c->f32) return fail("mvgpu_louvain32 needs a shard uploaded with mvgpu_upload_shard32");
  if (c->have_init || c->opt_stop_after) return fail("mvgpu_louvain32 supports neither an initial assignment nor stop_after");
  if (c->have_mov) return fail("mvgpu_louvain32 does not support a movable set (mvgpu_set_movable)");
  double mod = 0.0;
  TRY(run_louvain(c, (double)lower, (double)thresh, iters, &mod));
  *modularity = (float)mod;
  return 0;
}

int mvgpu_get_communities32(mvgpu_ctx *c, int32_t *out) {
  if (!c || !out) return fail("null argument");
  if (!c->final_on_shard) return fail(kNoRunOnShard);
  if (c->lnv == 0) return 0;
  TRY(final_in_caller_order(c));
  CK(cudaMemcpyAsync(out, c->final_orig.p, sizeof(int32_t) * c->lnv, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int mvgpu_dist_louvain_method(int device, int64_t nv, int64_t ne_local, const int64_t *edge_indices, const void *edge_list,
                              double lower, double thresh, int *iters, double *modularity, int64_t *comm_out) {
  mvgpu_ctx *c = nullptr;
  TRY(mvgpu_create(&c, device, 0, 1));
  const int64_t parts[2] = {0, nv};
  int rc = mvgpu_upload_shard(c, nv, parts, nv, ne_local, edge_indices, edge_list);
  if (!rc) rc = mvgpu_louvain(c, lower, thresh, iters, modularity);
  if (!rc && comm_out) rc = mvgpu_get_communities(c, comm_out);
  const std::string keep = g_err;
  mvgpu_destroy(c);
  if (rc) g_err = keep;
  return rc;
}

}  // extern "C"
