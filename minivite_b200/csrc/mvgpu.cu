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
// one ncclAllReduce of two doubles.  The setup exchanges (ghost lists, counts, IPC handles) always use NCCL.
#include <cuda_runtime.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cub/cub.cuh>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include "../../include/mvgpu.h"
#include "host_comm.hpp"
#include "kernels.cuh"
#include "scan_pipe.cuh"
#include "scan_queue.cuh"
#include "nccl_dyn.h"
#include "rgg_gpu.cuh"

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

struct PeerBlob {            // what every rank publishes about its community arrays
  cudaIpcMemHandle_t h[10];
  unsigned long long raw[10];
  int pid, device, unit, pad;
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
  DevBuf<long long> wide;
  void *h_bounce[2] = {nullptr, nullptr};
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
  int peers_unit = -1;
  void *last_ptrs[10] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  unsigned last_gens[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  // options
  int opt_trace = 0, opt_force_weighted = 0, opt_scan_variant = 6, opt_cache_policy = 5, opt_reorder = 2, opt_region = 512, opt_comm_mode = 1, opt_compact_upload = 0, opt_host_threads = 8, opt_first_iter = 1, opt_host_transport = 0;
  long long opt_upload_chunk = 4LL << 20;
  long long opt_max_iters = 10000, opt_force_heavy_deg = 0;
  // results
  bool unit = true;
  bool f32 = false;                    // shard came through mvgpu_upload_shard32: float-build arithmetic (see mvgpu.h)
  double constant = 0.0;
  int32_t *d_final = nullptr;          // currComm at exit (points into comm_a/comm_b)
  bool final_ready = false;            // final_orig holds the assignment of the last run in the caller's numbering
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
};

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
  long long *d = reinterpret_cast<Scalars *>(c->scratch.p)->counts;
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
  long long *d = reinterpret_cast<Scalars *>(c->scratch.p)->counts;
  NK(g_nccl.AllReduce(d, d, 1, ncclInt64, ncclSum, c->comm, c->stream));
  return coll_sync(c);
}

int set_graph(mvgpu_ctx *c, long long nv_global, const int64_t *parts, long long lnv, long long lne) {
  if (c->nranks > kMaxRanks) return fail("too many ranks");
  if (nv_global < 0 || lnv < 0 || lne < 0) return fail("negative graph size");
  if (nv_global >= (1LL << 31)) return fail("nv_global >= 2^31: 32-bit community ids would overflow (not supported)");
  if (lne >= (1LL << 32)) return fail("lne >= 2^32 per shard: 32-bit edge offsets would overflow (not supported)");
  c->parts.assign(parts, parts + c->nranks + 1);
  if (c->parts[0] != 0 || c->parts[c->nranks] != nv_global) return fail("parts[] must run from 0 to nv_global");
  for (int r = 0; r < c->nranks; r++) if (c->parts[r + 1] < c->parts[r]) return fail("parts[] not monotone");
  c->base = c->parts[c->rank];
  c->bound = c->parts[c->rank + 1];
  if (c->bound - c->base != lnv) return fail("lnv does not match parts[rank+1]-parts[rank]");
  c->nv_global = nv_global; c->lnv = lnv; c->lne = lne;
  c->have_graph = true;
  c->peers_ready = false;
  return 0;
}

// ---- multi-GPU: publish/obtain peer pointers for the community arrays -------------------------
int setup_peers(mvgpu_ctx *c, int unit) {
  PeerTable &pt = c->pt;
  pt.nranks = c->nranks; pt.rank = c->rank;
  for (int r = 0; r <= c->nranks; r++) pt.parts[r] = c->parts[r];
  if (c->nranks == 1) {
    pt.lab[0] = c->relabel ? c->lab.p : nullptr;
    pt.cdeg[0] = c->cdeg.p; pt.csize[0] = c->csize.p; pt.upd[0] = c->upd.p; pt.cinfo_w[0] = c->cinfo_w.p; pt.usize[0] = c->usize.p; pt.udeg[0] = c->udeg.p;
    return 0;
  }
  void *ptrs[10] = {unit ? (void *)c->cdeg.p : nullptr, unit ? (void *)c->csize.p : nullptr, unit ? (void *)c->upd.p : nullptr,
                    unit ? nullptr : (void *)c->cinfo_w.p, unit ? nullptr : (void *)c->usize.p,
                    unit ? nullptr : (void *)c->udeg.p, c->relabel ? (void *)c->lab.p : nullptr,
                    (void *)c->comm_a.p, (void *)c->comm_b.p, (void *)c->p2p.p};
  if (c->peers_ready) return 0;            // same graph, same buffers: tables are still valid
  // IPC handles are expensive to (re)open: skip the exchange when no rank's buffers moved since the last one
  const unsigned gens[10] = {c->cdeg.gen, c->csize.gen, c->upd.gen, c->cinfo_w.gen, c->usize.gen, c->udeg.gen, c->lab.gen,
                             c->comm_a.gen, c->comm_b.gen, c->p2p.gen};
  long long changed = c->ipc_valid ? 0 : 1;
  for (int k = 0; k < 10; k++) if (ptrs[k] != c->last_ptrs[k] || (ptrs[k] && gens[k] != c->last_gens[k])) changed = 1;
  TRY(coll_allreduce_i64(c, &changed, 1, true));
  if (changed) {
  for (void *p : c->ipc_opened) cudaIpcCloseMemHandle(p);
  c->ipc_opened.clear();
  c->ipc_valid = false;
  PeerBlob mine;
  memset(&mine, 0, sizeof mine);
  for (int k = 0; k < 10; k++) {
    mine.raw[k] = (unsigned long long)ptrs[k];
    if (ptrs[k]) CK(cudaIpcGetMemHandle(&mine.h[k], ptrs[k]));
  }
  mine.pid = (int)getpid(); mine.device = c->device; mine.unit = unit;
  std::vector<PeerBlob> all(c->nranks);
  TRY(coll_allgather(c, &mine, all.data(), sizeof(PeerBlob)));
  for (int r = 0; r < c->nranks; r++) {
    void *q[10] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    if (all[r].unit != unit) return fail("ranks disagree on the unit-weight path");
    if (r == c->rank) { for (int k = 0; k < 10; k++) q[k] = ptrs[k]; }
    else if (all[r].pid == mine.pid) {           // same process (threads): plain UVA pointers + peer access
      if (all[r].device != c->device) {          // ranks sharing one device need no peer mapping at all
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, c->device, all[r].device));
        if (!can) return fail("GPU " + std::to_string(c->device) + " cannot access peer GPU " + std::to_string(all[r].device));
        cudaError_t e = cudaDeviceEnablePeerAccess(all[r].device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e);
        cudaGetLastError();
      }
      for (int k = 0; k < 10; k++) q[k] = (void *)all[r].raw[k];
    } else {
      for (int k = 0; k < 10; k++)
        if (all[r].raw[k]) {
          CK(cudaIpcOpenMemHandle(&q[k], all[r].h[k], cudaIpcMemLazyEnablePeerAccess));
          c->ipc_opened.push_back(q[k]);
        }
    }
    pt.cdeg[r] = (const uint32_t *)q[0]; pt.csize[r] = (const int32_t *)q[1]; pt.upd[r] = (unsigned long long *)q[2];
    pt.cinfo_w[r] = (const CommW *)q[3]; pt.usize[r] = (long long *)q[4]; pt.udeg[r] = (double *)q[5];
    pt.lab[r] = (const int32_t *)q[6];
    c->peer_comm[0][r] = (int32_t *)q[7]; c->peer_comm[1][r] = (int32_t *)q[8];
    c->pp.st[r] = (P2PState *)q[9];
  }
  for (int k = 0; k < 10; k++) { c->last_ptrs[k] = ptrs[k]; c->last_gens[k] = gens[k]; }
  c->ipc_valid = true;
  }
  // where my send segments land in each peer's community array: its lnv + its receive offset for me
  {
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
  }
  c->peers_ready = true;
  c->peers_unit = unit * 2 + c->relabel;
  return 0;
}

template <bool UNIT, bool MULTI, bool TRACE>
int launch_scan_t(mvgpu_ctx *c, const ScanParams &sp, bool first) {
  const size_t smem = UNIT ? sizeof(int32_t) * 2 * kECap : sizeof(int32_t) * kECap + sizeof(double) * kECap;
  static bool attr_done = false;
  if (!attr_done) {
    CK(cudaFuncSetAttribute(k_scan_ws<UNIT, MULTI, TRACE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  const int tiles = (int)((c->lnv + kTileV - 1) / kTileV);
  if (tiles > 0 && c->opt_scan_variant >= 5 && c->scan_kernel == 5 && UNIT && !first) {
    // k_scan_pw's pipeline with a per-warp ring of hard vertices (scan_queue.cuh); iteration 1 and the weighted path
    // stay with k_scan_pw
    static int pq_ctas_per_sm = 0;
    if (!pq_ctas_per_sm) {
      CK(cudaFuncSetAttribute(k_scan_pq<MULTI, TRACE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pq_smem_bytes()));
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pq_ctas_per_sm, k_scan_pq<MULTI, TRACE>, kPwWarps * 32, pq_smem_bytes()));
      if (pq_ctas_per_sm < 1) return fail("k_scan_pq cannot be made resident");
    }
    const int ngroups = (int)((c->lnv + 31) / 32);
    const int grid = std::min((ngroups + kPwWarps - 1) / kPwWarps, pq_ctas_per_sm * c->num_sms);
    k_scan_pq<MULTI, TRACE><<<grid, kPwWarps * 32, pq_smem_bytes(), c->stream>>>(sp, ngroups);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  } else if (tiles > 0 && c->opt_scan_variant >= 4) {
    // persistent warps, TMA-fed double buffer (scan_pipe.cuh): one CTA slot per resident block, warps stride over groups
    static int pw_ctas_per_sm = 0;
    if (!pw_ctas_per_sm) {
      CK(cudaFuncSetAttribute(k_scan_pw<UNIT, MULTI, TRACE, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pw_smem_bytes<UNIT>()));
      CK(cudaFuncSetAttribute(k_scan_pw<UNIT, MULTI, TRACE, UNIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pw_smem_bytes<UNIT>()));
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pw_ctas_per_sm, k_scan_pw<UNIT, MULTI, TRACE, false>, kPwWarps * 32, pw_smem_bytes<UNIT>()));
      if (pw_ctas_per_sm < 1) return fail("k_scan_pw cannot be made resident");
    }
    const int ngroups = (int)((c->lnv + 31) / 32);
    const int grid = std::min((ngroups + kPwWarps - 1) / kPwWarps, pw_ctas_per_sm * c->num_sms);
    if (UNIT && first) k_scan_pw<UNIT, MULTI, TRACE, UNIT><<<grid, kPwWarps * 32, pw_smem_bytes<UNIT>(), c->stream>>>(sp, ngroups);
    else k_scan_pw<UNIT, MULTI, TRACE, false><<<grid, kPwWarps * 32, pw_smem_bytes<UNIT>(), c->stream>>>(sp, ngroups);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  } else if (tiles > 0) {
    k_scan_ws<UNIT, MULTI, TRACE><<<tiles, kTileV, UNIT ? sizeof(int32_t) * kECap : smem, c->stream>>>(sp);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  }
  if (c->nheavy > 0) {
    k_scan_heavy<UNIT, MULTI, TRACE><<<(int)c->nheavy, 256, 0, c->stream>>>(sp);
    c->tm.kernel_launches++; c->tm.scan_launches++;
  }
  CK(cudaGetLastError());
  return 0;
}

int launch_scan(mvgpu_ctx *c, const ScanParams &sp, bool first) {
  const bool multi = c->nranks > 1, tr = c->opt_trace != 0;
#define MV_CASE(U, M, T) if (c->unit == U && multi == M && tr == T) return launch_scan_t<U, M, T>(c, sp, first);
  MV_CASE(true, false, false) MV_CASE(true, false, true) MV_CASE(true, true, false) MV_CASE(true, true, true)
  MV_CASE(false, false, false) MV_CASE(false, false, true) MV_CASE(false, true, false) MV_CASE(false, true, true)
#undef MV_CASE
  return fail("unreachable");
}

int exchange_ghosts(mvgpu_ctx *c, int32_t *comm);
int final_in_caller_order(mvgpu_ctx *c);

// ---- setup: reference-format arrays -> compact graph, ghosts, init ------------------------------
int setup_run(mvgpu_ctx *c) {
  cudaStream_t s = c->stream;
  const int nsm = c->num_sms;
  TRY(c->scratch.ensure(sizeof(Scalars)));
  Scalars *d_sc = reinterpret_cast<Scalars *>(c->scratch.p);
  Scalars h;
  CK(cudaMemsetAsync(d_sc, 0, sizeof(Scalars), s));
  const long long lnv = c->lnv, lne = c->lne;

  // pass 1 over the edges: unit weights? how many non-owned tails? (+ input validation).  The compact upload
  // format has answered all of that on the host already.
  const bool compact_in = c->d_tails32 != nullptr;
  const bool fused_stats = !compact_in && c->nranks == 1;      // single rank: statistics ride on the conversion pass
  if (fused_stats) {
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
  // input errors are agreed on across ranks before anybody returns: a rank that left alone would leave its peers
  // blocked in the next collective
  std::string input_err;
  if (h.st.bad_tail) input_err = "edge tail outside [0, nv)";
  else if (h.bad_rowptr) input_err = "edge_indices malformed (must start at 0, end at lne and never decrease)";
  else if (c->nranks == 1 && h.st.nremote) input_err = "non-local tail in a single-rank graph";
  c->maxdeg = h.maxdeg;
  int unit = (!h.st.nonunit && !c->opt_force_weighted) ? 1 : 0;
  if (input_err.empty() && compact_in && !unit) input_err = "force_weighted needs the full edge records: set compact_upload=0";

  // global agreement on the path + on 2m < 2^31 needs the total weight; the weight total itself comes
  // from the vertex-init kernel below, so first settle `unit` from the flags (ne bound checked after).
  long long ne_global = lne;
  if (c->nranks > 1) {
    // exported (peer-mapped) arrays that this run may have to grow: CUDA IPC requires every peer to close its
    // mapping before the owner frees the block, so that is agreed on here and done collectively
    const size_t need_v = (size_t)lnv, need_s = (size_t)(lnv + (long long)h.st.nremote);
    const bool grow = c->ipc_valid && ((c->cdeg.p && c->cdeg.cap < need_v) || (c->cinfo_w.p && c->cinfo_w.cap < need_v) ||
                                       (c->lab.p && c->lab.cap < need_v) || c->comm_a.cap < need_s || c->comm_b.cap < need_s);
    long long hv[4] = {unit ? 0 : 1, lne, input_err.empty() ? 0 : 1, grow ? 1 : 0};
    TRY(coll_allreduce_i64(c, hv, 4, false));
    unit = hv[0] == 0;
    ne_global = hv[1];
    if (hv[2] && input_err.empty()) input_err = "another rank rejected its shard";
    if (hv[3]) {
      for (void *q : c->ipc_opened) cudaIpcCloseMemHandle(q);
      c->ipc_opened.clear();
      c->ipc_valid = false;
      c->peers_ready = false;
      TRY(coll_barrier(c));                       // all mappings are closed before any owner reallocates
    }
  }
  if (!input_err.empty()) return fail(input_err);
  if (unit && ne_global >= (1LL << 31)) unit = 0;   // packed 32-bit degree deltas need 2m < 2^31
  c->unit = unit != 0;

  // pass 2: tails -> slots, weights split off, remote tails listed
  const long long nremote = (long long)h.st.nremote;
  if (nremote) { TRY(c->remote_list.ensure(nremote)); TRY(c->remote_pos.ensure(nremote)); }
  const uint32_t *src_rowptr = c->rowptr.p;
  const int32_t *src_tails = nullptr;
  const double *src_weights = nullptr;
  if (compact_in && c->nranks == 1) {
    src_tails = c->d_tails32;                       // global id == local slot: the uploaded array is used as is (read-only)
    if (!c->unit) {                                 // 2m >= 2^31: fp64 path on a shard that arrived without weights
      TRY(c->weights.ensure(lne + 4));
      k_fill_ones<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->weights.p, lne);
      c->tm.kernel_launches++;
      src_weights = c->weights.p;
    }
  } else if (fused_stats) {
    src_tails = c->tails.p;                         // converted by the fused pass above
    if (!c->unit) {
      TRY(c->weights.ensure(lne + 4));
      k_extract_weights<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->d_edges, lne, c->weights.p);
      c->tm.kernel_launches++;
      src_weights = c->weights.p;
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
    if (compact_in && !c->unit) {                   // a peer's shard is weighted (or 2m >= 2^31): this one's weights are all 1.0
      k_fill_ones<<<grid_for(lne, 256, nsm, 16), 256, 0, s>>>(c->weights.p, lne);
      c->tm.kernel_launches++;
    }
    src_tails = c->tails.p;
    src_weights = c->unit ? nullptr : c->weights.p;
  }

  // ghost discovery (exchangeVertexReqs, dspl.hpp:1106-1272): sorted unique non-owned tails
  c->nghost = 0; c->nsend = 0;
  c->rcount.assign(c->nranks, 0); c->scount.assign(c->nranks, 0);
  c->roff.assign(c->nranks + 1, 0); c->soff.assign(c->nranks + 1, 0);
  if (c->nranks > 1) {
    if (nremote) {
      DevBuf<long long> &sorted = c->sorted_tmp;   // grow-only: no cudaMalloc/cudaFree inside the timed setup after the first run
      TRY(sorted.ensure(nremote));
      TRY(c->ghost_gid.ensure(nremote));
      size_t tb1 = 0, tb2 = 0;
      int bits = 1;
      while ((1LL << bits) < c->nv_global && bits < 63) bits++;
      cub::DeviceRadixSort::SortKeys(nullptr, tb1, c->remote_list.p, sorted.p, nremote, 0, bits, s);
      cub::DeviceSelect::Unique(nullptr, tb2, sorted.p, c->ghost_gid.p, &d_sc->nunique, nremote, s);
      TRY(c->cub_tmp.ensure(std::max(tb1, tb2)));
      size_t tb = c->cub_tmp.cap;
      CK(cub::DeviceRadixSort::SortKeys(c->cub_tmp.p, tb, c->remote_list.p, sorted.p, nremote, 0, bits, s));
      tb = c->cub_tmp.cap;
      CK(cub::DeviceSelect::Unique(c->cub_tmp.p, tb, sorted.p, c->ghost_gid.p, &d_sc->nunique, nremote, s));
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
    {
      std::vector<long long> allc((size_t)c->nranks * c->nranks);
      TRY(coll_allgather(c, c->rcount.data(), allc.data(), sizeof(long long) * c->nranks));
      for (int r = 0; r < c->nranks; r++) c->scount[r] = allc[(size_t)r * c->nranks + c->rank];
    }
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
  }

  // ---- locality renumbering (see kernels.cuh): decide, then BFS regions -> sort -> permute the compact CSR
  c->reordered = false;
  c->relabel = 0;
  {
    int want = c->opt_reorder == 1 ? 1 : 0;
    if (c->opt_reorder == 2 && lnv >= 65536) {
      // auto: renumber when the given numbering has no locality (mean |tail - v| above lnv/64 on a vertex sample)
      k_span_sample<<<grid_for(lnv / 64 + 1, 256, nsm), 256, 0, s>>>((int)lnv, src_rowptr, src_tails, 64, &d_sc->span_sum, &d_sc->span_cnt);
      c->tm.kernel_launches++;
      unsigned long long sp2[2];
      CK(cudaMemcpyAsync(sp2, &d_sc->span_sum, sizeof sp2, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      if (sp2[1] > 0 && (double)sp2[0] / (double)sp2[1] > (double)lnv / 64.0) want = 1;
    }
    int any = want;
    if (c->nranks > 1) {
      long long hv = want;
      TRY(coll_allreduce_i64(c, &hv, 1, true));
      any = hv != 0;
    }
    c->relabel = any;                       // labels are needed everywhere as soon as one rank renumbers
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
        int ilnv = (int)lnv, stride = c->opt_region, ml = max_levels;
        const uint32_t *rp = src_rowptr; const int32_t *tl = src_tails; uint32_t *key = c->bfs_key.p;
        // the BFS queue and its level bitmaps (4 bits per vertex) live in ids and sortkey2, which k_bfs_sortkeys and the
        // sort only write after the BFS
        int32_t *q = c->ids.p; unsigned int *lc = c->bfs_level_count.p; uint32_t *lm = c->sortkey2.p;
        void *args[] = {&ilnv, &rp, &tl, &key, &stride, &ml, &q, &lc, &lm};
        CK(cudaLaunchCooperativeKernel((void *)k_msbfs, dim3(occ * nsm), dim3(256), args, 0, s));
        // sort by (region, level): only the bits that can be set take part (one radix pass less than a 32-bit sort)
        const long long nregions = (lnv + stride - 1) / stride;
        int sort_bits = (int)kBfsLevelBits;
        while ((1LL << (sort_bits - (int)kBfsLevelBits)) <= nregions && sort_bits < 32) sort_bits++;
        const unsigned int unreached_key = sort_bits >= 32 ? 0xFFFFFFFFu : ((1u << sort_bits) - 1u);
        k_bfs_sortkeys<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->bfs_key.p, c->sortkey.p, c->ids.p, unreached_key);
        size_t tb = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tb, c->sortkey.p, c->sortkey2.p, c->ids.p, c->perm.p, (int)lnv, 0, sort_bits, s);
        TRY(c->cub_tmp.ensure(tb));
        tb = c->cub_tmp.cap;
        CK(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, c->sortkey.p, c->sortkey2.p, c->ids.p, c->perm.p, (int)lnv, 0, sort_bits, s));
        c->tm.kernel_launches += 3;
      } else {
        // another rank renumbers, this one keeps its order: identity permutation, labels still required
        k_bfs_sortkeys<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->bfs_key.p, c->sortkey.p, c->perm.p, 0xFFFFFFFFu);
        c->tm.kernel_launches++;
      }
      k_perm_inverse<<<grid_for(lnv + 1, 256, nsm), 256, 0, s>>>((int)lnv, c->perm.p, c->base, want ? nullptr : c->inv.p, c->lab.p, src_rowptr, c->deg_new.p);
      c->tm.kernel_launches++;
      if (want) {
        // inv[old] = new as a second radix sort (keys perm, values the ids 0..lnv-1 still in c->ids): lnv random 4-byte
        // stores inv[perm[i]] = i cost more than twice as much as the sort's bucketed scatters (DESIGN.md §3.3)
        int bits = 1;
        while ((1LL << bits) < lnv && bits < 31) bits++;
        const uint32_t *pk = reinterpret_cast<const uint32_t *>(c->perm.p);
        size_t tb = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tb, pk, c->sortkey2.p, c->ids.p, c->inv.p, (int)lnv, 0, bits, s);
        TRY(c->cub_tmp.ensure(tb));
        tb = c->cub_tmp.cap;
        CK(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, pk, c->sortkey2.p, c->ids.p, c->inv.p, (int)lnv, 0, bits, s));
        tb = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tb, c->deg_new.p, c->rowptr2.p, (int)lnv + 1, s);
        TRY(c->cub_tmp.ensure(tb));
        tb = c->cub_tmp.cap;
        CK(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, tb, c->deg_new.p, c->rowptr2.p, (int)lnv + 1, s));
        k_permute_adj<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->perm.p, c->inv.p, src_rowptr, src_tails, src_weights,
                                                               c->rowptr2.p, c->tails2.p, c->unit ? nullptr : c->weights2.p,
                                                               (int)c->roff[c->rank], &d_sc->unordered);
        c->tm.kernel_launches += 3;
        src_rowptr = c->rowptr2.p;
        src_tails = c->tails2.p;
        src_weights = c->unit ? nullptr : c->weights2.p;
        c->reordered = true;
      }
      CK(cudaEventRecord(r1, s));
    }
    // peers asked for my vertices by ORIGINAL id: the send list holds their current (internal) local index
    if (c->relabel && c->nsend) {
      k_apply_inv<<<grid_for(c->nsend, 256, nsm), 256, 0, s>>>(c->send_lid.p, (int)c->nsend, c->inv.p);
      c->tm.kernel_launches++;
    }
  }

  c->a_rowptr = src_rowptr; c->a_tails = src_tails; c->a_weights = src_weights;

  // state arrays
  // sized for the bound the collective "does an exported array have to grow?" test can evaluate before the ghosts are
  // known (lnv + #non-owned edge tails >= lnv + nghost), so that a repeated run never looks like a growing one
  const long long nslots = lnv + c->nghost;
  TRY(c->comm_a.ensure(std::max(nslots, lnv + nremote)));
  TRY(c->comm_b.ensure(std::max(nslots, lnv + nremote)));
  if (c->unit) { TRY(c->cdeg.ensure(lnv)); TRY(c->csize.ensure(lnv)); TRY(c->upd.ensure(lnv)); TRY(c->self_i.ensure(lnv)); }
  else { TRY(c->cinfo_w.ensure(lnv)); TRY(c->usize.ensure(lnv)); TRY(c->udeg.ensure(lnv)); TRY(c->vdeg.ensure(lnv)); TRY(c->self_d.ensure(lnv)); }
  TRY(c->acc.ensure((size_t)c->opt_max_iters + 2));
  CK(cudaMemsetAsync(c->acc.p, 0, sizeof(Acc) * ((size_t)c->opt_max_iters + 2), s));

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
  // fetch it with the same all-to-all-v the iterations use
  if (c->nranks > 1) TRY(exchange_ghosts(c, c->comm_a.p));

  // high-degree vertices
  // largest degree the tile kernels take: one staging buffer (minus the 16-byte alignment slack of the bulk copies)
  const long long tile_cap = c->opt_scan_variant >= 4 ? (c->unit ? PwCap<true>::value : PwCap<false>::value) - 4 : kECap;
  const long long heavy_deg = (c->opt_force_heavy_deg > 0) ? std::min<long long>(c->opt_force_heavy_deg, tile_cap) : tile_cap;
  c->nheavy = 0;
  if (c->maxdeg > heavy_deg) {
    TRY(c->heavy_list.ensure(lnv));
    k_collect_heavy<<<grid_for(lnv, 256, nsm), 256, 0, s>>>((int)lnv, c->a_rowptr, (unsigned int)heavy_deg, c->heavy_list.p, &d_sc->heavy_count);
    c->tm.kernel_launches++;
  }

  // 1/(2m): MPI_Allreduce of the local degree sums (dspl.hpp:109-130)
  if (c->nranks > 1 && !c->hc.is_open()) NK(g_nccl.AllReduce(&d_sc->total_weight, &d_sc->total_weight, 1, ncclDouble, ncclSum, c->comm, s));
  CK(cudaMemcpyAsync(&h, d_sc, sizeof h, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (c->nranks > 1 && c->hc.is_open()) c->hc.allreduce(&h.total_weight, 1, [](double a, double b) { return a + b; });
  c->constant = 1.0 / h.total_weight;
  if (c->f32) c->constant = (double)(float)(1.0 / (double)(float)h.total_weight);   // dspl.hpp:129 with GraphWeight = float
  const int has_self = h.has_self ? 1 : 0;
  c->simple_sorted = c->unit && !h.unordered && !has_self;
  if (c->maxdeg > heavy_deg) {
    c->nheavy = h.heavy_count;
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
  }
  if (c->nranks > 1) {
    TRY(c->p2p.ensure(1));
    if (!c->p2p_zeroed) { CK(cudaMemsetAsync(c->p2p.p, 0, sizeof(P2PState), s)); CK(cudaStreamSynchronize(s)); c->p2p_zeroed = true; }
  }
  TRY(setup_peers(c, c->unit ? 1 : 0));
  c->tm.unit_weight = c->unit ? 1 : 0;
  c->scan_has_self = has_self;
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

int run_louvain(mvgpu_ctx *c, double lower, double thresh, int *iters_out, double *mod_out) {
  if (!c->have_graph) return fail("no graph uploaded");
  if (c->nranks > 1 && !c->comm && !c->hc.is_open()) return fail("mvgpu_comm_init has not been called");
  if (c->nranks > 1 && !c->comm && c->opt_comm_mode != 1) return fail("comm_mode=0 (NCCL data plane) needs the NCCL communicator: host_transport=1 supports comm_mode=1 only");
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

  Scalars *d_sc = reinterpret_cast<Scalars *>(c->scratch.p);
  int32_t *cur = c->comm_a.p, *tgt = c->comm_b.p;
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
  c->last_sp = sp;

  struct HostMail { Acc acc; double red2[2]; unsigned long long tr2[2]; unsigned int p2p_error; };
  HostMail *mail = reinterpret_cast<HostMail *>(c->h_pin);
  const size_t ev_iter0 = ev;
  double prevMod = lower, currMod = -1.0;
  int numIters = 0, auto_choice = 4;
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
    TRY(launch_scan(c, sp, numIters == 1 && c->simple_sorted && c->opt_first_iter && c->opt_scan_variant >= 4 && !c->f32));
    CK(cudaEventRecord(e1, s));
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
        NK(g_nccl.AllReduce(d_sc->counts, d_sc->counts, 1, ncclInt64, ncclSum, c->comm, s));
      }
    }
    CK(cudaEventRecord(e2, s));
    if (c->unit) k_fold_unit<<<grid_for((c->lnv >> 2) + 1, 256, c->num_sms, 8), 256, 0, s>>>((int)c->lnv, c->cdeg.p, c->csize.p, c->upd.p, acc, acc - 1);
    else k_fold_w<<<fold_grid, 256, 0, s>>>((int)c->lnv, c->cinfo_w.p, c->usize.p, c->udeg.p, acc);
    c->tm.kernel_launches++;
    CK(cudaEventRecord(e3, s));
    double e_xx, a2_x;
    unsigned long long moved = 0, hash = 0;
    if (p2p) {
      k_p2p_allreduce<<<1, 32, 0, s>>>(c->pp, ++c->p2p_epoch, acc, c->unit ? 1 : 0, d_sc->red2, d_sc->tr2);   // dspl.hpp:441
      c->tm.kernel_launches++;
      CK(cudaMemcpyAsync(mail->red2, d_sc->red2, sizeof mail->red2 + sizeof mail->tr2, cudaMemcpyDeviceToHost, s));
      CK(cudaMemcpyAsync(&mail->p2p_error, &c->p2p.p->error, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      if (mail->p2p_error) return fail("peer-memory collective timed out (a peer rank is gone)");
      e_xx = mail->red2[0]; a2_x = mail->red2[1];
      moved = mail->tr2[0]; hash = mail->tr2[1];
    } else if (c->nranks > 1) {
      k_acc_to_double<<<1, 32, 0, s>>>(acc, c->unit ? 1 : 0, d_sc->red2);
      c->tm.kernel_launches++;
      NK(g_nccl.AllReduce(d_sc->red2, d_sc->red2, 2, ncclDouble, ncclSum, c->comm, s));   // dspl.hpp:441
      CK(cudaMemcpyAsync(mail->red2, d_sc->red2, sizeof mail->red2, cudaMemcpyDeviceToHost, s));
      if (c->opt_trace) {
        k_trace_to_u64<<<1, 32, 0, s>>>(acc, d_sc->tr2);
        c->tm.kernel_launches++;
        NK(g_nccl.AllReduce(d_sc->tr2, d_sc->tr2, 2, ncclUint64, ncclSum, c->comm, s));
        CK(cudaMemcpyAsync(mail->tr2, d_sc->tr2, sizeof mail->tr2, cudaMemcpyDeviceToHost, s));
      }
      CK(cudaStreamSynchronize(s));
      e_xx = mail->red2[0]; a2_x = mail->red2[1];
      moved = mail->tr2[0]; hash = mail->tr2[1];
    } else {
      CK(cudaMemcpyAsync(&mail->acc, acc, sizeof(Acc), cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      e_xx = c->unit ? (double)mail->acc.le_u : mail->acc.le_d;
      a2_x = c->unit ? (double)mail->acc.la2_u : mail->acc.la2_d;
      moved = mail->acc.moved; hash = mail->acc.hash;
    }
    if (c->opt_scan_variant == 6 && numIters == 4) {           // iterations 2..4 have completed (the stream was just synchronised)
      float t2 = 0, t3 = 0, t4 = 0;
      CK(cudaEventElapsedTime(&t2, c->events[ev_iter0 + 4 * 1], c->events[ev_iter0 + 4 * 1 + 1]));
      CK(cudaEventElapsedTime(&t3, c->events[ev_iter0 + 4 * 2], c->events[ev_iter0 + 4 * 2 + 1]));
      CK(cudaEventElapsedTime(&t4, c->events[ev_iter0 + 4 * 3], c->events[ev_iter0 + 4 * 3 + 1]));
      auto_choice = ((double)t3 * t3 < (double)t2 * t4) ? 5 : 4;
      c->tm.scan_kernel_chosen = auto_choice;
    }
    // dspl.hpp:447-448
    const double cst = c->constant;
    if (c->f32) {                      // GraphWeight = float: every product and the difference round to float
      const float cf = (float)cst;
      volatile float t1f = (float)e_xx * cf;
      volatile float t2af = (float)a2_x * cf;
      volatile float t2f = t2af * cf;
      volatile float df = t1f - t2f;
      currMod = (double)std::fabs(df);
    } else {
    volatile double term1 = e_xx * cst;
    volatile double term2a = a2_x * cst;
    volatile double term2 = term2a * cst;
    currMod = std::fabs(term1 - term2);
    }
    if (c->opt_trace) {
      mvgpu_iter_trace t;
      t.modularity = currMod; t.moved = (int64_t)moved; t.chash = hash;
      c->trace.push_back(t);
    }
    if (c->f32 ? ((float)currMod - (float)prevMod < (float)thresh) : (currMod - prevMod < thresh)) break;   // dspl.hpp:1401-1402
    prevMod = currMod;
    if (prevMod < lower) prevMod = lower;                      // dspl.hpp:1404-1406
    std::swap(cur, tgt);                                       // rotation (dspl.hpp:1408-1422) is a pointer swap
  }
  cudaEvent_t e_end = get_event(c, ev++);
  CK(cudaEventRecord(e_end, s));
  c->d_final = cur;
  c->final_ready = false;
  if (c->nranks > 1) {
    // the assignment in the caller's numbering needs the label arrays of the PEERS (a community may be owned by another
    // rank): resolve it now, while every rank is still inside this call, and leave together -- afterwards a rank may
    // free its arrays (mvgpu_destroy) without a peer still reading them.  Outside the timed region, like the
    // reference's output code is outside its timer.
    TRY(final_in_caller_order(c));
    if (c->opt_comm_mode == 1) { k_p2p_barrier<<<1, 32, 0, s>>>(c->pp, ++c->p2p_epoch); c->tm.kernel_launches++; }
    else TRY(coll_barrier(c));
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

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
// `-p`: random long edges on top of the generated strip (graph.hpp:939-1122; host/rgg.hpp add_random_edges is the
// restatement this follows, including its fixed seed).  Every rank replays all p draw streams (they are cheap and
// sequential) and keeps the records that touch its strip.
static int add_random_edges(mvgpu_ctx *c, const RggParams &P, int64_t nv, int unit, double pct, const double *X3, const double *Y3,
                            long long *lne_io) {
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
  DevBuf<unsigned int> qidx, sq, emit, epos, xidx, sxidx, add, xstart;
  DevBuf<double> xw;
  TRY(dsoff.ensure(p + 1)); TRY(di.ensure(nrande)); TRY(dgj.ensure(nrande));
  TRY(key.ensure(nrande)); TRY(skey.ensure(nrande)); TRY(qidx.ensure(nrande)); TRY(sq.ensure(nrande));
  TRY(emit.ensure(nrande + 1)); TRY(epos.ensure(nrande + 1));
  CK(cudaMemcpyAsync(dsoff.p, soff.data(), sizeof(long long) * (p + 1), cudaMemcpyHostToDevice, s));
  k_rande_draws<<<p, 32, 0, s>>>(R, dsoff.p, di.p, dgj.p);
  k_rande_keys<<<grid_for(nrande, 256, nsm), 256, 0, s>>>(R, dsoff.p, di.p, dgj.p, nrande, c->gen_rowptr.p, c->gen_edges.p, key.p, qidx.p);
  size_t tb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, key.p, skey.p, qidx.p, sq.p, (int)nrande, 0, 64, s);
  TRY(c->cub_tmp.ensure(tb));
  tb = c->cub_tmp.cap;
  CK(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, key.p, skey.p, qidx.p, sq.p, (int)nrande, 0, 64, s));
  CK(cudaMemsetAsync(emit.p + nrande, 0, sizeof(unsigned int), s));
  k_rande_first<<<grid_for(nrande, 256, nsm), 256, 0, s>>>(skey.p, sq.p, nrande, R, dsoff.p, dgj.p, emit.p);
  tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, emit.p, epos.p, (int)(nrande + 1), s);
  TRY(c->cub_tmp.ensure(tb));
  tb = c->cub_tmp.cap;
  CK(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, tb, emit.p, epos.p, (int)(nrande + 1), s));
  unsigned int nextra = 0;
  CK(cudaMemcpyAsync(&nextra, epos.p + nrande, sizeof nextra, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (!nextra) return 0;
  TRY(xkey.ensure(nextra)); TRY(sxkey.ensure(nextra)); TRY(xidx.ensure(nextra)); TRY(sxidx.ensure(nextra)); TRY(xw.ensure(nextra));
  TRY(add.ensure(P.n + 1)); TRY(xstart.ensure(P.n + 1)); TRY(nrow.ensure(P.n + 1));
  CK(cudaMemsetAsync(add.p, 0, sizeof(unsigned int) * (P.n + 1), s));
  k_rande_emit<<<grid_for(nrande, 256, nsm), 256, 0, s>>>(R, P, dsoff.p, di.p, dgj.p, nrande, emit.p, epos.p, unit, X3, Y3, xkey.p, xw.p,
                                                        xidx.p, add.p);
  tb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, xkey.p, sxkey.p, xidx.p, sxidx.p, (int)nextra, 0, 62, s);
  TRY(c->cub_tmp.ensure(tb));
  tb = c->cub_tmp.cap;
  CK(cub::DeviceRadixSort::SortPairs(c->cub_tmp.p, tb, xkey.p, sxkey.p, xidx.p, sxidx.p, (int)nextra, 0, 62, s));
  tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, add.p, xstart.p, (int)(P.n + 1), s);
  TRY(c->cub_tmp.ensure(tb));
  tb = c->cub_tmp.cap;
  CK(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, tb, add.p, xstart.p, (int)(P.n + 1), s));
  k_rande_rowptr<<<grid_for(P.n + 1, 256, nsm), 256, 0, s>>>(c->gen_rowptr.p, xstart.p, P.n, nrow.p);
  const long long lne2 = *lne_io + (long long)nextra;
  DevBuf<Edge16> merged;
  TRY(merged.ensure(lne2));
  k_rande_merge<<<grid_for(P.n, 256, nsm, 16), 256, 0, s>>>(c->gen_rowptr.p, c->gen_edges.p, xstart.p, sxkey.p, sxidx.p, xw.p, P.n, nrow.p,
                                                          merged.p);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  std::swap(c->gen_edges.p, merged.p); std::swap(c->gen_edges.cap, merged.cap); c->gen_edges.gen++;
  std::swap(c->gen_rowptr.p, nrow.p); std::swap(c->gen_rowptr.cap, nrow.cap); c->gen_rowptr.gen++;
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
  for (void *p : c->ipc_opened) cudaIpcCloseMemHandle(p);
  if (c->comm) g_nccl.CommDestroy(c->comm);
  c->hc.close_comm();
  for (cudaEvent_t e : c->events) cudaEventDestroy(e);
  if (c->h_stage) cudaFreeHost(c->h_stage);
  c->in_tails32.release(); c->wide.release(); c->raw_ring.release();
  for (int b = 0; b < 2; b++) if (c->h_bounce[b]) cudaFreeHost(c->h_bounce[b]);
  c->gen_rowptr.release(); c->gen_edges.release();
  c->in_rowptr.release(); c->in_edges.release(); c->rowptr.release(); c->tails.release(); c->weights.release();
  c->self_i.release(); c->self_d.release(); c->vdeg.release(); c->comm_a.release(); c->comm_b.release();
  c->cdeg.release(); c->csize.release(); c->upd.release(); c->cinfo_w.release(); c->usize.release(); c->udeg.release(); c->acc.release();
  c->scratch.release(); c->cub_tmp.release(); c->coll_tmp.release(); c->sorted_tmp.release(); c->remote_list.release(); c->remote_pos.release(); c->ghost_gid.release(); c->send_gid.release();
  c->bfs_key.release(); c->sortkey.release(); c->sortkey2.release(); c->deg_new.release(); c->rowptr2.release();
  c->ids.release(); c->perm.release(); c->inv.release(); c->lab.release(); c->tails2.release(); c->final_orig.release();
  c->weights2.release(); c->bfs_level_count.release();
  c->p2p.release();
  c->send_lid.release(); c->send_buf.release(); c->heavy_list.release(); c->hkeys.release(); c->hvals_i.release();
  c->hvals_d.release(); c->heavy_off.release();
  if (c->h_pin) cudaFreeHost(c->h_pin);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
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
  Scalars *d_sc = reinterpret_cast<Scalars *>(c->scratch.p);
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
  c->f32 = false;
  TRY(c->in_rowptr.ensure(lnv + 1));
  cudaEvent_t a = get_event(c, 0), b = get_event(c, 1);
  CK(cudaEventRecord(a, c->stream));
  CK(cudaMemcpyAsync(c->in_rowptr.p, edge_indices, sizeof(long long) * (lnv + 1), cudaMemcpyHostToDevice, c->stream));
  c->d_tails32 = nullptr;
  c->d_edges = nullptr;
  int compact = 1;
  long long compact_bytes = 0;
  if (c->opt_compact_upload && !c->opt_force_weighted && lne > 0) {
    compact = upload_compact(c, nv_global, lne, edge_list, &compact_bytes);
    if (compact < 0) return fail(std::string("compact upload: ") + cudaGetErrorString(cudaGetLastError()));
  }
  if (compact == 0) c->d_tails32 = c->in_tails32.p;
  else {
    TRY(c->in_edges.ensure(lne));
    if (lne) CK(cudaMemcpyAsync(c->in_edges.p, edge_list, sizeof(Edge16) * lne, cudaMemcpyHostToDevice, c->stream));
    c->d_edges = c->in_edges.p;
  }
  CK(cudaEventRecord(b, c->stream));
  CK(cudaEventSynchronize(b));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, a, b));
  c->h2d_s = ms * 1e-3;
  c->h2d_bytes = (long long)sizeof(long long) * (lnv + 1) + (compact == 0 ? compact_bytes : (long long)sizeof(Edge16) * lne);
  c->d_rowptr64 = c->in_rowptr.p;
  return 0;
}

int mvgpu_attach_shard_device(mvgpu_ctx *c, int64_t nv_global, const int64_t *parts, int64_t lnv, int64_t lne,
                              const int64_t *d_edge_indices, const void *d_edge_list) {
  if (!c || !parts || !d_edge_indices || (lne && !d_edge_list)) return fail("null argument");
  if (((uintptr_t)d_edge_list & 15) || ((uintptr_t)d_edge_indices & 7)) return fail("device arrays must be 16/8-byte aligned");
  CK(cudaSetDevice(c->device));
  TRY(set_graph(c, nv_global, parts, lnv, lne));
  c->f32 = false;
  c->d_rowptr64 = reinterpret_cast<const long long *>(d_edge_indices);
  c->d_edges = reinterpret_cast<const Edge16 *>(d_edge_list);
  c->d_tails32 = nullptr;
  c->h2d_bytes = 0;
  c->h2d_s = 0.0;
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
  TRY(X.ensure(3 * P.n)); TRY(UY.ensure(3 * P.n)); TRY(cnt.ensure(ncells + 1)); TRY(cstart.ensure(ncells + 1)); TRY(deg.ensure(P.n + 1));
  k_rgg_points<<<grid_for(P.n, 256, nsm), 256, 0, s>>>(P, X.p, UY.p);
  CK(cudaMemsetAsync(cnt.p, 0, sizeof(unsigned int) * (ncells + 1), s));
  k_rgg_bin<<<grid_for(P.n, 256, nsm), 256, 0, s>>>(P, X.p, UY.p, 0, cnt.p, nullptr, nullptr, nullptr, nullptr);
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt.p, cstart.p, (int)(ncells + 1), s);
  TRY(c->cub_tmp.ensure(tb));
  tb = c->cub_tmp.cap;
  CK(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, tb, cnt.p, cstart.p, (int)(ncells + 1), s));
  unsigned int ncand = 0;
  CK(cudaMemcpyAsync(&ncand, cstart.p + ncells, sizeof ncand, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  TRY(cx.ensure(ncand)); TRY(cy.ensure(ncand)); TRY(cgid.ensure(ncand));
  CK(cudaMemsetAsync(cnt.p, 0, sizeof(unsigned int) * (ncells + 1), s));
  k_rgg_bin<<<grid_for(P.n, 256, nsm), 256, 0, s>>>(P, X.p, UY.p, 1, cnt.p, cstart.p, cx.p, cy.p, cgid.p);
  CK(cudaMemsetAsync(deg.p + P.n, 0, sizeof(long long), s));
  k_rgg_neighbours<false><<<grid_for(P.n, 128, nsm, 16), 128, 0, s>>>(P, X.p, UY.p, cstart.p, cx.p, cy.p, cgid.p, unit_weight, deg.p, nullptr);
  TRY(c->gen_rowptr.ensure(P.n + 1));
  tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, deg.p, c->gen_rowptr.p, (int)(P.n + 1), s);
  TRY(c->cub_tmp.ensure(tb));
  tb = c->cub_tmp.cap;
  CK(cub::DeviceScan::ExclusiveSum(c->cub_tmp.p, tb, deg.p, c->gen_rowptr.p, (int)(P.n + 1), s));
  long long lne = 0;
  CK(cudaMemcpyAsync(&lne, c->gen_rowptr.p + P.n, sizeof lne, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  TRY(c->gen_edges.ensure(lne));
  k_rgg_neighbours<true><<<grid_for(P.n, 128, nsm, 16), 128, 0, s>>>(P, X.p, UY.p, cstart.p, cx.p, cy.p, cgid.p, unit_weight, c->gen_rowptr.p, c->gen_edges.p);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(s));
  cx.release(); cy.release(); cgid.release(); deg.release(); cnt.release(); cstart.release();
  if (random_edge_percent > 0.0) TRY(add_random_edges(c, P, nv_global, unit_weight, random_edge_percent, X.p, UY.p, &lne));
  X.release(); UY.release();
  std::vector<int64_t> parts(p + 1);
  for (int q = 0; q <= p; q++) parts[q] = (nv_global * q) / p;
  TRY(set_graph(c, nv_global, parts.data(), P.n, lne));
  c->f32 = false;
  c->d_rowptr64 = c->gen_rowptr.p;
  c->d_edges = c->gen_edges.p;
  c->d_tails32 = nullptr;
  c->h2d_bytes = 0;
  c->h2d_s = 0.0;
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

int mvgpu_louvain(mvgpu_ctx *c, double lower, double thresh, int *iters, double *modularity) {
  if (!c || !iters || !modularity) return fail("null argument");
  return run_louvain(c, lower, thresh, iters, modularity);
}

int mvgpu_get_communities_device(mvgpu_ctx *c, const int32_t **d_out) {
  if (!c || !c->d_final) return fail("no result yet");
  TRY(final_in_caller_order(c));
  CK(cudaStreamSynchronize(c->stream));
  *d_out = c->final_orig.p;
  return 0;
}

int mvgpu_get_communities(mvgpu_ctx *c, int64_t *out) {
  if (!c || !c->d_final) return fail("no result yet");
  if (c->lnv == 0) return 0;
  TRY(final_in_caller_order(c));
  TRY(c->wide.ensure(c->lnv));
  k_widen<<<grid_for(c->lnv, 256, c->num_sms), 256, 0, c->stream>>>(c->final_orig.p, c->lnv, c->wide.p);
  // pageable destinations are copied through a pinned bounce buffer in chunks (full PCIe rate instead of the
  // driver's staged pageable path); a pinned destination is detected and written directly
  cudaPointerAttributes attr;
  const bool pinned = cudaPointerGetAttributes(&attr, out) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  if (pinned) {
    CK(cudaMemcpyAsync(out, c->wide.p, sizeof(long long) * c->lnv, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return 0;
  }
  const long long CH = 4LL << 20;                                  // 4 Mi entries = 32 MB per bounce buffer
  for (int b = 0; b < 2; b++)
    if (!c->h_bounce[b]) CK(cudaMallocHost(&c->h_bounce[b], CH * sizeof(long long)));
  struct { long long off, n; } pend[2] = {{0, 0}, {0, 0}};
  cudaEvent_t ev[2] = {get_event(c, 0), get_event(c, 1)};
  long long off = 0;
  for (int k = 0; off < c->lnv || pend[0].n || pend[1].n; k++) {
    const int b = k & 1;
    if (pend[b].n) {                                               // drain this buffer (its DMA was issued two steps ago,
      CK(cudaEventSynchronize(ev[b]));                             //  the other buffer's DMA is in flight meanwhile)
      memcpy(out + pend[b].off, c->h_bounce[b], sizeof(long long) * pend[b].n);
      pend[b].n = 0;
    }
    if (off < c->lnv) {
      const long long n = std::min<long long>(CH, c->lnv - off);
      CK(cudaMemcpyAsync(c->h_bounce[b], c->wide.p + off, sizeof(long long) * n, cudaMemcpyDeviceToHost, c->stream));
      CK(cudaEventRecord(ev[b], c->stream));
      pend[b].off = off; pend[b].n = n;
      off += n;
    }
  }
  return 0;
}

int mvgpu_set_option(mvgpu_ctx *c, const char *name, int64_t value) {
  if (!c || !name) return fail("null argument");
  const std::string n(name);
  c->peers_ready = false;          // options may change which arrays exist: re-validate the peer tables
  if (n == "trace") c->opt_trace = value != 0;
  else if (n == "max_iters") { if (value < 1) return fail("max_iters < 1"); c->opt_max_iters = value; }
  else if (n == "force_weighted") c->opt_force_weighted = value != 0;
  else if (n == "force_heavy_deg") c->opt_force_heavy_deg = value;
  else if (n == "scan_variant") { if (value < 3 || value > 6) return fail("scan_variant must be 6 (measure and choose, default), 5 (k_scan_pq), 4 (k_scan_pw) or 3 (k_scan_ws)"); c->opt_scan_variant = (int)value; }
  else if (n == "cache_policy") c->opt_cache_policy = (int)value;
  else if (n == "reorder") c->opt_reorder = (int)value;
  else if (n == "comm_mode") c->opt_comm_mode = (int)value;
  else if (n == "compact_upload") c->opt_compact_upload = (int)value;
  else if (n == "host_threads") c->opt_host_threads = (int)value;
  else if (n == "first_iter") c->opt_first_iter = value != 0;
  else if (n == "upload_chunk") { if (value < 256 || (value & 3)) return fail("upload_chunk must be a multiple of 4, >= 256"); c->opt_upload_chunk = value; }
  else if (n == "host_transport") {
    if ((c->comm || c->hc.is_open()) && c->opt_host_transport != (value != 0)) return fail("host_transport must be set before mvgpu_comm_init");
    c->opt_host_transport = value != 0;
  }
  else if (n == "region_size") { if (value < 32) return fail("region_size < 32"); c->opt_region = (int)value; }
  else return fail("unknown option " + n);
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
  info6[0] = c->lnv; info6[1] = c->lne; info6[2] = c->nghost; info6[3] = c->nsend; info6[4] = c->nheavy; info6[5] = c->maxdeg;
  return 0;
}

// ---- USE_32_BIT_GRAPH surface (utils.hpp:72-82): int32 offsets, {int32 tail; float weight} records, float results ----
int mvgpu_upload_shard32(mvgpu_ctx *c, int32_t nv_global, const int32_t *parts, int32_t lnv, int32_t lne,
                         const int32_t *edge_indices, const void *edge_list8) {
  if (!c || !parts || !edge_indices || (lne && !edge_list8)) return fail("null argument");
  CK(cudaSetDevice(c->device));
  std::vector<int64_t> parts64(parts, parts + c->nranks + 1);
  TRY(set_graph(c, nv_global, parts64.data(), lnv, lne));
  c->f32 = true;
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
  c->h2d_s = ms * 1e-3;
  c->h2d_bytes = (long long)sizeof(int32_t) * (lnv + 1) + (long long)sizeof(Edge8) * lne;
  c->d_rowptr64 = c->in_rowptr.p;
  c->d_edges = c->in_edges.p;
  c->d_tails32 = nullptr;
  return 0;
}

int mvgpu_louvain32(mvgpu_ctx *c, float lower, float thresh, int *iters, float *modularity) {
  if (!c || !iters || !modularity) return fail("null argument");
  if (!c->f32) return fail("mvgpu_louvain32 needs a shard uploaded with mvgpu_upload_shard32");
  double mod = 0.0;
  TRY(run_louvain(c, (double)lower, (double)thresh, iters, &mod));
  *modularity = (float)mod;
  return 0;
}

int mvgpu_get_communities32(mvgpu_ctx *c, int32_t *out) {
  if (!c || !c->d_final) return fail("no result yet");
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
