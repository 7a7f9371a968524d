// Host replacement for the reference's distLouvainMethod (dspl.hpp:1280-1283): same parameter list,
// same return value / `iters` semantics; the body marshals the Graph's arrays across the C ABI
// (include/mvgpu.h) to the CUDA library instead of running the OpenMP/MPI loops.
#pragma once
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

#include "graph.hpp"
#include "mvgpu.h"

// What MPI_Comm carried in the reference: which GPU to use and (for nprocs > 1) the communicator id
// every rank received from rank 0.
struct GpuRankContext {
  int device = 0;
  unsigned char unique_id[MVGPU_UNIQUE_ID_BYTES] = {0};
  bool trace = false;
  std::vector<GraphElem> *comm_out = nullptr;     // final currComm of this rank (the reference drops it, dspl.hpp:1432-1438)
  mvgpu_timings timings{};
  std::vector<mvgpu_iter_trace> iter_trace;
  const std::vector<GraphElem> *init_comm = nullptr;   // -i: starting assignment of this rank's vertices (global ids)
  int stop_after = 0;                                  // -k: stop after that many accepted iterations (0 = off)
  bool stopped = false;                                // the run ended by stop_after, not by the exit test
  bool quality = false;                                // -q: evaluate the returned assignment after the run
  const std::vector<GraphElem> *eval_comm = nullptr;   // -E: evaluate this assignment instead of running the phase
  mvgpu_quality q{};                                   // -q / -E: the evaluation (global values)
  bool split = false;                                  // -C: split the run's (or -E's) assignment into connected pieces
  mvgpu_split_report split_rep{};                      // -C: the split's counts (global values)
  std::vector<GraphElem> split_comm;                   // -C: the split assignment of this rank's vertices
  const std::vector<GraphElem> *cmp_comm = nullptr;    // -M: compare the assignment -q would evaluate with this one
  mvgpu_compare_report cmp{};                          // -M: the comparison (global values)
  const std::vector<unsigned char> *movable = nullptr; // -V: movable set of this rank's vertices (nonzero = movable)
  bool frontier = false;                               // -F: grow the movable set from the vertices that move
  std::vector<unsigned char> *movable_out = nullptr;   // -o: the set the next iteration would use (for -V on resume)
  bool probe = false;                                  // -U: probe the assignment -q would evaluate
  mvgpu_probe_report probe_rep{};                      // -U: the probe's counts (global values)
  std::vector<unsigned char> unsettled;                // -U with -o: 1 where the probe's target differs from the assignment
};

[[noreturn]] inline void mv_abort(const std::string &where) {
  // the reference's only error behaviour on this path is MPI_Abort(comm, -99) (main.cpp:90,251-276)
  std::fprintf(stderr, "[miniVite_b200] %s: %s\n", where.c_str(), mvgpu_last_error());
  std::exit(99);
}

// Developer knobs, not part of the reference's surface: MVGPU_OPTIONS="name=value,name=value" is handed to
// mvgpu_set_option (unknown names abort), MVGPU_REPEAT=n runs the phase n times (same result; timings of the last,
// warm, run are reported).
inline void mv_apply_env_options(mvgpu_ctx *ctx) {
  const char *e = std::getenv("MVGPU_OPTIONS");
  if (!e) return;
  std::string s(e);
  size_t pos = 0;
  while (pos < s.size()) {
    size_t end = s.find(',', pos);
    if (end == std::string::npos) end = s.size();
    const std::string kv = s.substr(pos, end - pos);
    pos = end + 1;
    if (kv.empty()) continue;
    const size_t eq = kv.find('=');
    if (eq == std::string::npos) { std::fprintf(stderr, "[miniVite_b200] MVGPU_OPTIONS: missing '=' in %s\n", kv.c_str()); std::exit(99); }
    if (mvgpu_set_option(ctx, kv.substr(0, eq).c_str(), std::atoll(kv.c_str() + eq + 1))) mv_abort("MVGPU_OPTIONS");
  }
}
inline int mv_env_repeat() {
  const char *e = std::getenv("MVGPU_REPEAT");
  const int n = e ? std::atoi(e) : 1;
  return n < 1 ? 1 : n;
}

// -i / -k: hand the starting assignment and the stop point to the library (after the shard exists)
inline void mv_apply_warm_start(mvgpu_ctx *ctx, const GpuRankContext &rc) {
  if (rc.init_comm && mvgpu_set_initial_communities(ctx, rc.init_comm->data())) mv_abort("mvgpu_set_initial_communities");
  if (rc.stop_after && mvgpu_set_option(ctx, "stop_after", rc.stop_after)) mv_abort("stop_after");
  if (rc.movable && mvgpu_set_movable(ctx, rc.movable->data())) mv_abort("mvgpu_set_movable");
  if (rc.frontier && mvgpu_set_option(ctx, "frontier", 1)) mv_abort("frontier");
}
// -C: split `comm` (NULL: the run's result) into rc.split_comm
inline void mv_split(mvgpu_ctx *ctx, GpuRankContext &rc, const GraphElem *comm, GraphElem lnv) {
  rc.split_comm.assign(lnv + 1, 0);                // never an empty array: the call takes a non-NULL out on every rank
  if (mvgpu_split_communities(ctx, comm, rc.split_comm.data(), &rc.split_rep)) mv_abort("mvgpu_split_communities");
  rc.split_comm.resize(lnv);
}
// -M: compare X (NULL: the run's result) with the assignment read from -M's files
inline void mv_compare(mvgpu_ctx *ctx, GpuRankContext &rc, const GraphElem *X) {
  if (!rc.cmp_comm) return;
  const GraphElem none = 0;                        // an empty shard still passes a non-NULL array
  const GraphElem *Y = rc.cmp_comm->empty() ? &none : rc.cmp_comm->data();
  if (mvgpu_compare_communities(ctx, X, Y, &rc.cmp)) mv_abort("mvgpu_compare_communities");
}
// -U: probe X (NULL: the run's result); with -o, mark the vertices whose target is not their community
inline void mv_probe(mvgpu_ctx *ctx, GpuRankContext &rc, const GraphElem *X, GraphElem lnv) {
  if (!rc.probe) return;
  std::vector<int64_t> target(lnv + 1);            // never an empty array
  if (mvgpu_probe_communities(ctx, X, target.data(), nullptr, nullptr, &rc.probe_rep)) mv_abort("mvgpu_probe_communities");
  if (!rc.comm_out) return;
  std::vector<int64_t> run;
  if (!X) {
    run.resize(lnv + 1);
    if (lnv && mvgpu_get_communities(ctx, run.data())) mv_abort("mvgpu_get_communities");
    X = run.data();
  }
  rc.unsettled.resize(lnv);
  for (GraphElem i = 0; i < lnv; i++) rc.unsettled[i] = target[i] != X[i] ? 1 : 0;
}
// -E: evaluate the given assignment (with -C: its split) and run no Louvain phase (true: done, the caller returns)
inline bool mv_evaluate_only(mvgpu_ctx *ctx, GpuRankContext &rc) {
  if (!rc.eval_comm) return false;
  const GraphElem *X = rc.eval_comm->data();
  if (rc.split) {
    mv_split(ctx, rc, X, (GraphElem)rc.eval_comm->size());
    X = rc.split_comm.data();
  }
  mv_compare(ctx, rc, X);
  mv_probe(ctx, rc, X, (GraphElem)rc.eval_comm->size());
  if (mvgpu_evaluate_communities(ctx, X, &rc.q)) mv_abort("mvgpu_evaluate_communities");
  mvgpu_destroy(ctx);
  return true;
}
// -C: split the assignment the run returned; -M: compare the run's assignment (with -C: its split); -U: probe it; -q:
// evaluate it
inline void mv_evaluate_run(mvgpu_ctx *ctx, GpuRankContext &rc, GraphElem lnv) {
  if (rc.split) mv_split(ctx, rc, nullptr, lnv);
  mv_compare(ctx, rc, rc.split ? rc.split_comm.data() : nullptr);
  mv_probe(ctx, rc, rc.split ? rc.split_comm.data() : nullptr, lnv);
  if (rc.quality && mvgpu_evaluate_communities(ctx, rc.split ? rc.split_comm.data() : nullptr, &rc.q))
    mv_abort("mvgpu_evaluate_communities");
}
// -o: the run's assignment (with -C: its split)
inline void mv_result(mvgpu_ctx *ctx, GpuRankContext &rc, GraphElem lnv) {
  if (rc.movable_out) {
    rc.movable_out->assign(lnv + 1, 1);
    if (mvgpu_get_movable(ctx, rc.movable_out->data())) mv_abort("mvgpu_get_movable");
    rc.movable_out->resize(lnv);
  }
  if (!rc.comm_out) return;
  if (rc.split) { *rc.comm_out = rc.split_comm; return; }
  rc.comm_out->resize(lnv);
  if (mvgpu_get_communities(ctx, rc.comm_out->data())) mv_abort("mvgpu_get_communities");
}
inline void mv_read_converged(mvgpu_ctx *ctx, GpuRankContext &rc) {
  int conv = 1;
  if (mvgpu_get_converged(ctx, &conv)) mv_abort("mvgpu_get_converged");
  rc.stopped = conv == 0;
}

// MVGPU_SCAN_TIMES=1: print the duration of every scan launch of the last phase (ms) on stderr
inline void mv_print_scan_times(mvgpu_ctx *ctx, int me) {
  if (me != 0 || !std::getenv("MVGPU_SCAN_TIMES")) return;
  int n = 0;
  mvgpu_get_scan_times(ctx, 0, nullptr, &n);
  std::vector<double> t(n);
  if (n) mvgpu_get_scan_times(ctx, n, t.data(), &n);
  std::fprintf(stderr, "SCAN_MS");
  for (double x : t) std::fprintf(stderr, " %.3f", x * 1e3);
  std::fprintf(stderr, "\n");
}

// The 6 scratch parameters (ssz ... rvdata) are caller-owned out-params that only the reference's
// exchangeVertexReqs filled (dspl.hpp:1106-1272); the ghost lists now live in device memory, so they
// are left empty.
inline GraphWeight distLouvainMethod(const int me, const int nprocs, const Graph &dg, size_t &ssz, size_t &rsz,
                                     std::vector<GraphElem> &ssizes, std::vector<GraphElem> &rsizes,
                                     std::vector<GraphElem> &svdata, std::vector<GraphElem> &rvdata,
                                     const GraphWeight lower, const GraphWeight thresh, int &iters,
                                     GpuRankContext &rc) {
  ssz = rsz = 0;
  ssizes.clear(); rsizes.clear(); svdata.clear(); rvdata.clear();
  mvgpu_ctx *ctx = nullptr;
  if (mvgpu_create(&ctx, rc.device, me, nprocs)) mv_abort("mvgpu_create");
  mv_apply_env_options(ctx);                       // before the communicator: host_transport decides how it is built
  if (nprocs > 1 && mvgpu_comm_init(ctx, rc.unique_id)) mv_abort("mvgpu_comm_init");
  if (rc.trace) mvgpu_set_option(ctx, "trace", 1);
  if (mvgpu_upload_shard(ctx, dg.get_nv(), dg.parts().data(), dg.get_lnv(), dg.get_lne(), dg.edge_indices_.data(),
                         dg.edge_list_.data()))
    mv_abort("mvgpu_upload_shard");
  mv_apply_warm_start(ctx, rc);
  if (mv_evaluate_only(ctx, rc)) return lower;
  double mod = 0.0;
  for (int rep = mv_env_repeat(); rep > 0; rep--)
    if (mvgpu_louvain(ctx, lower, thresh, &iters, &mod)) mv_abort("mvgpu_louvain");
  mv_evaluate_run(ctx, rc, dg.get_lnv());
  mvgpu_get_timings(ctx, &rc.timings);
  mv_read_converged(ctx, rc);
  mv_print_scan_times(ctx, me);
  if (rc.trace) {
    int n = 0;
    mvgpu_get_trace(ctx, 0, nullptr, &n);
    rc.iter_trace.resize(n);
    if (n) mvgpu_get_trace(ctx, n, rc.iter_trace.data(), &n);
  }
  mv_result(ctx, rc, dg.get_lnv());
  mvgpu_destroy(ctx);
  return mod;
}

// Variant for `-D`: the shard never exists on the host -- GenerateRGG runs on the device (mvgpu_generate_rgg_shard,
// the reference's generator of graph.hpp:584-1213 bit for bit) and the Louvain phase consumes it in place.
// `gen_seconds` receives the generation time, `lne` the local edge count.
inline GraphWeight distLouvainMethodOnDeviceRGG(const int me, const int nprocs, const GraphElem nv, const bool unitEdgeWeight,
                                                const bool lcg, const GraphWeight randomEdgePercent, const GraphWeight lower, const GraphWeight thresh, int &iters,
                                                GpuRankContext &rc, GraphElem &lne, double &gen_seconds,
                                                const std::function<void()> &before_louvain) {
  mvgpu_ctx *ctx = nullptr;
  if (mvgpu_create(&ctx, rc.device, me, nprocs)) mv_abort("mvgpu_create");
  mv_apply_env_options(ctx);                       // before the communicator: host_transport decides how it is built
  if (nprocs > 1 && mvgpu_comm_init(ctx, rc.unique_id)) mv_abort("mvgpu_comm_init");
  if (rc.trace) mvgpu_set_option(ctx, "trace", 1);
  const auto t0 = std::chrono::steady_clock::now();
  int64_t lne64 = 0;
  if (mvgpu_generate_rgg_shard_ex(ctx, nv, unitEdgeWeight ? 1 : 0, lcg ? 1 : 0, randomEdgePercent, &lne64)) mv_abort("mvgpu_generate_rgg_shard");
  gen_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  lne = lne64;
  mv_apply_warm_start(ctx, rc);
  before_louvain();
  if (mv_evaluate_only(ctx, rc)) return lower;
  double mod = 0.0;
  for (int rep = mv_env_repeat(); rep > 0; rep--)
    if (mvgpu_louvain(ctx, lower, thresh, &iters, &mod)) mv_abort("mvgpu_louvain");
  mv_evaluate_run(ctx, rc, nv / nprocs);
  mvgpu_get_timings(ctx, &rc.timings);
  mv_read_converged(ctx, rc);
  mv_print_scan_times(ctx, me);
  if (rc.trace) {
    int n = 0;
    mvgpu_get_trace(ctx, 0, nullptr, &n);
    rc.iter_trace.resize(n);
    if (n) mvgpu_get_trace(ctx, n, rc.iter_trace.data(), &n);
  }
  mv_result(ctx, rc, nv / nprocs);
  mvgpu_destroy(ctx);
  return mod;
}
