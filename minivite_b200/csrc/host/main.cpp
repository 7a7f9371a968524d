// miniVite_b200: command-line driver with the reference's options and report block (main.cpp:75-278),
// running the Louvain phase on H100 GPUs.  "Processes" of the reference == GPU ranks here: `-g N`
// forks one host process per GPU (the reference gets its ranks from mpirun); each rank builds or
// reads its own vertex-range shard exactly as reference rank r would.
//
//   -f <file>  binary graph file          -b  edge-balanced partition      -r <n> ranks per node (accepted, unused)
//   -t <thr>   convergence threshold      -n <nv> generate an RGG          -w  Euclidean edge weights
//   -l         LCG random numbers         -p <pct> extra random edges      -s  print the graph
// additions: -g <gpus> (default 1)   -o <prefix> dump final communities per rank   -T per-iteration trace on stderr
//            -D generate the RGG on the GPU (same graph; with -n, also -w, -l and -p; without -s)
//            -i <prefix> start from the communities an earlier -o <prefix> wrote   -k <n> stop after n accepted
//            iterations (prints STOPPED iters=<n> prevMod=<v>)   -L <v> starting `lower` (default -1; resume: -L <v>)
//            -q evaluate the returned assignment (prints QUALITY mod=.. e=.. a2=.. communities=.. singletons=.. maxsize=..)
//            -E <prefix> evaluate the communities an earlier -o <prefix> wrote, without a Louvain phase (prints QUALITY)
//            -C split every community of the returned (or -E) assignment into its connected pieces; -q evaluates and -o
//            writes the split assignment (prints SPLIT communities=.. components=.. disconnected=.. rounds=..)
//            -M <prefix> compare the assignment -q would evaluate with the communities an earlier -o <prefix> wrote
//            (prints COMPARE ari=.. nmi=.. vi=.. rand=.. mi=.. hx=.. hy=.. cells=.. communities_x=.. communities_y=..)
//            -U probe the assignment -q would evaluate: what every vertex would do under the Louvain rule from it (prints
//            PROBE vertices=.. moves=.. vetoed=.. interior=.. max_gain=..); with -o also <o>.unsettled.<rank>, lnv bytes,
//            1 where the vertex would move, in the -V format: -i <o> -V <o>.unsettled -F re-clusters from those vertices
#include <getopt.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>

#include <atomic>
#include <cassert>
#include <chrono>
#include <cstring>
#include <iostream>
#include <new>
#include <sstream>
#include <string>

#include "binio.hpp"
#include "graph.hpp"
#include "louvain.hpp"
#include "rgg.hpp"

static std::string inputFileName, dumpPrefix, initPrefix, evalPrefix, comparePrefix, movablePrefix;
static bool frontierGrow = false;
static int stopAfter = 0;
static GraphWeight lowerStart = -1.0;
static int me = 0, nprocs = 1;
static int ranksPerNode = 1;
static GraphElem nvRGG = 0;
static bool generateGraph = false, readBalanced = false, showGraph = false, traceIters = false, deviceGenerate = false,
            evalQuality = false, splitComm = false, probeComm = false;
static GraphWeight randomEdgePercent = 0.0;
static bool randomNumberLCG = false, isUnitEdgeWeight = true;
static GraphWeight threshold = 1.0E-6;

// ---- the handful of collectives main() needs, over a shared page (ranks are forked processes) ----
struct Shared {
  std::atomic<int> arrived[8];
  std::atomic<int> id_ready;
  unsigned char unique_id[MVGPU_UNIQUE_ID_BYTES];
  double dbl[64];
  long long i64[64];
};
static Shared *shm = nullptr;
static int barrier_epoch = 0;

static void rank_barrier() {
  const int slot = barrier_epoch++ & 7;
  shm->arrived[slot].fetch_add(1);
  while (shm->arrived[slot].load() < nprocs) usleep(50);
  // slot is reused 8 barriers later; reset by the last rank to leave the *next* barrier
  if (me == 0) shm->arrived[(slot + 4) & 7].store(0);
}
static double wtime() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
static double reduce_sum(double v) {
  shm->dbl[me] = v;
  rank_barrier();
  double s = 0;
  for (int r = 0; r < nprocs; r++) s += shm->dbl[r];
  rank_barrier();
  return s;
}
static long long reduce_sum_ll(long long v) {
  shm->i64[me] = v;
  rank_barrier();
  long long s = 0;
  for (int r = 0; r < nprocs; r++) s += shm->i64[r];
  rank_barrier();
  return s;
}
[[noreturn]] static void abort_all(int code) {
  if (me == 0) kill(0, SIGTERM);
  _exit(code);
}

static void parseCommandLine(const int argc, char *const argv[]) {
  int ret;
  while ((ret = getopt(argc, argv, "f:br:t:n:wlp:sg:o:TDi:k:L:qE:CM:V:FU")) != -1) {
    switch (ret) {
      case 'f': inputFileName.assign(optarg); break;
      case 'b': readBalanced = true; break;
      case 'r': ranksPerNode = atoi(optarg); break;
      case 't': threshold = atof(optarg); break;
      case 'n': nvRGG = atol(optarg); if (nvRGG > 0) generateGraph = true; break;
      case 'w': isUnitEdgeWeight = false; break;
      case 'l': randomNumberLCG = true; break;
      case 'p': randomEdgePercent = atof(optarg); break;
      case 's': showGraph = true; break;
      case 'g': nprocs = atoi(optarg); break;
      case 'o': dumpPrefix.assign(optarg); break;
      case 'T': traceIters = true; break;
      case 'D': deviceGenerate = true; break;
      case 'i': initPrefix.assign(optarg); break;
      case 'k': stopAfter = atoi(optarg); break;
      case 'L': lowerStart = atof(optarg); break;
      case 'q': evalQuality = true; break;
      case 'E': evalPrefix.assign(optarg); break;
      case 'C': splitComm = true; break;
      case 'M': comparePrefix.assign(optarg); break;
      case 'V': movablePrefix.assign(optarg); break;
      case 'F': frontierGrow = true; break;
      case 'U': probeComm = true; break;
      default: assert(0 && "Option not recognized!!!"); break;
    }
  }
  // same validation messages as the reference (main.cpp:249-277)
  if (argc == 1) { std::cerr << "Must specify some options." << std::endl; exit(99); }
  if (!generateGraph && inputFileName.empty()) {
    std::cerr << "Must specify a binary file name with -f or provide parameters for generating a graph." << std::endl;
    exit(99);
  }
  if (!generateGraph && randomNumberLCG) { std::cerr << "Must specify -g for graph generation using LCG." << std::endl; exit(99); }
  if (!generateGraph && (randomEdgePercent > 0.0)) {
    std::cerr << "Must specify -g for graph generation first to add random edges to it." << std::endl; exit(99);
  }
  if (!generateGraph && !isUnitEdgeWeight) {
    std::cerr << "Must specify -g for graph generation first before setting edge weights." << std::endl; exit(99);
  }
  if (generateGraph && ((randomEdgePercent < 0) || (randomEdgePercent >= 100))) {
    std::cerr << "Invalid random edge percentage for generated graph!" << std::endl; exit(99);
  }
  if (nprocs < 1 || nprocs > 16) { std::cerr << "Invalid number of GPUs (-g)." << std::endl; exit(99); }
  if (deviceGenerate && (!generateGraph || showGraph)) {
    std::cerr << "-D (generate the RGG on the GPU) needs -n and excludes -s." << std::endl; exit(99);
  }
  if (stopAfter < 0) { std::cerr << "-k needs a number of iterations >= 0." << std::endl; exit(99); }
  if (!evalPrefix.empty() && (!initPrefix.empty() || !dumpPrefix.empty() || stopAfter)) {
    std::cerr << "-E runs no Louvain phase: it excludes -i, -o and -k." << std::endl; exit(99);
  }
}

int main(int argc, char *argv[]) {
  parseCommandLine(argc, argv);
  (void)ranksPerNode;

  shm = (Shared *)mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  if (shm == (Shared *)MAP_FAILED) { perror("mmap"); return 99; }
  new (shm) Shared();
  setpgid(0, 0);
  fflush(stdout); fflush(stderr);
  for (int r = 1; r < nprocs; r++) {            // ranks = processes, like mpirun -n nprocs (no CUDA touched yet)
    pid_t p = fork();
    if (p < 0) { perror("fork"); return 99; }
    if (p == 0) { me = r; break; }
  }

  // the reference prints these with -DPRINT_DIST_STATS (its Makefile default, Makefile:10-16)
  auto print_stats = [&](long lne, GraphElem nv, GraphElem ne) {
    const double sumdeg = reduce_sum((double)lne), sum_sq = reduce_sum((double)lne * (double)lne);
    shm->i64[32 + me] = lne;
    rank_barrier();
    if (me == 0) {
      long maxdeg = 0;
      for (int r = 0; r < nprocs; r++) maxdeg = std::max<long>(maxdeg, shm->i64[32 + r]);
      const double average = sumdeg / nprocs, avg_sq = sum_sq / nprocs, var = avg_sq - average * average;
      std::cout << std::endl;
      std::cout << "-------------------------------------------------------" << std::endl;
      std::cout << "Graph edge distribution characteristics" << std::endl;
      std::cout << "-------------------------------------------------------" << std::endl;
      std::cout << "Number of vertices: " << nv << std::endl;
      std::cout << "Number of edges: " << ne << std::endl;
      std::cout << "Maximum number of edges: " << maxdeg << std::endl;
      std::cout << "Average number of edges: " << average << std::endl;
      std::cout << "Expected value of X^2: " << avg_sq << std::endl;
      std::cout << "Variance: " << var << std::endl;
      std::cout << "Standard deviation: " << std::sqrt(var) << std::endl;
      std::cout << "-------------------------------------------------------" << std::endl;
    }
    rank_barrier();
  };

  rank_barrier();
  const double td0 = wtime();
  Graph *g = nullptr;
  if (!deviceGenerate) {
  try {
    if (generateGraph) {
      mvhost::GenerateRGG gr(nvRGG, nprocs);
      if (randomEdgePercent > 0.0) {
        // random edges couple all strips (graph.hpp:939-1122): every rank builds all strips, keeps its own
        std::vector<Graph *> all = gr.generate(randomNumberLCG, isUnitEdgeWeight, randomEdgePercent);
        g = all[me];
        for (int r = 0; r < nprocs; r++) if (r != me) delete all[r];
      } else {
        g = gr.generate(randomNumberLCG, isUnitEdgeWeight, 0.0, me, me + 1)[0];
      }
    } else {
      mvhost::BinaryEdgeList rm;
      g = readBalanced ? rm.read_balanced(me, nprocs, ranksPerNode, inputFileName) : rm.read(me, nprocs, ranksPerNode, inputFileName);
      if (readBalanced && me == 0) std::cout << "Trying to achieve equal edge distribution across processes." << std::endl;
    }
  } catch (const std::exception &e) {
    if (me == 0) std::cout << e.what() << std::endl << "Exiting..." << std::endl;
    abort_all(99);
  }
  assert(g != nullptr);
  const long long ne_global = reduce_sum_ll(g->get_lne());
  g->set_nedges(g->get_lne(), ne_global);
  if (showGraph) {
    for (int p = 0; p < nprocs; p++) { rank_barrier(); if (p == me) g->print(); }
  }
  print_stats((long)g->get_lne(), g->get_nv(), g->get_ne());
  const double tdt = reduce_sum(wtime() - td0);
  if (me == 0) {
    if (!generateGraph)
      std::cout << "Time to read input file and create distributed graph (in s): " << (tdt / nprocs) << std::endl;
    else
      std::cout << "Time to generate distributed graph of " << nvRGG << " vertices (in s): " << (tdt / nprocs) << std::endl;
  }
  }

  // ---- communicator bootstrap (stands in for MPI_Init + createCommunityMPIType, main.cpp:78-102)
  GpuRankContext rc;
  {
    // one GPU per rank; with more ranks than GPUs the ranks wrap around (only the host transport, MVGPU_OPTIONS=
    // host_transport=1, lets several ranks share a device: NCCL refuses)
    const int ngpu = mvgpu_device_count();
    rc.device = ngpu > 0 ? me % ngpu : me;
  }
  rc.trace = traceIters;
  std::vector<GraphElem> comm;
  std::vector<unsigned char> movableOut;
  if (!dumpPrefix.empty()) { rc.comm_out = &comm; rc.movable_out = &movableOut; }
  if (nprocs > 1) {
    if (me == 0) {
      if (mvgpu_get_unique_id(shm->unique_id)) mv_abort("mvgpu_get_unique_id");
      shm->id_ready.store(1);
    }
    while (!shm->id_ready.load()) usleep(50);
    memcpy(rc.unique_id, shm->unique_id, sizeof rc.unique_id);
  }

  // -i / -E: this rank's slice of an earlier run's -o dump ({base, lnv} header, then lnv global community ids)
  auto read_assignment = [&](const char *flag, const std::string &prefix, std::vector<GraphElem> &comm) {
    const long long want_base = deviceGenerate ? (long long)(nvRGG / nprocs) * me : (long long)g->get_base(me);
    const long long want_lnv = deviceGenerate ? (long long)(nvRGG / nprocs) : (long long)g->get_lnv();
    const std::string fn = prefix + "." + std::to_string(me);
    FILE *f = fopen(fn.c_str(), "rb");
    long long hdr[2] = {-1, -1};
    bool ok = f && fread(hdr, 8, 2, f) == 2 && hdr[0] == want_base && hdr[1] == want_lnv;
    if (ok) {
      comm.resize((size_t)want_lnv);
      ok = fread(comm.data(), sizeof(GraphElem), comm.size(), f) == comm.size();
    }
    if (f) fclose(f);
    if (!ok)
      fprintf(stderr, "[miniVite_b200] %s %s: cannot read %s or its header {base %lld, lnv %lld} does not match this rank's "
              "shard {base %lld, lnv %lld}\n", flag, prefix.c_str(), fn.c_str(), hdr[0], hdr[1], want_base, want_lnv);
    if (reduce_sum_ll(ok ? 0 : 1)) abort_all(99);       // every rank leaves, not only the one with the bad file
  };
  std::vector<GraphElem> initComm, evalComm, cmpComm;
  if (!initPrefix.empty()) {
    read_assignment("-i", initPrefix, initComm);
    rc.init_comm = &initComm;
  }
  if (!evalPrefix.empty()) {
    read_assignment("-E", evalPrefix, evalComm);
    rc.eval_comm = &evalComm;
  }
  if (!comparePrefix.empty()) {
    read_assignment("-M", comparePrefix, cmpComm);
    rc.cmp_comm = &cmpComm;
  }
  // -V: this rank's movable set, PREFIX.<rank> = lnv raw bytes (what -o writes to <o>.mask.<rank>)
  std::vector<unsigned char> movableIn;
  if (!movablePrefix.empty()) {
    const long long want_lnv = deviceGenerate ? (long long)(nvRGG / nprocs) : (long long)g->get_lnv();
    const std::string fn = movablePrefix + "." + std::to_string(me);
    FILE *f = fopen(fn.c_str(), "rb");
    movableIn.assign((size_t)want_lnv + 1, 0);
    const size_t got = f ? fread(movableIn.data(), 1, movableIn.size(), f) : 0;
    if (f) fclose(f);
    const bool ok = f && (long long)got == want_lnv;
    if (!ok) fprintf(stderr, "[miniVite_b200] -V %s: cannot read %s or it does not hold lnv = %lld bytes\n", movablePrefix.c_str(),
                     fn.c_str(), want_lnv);
    if (reduce_sum_ll(ok ? 0 : 1)) abort_all(99);
    rc.movable = &movableIn;
  }
  rc.frontier = frontierGrow;
  rc.stop_after = stopAfter;
  rc.quality = evalQuality;
  rc.split = splitComm;
  rc.probe = probeComm;

  GraphWeight currMod = lowerStart;
  std::vector<GraphElem> ssizes, rsizes, svdata, rvdata;
  size_t ssz = 0, rsz = 0;
  int iters = 0;

  GraphElem nv_rep = 0, ne_rep = 0, base_rep = 0, lnv_rep = 0;
  double t1 = 0.0;
  if (deviceGenerate) {
    GraphElem lne = 0;
    double gen_s = 0.0;
    currMod = distLouvainMethodOnDeviceRGG(me, nprocs, nvRGG, isUnitEdgeWeight, randomNumberLCG, randomEdgePercent, currMod, threshold, iters, rc, lne, gen_s, [&]() {
      ne_rep = reduce_sum_ll(lne);                 // between generation and the Louvain phase: the reference's report + timer start
      print_stats((long)lne, nvRGG, ne_rep);
      const double tdt = reduce_sum(gen_s);
      if (me == 0)
        std::cout << "Time to generate distributed graph of " << nvRGG << " vertices (in s): " << (tdt / nprocs) << std::endl;
      rank_barrier();
      t1 = wtime();
    });
    nv_rep = nvRGG; lnv_rep = nvRGG / nprocs; base_rep = lnv_rep * me;
  } else {
    rank_barrier();
    t1 = wtime();
    currMod = distLouvainMethod(me, nprocs, *g, ssz, rsz, ssizes, rsizes, svdata, rvdata, currMod, threshold, iters, rc);
    nv_rep = g->get_nv(); ne_rep = g->get_ne(); base_rep = g->get_base(me); lnv_rep = g->get_lnv();
  }
  rank_barrier();
  const double total = wtime() - t1;
  const double tot_time = reduce_sum(total);
  const double dev_time = reduce_sum(rc.timings.total_s);
  if (me == 0 && splitComm)
    fprintf(stderr, "SPLIT communities=%ld components=%ld disconnected=%ld rounds=%d\n", (long)rc.split_rep.communities,
            (long)rc.split_rep.components, (long)rc.split_rep.disconnected, (int)rc.split_rep.rounds);
  if (me == 0 && !comparePrefix.empty())
    fprintf(stderr, "COMPARE ari=%.17g nmi=%.17g vi=%.17g rand=%.17g mi=%.17g hx=%.17g hy=%.17g cells=%ld communities_x=%ld "
            "communities_y=%ld\n", rc.cmp.ari, rc.cmp.nmi, rc.cmp.vi, rc.cmp.rand, rc.cmp.mi, rc.cmp.h_x, rc.cmp.h_y,
            (long)rc.cmp.cells, (long)rc.cmp.communities_x, (long)rc.cmp.communities_y);
  if (me == 0 && probeComm)
    fprintf(stderr, "PROBE vertices=%ld moves=%ld vetoed=%ld interior=%ld max_gain=%.17g\n", (long)rc.probe_rep.vertices,
            (long)rc.probe_rep.moves, (long)rc.probe_rep.vetoed, (long)rc.probe_rep.interior, rc.probe_rep.max_gain);
  if (me == 0 && (evalQuality || !evalPrefix.empty()))
    fprintf(stderr, "QUALITY mod=%.17g e=%.17g a2=%.17g communities=%ld singletons=%ld maxsize=%ld\n", rc.q.modularity,
            rc.q.e_in, rc.q.a2, (long)rc.q.communities, (long)rc.q.singletons, (long)rc.q.max_size);

  if (traceIters && me == 0)
    for (size_t k = 0; k < rc.iter_trace.size(); k++)
      fprintf(stderr, "ITER %zu mod=%.17g moved=%ld chash=%016llx\n", k + 1, rc.iter_trace[k].modularity,
              (long)rc.iter_trace[k].moved, (unsigned long long)rc.iter_trace[k].chash);
  if (!dumpPrefix.empty()) {
    const std::string fn = dumpPrefix + "." + std::to_string(me);
    FILE *f = fopen(fn.c_str(), "wb");
    long long hdr[2] = {(long long)base_rep, (long long)lnv_rep};
    fwrite(hdr, 8, 2, f);
    fwrite(comm.data(), sizeof(GraphElem), comm.size(), f);
    fclose(f);
    FILE *fm = fopen((dumpPrefix + ".mask." + std::to_string(me)).c_str(), "wb");
    fwrite(movableOut.data(), 1, movableOut.size(), fm);
    fclose(fm);
    if (probeComm) {
      FILE *fu = fopen((dumpPrefix + ".unsettled." + std::to_string(me)).c_str(), "wb");
      fwrite(rc.unsettled.data(), 1, rc.unsettled.size(), fu);
      fclose(fu);
    }
  }
  if (me == 0 && evalPrefix.empty()) {            // (-E ran no Louvain phase: nothing to report)
    const double avgt = tot_time / nprocs, avgd = dev_time / nprocs;
    if (!generateGraph) {
      std::cout << "-------------------------------------------------------" << std::endl;
      std::cout << "File: " << inputFileName << std::endl;
      std::cout << "-------------------------------------------------------" << std::endl;
    }
    std::cout << "-------------------------------------------------------" << std::endl;
    std::cout << "64-bit datatype" << std::endl;
    std::cout << "-------------------------------------------------------" << std::endl;
    std::cout << "Average total time (in s), #Processes: " << avgt << ", " << nprocs << std::endl;
    std::cout << "Modularity, #Iterations: " << currMod << ", " << iters << std::endl;
    std::cout << "MODS (final modularity * average time): " << (currMod * avgt) << std::endl;
    std::cout << "-------------------------------------------------------" << std::endl;
    // additions of this build: device-side phase time (H2D upload excluded) and throughput
    std::cout << "GPU Louvain phase (in s), H2D upload (in s): " << avgd << ", " << rc.timings.h2d_s << std::endl;
    std::cout << "Edges/s (ne*iters/t), s/iter: " << (double)ne_rep * iters / avgd << ", " << avgd / iters << std::endl;
    std::cout << "-------------------------------------------------------" << std::endl;
    fprintf(stderr, "TIMINGS_MS total=%.3f setup=%.3f reorder=%.3f scan=%.3f fold=%.3f exchange=%.3f launches=%d reordered=%d\n",
            rc.timings.total_s * 1e3, rc.timings.setup_s * 1e3, rc.timings.reorder_s * 1e3, rc.timings.scan_s * 1e3,
            rc.timings.fold_s * 1e3, rc.timings.exchange_s * 1e3, (int)rc.timings.kernel_launches, (int)rc.timings.reordered);
    fprintf(stderr, "RESULT mod=%.17g iters=%d time=%.9g nv=%ld ne=%ld nprocs=%d threads=0\n", currMod, iters, avgd,
            (long)nv_rep, (long)ne_rep, nprocs);
    if (rc.stopped) fprintf(stderr, "STOPPED iters=%d prevMod=%.17g\n", iters, currMod);
  }
  rank_barrier();
  delete g;   // nullptr with -D
  fflush(stdout); fflush(stderr);
  if (me != 0) _exit(0);
  int st;
  while (wait(&st) > 0) {}
  return 0;
}
