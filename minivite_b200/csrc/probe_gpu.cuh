// Probing an assignment (mvgpu_probe_communities, DESIGN.md §3.15): what every vertex would do under the Louvain rule
// from assignment X, without moving anything.  The driver sets up like an evaluation (setup_run with an EvalSetup: warm
// init from X, no renumbering), so cur[] holds X on every own and ghost slot, the Comm records are X's, and internal ids
// are caller ids.  Per vertex the kernels give
//   best   the candidate community (a neighbour's community other than the own one) of largest gain, equal gains of any
//          value to the smaller id; -1 without a candidate;
//   gain   its gain (-inf without a candidate): the stability margin;
//   target the reference's decision (dspl.hpp:174-228, 309-324): best if gain > 0 and the singleton veto does not fire,
//          else the own community;
// and four global counters: moves (target != X), vetoed (gain > 0 but held by the veto), interior (records, no
// candidate) and the largest gain as an order-preserving key.
// k_probe is k_scan_ws's tile layout around the shared per-vertex helpers of kernels.cuh (vertex_load, pass0, pass1 with
// MARGIN, singleton_veto); k_probe_heavy takes the vertices above heavy_deg on k_scan_heavy's hash table (HeavyTable,
// kernels.cuh) with its own argmax.
#pragma once
#include "kernels.cuh"

namespace mv {

struct ProbeOut {
  int32_t *target, *best;            // lnv each, caller ids
  double *gain;                      // lnv
  unsigned long long *agg;           // [0] moves, [1] vetoed, [2] interior, [3] largest gain as probe_key (0: none)
};

// doubles -> unsigned keys in the same order (0 is the key of no double that a gain can be)
__device__ __forceinline__ unsigned long long probe_key(double g) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(g);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
}

struct ProbeCounts { unsigned long long moves = 0, vetoed = 0, interior = 0, kmax = 0; };

// the decision of vertex v (degree d, community cc) from its best candidate and that candidate's gain; stores the
// three per-vertex values and counts
template <bool UNIT, bool MULTI>
__device__ __forceinline__ void probe_decide(const ScanParams &p, const ProbeOut &o, int v, int cc, int d, int best, int lbest,
                                             double bg, ProbeCounts &n) {
  int t = cc;
  if (bg > 0.0) {
    t = singleton_veto<UNIT, MULTI>(p, cc, best, lbest, d);
    n.vetoed += t == cc;
  }
  n.moves += t != cc;
  n.interior += d > 0 && best < 0;
  n.kmax = max(n.kmax, probe_key(bg));
  o.target[v] = t;
  o.best[v] = best;
  o.gain[v] = bg;
}

__device__ __forceinline__ void probe_flush(const ProbeOut &o, const ProbeCounts &n) {
  const unsigned long long a = warp_sum(n.moves), b = warp_sum(n.vetoed), i = warp_sum(n.interior);
  unsigned long long k = n.kmax;
#pragma unroll
  for (int off = 16; off; off >>= 1) k = max(k, __shfl_xor_sync(0xffffffffu, k, off));
  if ((threadIdx.x & 31) == 0) {
    if (a) atomicAdd(o.agg + 0, a);
    if (b) atomicAdd(o.agg + 1, b);
    if (i) atomicAdd(o.agg + 2, i);
    if (k) atomicMax(o.agg + 3, k);
  }
}

// one CTA per tile of kTileV vertices: the neighbour communities (and weights) of the longest run of vertices that fits
// kECap staged edges go to shared memory edge-parallel, then every lane decides its own vertex.  Vertices above
// heavy_deg (<= kECap) are skipped here.
template <bool UNIT, bool MULTI>
__global__ void __launch_bounds__(kTileV) k_probe(const ScanParams p, const ProbeOut o) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int32_t *s_comm = reinterpret_cast<int32_t *>(smem_raw);
  double *s_w = reinterpret_cast<double *>(smem_raw + sizeof(int32_t) * kECap);
  __shared__ int s_next, s_end, s_skip;
  __shared__ uint32_t s_e0;

  const int tid = threadIdx.x;
  const int v0 = blockIdx.x * kTileV;
  const int v1 = min(p.lnv, v0 + kTileV);
  const int v = v0 + tid;
  uint32_t r0 = 0, r1 = 0;
  if (v < v1) { r0 = p.rowptr[v]; r1 = p.rowptr[v + 1]; }
  const uint32_t deg = r1 - r0;
  const bool is_heavy = deg > (uint32_t)p.heavy_deg;
  ProbeCounts n;

  int start = v0;
  while (start < v1) {
    if (tid == start - v0) { s_e0 = r0; s_skip = is_heavy ? 1 : 0; s_end = v1; }
    __syncthreads();
    if (s_skip) { start++; __syncthreads(); continue; }
    const uint32_t E0 = s_e0;
    if (v > start && v < v1 && (is_heavy || (r1 - E0 > (uint32_t)kECap))) atomicMin(&s_end, v);
    __syncthreads();
    const int end = s_end;
    if (tid == end - 1 - v0) s_next = (int)r1;
    __syncthreads();
    const int ne = (int)((uint32_t)s_next - E0);

    // edge-parallel staging: all tail loads of a pass before the first gather, all gathers before the first store
    {
      const int32_t *tl = p.tails + E0;
      for (int i0 = 0; i0 < ne; i0 += kStageU * kTileV) {
        int t[kStageU], cm[kStageU];
#pragma unroll
        for (int u = 0; u < kStageU; u++) {
          const int i = i0 + u * kTileV + tid;
          t[u] = (i < ne) ? ld_stream(tl + i) : -1;
        }
#pragma unroll
        for (int u = 0; u < kStageU; u++) cm[u] = (t[u] >= 0) ? __ldg(p.cur + t[u]) : 0;
#pragma unroll
        for (int u = 0; u < kStageU; u++) {
          const int i = i0 + u * kTileV + tid;
          if (i < ne) s_comm[i] = cm[u];
        }
      }
      if (!UNIT) {
        const double *wl = p.weights + E0;
        for (int k = tid; k < ne; k += kTileV) s_w[k] = ld_stream(wl + k);
      }
    }
    __syncthreads();

    const bool mine = (v >= start && v < end);
    const int d = mine ? (int)deg : 0;
    const int o0 = mine ? (int)(r0 - E0) : 0;
    int cc = 0;
    if (mine) cc = __ldg(p.cur + v);
    double cc_deg = 0.0, vdeg = 0.0, sl = 0.0;
    if (d) vertex_load<UNIT, MULTI>(p, v, cc, d, cc_deg, vdeg, sl);
    double w0;
    const int m = pass0<UNIT>(s_comm + o0, s_w + o0, d, cc, w0);
    const double eix = __dsub_rn(w0, sl), ax = __dsub_rn(cc_deg, vdeg);
    int best = -1, lbest = kNoLabel;
    double bg;
    pass1<UNIT, MULTI, true>(p, s_comm + o0, s_w + o0, m, eix, vdeg, ax, best, lbest, &bg);
    if (mine) probe_decide<UNIT, MULTI>(p, o, v, cc, d, best, lbest, bg, n);
    start = end;
    __syncthreads();
  }
  probe_flush(o, n);
}

// one CTA per vertex above heavy_deg: its HeavyTable (kernels.cuh), then a CTA-wide argmax that starts at -inf and
// sends equal gains of any value to the smaller id.
template <bool UNIT, bool MULTI>
__global__ void __launch_bounds__(256) k_probe_heavy(const ScanParams p, const ProbeOut o) {
  const int v = p.heavy_list[blockIdx.x];
  const HeavyTable<UNIT> tab(p);
  const int tid = threadIdx.x;
  const uint32_t e0 = p.rowptr[v], e1 = p.rowptr[v + 1];
  const int d = (int)(e1 - e0);
  const int cc = p.cur[v];
  __shared__ double s_w0;
  tab.fill(p, e0, e1, cc, s_w0);
  __shared__ double s_g[8];
  __shared__ int s_y[8], s_l[8];
  double cc_deg, vdeg, sl;
  vertex_load<UNIT, MULTI>(p, v, cc, d, cc_deg, vdeg, sl);
  const double eix = __dsub_rn(s_w0, sl), ax = __dsub_rn(cc_deg, vdeg);
  double bg = -INFINITY;
  int by = -1, lby = kNoLabel;
  for (unsigned int i = tid; i < tab.T; i += blockDim.x) {
    const int y = tab.keys[i];
    if (y < 0 || y == cc) continue;
    const double ay = UNIT ? (double)__ldg(at_cdeg<MULTI>(p, y)) : __ldg(&at_cinfo_w<MULTI>(p, y)->degree);
    const double eiy = tab.val(i);
    const double g = gain_of(eiy, eix, vdeg, ay, ax, p.constant, p.f32);
    if (better_l<MULTI, true>(p, g, y, bg, by, lby)) { bg = g; by = y; }
  }
  if (by >= 0 && lby == kNoLabel) lby = label_of<MULTI>(p, by);   // partial winners carry their label into the reduction
  auto wins = [](double og, int oy, int ol, double g, int y, int l) { return oy >= 0 && (y < 0 || og > g || (og == g && ol < l)); };
#pragma unroll
  for (int s = 16; s; s >>= 1) {
    const double og = __shfl_xor_sync(0xffffffffu, bg, s);
    const int oy = __shfl_xor_sync(0xffffffffu, by, s);
    const int ol = __shfl_xor_sync(0xffffffffu, lby, s);
    if (wins(og, oy, ol, bg, by, lby)) { bg = og; by = oy; lby = ol; }
  }
  if ((tid & 31) == 0) { s_g[tid >> 5] = bg; s_y[tid >> 5] = by; s_l[tid >> 5] = lby; }
  __syncthreads();
  if (tid < 32) {
    bg = -INFINITY; by = -1; lby = kNoLabel;
    if (tid == 0)
      for (int w = 0; w < (int)(blockDim.x >> 5); w++)
        if (wins(s_g[w], s_y[w], s_l[w], bg, by, lby)) { bg = s_g[w]; by = s_y[w]; lby = s_l[w]; }
    ProbeCounts n;
    if (tid == 0) probe_decide<UNIT, MULTI>(p, o, v, cc, d, by, lby, bg, n);
    probe_flush(o, n);
  }
}

}  // namespace mv
