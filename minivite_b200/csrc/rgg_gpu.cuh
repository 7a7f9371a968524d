// Device-side random geometric graph generator: SURVEY.md section 8(f) rank 1, the step *before* the Louvain path.
//
// Builds strip `rank` of the graph `miniVite -n nv` creates on `nranks` ranks (reference GenerateRGG,
// graph.hpp:584-1213, default RNG path, no -l / -p) directly in HBM, in the reference's own array format
// (int64 rowptr[lnv+1], {int64 tail; double weight}[lne]), bit-identical to the reference generator and to this
// repo's host generator (host/rgg.hpp).  `-l` (the reference's LCG class, utils.hpp:118-303) is supported too: rank r's
// coordinates are entries [2 n r, 2 n (r+1)) of x <- 16807 x mod 2^31-1, its first entry coming from the reference's
// wrapping 64-bit matrix power (evaluated on the host, handed over as |first|); every strip has its own point pattern
// there, so coordinates are kept per strip.  Default RNG path:
//   * coordinates: minstd_rand0 (x <- 16807 x mod 2^31-1) seeded with reseeder(1); vertex i consumes outputs
//     4i+1..4i+4 (two per double, std::generate_canonical<double,53>); every strip restarts from the same seed
//     (graph.hpp:680-700).  The generator is a pure multiplicative LCG, so thread i jumps to its position with one
//     modular power instead of replaying the stream;
//   * radius and predicate: rn of graph.hpp:629-631, sqrt(dx*dx+dy*dy) <= rn in fp64 with explicit _rn operations
//     (no FMA contraction), pairs between adjacent strips skipped when the local indices are equal
//     (graph.hpp:817,849);
//   * uniform cell grid (cell width >= rn) instead of the reference's O((n/p)^2) loops; adjacency sorted by tail
//     (graph.hpp:1145-1153).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace mv {

struct RggParams {
  long long n;               // vertices per strip
  int rank, nranks;
  unsigned int seed;         // (unsigned)reseeder(1)
  double rn;                 // radius
  double rec_np;             // 1/nranks as the reference computes it
  double r_range;            // 2147483646.0  (urng.max() - urng.min() + 1)
  double r_range2;           // (double)(r_range * r_range evaluated in long double), the divisor of generate_canonical
  long long ncell;           // cells per unit length
  long long row0, nrows;     // slab of cell rows this strip can reach
  double ylo, yhi;           // candidate band
  int lcg;                   // -l: coordinates from the reference's LCG stream instead of minstd_rand0 + generate_canonical
  unsigned long long lcg_first[3];   // |first entry| of the strips rank-1, rank, rank+1 (utils.hpp:146-218)
  double lcg_mult;           // 1 / (1 + (M - 1)) as the reference evaluates it
};

__device__ __forceinline__ unsigned long long mulmod31(unsigned long long a, unsigned long long b) {
  return (a * b) % 2147483647ULL;
}
__device__ __forceinline__ unsigned long long powmod31(unsigned long long a, unsigned long long e) {
  unsigned long long r = 1;
  while (e) { if (e & 1) r = mulmod31(r, a); a = mulmod31(a, a); e >>= 1; }
  return r;
}
// std::generate_canonical<double,53>(minstd_rand0): two draws; sum and divisor rounded exactly as libstdc++ does
__device__ __forceinline__ double canonical2(unsigned long long o1, unsigned long long o2, const RggParams &p) {
  double sum = (double)(o1 - 1ULL);                                   // * tmp (= 1.0)
  sum = __dadd_rn(sum, __dmul_rn((double)(o2 - 1ULL), p.r_range));
  double ret = __ddiv_rn(sum, p.r_range2);
  if (ret >= 1.0) ret = 0.99999999999999988898;                       // nextafter(1.0, 0.0)
  return ret;
}
// canonical X and canonical Y of local index i (identical for every strip)
__device__ __forceinline__ void point_canon(long long i, const RggParams &p, double &ux, double &uy) {
  unsigned long long x0 = (unsigned long long)p.seed % 2147483647ULL;
  if (x0 == 0) x0 = 1;
  unsigned long long x = mulmod31(x0, powmod31(16807ULL, (unsigned long long)(4 * i)));
  const unsigned long long o1 = mulmod31(x, 16807ULL), o2 = mulmod31(o1, 16807ULL), o3 = mulmod31(o2, 16807ULL),
                           o4 = mulmod31(o3, 16807ULL);
  ux = canonical2(o1, o2, p);
  uy = canonical2(o3, o4, p);
}
__device__ __forceinline__ double strip_y(double uy, int s, const RggParams &p) {
  const double lo = __dmul_rn((double)s, p.rec_np), hi = __dadd_rn(lo, p.rec_np);
  return __dadd_rn(__dmul_rn(uy, __dsub_rn(hi, lo)), lo);           // uniform_real_distribution: u*(b-a)+a
}
__device__ __forceinline__ long long cell_of(double v, long long ncell) {
  long long c = (long long)floor(__dmul_rn(v, (double)ncell));
  return c < 0 ? 0 : (c >= ncell ? ncell - 1 : c);
}

// coordinates of local index i of strip s (s in [rank-1, rank+1]): x and absolute y
__device__ __forceinline__ void strip_point(long long i, int s, const RggParams &p, double &x, double &y) {
  if (!p.lcg) {
    double ux, uy;
    point_canon(i, p, ux, uy);
    x = __dadd_rn(__dmul_rn(ux, 1.0), 0.0);
    y = strip_y(uy, s, p);
    return;
  }
  // utils.hpp:118-303 as the host generator restates it (host/rgg.hpp strip_points): entry k of the strip's stream is
  // first * 16807^k mod M with C++'s sign-preserving %, only its magnitude is used
  const unsigned long long f = p.lcg_first[s - p.rank + 1];
  const unsigned long long ax = mulmod31(f, powmod31(16807ULL, (unsigned long long)i));
  const unsigned long long ay = mulmod31(f, powmod31(16807ULL, (unsigned long long)(p.n + i)));
  x = __dmul_rn((double)ax, p.lcg_mult);
  const double lo = __dmul_rn((double)s, p.rec_np);
  y = __dadd_rn(lo, __dmul_rn(p.rec_np, __dmul_rn((double)ay, p.lcg_mult)));
}

// coordinates of the own and the two adjacent strips: X3/Y3[(s - s0) * n + i]
__global__ void __launch_bounds__(256) k_rgg_points(RggParams p, double *X3, double *Y3) {
  const int s0 = max(0, p.rank - 1), s1 = min(p.nranks - 1, p.rank + 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x)
    for (int s = s0; s <= s1; s++) {
      double x, y;
      strip_point(i, s, p, x, y);
      X3[(long long)(s - s0) * p.n + i] = x;
      Y3[(long long)(s - s0) * p.n + i] = y;
    }
}

// candidates = all points of the own strip + the points of the adjacent strips inside the band [ylo, yhi];
// pass 0 counts per cell, pass 1 scatters (cell-sorted arrays cx, cy, cgid)
__global__ void __launch_bounds__(256) k_rgg_bin(RggParams p, const double *X3, const double *Y3, int pass, unsigned int *cell_cnt,
                                                 const unsigned int *cell_start, double *cx, double *cy, long long *cgid) {
  const int s0 = max(0, p.rank - 1), s1 = min(p.nranks - 1, p.rank + 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    for (int s = s0; s <= s1; s++) {
      const double x = X3[(long long)(s - s0) * p.n + i], y = Y3[(long long)(s - s0) * p.n + i];
      if (y < p.ylo || y > p.yhi) continue;
      const long long row = cell_of(y, p.ncell);
      if (row < p.row0 || row >= p.row0 + p.nrows) continue;
      const long long c = (row - p.row0) * p.ncell + cell_of(x, p.ncell);
      if (pass == 0) atomicAdd(&cell_cnt[c], 1u);
      else {
        const unsigned int pos = cell_start[c] + atomicAdd(&cell_cnt[c], 1u);
        cx[pos] = x; cy[pos] = y; cgid[pos] = (long long)s * p.n + i;
      }
    }
  }
}

// neighbours of local vertex i: pass 0 counts (deg), pass 1 writes {tail, weight} records, then sorts them by tail
template <bool FILL>
__global__ void __launch_bounds__(128) k_rgg_neighbours(RggParams p, const double *X3, const double *Y3, const unsigned int *cell_start,
                                                        const double *cx, const double *cy, const long long *cgid, int unit,
                                                        long long *deg_or_rowptr, Edge16 *edges) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    const long long own = (long long)(p.rank - max(0, p.rank - 1)) * p.n;
    const double xi = X3[own + i], yi = Y3[own + i];
    const long long row = cell_of(yi, p.ncell), col = cell_of(xi, p.ncell);
    const long long c0 = max(0LL, col - 1), c1 = min(p.ncell - 1, col + 1);
    long long cnt = 0;
    Edge16 *out = FILL ? edges + deg_or_rowptr[i] : nullptr;
    for (long long rr = max(p.row0, row - 1); rr <= min(p.row0 + p.nrows - 1, row + 1); rr++) {
      const unsigned int b = cell_start[(rr - p.row0) * p.ncell + c0], e = cell_start[(rr - p.row0) * p.ncell + c1 + 1];
      for (unsigned int k = b; k < e; k++) {
        const double dx = __dsub_rn(xi, cx[k]), dy = __dsub_rn(yi, cy[k]);
        const double ed = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
        if (!(ed <= p.rn)) continue;
        const long long g = cgid[k];
        if (g % p.n == i) continue;          // the vertex itself, or the equal-index vertex of an adjacent strip
        if (FILL) { out[cnt].tail = g; out[cnt].weight = unit ? 1.0 : ed; }
        cnt++;
      }
    }
    if (!FILL) deg_or_rowptr[i] = cnt;
    else {
      for (long long a = 1; a < cnt; a++) {              // insertion sort by tail (a few dozen entries at most)
        const Edge16 key = out[a];
        long long b2 = a - 1;
        while (b2 >= 0 && out[b2].tail > key.tail) { out[b2 + 1] = out[b2]; b2--; }
        out[b2 + 1] = key;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Random long edges (`-p`, GenerateRGG graph.hpp:939-1122 as host/rgg.hpp add_random_edges restates it with a fixed
// seed). Stream s (= generating rank s) draws pnrande(s) pairs (i, g_j) from minstd_rand0(seed + s); a pair becomes an
// edge unless i == j, i -> g_j is an RGG edge of strip s, or stream s added the same pair before. The draws are
// sequential per stream (one thread each, p streams); everything after them is data parallel.
// ---------------------------------------------------------------------------------------------------------------
struct RandeParams {
  long long n, nv;           // vertices per strip, in total
  int p, me;
  unsigned int seed;         // stream s is seeded with seed + s
};

// libstdc++ uniform_int_distribution over a generator whose range (2147483646 values) is not a power of two:
// scale down with rejection (bits/uniform_int_dist.h, the "downscaling" branch)
__device__ __forceinline__ unsigned long long minstd_below(unsigned long long &x, unsigned long long scaling, unsigned long long past) {
  unsigned long long ret;
  do {
    x = mulmod31(x, 16807ULL);
    ret = x - 1ULL;
  } while (ret >= past);
  return ret / scaling;
}

__global__ void k_rande_draws(RandeParams rp, const long long *soff, int *di, int *dgj) {
  if (threadIdx.x) return;
  const int s = blockIdx.x;
  unsigned long long x = (unsigned long long)(rp.seed + (unsigned int)s) % 2147483647ULL;
  if (x == 0) x = 1;
  const unsigned long long sc_i = 2147483645ULL / (unsigned long long)rp.n, past_i = (unsigned long long)rp.n * sc_i;
  const unsigned long long sc_j = 2147483645ULL / (unsigned long long)rp.nv, past_j = (unsigned long long)rp.nv * sc_j;
  for (long long q = soff[s]; q < soff[s + 1]; q++) {
    di[q] = (int)minstd_below(x, sc_i, past_i);
    dgj[q] = (int)minstd_below(x, sc_j, past_j);
  }
}

__device__ __forceinline__ int rande_stream_of(const long long *soff, int p, long long q) {
  int s = 0;
  while (s + 1 < p && q >= soff[s + 1]) s++;
  return s;
}

// key[q] = (g_i, g_j) packed for the draws that touch this strip and are not RGG edges, ~0 for the rest.
// RGG adjacency is symmetric, so "i -> g_j is an edge of strip s" is answered from g_j's own list when s is remote.
__global__ void __launch_bounds__(256) k_rande_keys(RandeParams rp, const long long *soff, const int *di, const int *dgj, long long nr,
                                                    const long long *rowptr, const Edge16 *edges, unsigned long long *key,
                                                    unsigned int *qidx) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nr; q += (long long)gridDim.x * blockDim.x) {
    const int s = rande_stream_of(soff, rp.p, q);
    const long long i = di[q], gj = dgj[q];
    const int target = (int)(gj / rp.n);
    const long long j = gj - (long long)target * rp.n, gi = (long long)s * rp.n + i;
    unsigned long long k = ~0ULL;
    if ((s == rp.me || target == rp.me) && i != j) {
      const long long lv = s == rp.me ? i : j, want = s == rp.me ? gj : gi;
      long long lo = rowptr[lv], hi = rowptr[lv + 1];
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (edges[mid].tail < want) lo = mid + 1; else hi = mid;
      }
      const bool in_rgg = lo < rowptr[lv + 1] && edges[lo].tail == want;
      if (!in_rgg) k = (unsigned long long)gi * (unsigned long long)rp.nv + (unsigned long long)gj;
    }
    key[q] = k;
    qidx[q] = (unsigned int)q;
  }
}

// after the stable sort by key: the first draw of every run of equal keys is the one the reference keeps
__global__ void __launch_bounds__(256) k_rande_first(const unsigned long long *skey, const unsigned int *sq, long long nr, RandeParams rp,
                                                     const long long *soff, const int *dgj, unsigned int *emit) {
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < nr; k += (long long)gridDim.x * blockDim.x) {
    const unsigned long long key = skey[k];
    const unsigned int q = sq[k];
    unsigned int cnt = 0;
    if (key != ~0ULL && (k == 0 || skey[k - 1] != key)) {
      const int s = rande_stream_of(soff, rp.p, q);
      const int target = (int)((long long)dgj[q] / rp.n);
      cnt = (s == rp.me ? 1u : 0u) + (target == rp.me ? 1u : 0u);
    }
    emit[q] = cnt;
  }
}

// the extra records of this strip in the reference's push order (stream, draw, forward before reverse):
// xkey = (local source vertex, tail) for the stable sort that follows, xw = weight
__global__ void __launch_bounds__(256) k_rande_emit(RandeParams rp, RggParams gp, const long long *soff, const int *di, const int *dgj,
                                                    long long nr, const unsigned int *emit, const unsigned int *epos, int unit,
                                                    const double *X3, const double *Y3, unsigned long long *xkey, double *xw,
                                                    unsigned int *xidx) {
  const int s0 = max(0, rp.me - 1);
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nr; q += (long long)gridDim.x * blockDim.x) {
    const unsigned int cnt = emit[q];
    if (!cnt) continue;
    const int s = rande_stream_of(soff, rp.p, q);
    const long long i = di[q], gj = dgj[q];
    const int target = (int)(gj / rp.n);
    const long long j = gj - (long long)target * rp.n, gi = (long long)s * rp.n + i;
    double w = 1.0;
    if (!unit) {
      if (target == s || target == s - 1 || target == s + 1) {
        const double dx = __dsub_rn(X3[(long long)(s - s0) * rp.n + i], X3[(long long)(target - s0) * rp.n + j]);
        const double dy = __dsub_rn(Y3[(long long)(s - s0) * rp.n + i], Y3[(long long)(target - s0) * rp.n + j]);
        w = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
      } else {
        // minstd_rand0((unsigned)hash(g_i * nv + g_j)) -> uniform_real_distribution(0.01, 1.0)
        unsigned long long x = (unsigned long long)(unsigned int)((unsigned long long)gi * (unsigned long long)rp.nv + (unsigned long long)gj) % 2147483647ULL;
        if (x == 0) x = 1;
        const unsigned long long o1 = mulmod31(x, 16807ULL), o2 = mulmod31(o1, 16807ULL);
        w = __dadd_rn(__dmul_rn(canonical2(o1, o2, gp), __dsub_rn(1.0, 0.01)), 0.01);
      }
    }
    unsigned int e = epos[q];
    if (s == rp.me) {
      xkey[e] = ((unsigned long long)i << 31) | (unsigned long long)gj;
      xw[e] = w; xidx[e] = e;
      e++;
    }
    if (target == rp.me) {
      xkey[e] = ((unsigned long long)j << 31) | (unsigned long long)gi;
      xw[e] = w; xidx[e] = e;
    }
  }
}

}  // namespace mv
