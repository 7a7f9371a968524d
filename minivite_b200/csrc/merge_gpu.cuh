// Edge-parallel merge of a batch of deletions and insertions into a reference-format shard (DESIGN.md §3.11).
//
// A batch record is a key (local row << 31 | tail); both lists arrive sorted by key, the insertions stably, so equal
// keys keep batch order.  Per row v:
//   1. every old record whose tail equals the tail of some deletion (v, tail) is dropped, the rest keep their order;
//   2. the insertions are merged into the survivors with the loop "emit the next old record while its tail <= the
//      next insertion's tail, otherwise emit the insertion" -- std::stable_sort of the concatenation when the row is
//      sorted by tail, and still fully defined when it is not.
// No thread walks a row.  With M(a) = the running maximum of the kept tails of row v up to and including record a,
// the loop emits insertion b before kept record a exactly when tail(b) < M(a), so
//   kept record a      -> newrow[v] + #kept before a in v + #{insertions of v with tail < M(a)}
//   j-th insertion (t) -> newrow[v] + j + #{kept a of v with M(a) <= t}
// and both counts are binary searches (M is non-decreasing along a row).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace mv {

constexpr int kKeyShift = 31;
constexpr unsigned long long kKeyTail = (1ULL << kKeyShift) - 1;
constexpr long long kNoTail = -(1LL << 62);   // M of a record with no kept record up to it (below every tail)

struct MaxLL {
  __device__ __forceinline__ long long operator()(long long a, long long b) const { return a > b ? a : b; }
};

__device__ __forceinline__ long long lower_bound_u64(const unsigned long long *a, long long lo, long long hi, unsigned long long x) {
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

constexpr unsigned int kBadBatch = 1, kBadRowptr = 2;   // what k_batch_keys / k_rowptr_check raise in *bad

// the shard's offsets start at 0, end at lne and never decrease: every merge kernel trusts [rowptr[v], rowptr[v+1]),
// and an uploaded or attached shard has not been checked before its first run
__global__ void __launch_bounds__(256) k_rowptr_check(const long long *rowptr, long long n, long long lne, unsigned int *bad) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v <= n; v += (long long)gridDim.x * blockDim.x) {
    const long long r = rowptr[v];
    if ((v == 0 && r != 0) || (v == n && r != lne) || (v < n && rowptr[v + 1] < r)) atomicOr(bad, kBadRowptr);
  }
}

// batch records (global ids) -> keys; raises *bad for a record outside this shard's rows or outside [0, nv)
__global__ void __launch_bounds__(256) k_batch_keys(const long long *src, const long long *dst, long long n, long long base, long long bound,
                                                    long long nv, unsigned long long *key, unsigned int *idx, unsigned int *bad) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long s = src[i], d = dst[i];
    const bool ok = s >= base && s < bound && d >= 0 && d < nv;
    key[i] = ok ? ((unsigned long long)(s - base) << kKeyShift) | (unsigned long long)d : 0ULL;
    if (idx) idx[i] = (unsigned int)i;
    if (!ok) atomicOr(bad, kBadBatch);
  }
}

// start[v] = first sorted key of row v, v in [0, n]
__global__ void __launch_bounds__(256) k_row_bounds(const unsigned long long *skey, long long m, long long n, unsigned int *start) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v <= n; v += (long long)gridDim.x * blockDim.x)
    start[v] = (unsigned int)lower_bound_u64(skey, 0, m, (unsigned long long)v << kKeyShift);
}

// per old record: its row, kept (no deletion of (row, tail)), and the value the row's max-scan starts from
__global__ void __launch_bounds__(256) k_merge_keep(const long long *rowptr, const Edge16 *edges, long long lne, long long n,
                                                    const unsigned long long *dkey, const unsigned int *dstart, int32_t *erow,
                                                    unsigned int *kept, long long *mval) {
  for (long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x; a < lne; a += (long long)gridDim.x * blockDim.x) {
    long long lo = 0, hi = n;                   // the row: last v with rowptr[v] <= a
    while (lo < hi) {
      const long long mid = (lo + hi + 1) >> 1;
      if (rowptr[mid] <= a) lo = mid; else hi = mid - 1;
    }
    const long long v = lo, t = edges[a].tail;
    bool keep = true;
    long long d0 = dstart[v], d1 = dstart[v + 1];
    while (d0 < d1) {                           // deletion tails of row v are ascending
      const long long mid = (d0 + d1) >> 1;
      if ((long long)(dkey[mid] & kKeyTail) < t) d0 = mid + 1; else d1 = mid;
    }
    if (d0 < dstart[v + 1] && (long long)(dkey[d0] & kKeyTail) == t) keep = false;
    erow[a] = (int32_t)v;
    kept[a] = keep ? 1u : 0u;
    mval[a] = keep ? t : kNoTail;
  }
}

// new degree of every row (entry n = 0, so that an exclusive sum of n + 1 entries ends with the new lne)
__global__ void __launch_bounds__(256) k_merge_degree(const long long *rowptr, const unsigned int *kscan, const unsigned int *istart,
                                                      long long n, long long *deg) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v <= n; v += (long long)gridDim.x * blockDim.x)
    deg[v] = v == n ? 0 : (long long)(kscan[rowptr[v + 1]] - kscan[rowptr[v]]) + (long long)(istart[v + 1] - istart[v]);
}

__global__ void __launch_bounds__(256) k_merge_old(const long long *rowptr, const Edge16 *edges, long long lne, const int32_t *erow,
                                                   const unsigned int *kscan, const long long *mscan, const unsigned long long *ikey,
                                                   const unsigned int *istart, const long long *nrow, Edge16 *out) {
  for (long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x; a < lne; a += (long long)gridDim.x * blockDim.x) {
    if (kscan[a + 1] == kscan[a]) continue;     // deleted
    const long long v = erow[a], m = mscan[a];
    long long b0 = istart[v], b1 = istart[v + 1];
    const long long first = b0;
    while (b0 < b1) {                           // insertions of v with tail < M(a)
      const long long mid = (b0 + b1) >> 1;
      if ((long long)(ikey[mid] & kKeyTail) < m) b0 = mid + 1; else b1 = mid;
    }
    out[nrow[v] + (long long)(kscan[a] - kscan[rowptr[v]]) + (b0 - first)] = edges[a];
  }
}

__global__ void __launch_bounds__(256) k_merge_ins(const unsigned long long *ikey, const unsigned int *iidx, const double *iw, long long nins,
                                                   const unsigned int *istart, const long long *rowptr, const unsigned int *kscan,
                                                   const long long *mscan, const long long *nrow, Edge16 *out) {
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < nins; j += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = ikey[j];
    const long long v = (long long)(k >> kKeyShift), t = (long long)(k & kKeyTail);
    long long a0 = rowptr[v], a1 = rowptr[v + 1];
    const long long first = a0;
    while (a0 < a1) {                           // old records of v with M <= t (kept or not)
      const long long mid = (a0 + a1) >> 1;
      if (mscan[mid] <= t) a0 = mid + 1; else a1 = mid;
    }
    Edge16 r;
    r.tail = t;
    r.weight = iw[iidx[j]];
    out[nrow[v] + (j - (long long)istart[v]) + (long long)(kscan[a0] - kscan[first])] = r;
  }
}

}  // namespace mv
