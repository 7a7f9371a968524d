// Comparing two community assignments X and Y (mvgpu_compare_communities, DESIGN.md §3.13).
//
// Everything here is integer counting, so every result is exact and independent of the thread order:
//   cell key     (x << shift) | y per vertex, shift = the bits of an id in [0, nv); sorted, run-length encoded, routed
//                to owner(x) (the key order is the owner order) and summed there: n_xy of every owned x, once each
//   rows         per owned x a CUB reduce-by-key over its cells: a_x = sum n_xy, and the best match as the maximum of
//                (n_xy << 32 | kIdMax - y) -- the largest overlap, ties to the smallest y
//   b_y          the same route for the key y alone, at owner(y)
//   best_size    b of every row's best match, fetched from owner(best) by one request / reply exchange
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"
#include "merge_gpu.cuh"

namespace mv {

constexpr unsigned long long kIdMax = 0x7fffffffULL;   // ids are < 2^31: kIdMax - y orders ties by the smallest y

struct CmpParts {                          // the vertex ranges, for routing keys to the owner of their top bits
  long long p[kMaxRanks + 1];
  int n;
};

// per owned community x: best = max over its cells of (n_xy << 32 | kIdMax - y), size = sum of n_xy
struct CmpRow {
  unsigned long long best, size;
};
struct CmpRowOp {
  __device__ __forceinline__ CmpRow operator()(const CmpRow &a, const CmpRow &b) const {
    return {a.best > b.best ? a.best : b.best, a.size + b.size};
  }
};
struct CmpSum {
  __device__ __forceinline__ uint32_t operator()(uint32_t a, uint32_t b) const { return a + b; }
};

// key[v] = X[v] << shift | Y[v]; X == NULL: key[v] = Y[v]
__global__ void __launch_bounds__(256) k_cmp_keys(int lnv, const int32_t *X, const int32_t *Y, int shift, unsigned long long *key) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < lnv; v += gridDim.x * blockDim.x)
    key[v] = (X ? (unsigned long long)X[v] << shift : 0ULL) | (unsigned long long)Y[v];
}

// off[r] = the first sorted key whose top bits (key >> shift) are >= parts[r], for r = 0..n: the keys of rank r's ids
// are [off[r], off[r+1])
__global__ void k_cmp_bounds(const unsigned long long *key, long long n, CmpParts parts, int shift, long long *off) {
  const int r = threadIdx.x;
  if (r <= parts.n) off[r] = lower_bound_u64(key, 0, n, (unsigned long long)parts.p[r] << shift);
}

// one cell (key, count) of an owned x -> its row slot x - base and its CmpRow
__global__ void __launch_bounds__(256) k_cmp_cell_rows(long long n, const unsigned long long *key, const uint32_t *cnt, int shift,
                                                       long long base, int32_t *slot, CmpRow *row) {
  const unsigned long long ymask = (1ULL << shift) - 1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = key[i];
    slot[i] = (int32_t)((long long)(k >> shift) - base);
    row[i] = {(unsigned long long)cnt[i] << 32 | (kIdMax - (k & ymask)), cnt[i]};
  }
}

// match arrays m = [size | best | overlap | best_size], lnv each: every slot starts as an empty community
__global__ void __launch_bounds__(256) k_cmp_match_init(int lnv, long long *m) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < lnv; s += gridDim.x * blockDim.x) {
    m[s] = 0; m[lnv + s] = -1; m[2 * (size_t)lnv + s] = 0; m[3 * (size_t)lnv + s] = 0;
  }
}

// the non-empty rows: size, best and overlap into m; their sizes (for the histogram) and the best-size requests
// (key = best y, value = the asking slot)
__global__ void __launch_bounds__(256) k_cmp_rows(int nrows, int lnv, const int32_t *slot, const CmpRow *row, long long *m,
                                                  uint32_t *size, unsigned long long *req, int32_t *req_slot) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nrows; j += gridDim.x * blockDim.x) {
    const int s = slot[j];
    const CmpRow r = row[j];
    const long long y = (long long)(kIdMax - (r.best & 0xffffffffULL));
    m[s] = (long long)r.size;
    m[lnv + s] = y;
    m[2 * (size_t)lnv + s] = (long long)(r.best >> 32);
    size[j] = (uint32_t)r.size;
    req[j] = (unsigned long long)y;
    req_slot[j] = s;
  }
}

// b_y of the owned ids y that occur (key = y, count = b_y) into the dense array b (zero elsewhere)
__global__ void __launch_bounds__(256) k_cmp_scatter_b(long long n, const unsigned long long *key, const uint32_t *cnt, long long base,
                                                       uint32_t *b) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    b[key[i] - base] = cnt[i];
}

// at owner(y): the reply to every request y is b_y
__global__ void __launch_bounds__(256) k_cmp_lookup(long long n, const unsigned long long *req, long long base, const uint32_t *b,
                                                    uint32_t *reply) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    reply[i] = b[req[i] - base];
}

// back at the asking rank: best_size of the asking slot
__global__ void __launch_bounds__(256) k_cmp_best_size(long long n, const int32_t *slot, const uint32_t *got, int lnv, long long *m) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m[3 * (size_t)lnv + slot[i]] = got[i];
}

}  // namespace mv
