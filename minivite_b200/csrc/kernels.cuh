// Device kernels of the Louvain phase for sm_90a (H100).  Hand-written CUDA; no tensor cores: the
// path is a sparse gather/scan (SURVEY.md section 8(d)).  With the reference's vertex numbering it is bound by HBM
// sector throughput (random 4-byte gathers); after the locality renumbering below it is instruction-issue bound.
//
// Data layout in HBM (per rank/GPU; built once per run by the setup kernels from the reference-format
// arrays int64 rowptr[lnv+1] + {int64 tail; double w}[lne]):
//   rowptr   uint32[lnv+1]          local edge offsets (lne < 2^32 per shard)
//   tails    int32[lne]             LOCAL SLOT of the neighbour: [0,lnv) own vertex, [lnv,lnv+nghost) ghost
//                                   (replaces the reference's per-edge owner test + unordered_map lookup,
//                                   dspl.hpp:251-260)
//   weights  double[lne]            only when some weight != 1.0
//   cur/tgt  int32[lnv+nghost]      community (global internal id) of every slot; ghosts are refreshed by the
//                                   per-iteration exchange (dspl.hpp:559-688)
//   lab      int32[lnv]             after renumbering: original global vertex id of every internal id (labels)
//   unit-weight fast path (all weights 1, 2m < 2^31): Comm{size,degree} (dspl.hpp:61-66) as exact integers, SoA:
//     cdeg   uint32[lnv]  community degree: the only field the gain needs (4 B gather per candidate)
//     csize  int32[lnv]   community size: read only for the singleton veto (dspl.hpp:224-225)
//     upd    uint64[lnv]  = dsize*2^32 + ddeg packed two's-complement delta: ONE 64-bit atomic per community
//                           update (dspl.hpp:339-346); fold decodes it (dspl.hpp:458-471)
//   weighted path: cinfo_w {int64 size; double degree}[lnv], usize int64[lnv], udeg double[lnv], vdeg double[lnv]
// With 32-bit ids the gathered arrays at 16M vertices are 64 MB (cur) + 64 MB (cdeg).  L2 policy hints alone did
// not keep them resident (measured); the renumbering makes the gathers local instead.  Streamed arrays (tails,
// rowptr, target writes) still carry an L2 evict_first policy.
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mv {

#ifndef MV_TILE_V
#define MV_TILE_V 128
#endif
#ifndef MV_ECAP
#define MV_ECAP 2048
#endif
constexpr int kTileV = MV_TILE_V;  // vertices per CTA tile == threads per CTA
constexpr int kECap = MV_ECAP;     // edges staged in shared memory per sub-range
#ifndef MV_STAGE_U
#define MV_STAGE_U 6
#endif
constexpr int kStageU = MV_STAGE_U;  // phase A: independent loads in flight per thread
constexpr int kMaxRanks = 16;

struct Edge16 { long long tail; double weight; };          // reference graph.hpp:60-66
struct CommW { long long size; double degree; };           // reference dspl.hpp:61-66

struct Acc {                       // per-iteration accumulators (one record per iteration, never reset)
  unsigned long long le_u;         // unit path: sum of counter[0] (dspl.hpp:318, 431)
  unsigned long long la2_u;        // unit path: sum of degree^2 (dspl.hpp:432)
  double le_d, la2_d;              // weighted path
  unsigned long long moved, hash;  // trace (optional)
};

struct PeerTable {                 // where community y lives: owner rank + that rank's arrays
  int nranks, rank;
  long long parts[kMaxRanks + 1];
  const uint32_t *cdeg[kMaxRanks];
  const int32_t *csize[kMaxRanks];
  unsigned long long *upd[kMaxRanks];
  const CommW *cinfo_w[kMaxRanks];
  long long *usize[kMaxRanks];
  double *udeg[kMaxRanks];
  const int32_t *lab[kMaxRanks];   // label (original global vertex id) of every internal vertex/community id
};

struct ScanParams {
  int lnv;
  int has_self;                    // any self loop in the shard (uniform branch)
  int heavy_deg;                   // degree > heavy_deg is left to the high-degree kernel (<= kECap)
  int has_heavy;                   // the shard has such vertices at all (uniform fast path when it has none)
  int relabel;                     // vertices were renumbered for locality: ids are internal, tie-breaks use labels
  int cache_policy;                // bit2: L2 evict_first on the streamed arrays (tails, target writes); bits 0-1 unused
                                   // (evict_last hints on the gathered arrays were measured without effect and removed)
  long long base;                  // global id of local vertex 0
  const uint32_t *rowptr;
  const int32_t *tails;
  const double *weights;
  const int32_t *cur;
  int32_t *tgt;
  const int32_t *self_i;           // unit: self-loop count per vertex
  const double *self_d;            // weighted: truncated self-loop weight (dspl.hpp:285)
  const double *vdeg;              // weighted: vertex degree (dspl.hpp:82-107)
  double constant;                 // 1/(2m) (dspl.hpp:129)
  int f32;                         // emulate the reference's USE_32_BIT_GRAPH arithmetic in the gain (see gain_of)
  Acc *acc;
  // high-degree scratch
  const int32_t *heavy_list;
  const unsigned long long *heavy_off;   // table offsets (entries), heavy_count+1
  int32_t *hkeys;
  double *hvals_d;
  int32_t *hvals_i;
  // this rank's own community arrays (the common case: no indexed constant-bank load)
  const uint32_t *loc_cdeg;
  const int32_t *loc_csize;
  unsigned long long *loc_upd;
  const CommW *loc_cinfo_w;
  long long *loc_usize;
  double *loc_udeg;
  const int32_t *loc_lab;
  PeerTable pt;
};

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
__device__ __forceinline__ unsigned long long vhash(long long gid, long long val) {
  return mix64(((unsigned long long)gid) * 0x9E3779B97F4A7C15ULL ^ (unsigned long long)val);
}

// streaming (read-once) and read-only gathers
__device__ __forceinline__ int ld_stream(const int32_t *p) { return __ldcs(p); }
__device__ __forceinline__ double ld_stream(const double *p) { return __ldcs(p); }

// L2 cache-policy descriptors (createpolicy) and loads/stores that carry them
__device__ __forceinline__ unsigned long long make_policy(int kind) {   // 0 normal, 1 evict_last, 2 evict_first
  unsigned long long pol;
  if (kind == 1) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  else if (kind == 2) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  else asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ int ld_pol_stream(const int32_t *p, unsigned long long pol) {
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_pol(int32_t *p, int v, unsigned long long pol) {
  asm volatile("st.global.L2::cache_hint.s32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}

template <bool MULTI>
__device__ __forceinline__ void locate_impl(const PeerTable &pt, long long base, int lnv, int y, int &owner, long long &idx) {
  if (!MULTI) { owner = 0; idx = (long long)y - base; return; }
  // almost every community a vertex meets is owned by its own rank: test that range first (plain kernel parameters,
  // no indexed constant-bank loads)
  const long long i = (long long)y - base;
  if ((unsigned long long)i < (unsigned long long)lnv) { owner = pt.rank; idx = i; return; }
  int o = 0;
#pragma unroll 1
  while (o + 1 < pt.nranks && (long long)y >= pt.parts[o + 1]) o++;
  owner = o;
  idx = (long long)y - pt.parts[o];
}

#define MV_PTR(field, type)                                                                          \
  template <bool MULTI>                                                                              \
  __device__ __forceinline__ type ptr_##field(const ScanParams &p, int o) {                          \
    return (!MULTI || o == p.pt.rank) ? p.loc_##field : p.pt.field[o];                               \
  }
MV_PTR(cdeg, const uint32_t *)
MV_PTR(csize, const int32_t *)
MV_PTR(upd, unsigned long long *)
MV_PTR(cinfo_w, const CommW *)
MV_PTR(usize, long long *)
MV_PTR(udeg, double *)
MV_PTR(lab, const int32_t *)
#undef MV_PTR

// element of a community array by (internal, global) community id: one 32-bit range test for the common case
// "owned by this rank", the owner search only for remote communities
__device__ __forceinline__ void locate_remote(const PeerTable &pt, int y, int &owner, long long &idx) {
  int o = 0;
#pragma unroll 1
  while (o + 1 < pt.nranks && (long long)y >= pt.parts[o + 1]) o++;
  owner = o;
  idx = (long long)y - pt.parts[o];
}
#define MV_AT(field, type)                                                                           \
  template <bool MULTI>                                                                              \
  __device__ __forceinline__ type at_##field(const ScanParams &p, int y) {                           \
    /* single rank: signed 64-bit index, so the compiler can fold "- base" into the array pointer */ \
    if (!MULTI) return p.loc_##field + ((long long)y - p.base);                                      \
    const unsigned int i = (unsigned int)(y - (int)p.base);                                          \
    if (i < (unsigned int)p.lnv) return p.loc_##field + i;                                           \
    int o; long long idx;                                                                            \
    locate_remote(p.pt, y, o, idx);                                                                  \
    return p.pt.field[o] + idx;                                                                      \
  }
MV_AT(cdeg, const uint32_t *)
MV_AT(csize, const int32_t *)
MV_AT(upd, unsigned long long *)
MV_AT(cinfo_w, const CommW *)
MV_AT(usize, long long *)
MV_AT(udeg, double *)
MV_AT(lab, const int32_t *)
#undef MV_AT

__device__ __forceinline__ unsigned long long pack_delta(int dsize, long long ddeg) {
  return (unsigned long long)(((long long)dsize << 32) + ddeg);
}

// dspl.hpp:212 with the reference's evaluation order and no FMA contraction:
//   curGain = 2.0*(eiy-eix) - ((2.0*vDegree)*(ay-ax))*constant
// f32 = the reference's USE_32_BIT_GRAPH build (utils.hpp:72-82): GraphWeight is float there, so (eiy-eix) and (ay-ax)
// are float subtractions, the 2.0 literals promote the rest to double, and the assignment to `GraphWeight curGain`
// rounds the result to float.  The values handed in are exact integers (or doubles made from floats), so rounding the
// two differences and the result to float reproduces that build's gain bit for bit.
__device__ __forceinline__ double gain_of(double eiy, double eix, double vdeg, double ay, double ax, double c, int f32 = 0) {
  double de = __dsub_rn(eiy, eix), da = __dsub_rn(ay, ax);
  if (f32) { de = (double)__double2float_rn(de); da = (double)__double2float_rn(da); }
  const double t1 = __dmul_rn(2.0, de);
  const double t2 = __dmul_rn(__dmul_rn(__dmul_rn(2.0, vdeg), da), c);
  const double g = __dsub_rn(t1, t2);
  return f32 ? (double)__double2float_rn(g) : g;
}

// (gain, id) ordering of dspl.hpp:214-215: larger gain wins; equal non-zero gains -> smaller id (better_l below).
// Locality renumbering keeps the reference's semantics by comparing LABELS (original global vertex ids of
// the community founders) wherever the reference compares community ids (dspl.hpp:215, 224).
constexpr int kNoLabel = (int)0x80000000;
template <bool MULTI>
__device__ __forceinline__ int label_of(const ScanParams &p, int c) {
  if (!p.relabel) return c;
  return __ldg(at_lab<MULTI>(p, c));
}
// better() with lazily fetched labels; lby caches the label of the current best (kNoLabel = not fetched)
template <bool MULTI>
__device__ __forceinline__ bool better_l(const ScanParams &p, double g, int y, double bg, int by, int &lby) {
  if (g > bg) { lby = kNoLabel; return true; }
  if ((g == bg) && (g != 0.0)) {
    const int ly = label_of<MULTI>(p, y);
    if (lby == kNoLabel) lby = label_of<MULTI>(p, by);
    if (ly < lby) { lby = ly; return true; }
  }
  return false;
}
// dspl.hpp:224: maxIndex > currComm, on labels
template <bool MULTI>
__device__ __forceinline__ bool label_greater(const ScanParams &p, int best, int lbest, int cc) {
  if (best == cc) return false;
  if (!p.relabel) return best > cc;
  if (lbest == kNoLabel) lbest = label_of<MULTI>(p, best);
  return lbest > label_of<MULTI>(p, cc);
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- helpers shared by the scan kernels ----------------------------------------------------------------
template <bool MULTI>
__device__ __forceinline__ void push_move_unit(const ScanParams &p, int cc, int best, int d) {
  atomicAdd(at_upd<MULTI>(p, best), pack_delta(1, (long long)d));
  atomicAdd(at_upd<MULTI>(p, cc), pack_delta(-1, -(long long)d));
}

template <bool MULTI>
__device__ __forceinline__ void push_move_w(const ScanParams &p, int cc, int best, double vdeg) {
  atomicAdd((unsigned long long *)at_usize<MULTI>(p, best), 1ULL);
  atomicAdd(at_udeg<MULTI>(p, best), vdeg);
  atomicAdd((unsigned long long *)at_usize<MULTI>(p, cc), ~0ULL);
  atomicAdd(at_udeg<MULTI>(p, cc), -vdeg);
}

// ----------------------------------------------------------------------------------------------
// Neighbour-scan kernel, second generation ("warp-synchronous loops"; option scan_variant=3, the default of round 1;
// the default is now k_scan_pw in scan_pipe.cuh, which keeps this kernel's phase B):
// distExecuteLouvainIteration + distBuildLocalMapCounter + distGetMaxIndex (dspl.hpp:276-405, 230-274, 174-228).
// One CTA owns a tile of kTileV (128) consecutive vertices; their CSR edges are one contiguous range.
//   phase A (edge-parallel, all lanes busy, coalesced): stream the int32 tails of the tile, gather cur[tail] (the only
//           random access per edge) and stage the neighbour communities (and weights) in shared memory;
//   phase B (vertex-parallel): the first kernel of round 1 let every lane run its own "count this community" loop and
//           was issue-bound at 12 of 32 lanes active, because the warp serialised them.  Here
// phase B is arranged so that the lanes of a warp run the same loop at the same time:
//   pass 0   counter[0] = weight towards the own community (one uniform walk over the staged segment); the other
//            neighbours are compacted to the front of the segment;
//   pass 1   repeat { all lanes take the first live entry's community and count it together in one walk over their
//            live list, compacting the rest to the front (stable: edge order survives, so weighted sums round like
//            the reference); the community degree gather issued before the walk is consumed after it; gain +
//            selection on registers }.
// The trip count of the outer loop is the largest number of distinct neighbour communities among the warp's 32
// vertices (about 4 after the first iterations) instead of the sum of all lanes' loops.  Sums are accumulated in
// edge order per community, exactly like k_scan, so the weighted path keeps the reference's rounding.
// ----------------------------------------------------------------------------------------------
template <bool UNIT, bool MULTI, bool TRACE>
__global__ void __launch_bounds__(kTileV) k_scan_ws(const ScanParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int32_t *s_comm = reinterpret_cast<int32_t *>(smem_raw);
  double *s_w = reinterpret_cast<double *>(smem_raw + sizeof(int32_t) * kECap);
  __shared__ int s_next, s_end, s_skip;
  __shared__ uint32_t s_e0;
  __shared__ unsigned long long s_red[3][kTileV / 32];
  __shared__ double s_redd[kTileV / 32];

  const int tid = threadIdx.x;
  const int v0 = blockIdx.x * kTileV;
  const int v1 = min(p.lnv, v0 + kTileV);
  const int v = v0 + tid;
  const unsigned long long pol_str = make_policy((p.cache_policy & 4) ? 2 : 0);
  uint32_t r0 = 0, r1 = 0;
  if (v < v1) { r0 = p.rowptr[v]; r1 = p.rowptr[v + 1]; }
  const uint32_t deg = r1 - r0;
  const bool is_heavy = deg > (uint32_t)p.heavy_deg;
  unsigned long long acc_le_u = 0, acc_moved = 0, acc_hash = 0;
  double acc_le_d = 0.0;

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

    // ---- phase A: coalesced stream of the tile's tails, gather cur[tail], stage in shared memory.  All loads of a
    // pass are issued before the first dependent gather, and all gathers before the first store (kStageU per thread)
    {
      const int32_t *tl = p.tails + E0;
      for (int i0 = 0; i0 < ne; i0 += kStageU * kTileV) {
        int t[kStageU], cm[kStageU];
#pragma unroll
        for (int u = 0; u < kStageU; u++) {
          const int i = i0 + u * kTileV + tid;
          t[u] = (i < ne) ? ld_pol_stream(tl + i, pol_str) : -1;
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

    // ---- phase B: all 32 lanes of a warp walk their segments in lock step
    const bool mine = (v >= start && v < end);
    const int d = mine ? (int)deg : 0;
    const int o0 = mine ? (int)(r0 - E0) : 0;
    int cc = 0, best = 0;
    if (mine) { cc = __ldg(p.cur + v); best = cc; }
    double cc_deg = 0.0, vdeg = 0.0, sl = 0.0;
    if (d) {
      if (UNIT) {
        cc_deg = (double)__ldg(at_cdeg<MULTI>(p, cc));
        vdeg = (double)d;
        sl = p.has_self ? (double)__ldg(p.self_i + v) : 0.0;
      } else {
        cc_deg = __ldg(&at_cinfo_w<MULTI>(p, cc)->degree);
        vdeg = __ldg(p.vdeg + v);
        sl = p.has_self ? __ldg(p.self_d + v) : 0.0;
      }
    }
    // pass 0: weight towards the own community, in edge order (counter[0], dspl.hpp:312-318); the other
    // neighbours are compacted to the front of the segment (stable, so edge order is kept)
    double w0 = 0.0;
    int cnt0 = 0, m = 0;
    for (int k = 0; k < d; k++) {
      const int x = s_comm[o0 + k];
      if (x == cc) { if (UNIT) cnt0++; else w0 += s_w[o0 + k]; }
      else {
        s_comm[o0 + m] = x;
        if (!UNIT) s_w[o0 + m] = s_w[o0 + k];
        m++;
      }
    }
    if (UNIT) w0 = (double)cnt0;
    const double eix = __dsub_rn(w0, sl), ax = __dsub_rn(cc_deg, vdeg);
    if (d) { if (UNIT) acc_le_u += (unsigned long long)cnt0; else acc_le_d += w0; }
    // pass 1: two distinct neighbour communities per lane per round.  The round's walk counts the community of the
    // first live entry and the first community that differs from it, and compacts everything else to the front, so
    // the live list only ever shrinks and no lane has to skip over already counted entries.
    double bg = 0.0;
    int lbest = kNoLabel;
    for (;;) {
      const bool has = m > 0;
      if (!__any_sync(0xffffffffu, has)) break;
      int ck1 = 0;
      double ay1 = 0.0;
      if (has) {
        ck1 = s_comm[o0];
        if (UNIT) ay1 = (double)__ldg(at_cdeg<MULTI>(p, ck1));
        else ay1 = __ldg(&at_cinfo_w<MULTI>(p, ck1)->degree);
      }
      int ck2 = -1, c1 = 0, c2 = 0, m2 = 0;
      double sum1 = 0.0, sum2 = 0.0;
      for (int j = 0; j < m; j++) {
        const int x = s_comm[o0 + j];
        if (x == ck1) { if (UNIT) c1++; else sum1 += s_w[o0 + j]; }
        else {
          if (ck2 < 0) ck2 = x;
          if (x == ck2) { if (UNIT) c2++; else sum2 += s_w[o0 + j]; }
          else {
            s_comm[o0 + m2] = x;
            if (!UNIT) s_w[o0 + m2] = s_w[o0 + j];
            m2++;
          }
        }
      }
      m = m2;
      if (has) {
        if (UNIT) sum1 = (double)c1;
        const double g1 = gain_of(sum1, eix, vdeg, ay1, ax, p.constant, p.f32);
        if (better_l<MULTI>(p, g1, ck1, bg, best, lbest)) { bg = g1; best = ck1; }
        if (ck2 >= 0) {
          double ay2;
          if (UNIT) { ay2 = (double)__ldg(at_cdeg<MULTI>(p, ck2)); sum2 = (double)c2; }
          else ay2 = __ldg(&at_cinfo_w<MULTI>(p, ck2)->degree);
          const double g2 = gain_of(sum2, eix, vdeg, ay2, ax, p.constant, p.f32);
          if (better_l<MULTI>(p, g2, ck2, bg, best, lbest)) { bg = g2; best = ck2; }
        }
      }
    }
    if (mine) {
      if (d && label_greater<MULTI>(p, best, lbest, cc)) {                   // singleton veto, dspl.hpp:224-225
        long long sz_cc, sz_b;
        if (UNIT) {
          sz_cc = __ldg(at_csize<MULTI>(p, cc));
          sz_b = __ldg(at_csize<MULTI>(p, best));
        } else {
          sz_cc = __ldg(&at_cinfo_w<MULTI>(p, cc)->size);
          sz_b = __ldg(&at_cinfo_w<MULTI>(p, best)->size);
        }
        if (sz_cc == 1 && sz_b == 1) best = cc;
      }
      if (best != cc) {                                                      // dspl.hpp:331-399
        if (UNIT) push_move_unit<MULTI>(p, cc, best, d);
        else push_move_w<MULTI>(p, cc, best, vdeg);
      }
      st_pol(p.tgt + v, best, pol_str);                                      // dspl.hpp:404
      if (TRACE) { acc_moved += (best != cc); acc_hash += vhash(label_of<MULTI>(p, (int)(p.base + v)), label_of<MULTI>(p, best)); }
    }
    start = end;
    __syncthreads();
  }

  const int lane = tid & 31, wid = tid >> 5;
  if (UNIT) { const unsigned long long s = warp_sum(acc_le_u); if (lane == 0) s_red[0][wid] = s; }
  else { const double s = warp_sum(acc_le_d); if (lane == 0) s_redd[wid] = s; }
  if (TRACE) {
    const unsigned long long a = warp_sum(acc_moved), b = warp_sum(acc_hash);
    if (lane == 0) { s_red[1][wid] = a; s_red[2][wid] = b; }
  }
  __syncthreads();
  if (tid == 0) {
    if (UNIT) {
      unsigned long long s = 0;
      for (int w = 0; w < kTileV / 32; w++) s += s_red[0][w];
      if (s) atomicAdd(&p.acc->le_u, s);
    } else {
      double s = 0;
      for (int w = 0; w < kTileV / 32; w++) s += s_redd[w];
      if (s != 0.0) atomicAdd(&p.acc->le_d, s);
    }
    if (TRACE) {
      unsigned long long a = 0, b = 0;
      for (int w = 0; w < kTileV / 32; w++) { a += s_red[1][w]; b += s_red[2][w]; }
      atomicAdd(&p.acc->moved, a);
      atomicAdd(&p.acc->hash, b);
    }
  }
}

// ----------------------------------------------------------------------------------------------
// High-degree vertices (degree > heavy_deg): one CTA per vertex, open-addressing table in HBM
// scratch (2x degree entries) keyed by neighbour community; same decision rule.  Weighted sums are
// accumulated with fp64 atomics here (order not fixed: weighted parity is tolerance-based anyway).
// ----------------------------------------------------------------------------------------------
template <bool UNIT, bool MULTI, bool TRACE>
__global__ void __launch_bounds__(256) k_scan_heavy(const ScanParams p) {
  const int v = p.heavy_list[blockIdx.x];
  const unsigned long long off = p.heavy_off[blockIdx.x];
  const unsigned int T = (unsigned int)(p.heavy_off[blockIdx.x + 1] - off);   // power of two
  int32_t *keys = p.hkeys + off;
  int32_t *vi = UNIT ? p.hvals_i + off : nullptr;
  double *vd = UNIT ? nullptr : p.hvals_d + off;
  const int tid = threadIdx.x;
  const uint32_t e0 = p.rowptr[v], e1 = p.rowptr[v + 1];
  const int cc = p.cur[v];
  for (unsigned int i = tid; i < T; i += blockDim.x) { keys[i] = -1; if (UNIT) vi[i] = 0; else vd[i] = 0.0; }
  __syncthreads();
  for (uint32_t e = e0 + tid; e < e1; e += blockDim.x) {
    const int c = __ldg(p.cur + p.tails[e]);
    unsigned int h = (unsigned int)mix64((unsigned long long)c) & (T - 1);
    for (;;) {
      const int old = atomicCAS(&keys[h], -1, c);
      if (old == -1 || old == c) {
        if (UNIT) atomicAdd(&vi[h], 1); else atomicAdd(&vd[h], p.weights[e]);
        break;
      }
      h = (h + 1) & (T - 1);
    }
  }
  __syncthreads();
  __shared__ double s_w0;
  __shared__ double s_g[8];
  __shared__ int s_y[8];
  __shared__ long long s_sz[8];
  __shared__ int s_l[8];
  if (tid == 0) s_w0 = 0.0;
  __syncthreads();
  for (unsigned int i = tid; i < T; i += blockDim.x)
    if (keys[i] == cc) s_w0 = UNIT ? (double)vi[i] : vd[i];
  __syncthreads();
  int owner; long long idx;
  locate_impl<MULTI>(p.pt, p.base, p.lnv, cc, owner, idx);
  double cc_deg, vdeg, sl; long long cc_size;
  if (UNIT) {
    cc_size = (long long)__ldg(ptr_csize<MULTI>(p, owner) + idx);
    cc_deg = (double)__ldg(ptr_cdeg<MULTI>(p, owner) + idx);
    vdeg = (double)(e1 - e0);
    sl = p.has_self ? (double)p.self_i[v] : 0.0;
  } else {
    const CommW cw = ptr_cinfo_w<MULTI>(p, owner)[idx];
    cc_size = cw.size; cc_deg = cw.degree;
    vdeg = p.vdeg[v];
    sl = p.has_self ? p.self_d[v] : 0.0;
  }
  const double w0 = s_w0;
  const double eix = __dsub_rn(w0, sl), ax = __dsub_rn(cc_deg, vdeg);
  double bg = 0.0; int by = cc; long long bsz = cc_size;
  int lby = kNoLabel;
  for (unsigned int i = tid; i < T; i += blockDim.x) {
    const int y = keys[i];
    if (y < 0 || y == cc) continue;
    int yo; long long yi;
    locate_impl<MULTI>(p.pt, p.base, p.lnv, y, yo, yi);
    double ay, eiy; long long ysz;
    if (UNIT) {
      ysz = (long long)__ldg(ptr_csize<MULTI>(p, yo) + yi);
      ay = (double)__ldg(ptr_cdeg<MULTI>(p, yo) + yi); eiy = (double)vi[i];
    } else {
      const CommW cw = ptr_cinfo_w<MULTI>(p, yo)[yi];
      ysz = cw.size; ay = cw.degree; eiy = vd[i];
    }
    const double g = gain_of(eiy, eix, vdeg, ay, ax, p.constant, p.f32);
    if (better_l<MULTI>(p, g, y, bg, by, lby)) { bg = g; by = y; bsz = ysz; }
  }
  if (by != cc && lby == kNoLabel) lby = label_of<MULTI>(p, by);   // partial winners carry their label into the reduction
  // CTA argmax under the same ordering (labels compared where the reference compares ids).  `better` needs care when combining partial winners that
  // still sit at the initial state (gain 0, id cc): an initial state never beats a real candidate.
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const double og = __shfl_xor_sync(0xffffffffu, bg, o);
    const int oy = __shfl_xor_sync(0xffffffffu, by, o);
    const long long os = __shfl_xor_sync(0xffffffffu, bsz, o);
    const int ol = __shfl_xor_sync(0xffffffffu, lby, o);
    if (oy != cc && (by == cc || (og > bg) || ((og == bg) && (og != 0.0) && (ol < lby)))) { bg = og; by = oy; bsz = os; lby = ol; }
  }
  if ((tid & 31) == 0) { s_g[tid >> 5] = bg; s_y[tid >> 5] = by; s_sz[tid >> 5] = bsz; s_l[tid >> 5] = lby; }
  __syncthreads();
  if (tid == 0) {
    bg = 0.0; by = cc; bsz = cc_size; lby = kNoLabel;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++)
      if (s_y[w] != cc && (by == cc || (s_g[w] > bg) || ((s_g[w] == bg) && (bg != 0.0) && (s_l[w] < lby)))) {
        bg = s_g[w]; by = s_y[w]; bsz = s_sz[w]; lby = s_l[w];
      }
    int best = by;
    if (bsz == 1 && cc_size == 1 && label_greater<MULTI>(p, best, lby, cc)) best = cc;
    if (best != cc) {
      int bo; long long bi;
      locate_impl<MULTI>(p.pt, p.base, p.lnv, best, bo, bi);
      if (UNIT) {
        atomicAdd(ptr_upd<MULTI>(p, bo) + bi, pack_delta(1, (long long)(e1 - e0)));
        atomicAdd(ptr_upd<MULTI>(p, owner) + idx, pack_delta(-1, -(long long)(e1 - e0)));
      } else {
        atomicAdd((unsigned long long *)(ptr_usize<MULTI>(p, bo) + bi), 1ULL);
        atomicAdd(ptr_udeg<MULTI>(p, bo) + bi, vdeg);
        atomicAdd((unsigned long long *)(ptr_usize<MULTI>(p, owner) + idx), ~0ULL);
        atomicAdd(ptr_udeg<MULTI>(p, owner) + idx, -vdeg);
      }
    }
    p.tgt[v] = best;
    if (UNIT) atomicAdd(&p.acc->le_u, (unsigned long long)w0); else atomicAdd(&p.acc->le_d, w0);
    if (TRACE) {
      atomicAdd(&p.acc->moved, (unsigned long long)(best != cc));
      atomicAdd(&p.acc->hash, vhash(label_of<MULTI>(p, (int)(p.base + v)), label_of<MULTI>(p, best)));
    }
  }
}

// ----------------------------------------------------------------------------------------------
// Fold kernel: localCinfo += localCupdate (+ the deltas remote ranks pushed with NVLink atomics,
// i.e. updateRemoteCommunities), zero the update array for the next iteration (distCleanCWandCU)
// and accumulate sum(degree^2) for the modularity (dspl.hpp:458-471, 978-1103, 473-486, 432).
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_fold_w(int lnv, CommW *cinfo_w, long long *usize, double *udeg, Acc *acc) {
  double a2d = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < lnv; i += gridDim.x * blockDim.x) {
    CommW c = cinfo_w[i];
    const long long us = usize[i];
    const double ud = udeg[i];
    if (us != 0 || ud != 0.0) {
      c.size += us; c.degree += ud;
      cinfo_w[i] = c; usize[i] = 0; udeg[i] = 0.0;
    }
    a2d += c.degree * c.degree;
  }
  __shared__ double sd[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const double s = warp_sum(a2d);
  if (lane == 0) sd[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < 8; w++) t += sd[w]; atomicAdd(&acc->la2_d, t); }
}

// Modularity partials as doubles for the cross-rank all-reduce (MPI_Allreduce of 2 doubles, dspl.hpp:441).
__global__ void k_acc_to_double(const Acc *acc, int unit, double *out2) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    out2[0] = unit ? (double)acc->le_u : acc->le_d;
    out2[1] = unit ? (double)acc->la2_u : acc->la2_d;
  }
}
__global__ void k_trace_to_u64(const Acc *acc, unsigned long long *out2) {
  if (threadIdx.x == 0 && blockIdx.x == 0) { out2[0] = acc->moved; out2[1] = acc->hash; }
}

// ----------------------------------------------------------------------------------------------
// Setup kernels (once per run): format conversion, ghost discovery, init (dspl.hpp:1106-1272, 151-172)
// ----------------------------------------------------------------------------------------------
struct EdgeStats { unsigned long long nremote; unsigned int nonunit; unsigned int bad_tail; };

__global__ void __launch_bounds__(256) k_edge_stats(const Edge16 *edges, long long lne, long long base, long long bound,
                                                    long long nv_global, EdgeStats *st) {
  unsigned long long nrem = 0;
  unsigned int nonunit = 0, bad = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < lne; e += (long long)gridDim.x * blockDim.x) {
    const double2 raw = __ldcs(reinterpret_cast<const double2 *>(edges + e));
    const long long t = __double_as_longlong(raw.x);
    if (raw.y != 1.0) nonunit = 1;
    if (t < 0 || t >= nv_global) bad = 1;
    else if (t < base || t >= bound) nrem++;
  }
  nrem = warp_sum(nrem);
  nonunit = __any_sync(0xffffffffu, nonunit);
  bad = __any_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    if (nrem) atomicAdd(&st->nremote, nrem);
    if (nonunit) atomicOr(&st->nonunit, 1u);
    if (bad) atomicOr(&st->bad_tail, 1u);
  }
}

// tails -> local slot (ghosts provisionally -1), weights split off, remote tails appended to a list.  With `st`
// the pass also gathers the statistics of k_edge_stats (single-rank runs need no separate statistics pass).
__global__ void __launch_bounds__(256) k_convert_edges(const Edge16 *edges, long long lne, long long base, long long bound,
                                                       long long nv_global, int32_t *tails, double *weights,
                                                       long long *remote_list, uint32_t *remote_pos,
                                                       unsigned long long *remote_cursor, EdgeStats *st) {
  unsigned long long nrem = 0;
  unsigned int nonunit = 0, bad = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < lne; e += (long long)gridDim.x * blockDim.x) {
    const double2 raw = __ldcs(reinterpret_cast<const double2 *>(edges + e));
    const long long t = __double_as_longlong(raw.x);
    const bool local = (t >= base && t < bound);
    tails[e] = local ? (int32_t)(t - base) : -1;
    if (weights) weights[e] = raw.y;
    if (st) {
      if (raw.y != 1.0) nonunit = 1;
      if (t < 0 || t >= nv_global) bad = 1;
      else if (!local) nrem++;
    }
    if (!local && remote_list) {
      const unsigned long long pos = atomicAdd(remote_cursor, 1ULL);
      remote_list[pos] = t;
      remote_pos[pos] = (uint32_t)e;              // where the ghost slot has to go (k_remap_ghost_tails)
    }
  }
  if (st) {
    nrem = warp_sum(nrem);
    nonunit = __any_sync(0xffffffffu, nonunit);
    bad = __any_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0) {
      if (nrem) atomicAdd(&st->nremote, nrem);
      if (nonunit) atomicOr(&st->nonunit, 1u);
      if (bad) atomicOr(&st->bad_tail, 1u);
    }
  }
}

__global__ void __launch_bounds__(256) k_extract_weights(const Edge16 *edges, long long lne, double *weights) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < lne; e += (long long)gridDim.x * blockDim.x)
    weights[e] = __ldcs(&edges[e].weight);
}

// USE_32_BIT_GRAPH input ({int32 tail; float weight} records, int32 offsets) -> the 64-bit layout the setup kernels read
struct Edge8 { int tail; float weight; };
__global__ void __launch_bounds__(256) k_widen_shard32(const Edge8 *e8, long long lne, const int32_t *rp32, long long lnv,
                                                       Edge16 *e16, long long *rp64) {
  const long long gsz = (long long)gridDim.x * blockDim.x, t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long e = t0; e < lne; e += gsz) {
    const Edge8 x = e8[e];
    Edge16 y; y.tail = x.tail; y.weight = (double)x.weight;
    e16[e] = y;
  }
  for (long long i = t0; i <= lnv; i += gsz) rp64[i] = rp32[i];
}

__global__ void __launch_bounds__(256) k_fill_ones(double *w, long long n) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) w[e] = 1.0;
}

// device half of the compact upload: a raw chunk of 16-byte records -> int32 global tails + the statistics the host
// pass (narrow.cpp) gathers for its chunks
__global__ void __launch_bounds__(256) k_narrow_records(const Edge16 *rec, long long n, long long nv_global, long long base,
                                                        long long bound, int32_t *dst, EdgeStats *st) {
  unsigned long long nrem = 0;
  unsigned int nonunit = 0, bad = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const double2 raw = __ldcs(reinterpret_cast<const double2 *>(rec + e));
    const long long t = __double_as_longlong(raw.x);
    dst[e] = (int32_t)t;
    if (raw.y != 1.0) nonunit = 1;
    if (t < 0 || t >= nv_global) bad = 1;
    else if (t < base || t >= bound) nrem++;
  }
  nrem = warp_sum(nrem);
  nonunit = __any_sync(0xffffffffu, nonunit);
  bad = __any_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    if (nrem) atomicAdd(&st->nremote, nrem);
    if (nonunit) atomicOr(&st->nonunit, 1u);
    if (bad) atomicOr(&st->bad_tail, 1u);
  }
}

// same conversion for the compact upload format (int32 global tails, unit weights; see mvgpu_upload_shard)
__global__ void __launch_bounds__(256) k_convert_tails32(const int32_t *gtails, long long lne, long long base, long long bound,
                                                         int32_t *tails, long long *remote_list, uint32_t *remote_pos,
                                                         unsigned long long *remote_cursor) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < lne; e += (long long)gridDim.x * blockDim.x) {
    const long long t = __ldcs(gtails + e);
    const bool local = (t >= base && t < bound);
    tails[e] = local ? (int32_t)(t - base) : -1;
    if (!local && remote_list) {
      const unsigned long long pos = atomicAdd(remote_cursor, 1ULL);
      remote_list[pos] = t;
      remote_pos[pos] = (uint32_t)e;
    }
  }
}

// ghosts: slot = lnv + rank of the tail in the sorted unique ghost list
__global__ void __launch_bounds__(256) k_remap_ghost_tails(const long long *remote_list, const uint32_t *remote_pos, long long nremote,
                                                           int32_t *tails, const long long *ghost_gid, int nghost, int lnv) {
  // one thread per NON-OWNED edge (their positions were recorded by the conversion pass), not one per edge of the shard
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < nremote; k += (long long)gridDim.x * blockDim.x) {
    const long long t = remote_list[k];
    int lo = 0, hi = nghost;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (ghost_gid[mid] < t) lo = mid + 1; else hi = mid; }
    tails[remote_pos[k]] = lnv + lo;
  }
}

__global__ void __launch_bounds__(256) k_rowptr32(const long long *rowptr64, int lnv, long long lne, uint32_t *rowptr,
                                                  unsigned int *maxdeg, unsigned int *bad) {
  unsigned int md = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= lnv; i += gridDim.x * blockDim.x) {
    const long long r = rowptr64[i];
    rowptr[i] = (uint32_t)r;
    if ((i == 0 && r != 0) || (i == lnv && r != lne)) *bad = 1;      // the scan kernels trust [rowptr[v], rowptr[v+1])
    if (i < lnv) {
      const long long d = rowptr64[i + 1] - r;
      if (d < 0) *bad = 1;
      else md = max(md, (unsigned int)min(d, (long long)0xffffffffu));
    }
  }
  for (int o = 16; o; o >>= 1) md = max(md, __shfl_xor_sync(0xffffffffu, md, o));
  if ((threadIdx.x & 31) == 0 && md) atomicMax(maxdeg, md);
}

// "Is this adjacency list strictly increasing by GLOBAL tail id?"  -- asked on slot ids: lower ranks' ghosts (slots
// [lnv, lnv+nlow)) precede the rank's own vertices ([0, lnv)), which precede higher ranks' ghosts.  A shard whose
// lists all pass has no parallel edges (duplicates would be adjacent), which the first-iteration kernel relies on.
__device__ __forceinline__ bool tails_ascend(int a, int b, int lnv, int nlow) {
  const int ka = a < lnv ? 1 : (a < lnv + nlow ? 0 : 2), kb = b < lnv ? 1 : (b < lnv + nlow ? 0 : 2);
  return ka < kb || (ka == kb && a < b);
}

// distSumVertexDegree + distInitComm + self-loop weights (dspl.hpp:82-107, 132-149, 247-248/285)
// Unit-weight fold (same job as k_fold_w on the packed integer arrays): four community slots per thread and
// iteration with 16-byte accesses (faster than one slot per thread).  u = dsize*2^32 + ddeg is the exact two's-complement sum of the deltas.
__device__ __forceinline__ uint32_t fold_apply_unit(uint32_t dg, unsigned long long u, int32_t *csize_i) {
  const int ddeg = (int)(uint32_t)u;
  const int dsize = (int)(((long long)u - (long long)ddeg) >> 32);
  if (dsize) *csize_i += dsize;
  return dg + (uint32_t)ddeg;
}
__global__ void __launch_bounds__(256) k_fold_unit(int lnv, uint32_t *cdeg, int32_t *csize, unsigned long long *upd, Acc *acc,
                                                   const Acc *prev) {
  // sum(degree^2) is carried from iteration to iteration (prev->la2_u; record 0 holds the initial sum, written by
  // k_vertex_init) and only corrected by new^2 - old^2 of the communities that changed -- exact in wrapping 64-bit
  // arithmetic --, so the pass streams the 8-byte delta array alone and touches cdeg / csize only where a delta is.
  unsigned long long a2u = 0;
  const int n4 = lnv >> 2;
  auto apply4 = [&](int q, const ulonglong2 ua, const ulonglong2 ub) {
    const int i = 4 * q;
    uint4 dg = reinterpret_cast<const uint4 *>(cdeg)[q];
    const uint4 old = dg;
    if (ua.x) dg.x = fold_apply_unit(dg.x, ua.x, csize + i);
    if (ua.y) dg.y = fold_apply_unit(dg.y, ua.y, csize + i + 1);
    if (ub.x) dg.z = fold_apply_unit(dg.z, ub.x, csize + i + 2);
    if (ub.y) dg.w = fold_apply_unit(dg.w, ub.y, csize + i + 3);
    reinterpret_cast<uint4 *>(cdeg)[q] = dg;
    const ulonglong2 z = make_ulonglong2(0ULL, 0ULL);
    if (ua.x | ua.y) reinterpret_cast<ulonglong2 *>(upd)[2 * q] = z;
    if (ub.x | ub.y) reinterpret_cast<ulonglong2 *>(upd)[2 * q + 1] = z;
    a2u += (unsigned long long)dg.x * dg.x + (unsigned long long)dg.y * dg.y + (unsigned long long)dg.z * dg.z +
           (unsigned long long)dg.w * dg.w;
    a2u -= (unsigned long long)old.x * old.x + (unsigned long long)old.y * old.y + (unsigned long long)old.z * old.z +
           (unsigned long long)old.w * old.w;
  };
  // (four groups per thread and step, eight 16-byte loads in flight, was measured: 1.41 -> 1.76 ms per phase; one group
  // per step it stays)
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n4; q += gridDim.x * blockDim.x) {
    const ulonglong2 ua = reinterpret_cast<const ulonglong2 *>(upd)[2 * q], ub = reinterpret_cast<const ulonglong2 *>(upd)[2 * q + 1];
    if (ua.x | ua.y | ub.x | ub.y) apply4(q, ua, ub);
  }
  if (blockIdx.x == 0) {                          // the up to three slots behind the last full group
    const int i = 4 * n4 + (int)threadIdx.x;
    if (i < lnv) {
      const unsigned long long u = upd[i];
      if (u) {
        const uint32_t old = cdeg[i];
        const uint32_t dg = fold_apply_unit(old, u, csize + i);
        cdeg[i] = dg; upd[i] = 0;
        a2u += (unsigned long long)dg * dg - (unsigned long long)old * old;
      }
    }
    if (threadIdx.x == 0) a2u += prev->la2_u;     // complete: the previous iteration's fold has finished
  }
  __shared__ unsigned long long su[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned long long s = warp_sum(a2u);
  if (lane == 0) su[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) { unsigned long long t = 0; for (int w = 0; w < 8; w++) t += su[w]; if (t) atomicAdd(&acc->la2_u, t); }
}
template <bool UNIT>
__global__ void __launch_bounds__(256) k_vertex_init(int lnv, long long base, const uint32_t *rowptr, const int32_t *tails,
                                                     const double *weights, int32_t *cur, uint32_t *cdeg, int32_t *csize,
                                                     unsigned long long *upd, CommW *cinfo_w, long long *usize, double *udeg,
                                                     double *vdeg, int32_t *self_i, double *self_d, double *total_weight,
                                                     unsigned int *has_self, int nlow, unsigned int *unordered, Acc *acc0) {
  double tw_sum = 0.0;
  unsigned long long sq_sum = 0;                 // unit path: initial sum(degree^2), the fold kernel's starting point
  unsigned int any_self = 0;
  bool bad = false;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < lnv; v += gridDim.x * blockDim.x) {
    const uint32_t e0 = rowptr[v], e1 = rowptr[v + 1];
    cur[v] = (int32_t)(base + v);
    if (UNIT) {
      int sl = 0;
      if (unordered) {                       // original numbering: the lists can still be checked for order (see tails_ascend)
        int prev = 0;
        for (uint32_t e = e0; e < e1; e++) {
          const int t = tails[e];
          sl += (t == v);
          if (e > e0 && !tails_ascend(prev, t, lnv, nlow)) bad = true;
          prev = t;
        }
      } else
      for (uint32_t e = e0; e < e1; e++) sl += (tails[e] == v);
      self_i[v] = sl;
      any_self |= (sl != 0);
      cdeg[v] = e1 - e0;
      csize[v] = 1;
      upd[v] = 0;
      tw_sum += (double)(e1 - e0);
      sq_sum += (unsigned long long)(e1 - e0) * (e1 - e0);
    } else {
      double tw = 0.0, sl = 0.0;
      for (uint32_t e = e0; e < e1; e++) {           // edge order, like dspl.hpp:97-100
        const double w = weights[e];
        tw += w;
        if (tails[e] == v) sl += w;
      }
      vdeg[v] = tw;
      self_d[v] = (double)(long long)sl;             // GraphWeight -> GraphElem truncation (dspl.hpp:285,315)
      any_self |= (sl != 0.0);
      CommW c; c.size = 1; c.degree = tw;
      cinfo_w[v] = c;
      usize[v] = 0; udeg[v] = 0.0;
      tw_sum += tw;
    }
  }
  tw_sum = warp_sum(tw_sum);
  if (UNIT) sq_sum = warp_sum(sq_sum);
  any_self = __any_sync(0xffffffffu, any_self);
  if (bad) *unordered = 1;
  if ((threadIdx.x & 31) == 0) {
    if (UNIT && sq_sum) atomicAdd(&acc0->la2_u, sq_sum);
    if (tw_sum != 0.0) atomicAdd(total_weight, tw_sum);
    if (any_self) atomicOr(has_self, 1u);
  }
}

__global__ void __launch_bounds__(256) k_collect_heavy(int lnv, const uint32_t *rowptr, unsigned int heavy_deg, int32_t *list,
                                                       unsigned int *count) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < lnv; v += gridDim.x * blockDim.x)
    if (rowptr[v + 1] - rowptr[v] > heavy_deg) list[atomicAdd(count, 1u)] = v;
}

// ----------------------------------------------------------------------------------------------
// Locality renumbering (GPU layout step, not in the reference).  miniVite numbers RGG vertices in
// generation order, i.e. randomly in space, so cur[tail] gathers have no locality and every edge costs a
// DRAM sector.  We grow lnv/region_size (default 512) regions simultaneously by breadth-first search from evenly spaced seed
// ids (one persistent cooperative kernel, one grid barrier per level) and renumber vertices by
// (region, BFS level): neighbours end up a few KB apart, so gathers hit L1/L2.  Results are unchanged:
// the algorithm is a synchronous (Jacobi) sweep, and wherever the reference compares community ids the
// kernels compare the original ids kept as labels.
// key = level << 22 | region  (atomicMin: lowest level wins, then lowest region -> deterministic)
// ----------------------------------------------------------------------------------------------
constexpr unsigned int kBfsRegionBits = 22;
constexpr unsigned int kBfsUnreached = 0xFFFFFFFFu;
// edges per lane whose loads are all issued before the first compare (BFS expansion and CSR permute); on H100 at
// config 2, 16 beat 8 and 4 in both kernels (DESIGN.md §3.3)
constexpr int kEdgeBatch = 16;

// A warp owns 32 rows whose edges form one range; `off` is this lane's row start within it (rows past the end hold the
// range's length).  Returns the row that edge j of the range belongs to: the last lane with off <= j.
__device__ __forceinline__ int row_of_edge(uint32_t off, uint32_t j) {
  int o = 0;
#pragma unroll
  for (int s = 16; s; s >>= 1)
    if (__shfl_sync(0xffffffffu, off, o + s) <= j) o += s;
  return o;
}

// Frontier-queue BFS.  queue[] holds the reached vertices in BFS order: level L is the segment [lo, hi), and
// level_count[L] counts the vertices level L appends (zeroed here, read only after the barrier that ends level L,
// so every CTA derives the same next segment).  A warp takes 32 frontier vertices, spreads their edges over its lanes
// and issues kEdgeBatch loads per lane at each step before any compare.  The vertex whose atomicMin finds it
// unreached appends it (once).  Only the order inside a level's segment depends on timing; keys do not (lowest level,
// then lowest region).
// Level bitmaps: lmap holds four bitmaps, interleaved per 32 vertices (one 16-byte word), bitmap l % 4 marking the
// vertices of level l.  Expanding level L skips every neighbour marked in the bitmaps of levels L-1 and L, whose keys
// are already below the new key, with a probe of the 8 MB lmap instead of the 64 MB key[] array; level L+1's claims
// are marked in bitmap (L+1) % 4, and bitmap (L+2) % 4 (level L-2, no longer read) is cleared for level L+1's claims.
__global__ void __launch_bounds__(256) k_msbfs(int lnv, const uint32_t *rowptr, const int32_t *tails, uint32_t *key,
                                               int region_stride, int max_levels, int32_t *queue,
                                               unsigned int *level_count, uint32_t *lmap) {
  namespace cg = cooperative_groups;
  cg::grid_group grid = cg::this_grid();
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  const int nwords = (lnv + 31) >> 5;
  for (int v = gtid; v < lnv; v += gsz) {
    const bool seed = v % region_stride == 0;
    key[v] = seed ? (unsigned int)(v / region_stride) : kBfsUnreached;
    if (seed) queue[v / region_stride] = v;
  }
  for (int q = gtid; q < nwords; q += gsz) {          // the seeds are level 0
    const long long end = min(32LL * q + 32, (long long)lnv);
    unsigned int seeds = 0;
    for (long long v = (32LL * q + region_stride - 1) / region_stride * region_stride; v < end; v += region_stride)
      seeds |= 1u << (v & 31);
    reinterpret_cast<uint4 *>(lmap)[q] = make_uint4(seeds, 0u, 0u, 0u);
  }
  for (int l = gtid; l < max_levels; l += gsz) level_count[l] = 0;
  grid.sync();
  const unsigned int full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const unsigned int gwarp = gtid >> 5, nwarps = gsz >> 5;
  unsigned int lo = 0, hi = (unsigned int)((lnv - 1) / region_stride + 1);
  for (int level = 0; level < max_levels && lo < hi; level++) {
    const unsigned int nk_level = (unsigned int)(level + 1) << kBfsRegionBits;
    const int m_prev = (level + 3) & 3, m_cur = level & 3, m_next = (level + 1) & 3;
    for (int q = gtid; q < nwords; q += gsz) lmap[4 * q + ((level + 2) & 3)] = 0u;
    for (unsigned int c = lo + gwarp * 32u; c < hi; c += nwarps * 32u) {
      uint32_t b = 0, d = 0, nk = 0;
      if (c + lane < hi) {
        const int v = __ldcg(queue + c + lane);                       // appended by other SMs: read through L2
        nk = nk_level | (__ldcg(key + v) & ((1u << kBfsRegionBits) - 1));
        b = rowptr[v];
        d = rowptr[v + 1] - b;
      }
      uint32_t incl = d;
#pragma unroll
      for (int s = 1; s < 32; s <<= 1) {
        const uint32_t y = __shfl_up_sync(full, incl, s);
        if (lane >= s) incl += y;
      }
      const uint32_t off = incl - d, total = __shfl_sync(full, incl, 31);
      for (uint32_t j0 = 0; j0 < total; j0 += 32 * kEdgeBatch) {
        int w[kEdgeBatch];
        uint32_t nkw[kEdgeBatch], kw[kEdgeBatch];
#pragma unroll
        for (int u = 0; u < kEdgeBatch; u++) {
          const uint32_t j = j0 + u * 32 + lane;
          const int o = row_of_edge(off, j);
          const uint32_t e = __shfl_sync(full, b, o) + (j - __shfl_sync(full, off, o));
          nkw[u] = __shfl_sync(full, nk, o);
          w[u] = j < total ? tails[e] : lnv;                          // ghosts (w >= lnv) are never probed
        }
        uint32_t mp[kEdgeBatch], mc[kEdgeBatch];
#pragma unroll
        for (int u = 0; u < kEdgeBatch; u++) {
          mp[u] = mc[u] = 0;
          if (w[u] < lnv) {
            mp[u] = __ldcg(lmap + 4 * (w[u] >> 5) + m_prev);
            mc[u] = __ldcg(lmap + 4 * (w[u] >> 5) + m_cur);
          }
        }
#pragma unroll
        for (int u = 0; u < kEdgeBatch; u++)
          if ((((mp[u] | mc[u]) >> (w[u] & 31)) & 1u)) w[u] = lnv;
#pragma unroll
        for (int u = 0; u < kEdgeBatch; u++) kw[u] = w[u] < lnv ? __ldcg(key + w[u]) : 0u;
        unsigned int nnew = 0;
#pragma unroll
        for (int u = 0; u < kEdgeBatch; u++) {
          bool claimed = false;
          if (w[u] < lnv && kw[u] > nkw[u]) claimed = atomicMin(&key[w[u]], nkw[u]) == kBfsUnreached;
          if (claimed) {
            nnew++;
            atomicOr(lmap + 4 * (w[u] >> 5) + m_next, 1u << (w[u] & 31));
          } else {
            w[u] = -1;
          }
        }
        // warp-aggregated append: one atomic per warp and batch
        unsigned int pos = nnew;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
          const unsigned int y = __shfl_up_sync(full, pos, s);
          if (lane >= s) pos += y;
        }
        const unsigned int cnt = __shfl_sync(full, pos, 31);
        if (cnt) {
          unsigned int base = 0;
          if (lane == 31) base = atomicAdd(level_count + level, cnt);
          pos = hi + __shfl_sync(full, base, 31) + pos - nnew;
#pragma unroll
          for (int u = 0; u < kEdgeBatch; u++)
            if (w[u] >= 0) queue[pos++] = w[u];
        }
      }
    }
    grid.sync();
    lo = hi;
    hi += __ldcg(level_count + level);
  }
}

// sort key: region major, level minor (8 bits, deeper levels clamp: layout quality only); unreached vertices (other
// components) carry `unreached_key` = all ones inside the sorted bit range and come last, in id order
constexpr unsigned int kBfsLevelBits = 8;
__global__ void __launch_bounds__(256) k_bfs_sortkeys(int lnv, const uint32_t *key, uint32_t *sortkey, int32_t *ids,
                                                      unsigned int unreached_key) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < lnv; v += gridDim.x * blockDim.x) {
    const unsigned int k = key[v];
    unsigned int sk;
    if (k == kBfsUnreached) sk = unreached_key;
    else {
      const unsigned int region = k & ((1u << kBfsRegionBits) - 1), level = min(k >> kBfsRegionBits, (1u << kBfsLevelBits) - 1u);
      sk = (region << kBfsLevelBits) | level;
    }
    sortkey[v] = sk;
    ids[v] = v;
  }
}

// perm[new] = old  ->  inv[old] = new (unless inv is null), lab[new] = global original id, deg_new[new] = degree
__global__ void __launch_bounds__(256) k_perm_inverse(int lnv, const int32_t *perm, long long base, int32_t *inv, int32_t *lab,
                                                      const uint32_t *rowptr_old, uint32_t *deg_new) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= lnv; i += gridDim.x * blockDim.x) {
    if (i == lnv) { deg_new[i] = 0; continue; }
    const int o = perm[i];
    if (inv) inv[o] = i;
    lab[i] = (int32_t)(base + o);
    deg_new[i] = rowptr_old[o + 1] - rowptr_old[o];
  }
}

// adjacency of new vertex i := adjacency of old vertex perm[i], tails renumbered (ghost slots unchanged),
// edge order preserved (weighted sums keep the reference's summation order).  A warp owns 32 consecutive new vertices,
// whose rows are one contiguous range of the new CSR; it walks that range edge-parallel, kEdgeBatch edges per lane, so
// the tails_old reads and then the inv[] gathers are issued kEdgeBatch at a time and the stores are coalesced.  Also
// checks that every old adjacency list is in tails_ascend order (sets *unordered otherwise).
__global__ void __launch_bounds__(256) k_permute_adj(int lnv, const int32_t *perm, const int32_t *inv, const uint32_t *rowptr_old,
                                                     const int32_t *tails_old, const double *w_old, const uint32_t *rowptr_new,
                                                     int32_t *tails_new, double *w_new, int nlow, unsigned int *unordered) {
  const unsigned int full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const long long gwarp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * (long long)blockDim.x) >> 5;
  bool bad = false;
  for (long long i0 = gwarp * 32; i0 < lnv; i0 += nwarps * 32) {
    const long long i = i0 + lane;
    const uint32_t d0 = rowptr_new[i0], total = rowptr_new[min(i0 + 32, (long long)lnv)] - d0;
    uint32_t off = total, s0 = 0;
    if (i < lnv) {
      off = rowptr_new[i] - d0;
      s0 = rowptr_old[perm[i]];
    }
    int carry = 0;                                     // lane 31's tail of the previous batch
    for (uint32_t j0 = 0; j0 < total; j0 += 32 * kEdgeBatch) {
      int t[kEdgeBatch];
      uint32_t k[kEdgeBatch];
#pragma unroll
      for (int u = 0; u < kEdgeBatch; u++) {
        const uint32_t j = j0 + u * 32 + lane;
        const int o = row_of_edge(off, j);
        k[u] = j - __shfl_sync(full, off, o);          // position inside the row
        const uint32_t src = __shfl_sync(full, s0, o) + k[u];
        t[u] = 0;
        if (j < total) {
          t[u] = tails_old[src];
          if (w_old) w_new[d0 + j] = w_old[src];
        }
      }
#pragma unroll
      for (int u = 0; u < kEdgeBatch; u++) {
        const int up = __shfl_up_sync(full, t[u], 1);
        const int prev = lane ? up : carry;            // the row's previous edge whenever k > 0
        carry = __shfl_sync(full, t[u], 31);
        if (j0 + u * 32 + lane < total && k[u] && !tails_ascend(prev, t[u], lnv, nlow)) bad = true;
      }
      int n[kEdgeBatch];
#pragma unroll
      for (int u = 0; u < kEdgeBatch; u++) n[u] = (j0 + u * 32 + lane < total && t[u] < lnv) ? inv[t[u]] : t[u];
#pragma unroll
      for (int u = 0; u < kEdgeBatch; u++)
        if (j0 + u * 32 + lane < total) tails_new[d0 + j0 + u * 32 + lane] = n[u];
    }
  }
  if (bad) *unordered = 1;
}

// average |tail - v| over a sample of edges: decides whether the given numbering already has locality
__global__ void __launch_bounds__(256) k_span_sample(int lnv, const uint32_t *rowptr, const int32_t *tails, int stride,
                                                     unsigned long long *span_sum, unsigned long long *span_cnt) {
  unsigned long long s = 0, c = 0;
  for (int v = (blockIdx.x * blockDim.x + threadIdx.x) * stride; v < lnv; v += gridDim.x * blockDim.x * stride) {
    const uint32_t e1 = rowptr[v + 1];
    for (uint32_t e = rowptr[v]; e < e1; e++) {
      const int t = tails[e];
      if (t < lnv) { s += (unsigned long long)abs(t - v); c++; }
    }
  }
  s = warp_sum(s); c = warp_sum(c);
  if ((threadIdx.x & 31) == 0 && c) { atomicAdd(span_sum, s); atomicAdd(span_cnt, c); }
}

// final assignment in the caller's numbering: out[old local vertex] = label of its community
template <bool MULTI>
__global__ void __launch_bounds__(256) k_final_labels(int lnv, const int32_t *cur, const int32_t *perm, ScanParams p, int32_t *out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < lnv; i += gridDim.x * blockDim.x) {
    const int c = cur[i];
    out[perm ? perm[i] : i] = label_of<MULTI>(p, c);
  }
}

// ----------------------------------------------------------------------------------------------
// Peer-memory collectives (comm_mode 1).  On one NVSwitch box every rank can store into every other rank's HBM,
// so the three per-iteration exchanges of the Louvain loop need no library round trips:
//   k_push_ghosts   my vertices' new communities are stored straight into the ghost tail of each peer's community
//                   array (the all-to-all-v of dspl.hpp:559-646 as NVLink stores from the producing GPU);
//   k_p2p_barrier   "every scan (and its remote atomics / ghost stores) has finished" before any fold;
//   k_p2p_allreduce the two modularity partial sums (MPI_Allreduce, dspl.hpp:441) plus the trace counters: every
//                   rank stores its contribution into every peer's mailbox, then each rank adds the mailbox up
//                   in rank order (bit-identical on all ranks); doubles as the barrier before the next scan.
// Synchronisation is an epoch counter per (destination, source) pair, written with st.release.sys after a
// system-scope fence and polled with ld.acquire.sys; epochs only grow, so a fast peer can never be missed.
// A watchdog turns a missing peer into an error flag instead of a hang.
// ----------------------------------------------------------------------------------------------
struct P2PState {                                   // one per rank, peer-mapped
  unsigned long long arrive[kMaxRanks];             // [src] = last epoch src announced to me
  unsigned long long vals[2][kMaxRanks][4];         // [epoch parity][src] = {le bits, la2 bits, moved, hash}
  unsigned int error;
  unsigned int pad_;
};
struct P2PPeers {
  int rank, nranks;
  P2PState *st[kMaxRanks];
};
struct PushTable {
  int nranks;
  long long soff[kMaxRanks + 1];                    // my send list, grouped by destination rank
  int32_t *dst[kMaxRanks];                          // where my values start in that rank's target array
};

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void p2p_wait(P2PState *mine, int src, unsigned long long epoch) {
  const long long t0 = clock64();
  while (ld_acquire_sys(&mine->arrive[src]) < epoch) {
    if (clock64() - t0 > 40000000000LL) { mine->error = 1; break; }     // ~20 s at 2 GHz: peer is gone
  }
}

__global__ void __launch_bounds__(256) k_push_ghosts(const int32_t *comm, const int32_t *send_lid, long long nsend, PushTable t) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nsend; i += (long long)gridDim.x * blockDim.x) {
    int q = 0;
    while (i >= t.soff[q + 1]) q++;
    t.dst[q][i - t.soff[q]] = comm[send_lid[i]];
  }
}

__global__ void k_p2p_barrier(P2PPeers pp, unsigned long long epoch) {
  const int t = threadIdx.x;
  P2PState *mine = pp.st[pp.rank];
  if (t < pp.nranks && t != pp.rank) {
    __threadfence_system();
    st_release_sys(&pp.st[t]->arrive[pp.rank], epoch);
    p2p_wait(mine, t, epoch);
  }
}

__global__ void k_p2p_allreduce(P2PPeers pp, unsigned long long epoch, const Acc *acc, int unit, double *out2,
                                unsigned long long *tr2) {
  const int t = threadIdx.x;
  P2PState *mine = pp.st[pp.rank];
  const int par = (int)((epoch >> 1) & 1);        // epochs alternate barrier/allreduce: bit 1 flips per iteration
  if (t < pp.nranks) {
    const double le = unit ? (double)acc->le_u : acc->le_d, la2 = unit ? (double)acc->la2_u : acc->la2_d;
    unsigned long long *dst = pp.st[t]->vals[par][pp.rank];
    dst[0] = (unsigned long long)__double_as_longlong(le);
    dst[1] = (unsigned long long)__double_as_longlong(la2);
    dst[2] = acc->moved;
    dst[3] = acc->hash;
    if (t != pp.rank) {
      __threadfence_system();
      st_release_sys(&pp.st[t]->arrive[pp.rank], epoch);
      p2p_wait(mine, t, epoch);
    }
  }
  __syncthreads();
  if (t == 0) {
    double e = 0.0, a = 0.0;
    unsigned long long mv = 0, hs = 0;
    for (int r = 0; r < pp.nranks; r++) {               // rank order: identical rounding on every rank
      const volatile unsigned long long *v = mine->vals[par][r];
      e += __longlong_as_double((long long)v[0]);
      a += __longlong_as_double((long long)v[1]);
      mv += v[2];
      hs += v[3];
    }
    out2[0] = e; out2[1] = a;
    tr2[0] = mv; tr2[1] = hs;
  }
}

// ghost exchange helpers (dspl.hpp:559-571): pack the communities peers asked for; global -> local ids
__global__ void __launch_bounds__(256) k_pack_send(const int32_t *comm, const int32_t *send_lid, int n, int32_t *out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = comm[send_lid[i]];
}
__global__ void __launch_bounds__(256) k_gid_to_lid(const long long *gid, int n, long long base, int32_t *lid) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) lid[i] = (int32_t)(gid[i] - base);
}
__global__ void __launch_bounds__(256) k_apply_inv(int32_t *lid, int n, const int32_t *inv) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) lid[i] = inv[lid[i]];
}

}  // namespace mv
