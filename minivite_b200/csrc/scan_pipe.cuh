// Neighbour-scan kernel, third generation: persistent warps fed by the TMA engine.
//
// Same per-vertex decision as k_scan_ws, from the helpers shared by the scan kernels in kernels.cuh (pass0, pass1,
// singleton_veto, commit) -- distExecuteLouvainIteration + distBuildLocalMapCounter + distGetMaxIndex,
// dspl.hpp:276-405, 230-274, 174-228 -- organised around what k_scan_ws's profile showed: it was
// instruction-issue bound with a share of the issue slots empty, because the four warps of a CTA staged, met at a block barrier, reduced and met again, and every tile
// started with a dependent chain "load row offsets -> load tails -> gather cur[tail]" of three memory latencies.  Here
//   * the unit of work is a GROUP of 32 consecutive vertices owned by ONE warp; warps never meet at a block barrier
//     (only __syncwarp), so a warp that waits for its gathers leaves the issue slots to the others;
//   * the kernel is persistent: gridDim = SMs x resident CTAs, every warp strides over its groups;
//   * both streamed inputs arrive in shared memory through the TMA engine (cp.async.bulk + mbarrier complete_tx),
//     issued by one lane and never waited for in the common case: the row offsets of group k+2 and the tails of
//     group k+1 are in flight while the warp reduces group k (a ring of 3 row buffers and 2 tail buffers per warp);
//   * phase A reads four tails per 16-byte shared-memory load, gathers, and writes the four communities back in
//     place (one 4-byte slot per edge);
//   * iteration 1 of a simple graph has its own reduction (FIRST): every vertex is a singleton, so each neighbour is
//     a distinct community with one edge, and the best move is the neighbour of smallest degree.
// Groups whose edges do not fit one buffer are processed in sub-ranges with synchronous bulk copies; vertices with
// more than heavy_deg (< CAP) edges are left to k_scan_heavy.
#pragma once
#include "kernels.cuh"

namespace mv {

#ifndef MV_WCAP_UNIT
#define MV_WCAP_UNIT 512
#endif
#ifndef MV_WCAP_W
#define MV_WCAP_W 320
#endif
#ifndef MV_PW_WARPS
#define MV_PW_WARPS 8
#endif
#ifndef MV_PW_RES_WARPS
#define MV_PW_RES_WARPS 32             // resident warps per SM the register budget is sized for (unit path): 64 registers
#endif
constexpr int kPwWarps = MV_PW_WARPS;                 // warps per CTA (no block-level cooperation between them)
constexpr int kPwRows = 40;                           // row-offset slots per ring entry: 33 used, 36 copied (16-byte multiple)
template <bool UNIT> struct PwCap { static constexpr int value = UNIT ? MV_WCAP_UNIT : MV_WCAP_W; };   // edges per warp buffer

// bytes of one warp's carve-out, a multiple of 128 so that every warp's buffers keep the 16-byte alignment the bulk copies
// and the 16-byte shared-memory accesses need
template <bool UNIT> struct PwWarpBytes {
  static constexpr int value = ((2 * PwCap<UNIT>::value * (UNIT ? 4 : 12) + 3 * kPwRows * 4 + 5 * 8) + 127) / 128 * 128;
};
template <bool UNIT>
constexpr size_t pw_smem_bytes() { return (size_t)kPwWarps * PwWarpBytes<UNIT>::value; }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// a bulk copy completes within microseconds; a wait that lasts seconds is a bug -> trap instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 4000000000LL) __trap();
}
// 1-D bulk copy global -> shared through the TMA engine; completion is counted in bytes on the mbarrier.
// dst, src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- the per-warp group pipeline of the persistent scan kernels, k_scan_pw below and k_scan_pq (scan_queue.cuh)
// Each kernel carves its own shared memory and hands the pipeline NT tail buffers of PwCap<UNIT> edges (k_scan_pw 2,
// k_scan_pq 1; weights beside them when !UNIT), 3 row-offset slots of kPwRows, and NT + 3 mbarriers at bar0: the tail
// buffers' at [0, NT), the row slots' at [NT, NT + 3).  Lane 0 issues the copies.  The state carried from group to
// group (ring positions, phase bits, what a tail buffer holds) stays with the kernel.
template <bool UNIT, int NT>
struct PwRing {
  static constexpr int CAP = PwCap<UNIT>::value;
  int32_t *s_c;                  // tails, then communities: [NT][CAP]
  double *s_wt;                  // weights [NT][CAP], read when !UNIT
  uint32_t *s_rows;              // row offsets [3][kPwRows]
  uint32_t bar0;
  int lane;

  __device__ __forceinline__ void init() const {
    if (lane == 0) {
#pragma unroll
      for (int b = 0; b < NT + 3; b++) mbar_init(bar0 + 8 * b, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
  }
  // row offsets rowptr[32*gg .. 32*gg + 36) -> ring slot
  __device__ __forceinline__ void issue_rows(const ScanParams &p, int gg, int slot) const {
    if (lane == 0) {
      mbar_expect_tx(bar0 + 8 * (NT + slot), 36 * 4);
      bulk_g2s(smem_u32(s_rows + slot * kPwRows), p.rowptr + (size_t)gg * 32, 36 * 4, bar0 + 8 * (NT + slot));
    }
  }
  // edges [lo4, lo4 + n4), both multiples of 4, n4 <= CAP -> tail buffer b
  __device__ __forceinline__ void issue_tails(const ScanParams &p, int b, uint32_t lo4, uint32_t n4) const {
    if (lane == 0) {
      mbar_expect_tx(bar0 + 8 * b, n4 * (UNIT ? 4u : 12u));
      bulk_g2s(smem_u32(s_c + b * CAP), p.tails + lo4, n4 * 4u, bar0 + 8 * b);
      if (!UNIT) bulk_g2s(smem_u32(s_wt + b * CAP), p.weights + lo4, n4 * 8u, bar0 + 8 * b);
    }
  }
  // phase_bits: bit b = parity the next wait on barrier b expects
  __device__ __forceinline__ void wait_bar(uint32_t &phase_bits, int b) const {
    mbar_wait(bar0 + 8 * b, (phase_bits >> b) & 1u);
    phase_bits ^= (1u << b);
  }
  // extent of a group's edge block from its (arrived) row offsets: [lo4, lo4 + n4), clipped to one buffer
  __device__ __forceinline__ void extent(const ScanParams &p, int gg, int slot, uint32_t &lo4, uint32_t &n4) const {
    const int nv = min(32, p.lnv - gg * 32);
    const uint32_t e0 = s_rows[slot * kPwRows], e1 = s_rows[slot * kPwRows + nv];
    lo4 = e0 & ~3u;
    n4 = (e1 > lo4) ? min((uint32_t)CAP, (e1 - lo4 + 3u) & ~3u) : 0u;
  }
  // prologue: rows of the warp's first two groups into slots 0 and 1, tails of the first into buffer 0
  __device__ __forceinline__ void prologue(const ScanParams &p, int g, int gstride, int ngroups, uint32_t &phase_bits,
                                           uint32_t &have_lo, uint32_t &have_n) const {
    if (g < ngroups) {
      issue_rows(p, g, 0);
      if (g + gstride < ngroups) issue_rows(p, g + gstride, 1);
      wait_bar(phase_bits, NT);
      extent(p, g, 0, have_lo, have_n);
      if (have_n) issue_tails(p, 0, have_lo, have_n);
    }
  }
  // the sub-range of a group that starts at lane `start` (ra, rb: this lane's row offsets, nvalid the group's size):
  // the longest run [start, end) of non-heavy vertices whose edges [e_lo, e_end) fit one buffer.  Tail buffer b, which
  // holds edges [have_lo, have_lo + have_n), is reloaded synchronously when it does not cover them (oversize group).
  // False when the start vertex is heavy: the caller steps over it, k_scan_heavy takes it.
  __device__ __forceinline__ bool sub_range(const ScanParams &p, int b, int start, int nvalid, uint32_t ra, uint32_t rb,
                                            bool is_heavy, int &end, uint32_t &e_lo, uint32_t &e_end, uint32_t &have_lo,
                                            uint32_t &have_n, uint32_t &phase_bits) const {
    const uint32_t heavy_mask = __ballot_sync(0xffffffffu, is_heavy);
    if ((heavy_mask >> start) & 1u) return false;
    e_lo = __shfl_sync(0xffffffffu, ra, start);
    const uint32_t a_sub = e_lo & ~3u;
    const bool fits = lane >= start && lane < nvalid && !is_heavy && (rb - a_sub) <= (uint32_t)CAP;
    const uint32_t stop_mask = ~__ballot_sync(0xffffffffu, fits) & (0xffffffffu << start);
    end = stop_mask ? (__ffs(stop_mask) - 1) : 32;               // > start: the start vertex always fits
    e_end = __shfl_sync(0xffffffffu, rb, end - 1);
    if (!(a_sub >= have_lo && e_end <= have_lo + have_n)) {
      have_lo = a_sub;
      have_n = (e_end - a_sub + 3u) & ~3u;
      if (have_n) { issue_tails(p, b, have_lo, have_n); wait_bar(phase_bits, b); }
    }
    return true;
  }
};

// MASKED (DESIGN.md §3.14): a vertex with movable[v] == 0 skips pass 1 and stays (counter[0] still counted).
template <bool UNIT, bool MULTI, bool TRACE, bool FIRST, bool MASKED = false>
__global__ void __launch_bounds__(kPwWarps * 32, UNIT ? MV_PW_RES_WARPS / kPwWarps : 24 / kPwWarps)
k_scan_pw(const ScanParams p, int ngroups, const uint8_t *movable) {
  static_assert(!FIRST || UNIT, "the first-iteration reduction exists for the unit-weight path only");
  static_assert(!(FIRST && MASKED), "a masked run takes the general reduction in iteration 1");
  constexpr int CAP = PwCap<UNIT>::value;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // per-warp carve-out: tails/communities [2][CAP] int32 | (weights [2][CAP] double) | row offsets [3][kPwRows] | 5 mbarriers
  constexpr int kWarpBytes = PwWarpBytes<UNIT>::value;
  static_assert(CAP % 4 == 0 && kPwRows % 4 == 0, "buffers must be 16-byte multiples");
  unsigned char *wbase = smem_raw + (size_t)wid * kWarpBytes;
  const PwRing<UNIT, 2> ring{reinterpret_cast<int32_t *>(wbase), reinterpret_cast<double *>(wbase + 2 * CAP * 4),
                             reinterpret_cast<uint32_t *>(wbase + 2 * CAP * (UNIT ? 4 : 12)),
                             smem_u32(wbase + 2 * CAP * (UNIT ? 4 : 12) + 3 * kPwRows * 4), lane};
  ring.init();
  const int gstride = gridDim.x * kPwWarps;
  int g = blockIdx.x * kPwWarps + wid;

  unsigned long long acc_le_u = 0, acc_moved = 0, acc_hash = 0;
  double acc_le_d = 0.0;
  uint32_t phase_bits = 0;

  int rslot = 0, buf = 0;                        // ring positions of the current group
  uint32_t have_lo = 0, have_n = 0;              // what the current tail buffer holds: edges [have_lo, have_lo + have_n)
  ring.prologue(p, g, gstride, ngroups, phase_bits, have_lo, have_n);

  for (; g < ngroups; g += gstride) {
    // ---- keep the rings full: rows of group k+2, tails of group k+1 (its rows arrived one iteration ago)
    const int rs1 = rslot == 2 ? 0 : rslot + 1, rs2 = rs1 == 2 ? 0 : rs1 + 1;
    if (g + 2 * gstride < ngroups) ring.issue_rows(p, g + 2 * gstride, rs2);
    uint32_t nx_lo = 0, nx_n = 0;
    if (g + gstride < ngroups) {
      ring.wait_bar(phase_bits, 2 + rs1);
      ring.extent(p, g + gstride, rs1, nx_lo, nx_n);
      if (nx_n) ring.issue_tails(p, buf ^ 1, nx_lo, nx_n);
    }
    if (have_n) ring.wait_bar(phase_bits, buf);

    const int v = g * 32 + lane;
    const int nvalid = min(32, p.lnv - g * 32);
    const uint32_t *rows = ring.s_rows + rslot * kPwRows;
    uint32_t ra = 0, rb = 0;
    if (lane < nvalid) { ra = rows[lane]; rb = rows[lane + 1]; }
    const uint32_t deg = rb - ra;
    const bool is_heavy = p.has_heavy && deg > (uint32_t)p.heavy_deg;
    int32_t *sc = ring.s_c + buf * CAP;
    double *sw = ring.s_wt + buf * CAP;
    const uint32_t g_e0 = rows[0], g_e1 = rows[nvalid];
    // the common case: no vertex of the shard is heavy and the whole group sits in the prefetched buffer
    const bool whole = !p.has_heavy && (g_e1 - have_lo) <= have_n;

    int start = 0;
    while (start < nvalid) {
      // ---- sub-range [start, end): longest run of non-heavy vertices whose edges fit the buffer
      int end = nvalid;
      uint32_t e_lo = g_e0, e_end = g_e1;
      if (!whole && !ring.sub_range(p, buf, start, nvalid, ra, rb, is_heavy, end, e_lo, e_end, have_lo, have_n, phase_bits)) {
        start++;
        continue;
      }
      const bool mine = lane >= start && lane < end;
      const int d = mine ? (int)deg : 0;
      const int o0 = (int)(ra - have_lo);
      const int ne = (int)(e_end - e_lo), eoff = (int)(e_lo - have_lo);

      // ---- phase A: tails (already in shared memory) -> communities, in place; 16-byte shared-memory accesses,
      // all gathers of a pass in flight before the first store.  FIRST: the neighbour's degree instead (every
      // neighbour is its own community).
      {
        int4 *sc4 = reinterpret_cast<int4 *>(sc);
        const int q0 = eoff >> 2, q1 = (eoff + ne + 3) >> 2;
        constexpr int U = 3;
        for (int qb = q0; qb < q1; qb += U * 32) {
          int4 t[U];
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int q = qb + u * 32 + lane;
            if (q < q1) t[u] = sc4[q];
          }
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int q = qb + u * 32 + lane;
            if (q < q1) {
              const int i0 = 4 * q - eoff;               // position of the quad's first entry inside the sub-range
              auto gat = [&](int tl) -> int {
                if (!FIRST) return __ldg(p.cur + tl);
                if (!MULTI || tl < p.lnv) return (int)__ldg(p.loc_cdeg + tl);
                return (int)__ldg(at_cdeg<MULTI>(p, __ldg(p.cur + tl)));
              };
              if ((unsigned)(i0 + 0) < (unsigned)ne) t[u].x = gat(t[u].x);
              if ((unsigned)(i0 + 1) < (unsigned)ne) t[u].y = gat(t[u].y);
              if ((unsigned)(i0 + 2) < (unsigned)ne) t[u].z = gat(t[u].z);
              if ((unsigned)(i0 + 3) < (unsigned)ne) t[u].w = gat(t[u].w);
            }
          }
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int q = qb + u * 32 + lane;
            if (q < q1) sc4[q] = t[u];
          }
        }
      }
      int cc = 0, best = 0;
      if (mine) { cc = __ldg(p.cur + v); best = cc; }
      double cc_deg = 0.0, vdeg = 0.0, sl = 0.0;
      if (d && !FIRST) vertex_load<UNIT, MULTI>(p, v, cc, d, cc_deg, vdeg, sl);
      __syncwarp();

      int lbest = kNoLabel;
      if (FIRST) {
        // ---- iteration 1 on a simple graph without self loops: cur[] is the identity, every community a singleton.
        // counter[0] = 0, eix = 0, ax = 0, and neighbour y offers gain_of(1, 0, d, deg(y), 0, c): the same expression
        // the general path evaluates, non-increasing in deg(y).  So the winner has the smallest degree; among equal
        // gains the smallest label wins (dspl.hpp:214-215).  sc[] holds the neighbours' degrees.
        int amin = 0x7fffffff;
        for (int k = 0; k < d; k++) amin = min(amin, sc[o0 + k]);
        if (d) {
          const double dd = (double)d;
          const double gmax = gain_of(1.0, 0.0, dd, (double)amin, 0.0, p.constant, p.f32);
          const double gnext = gain_of(1.0, 0.0, dd, (double)amin + 1.0, 0.0, p.constant, p.f32);
          if (gmax > 0.0) {                                   // maxGain starts at 0: only a positive gain moves (dspl.hpp:214)
            const bool collide = !(gnext < gmax);             // never seen: two degrees rounding to one gain -> compare gains
            int by = cc, lb = 0x7fffffff;
            for (int k = 0; k < d; k++) {
              const int a = sc[o0 + k];
              if (a == amin || (collide && gain_of(1.0, 0.0, dd, (double)a, 0.0, p.constant, p.f32) == gmax)) {
                const int tl = __ldg(p.tails + ra + k);
                const int y = (!MULTI || tl < p.lnv) ? (int)p.base + tl : __ldg(p.cur + tl);
                const int ly = label_of<MULTI>(p, y);
                if (ly < lb) { lb = ly; by = y; }
              }
            }
            best = by; lbest = lb;
            // singleton veto (dspl.hpp:224-225): both communities have size 1 in this iteration
            if (lbest > label_of<MULTI>(p, cc)) best = cc;
          }
        }
      } else {
        // ---- phase B: the shared per-vertex decision (kernels.cuh)
        double w0;
        int m = pass0<UNIT>(sc + o0, sw + o0, d, cc, w0);
        const double eix = __dsub_rn(w0, sl), ax = __dsub_rn(cc_deg, vdeg);
        if (d) { if (UNIT) acc_le_u += (unsigned long long)(d - m); else acc_le_d += w0; }
        if (MASKED && d && !movable[v]) m = 0;                               // frozen: no candidate, best stays cc
        pass1<UNIT, MULTI>(p, sc + o0, sw + o0, m, eix, vdeg, ax, best, lbest);
        if (mine) best = singleton_veto<UNIT, MULTI>(p, cc, best, lbest, d);
      }
      if (mine) {
        p.tgt[v] = best;                                                       // dspl.hpp:404
        commit<UNIT, MULTI, TRACE>(p, v, cc, best, d, vdeg, acc_moved, acc_hash);
      }
      start = end;
      fence_proxy_async_smem();                  // this lane's generic-proxy accesses to the buffer are ordered before
      __syncwarp();                              // the TMA write that reuses it (issued by lane 0 after the barrier)
    }
    // rotate the rings
    rslot = rs1;
    buf ^= 1;
    have_lo = nx_lo; have_n = nx_n;
  }

  flush_acc<UNIT, TRACE, kPwWarps>(p, acc_le_u, acc_le_d, acc_moved, acc_hash);
}

}  // namespace mv
