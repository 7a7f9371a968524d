// Neighbour-scan kernel with a per-warp queue of "hard" vertices (unit-weight path, option scan_variant=5).
//
// k_scan_pw spends a large share of its instructions in pass 1 and the gain arithmetic of phase B, executed with few
// of the 32 lanes active: in a converged sweep most vertices have nearly all of
// their neighbours in their own community, but the few boundary vertices of a group keep the whole warp in the pass-1
// loops.  Two observations make that cheaper without changing a single result:
//   * a vertex whose leftover neighbours (those outside its community) number m can only see gains
//       curGain <= fl( 2 (m - e_ix) + fl(fl(fl(2 k_i) a_x) c) )            (dspl.hpp:212, fl = round to nearest)
//     because every candidate community holds at most m of its edges, its degree a_y is >= 0, and rounding is monotone.
//     If that bound is <= 0 no candidate can beat maxGain = 0 (dspl.hpp:214-215) and the vertex stays where it is:
//     pass 1 is skipped for it, exactly.  At convergence that covers ~84 % of the vertices (CPU count on n = 524 288);
//   * the remaining hard vertices (5 of 32 on average) are parked -- community list, vertex, community, degree -- in a
//     small per-warp ring in shared memory, and pass 1 runs once 32 of them are waiting: one lane per hard vertex,
//     every lane busy, about every sixth group.  While the ring absorbs the leftovers the tail buffer is already
//     free, so ONE buffer suffices (the next group's bulk copy is issued right after pass 0): 6.5 KB of shared memory
//     per warp against k_scan_pw's 4.8 KB.
// A group that holds a hard vertex with more leftovers than a ring slot takes (early iterations: every neighbour is a
// different community) runs pass 1 in place like k_scan_pw.  Groups of 32 vertices per warp, the persistent grid, the
// row offsets and tails through cp.async.bulk + mbarrier, the sub-ranges and the heavy vertices come from the pipeline
// it shares with k_scan_pw (PwRing, scan_pipe.cuh), here with one tail buffer.  The 16-byte phase A is k_scan_pw's,
// written out again: as a shared helper it costs k_scan_pw registers and spills.
#pragma once
#include "scan_pipe.cuh"

namespace mv {

#ifndef MV_Q_ENT
#define MV_Q_ENT 12                    // leftover communities a ring slot holds
#endif
#ifndef MV_Q_SLOTS
#define MV_Q_SLOTS 64                   // ring slots per warp: up to (drain threshold - 1) waiting + 32 from one group
#endif
#ifndef MV_Q_DRAIN
#define MV_Q_DRAIN 32                   // parked vertices that trigger a pass-1 round (<= 32, MV_Q_SLOTS >= MV_Q_DRAIN + 31)
#endif
constexpr int kQSlots = MV_Q_SLOTS;
constexpr int kQDrain = MV_Q_DRAIN;
static_assert(kQDrain <= 32 && kQSlots >= kQDrain + 31, "ring too small");
constexpr int kQEnt = MV_Q_ENT;
constexpr int kPqCap = MV_WCAP_UNIT;   // edges in the (single) tail buffer
constexpr int kPqWarpBytes = ((kPqCap * 4 + 3 * kPwRows * 4 + kQSlots * kQEnt * 4 + kQSlots * 16 + 4 * 8) + 127) / 128 * 128;
constexpr size_t pq_smem_bytes() { return (size_t)kPwWarps * kPqWarpBytes; }

// MASKED (DESIGN.md §3.14): a vertex with movable[v] == 0 is treated like one whose bound is <= 0: never hard, never
// parked, it stays.
template <bool MULTI, bool TRACE, bool MASKED = false>
__global__ void __launch_bounds__(kPwWarps * 32, MV_PW_RES_WARPS / kPwWarps) k_scan_pq(const ScanParams p, int ngroups, const uint8_t *movable) {
  constexpr int CAP = kPqCap;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // per-warp carve-out: tails/communities [CAP] | row offsets [3][kPwRows] | ring entries [kQSlots][kQEnt] | ring headers
  // int4 [kQSlots] {vertex, community, m | degree << 16, community degree} | 4 mbarriers (tails, rows x3)
  unsigned char *wbase = smem_raw + (size_t)wid * kPqWarpBytes;
  int32_t *sc = reinterpret_cast<int32_t *>(wbase);
  const PwRing<true, 1> ring{sc, nullptr, reinterpret_cast<uint32_t *>(wbase + CAP * 4),
                             smem_u32(wbase + CAP * 4 + 3 * kPwRows * 4 + kQSlots * kQEnt * 4 + kQSlots * 16), lane};
  int32_t *q_ent = reinterpret_cast<int32_t *>(wbase + CAP * 4 + 3 * kPwRows * 4);
  int4 *q_hdr = reinterpret_cast<int4 *>(wbase + CAP * 4 + 3 * kPwRows * 4 + kQSlots * kQEnt * 4);
  ring.init();
  const int gstride = gridDim.x * kPwWarps;
  int g = blockIdx.x * kPwWarps + wid;

  unsigned long long acc_le_u = 0, acc_moved = 0, acc_hash = 0;
  uint32_t phase_bits = 0;
  int qhead = 0, qcount = 0;                     // ring state (warp-uniform)

  // pass 1 + singleton veto (kernels.cuh) for one vertex whose leftover communities sit in seg[0..m).  All lanes call
  // it; lanes without work pass m = 0.  Returns the chosen community.
  // (The same bound per candidate -- skip the exact gain when fl(2 (c - e_ix) + gB) is below the best gain so far -- was
  // measured and removed: the test costs more double-precision instructions than it saves, scan 15.30 -> 15.68 ms.)
  auto decide = [&](int32_t *seg, int m, int cc, int d, double eix, double vdeg, double ax) -> int {
    int best = cc, lbest = kNoLabel;
    pass1<true, MULTI>(p, seg, nullptr, m, eix, vdeg, ax, best, lbest);
    return singleton_veto<true, MULTI>(p, cc, best, lbest, d);
  };
  // targetComm, deltas, trace for one vertex (dspl.hpp:331-404)
  auto finish = [&](int v, int cc, int best, int d) {
    p.tgt[v] = best;
    commit<true, MULTI, TRACE>(p, v, cc, best, d, 0.0, acc_moved, acc_hash);
  };
  // run pass 1 for up to 32 parked vertices, one per lane
  auto drain = [&](int n) {
    const bool on = lane < n;
    const int slot = (qhead + lane) % kQSlots;
    int4 h = make_int4(0, 0, 0, 0);
    if (on) h = q_hdr[slot];
    const int m = on ? (h.z & 0xffff) : 0, d = h.z >> 16;
    const double vdeg = (double)d, sl = (on && p.has_self) ? (double)__ldg(p.self_i + h.x) : 0.0;
    const double eix = __dsub_rn((double)(d - m), sl), ax = __dsub_rn((double)(unsigned int)h.w, vdeg);
    const int best = decide(q_ent + slot * kQEnt, m, h.y, d, eix, vdeg, ax);
    if (on) finish(h.x, h.y, best, d);
    qhead = (qhead + n) % kQSlots;
    qcount -= n;
    __syncwarp();
  };

  int rslot = 0;
  uint32_t have_lo = 0, have_n = 0;
  ring.prologue(p, g, gstride, ngroups, phase_bits, have_lo, have_n);

  for (; g < ngroups; g += gstride) {
    const int rs1 = rslot == 2 ? 0 : rslot + 1, rs2 = rs1 == 2 ? 0 : rs1 + 1;
    if (g + 2 * gstride < ngroups) ring.issue_rows(p, g + 2 * gstride, rs2);
    if (have_n) ring.wait_bar(phase_bits, 0);

    const int v = g * 32 + lane;
    const int nvalid = min(32, p.lnv - g * 32);
    const uint32_t *rows = ring.s_rows + rslot * kPwRows;
    uint32_t ra = 0, rb = 0;
    if (lane < nvalid) { ra = rows[lane]; rb = rows[lane + 1]; }
    const uint32_t deg = rb - ra;
    const bool is_heavy = p.has_heavy && deg > (uint32_t)p.heavy_deg;
    const uint32_t g_e0 = rows[0], g_e1 = rows[nvalid];
    const bool whole = !p.has_heavy && (g_e1 - have_lo) <= have_n;

    int start = 0;
    while (start < nvalid) {
      int end = nvalid;
      uint32_t e_lo = g_e0, e_end = g_e1;
      if (!whole && !ring.sub_range(p, 0, start, nvalid, ra, rb, is_heavy, end, e_lo, e_end, have_lo, have_n, phase_bits)) {
        start++;
        continue;
      }
      const bool mine = lane >= start && lane < end;
      const int d = mine ? (int)deg : 0;
      const int o0 = (int)(ra - have_lo);
      const int ne = (int)(e_end - e_lo), eoff = (int)(e_lo - have_lo);

      // ---- phase A: tails -> communities in place (16-byte shared-memory accesses)
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
              const int i0 = 4 * q - eoff;
              if ((unsigned)(i0 + 0) < (unsigned)ne) t[u].x = __ldg(p.cur + t[u].x);
              if ((unsigned)(i0 + 1) < (unsigned)ne) t[u].y = __ldg(p.cur + t[u].y);
              if ((unsigned)(i0 + 2) < (unsigned)ne) t[u].z = __ldg(p.cur + t[u].z);
              if ((unsigned)(i0 + 3) < (unsigned)ne) t[u].w = __ldg(p.cur + t[u].w);
            }
          }
#pragma unroll
          for (int u = 0; u < U; u++) {
            const int q = qb + u * 32 + lane;
            if (q < q1) sc4[q] = t[u];
          }
        }
      }
      int cc = 0;
      unsigned int cc_deg_u = 0;
      if (mine) cc = __ldg(p.cur + v);
      double sl = 0.0;
      if (d) {
        cc_deg_u = __ldg(at_cdeg<MULTI>(p, cc));
        sl = p.has_self ? (double)__ldg(p.self_i + v) : 0.0;
      }
      __syncwarp();

      // ---- pass 0 (kernels.cuh): count the own community, compact the others to the front
      int32_t *const seg = sc + o0;
      double w0;
      const int m = pass0<true>(seg, nullptr, d, cc, w0);
      if (d) acc_le_u += (unsigned long long)(d - m);
      const double vdeg = (double)d;
      const double eix = __dsub_rn(w0, sl), ax = __dsub_rn((double)cc_deg_u, vdeg);
      // ---- can any candidate beat maxGain = 0?  (see the header: exact upper bound on curGain)
      const double gB = __dmul_rn(__dmul_rn(__dmul_rn(2.0, vdeg), ax), p.constant);
      const double bound = __dadd_rn(__dmul_rn(2.0, __dsub_rn((double)m, eix)), gB);
      const bool hard = m > 0 && (p.f32 || !(bound <= 0.0))     // the bounds are derived for the double-precision gain
                        && (!MASKED || movable[v]);
      const uint32_t hmask = __ballot_sync(0xffffffffu, hard);
      const bool in_place = __any_sync(0xffffffffu, hard && m > kQEnt);
      if (in_place) {
        // early iterations: long leftover lists everywhere -> pass 1 where the lists are, like k_scan_pw
        const int best = decide(seg, hard ? m : 0, cc, d, eix, vdeg, ax);
        if (mine) finish(v, cc, best, d);
      } else {
        if (mine && !hard) finish(v, cc, cc, d);
        if (hmask) {
          // park the hard vertices: header + leftover list into the ring
          if (hard) {
            const int slot = (qhead + qcount + __popc(hmask & ((1u << lane) - 1u))) % kQSlots;
            q_hdr[slot] = make_int4(v, cc, m | (d << 16), (int)cc_deg_u);
            int32_t *dst = q_ent + slot * kQEnt;
            for (int j = 0; j < m; j++) dst[j] = seg[j];
          }
          qcount += __popc(hmask);
        }
      }
      start = end;
      fence_proxy_async_smem();                  // generic-proxy accesses to the tail buffer end here; the next bulk copy
      __syncwarp();                              // into it is issued by lane 0 after this barrier
    }
    // ---- the tail buffer is free: next group's tails (its rows arrived while this group was reduced)
    have_lo = 0; have_n = 0;
    if (g + gstride < ngroups) {
      ring.wait_bar(phase_bits, 1 + rs1);
      ring.extent(p, g + gstride, rs1, have_lo, have_n);
      if (have_n) ring.issue_tails(p, 0, have_lo, have_n);
    }
    // ---- enough hard vertices waiting: pass 1 with one vertex per lane while the copy is in flight
    while (qcount >= kQDrain) drain(min(qcount, 32));
    rslot = rs1;
  }
  while (qcount > 0) drain(min(qcount, 32));

  flush_acc<true, TRACE, kPwWarps>(p, acc_le_u, 0.0, acc_moved, acc_hash);
}

}  // namespace mv
