// One association + reduction pass over the queries of EVERY resident unit of the CTA at each unit's current
// linearisation point (rows A2-A9 of SURVEY.md §8; reference findCorrespondingSurfFeatures /
// findCorrespondingCornerFeatures, lins/include/StateEstimator.hpp:829-1063, + the measurement assembly :499-532
// folded into 28 sums per unit).
//
// Queries live in a virtual index space v = slot * qtile + i (qtile a multiple of 32, so a warp never straddles two
// units).  Thread-per-query phases sweep v, warp-per-search phases pull v from one work list shared by all slots.
//
// Fast path (sm.az_ok): targets are ring-sorted, the (ring, azimuth) index of lins_assoc_az.cuh is valid.
// Legacy path: any ring order / ring values / a 1-NN cloud that differs from the walk cloud (the stale-index
// quirk of :1156-1160): brute-force exact 1-NN + the literal sequential walks over global memory.
#pragma once
#include "lins_assoc_az.cuh"

namespace lins_dev {

// Probe-first search (lins_assoc_az.cuh: az_probe_window) is used for the closest-point search of a unit's FIRST pass
// only: there every query is unseeded and the gate-wide window is much larger than the neighbourhood that holds the
// answer.
// widest windows (azimuth bins per ring) a group of kGroupLanes lanes scans; wider ones go to a whole warp
constexpr int kGroupLanes = 4;
constexpr int kThreadScanBins = 16, kThreadWalkBins = 48;

// Certificate and pass counters of the phase timers (bv.timers, read by lins_gpu_debug_phase_cycles; tools/phase_profile.py
// prints them).  Slots kCertSlots + k, k = 0..7, count the certificates of seeded queries: checked, accepted, failed because
// the runner-up now beats the winner (and the bound does not certify it), because winner + moved + slack >= bound, because
// the answer left the gate, because a rejected search's slack is used up, failed although the fresh search returned one of
// the stored front-runners, accepted by a swap.  Each slot holds two 32-bit counts: the closest point's certificates in
// the low half, the walks' (one per query: Ind2 and, for surf, Ind3) in the high half.  Slots kPassSlots + 0..13: later
// passes (no unit in its first pass) by their number of closest-point searches (0 / 1-16 / > 16: 3 counts, then the P2
// cycles of each) and of walk searches (0 / 1-16 / 17-32 / > 32: 4 counts, then the P3 + P4 cycles of each).
constexpr int kCertSlots = 40, kPassSlots = 48;
__device__ __forceinline__ void count_cert_events(long long* timers, unsigned ev) {  // warp-wide; ev: bit k / 8 + k
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const unsigned n1 = __popc(__ballot_sync(0xffffffffu, (ev >> k) & 1u)), n2 = __popc(__ballot_sync(0xffffffffu, (ev >> (8 + k)) & 1u));
    if ((threadIdx.x & 31) == 0 && (n1 | n2)) atomicAdd((unsigned long long*)&timers[kCertSlots + k], ((unsigned long long)n2 << 32) | n1);
  }
}

struct PassBuffers {           // per-query arrays, indexed by v = slot * qtile + i (shared memory, or the CTA's global scratch)
  float4* qpt;               // staged queries (x, y, z, intensity)
  float4* sel;               // de-skewed queries (pointSel)
  unsigned long long* key;   // legacy path: 1-NN keys; fast path: (B2, B3) of the walk windows
  int* pos;                  // 3 per query.  fast path: slots in the sorted copies (closest, Ind2, Ind3);
                             //               legacy path / reloaded correspondences: original indices
  float4* qa;                // fast path: (azimuth, rho, -, bound of everything outside the window) of the de-skewed query
  int4* qw;                  // fast path: level / search windows w1 / w2 / w3 and (ring << 24 | index) of the closest point
  float4* qref;              // fast path: pointSel at the last closest-point search + the certificate bound of its answer
  float4* qref2;             // fast path: pointSel at the last walk search + the bound of Ind2
  int* qccr;                 // fast path: (ring << 24 | original index) of the closest point, -1 = none
  float4* qext;              // fast path: (bound of Ind3, runner-up slots of closest / Ind2 / Ind3 as int bits)
  int* wl;                   // work list of the queries that need a closest-point search / ring walks this pass
  double* wacc;              // [slot][warp of the slot][28] partial folds of the pass
  int* wcnt;                 // [slot][warp of the slot][2] accepted surf / corner measurements
  int nvw;                   // warps per slot = qtile / 32
};

// The fused kernel's dynamic shared memory, in this order, every region starting 16-byte aligned:
//   CtaMem | Smem x nslots | wacc | wcnt | per-query arrays
// The per-query arrays hold NQ = nslots * qtile entries each, back to back in the order pass_layout carves them (qtile
// is a multiple of 32, so each of them starts 16-byte aligned).  When even one slot's arrays do not fit shared memory,
// they live in a per-CTA global scratch instead (BatchView::qscratch) and the launch asks only for fixed_bytes.
struct PassLayout {
  size_t slots;        // offset of slot 0 (CtaMem is at offset 0)
  size_t fixed_bytes;  // CtaMem, slots, wacc, wcnt
  size_t query_bytes;  // the per-query arrays
};

__host__ __device__ constexpr size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// The layout for nslots units of qtile queries.  With pb, also fills *pb for CTA `cta`, whose dynamic shared memory starts
// at smem: its per-query arrays follow wcnt there or, when qscratch is not null, start at qscratch + cta * qscratch_stride.
__host__ __device__ __forceinline__ PassLayout pass_layout(int nslots, int qtile, PassBuffers* pb = nullptr, unsigned char* smem = nullptr,
                                                           unsigned char* qscratch = nullptr, unsigned cta = 0, size_t qscratch_stride = 0) {
  static_assert(sizeof(Smem) % 16 == 0, "slots are indexed as an array");
  const int NQ = nslots * qtile;
  const size_t nvw_all = (size_t)nslots * (qtile / 32);
  const size_t wacc_bytes = align16(nvw_all * kNAcc * sizeof(double)), wcnt_bytes = align16(nvw_all * 2 * sizeof(int));
  PassLayout lay;
  lay.slots = align16(sizeof(CtaMem));
  lay.fixed_bytes = lay.slots + nslots * sizeof(Smem) + wacc_bytes + wcnt_bytes;
  // one entry of every per-query array the carve below takes, in its order (pos holds three per query); the carve is a
  // pointer chain so that the kernel's address set-up stays as before
  lay.query_bytes = align16((size_t)NQ * (sizeof(*pb->qpt) + sizeof(*pb->sel) + sizeof(*pb->qa) + sizeof(*pb->qw) + sizeof(*pb->qref) +
                                          sizeof(*pb->qref2) + sizeof(*pb->qext) + sizeof(*pb->key) + 3 * sizeof(*pb->pos) +
                                          sizeof(*pb->qccr) + sizeof(*pb->wl)));
  if (pb) {
    PassBuffers& b = *pb;
    b.nvw = qtile / 32;
    unsigned char* p = smem + lay.slots;
    p += nslots * sizeof(Smem);
    b.wacc = reinterpret_cast<double*>(p); p += wacc_bytes;
    b.wcnt = reinterpret_cast<int*>(p); p += wcnt_bytes;
    if (qscratch) p = qscratch + (size_t)cta * qscratch_stride;
    b.qpt = reinterpret_cast<float4*>(p); p = reinterpret_cast<unsigned char*>(b.qpt + NQ);
    b.sel = reinterpret_cast<float4*>(p); p = reinterpret_cast<unsigned char*>(b.sel + NQ);
    b.qa = reinterpret_cast<float4*>(p); p = reinterpret_cast<unsigned char*>(b.qa + NQ);
    b.qw = reinterpret_cast<int4*>(p); p = reinterpret_cast<unsigned char*>(b.qw + NQ);
    b.qref = reinterpret_cast<float4*>(p); p = reinterpret_cast<unsigned char*>(b.qref + NQ);
    b.qref2 = reinterpret_cast<float4*>(p); p = reinterpret_cast<unsigned char*>(b.qref2 + NQ);
    b.qext = reinterpret_cast<float4*>(p); p = reinterpret_cast<unsigned char*>(b.qext + NQ);
    b.key = reinterpret_cast<unsigned long long*>(p); p = reinterpret_cast<unsigned char*>(b.key + NQ);
    b.pos = reinterpret_cast<int*>(p); p = reinterpret_cast<unsigned char*>(b.pos + 3 * NQ);
    b.qccr = reinterpret_cast<int*>(p); p = reinterpret_cast<unsigned char*>(b.qccr + NQ);
    b.wl = reinterpret_cast<int*>(p);
  }
  return lay;
}

__device__ __forceinline__ AzIndex az_index_of(const Smem& sm, const BatchView& bv, bool surf) {
  AzIndex ix;
  if (surf) { ix.pts = bv.az_s + sm.ts0; ix.bstart = sm.azTabS; ix.elev = sm.elevS; ix.nb = sm.nbS; ix.nrings = sm.nringsS; ix.T = sm.Ts; }
  else { ix.pts = bv.az_c + sm.tc0; ix.bstart = sm.azTabC; ix.elev = sm.elevC; ix.nb = sm.nbC; ix.nrings = sm.nringsC; ix.T = sm.Tc; }
  return ix;
}

// slot of a virtual query index (nslots <= kMaxSlots = 4)
__device__ __forceinline__ int slot_of(int v, int Q) { return (v >= Q) + (v >= 2 * Q) + (v >= 3 * Q); }

template <int MODE>
__device__ void association_pass(CtaMem& cta, Smem* slots, const BatchView& bv, const KParams& kp, const PassBuffers& pb) {
  const int Q = bv.qtile, NQ = bv.nslots * Q;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // ---- A2: de-skew, fused with phase P1 of the association (same thread-per-query mapping; P1 touches only its own
  // query's state and the read-only index): per-query level -2 everything certified, -3 closest point certified (walks
  // only), -4 closest point certified by a swap (walks only, around the new closest point), >= 0 full search (= window),
  // -1 cannot match.  The work-list counters were reset after the previous pass.
  for (int v = threadIdx.x; v < NQ; v += kThreads) {  // (NQ is a multiple of 32: every lane of a warp runs every trip)
    unsigned ev = 0u;  // diagnostics: certificate events of this query (bit k: closest point, slot 40 + k; bit 8 + k: walks)
    do {  // (a `continue` below leaves this block, not the loop: the events of every query are counted after it)
    const int sl = slot_of(v, Q), i = v - sl * Q;
    Smem& sm = slots[sl];
    if (!sm.run || i >= sm.ns + sm.nc) continue;
    const float4 s = transform_to_start(pb.qpt[v], sm, sm.period);
    pb.sel[v] = s;
    pb.key[v] = kKeyMax;
    if (!sm.search) {
      // iter % ICP_FREQ != 0: reuse pointSearch*Ind (StateEstimator.hpp:844, :970); a unit that has not searched in this
      // launch takes them from global memory (they persist between calls like the reference's arrays)
      if (!sm.pos_valid) {
        if (i < sm.ns) { const int* o = bv.ind_s + 3 * (size_t)(sm.qs0 + i); pb.pos[3 * v] = o[0]; pb.pos[3 * v + 1] = o[1]; pb.pos[3 * v + 2] = o[2]; }
        else { const int* o = bv.ind_c + 2 * (size_t)(sm.qc0 + i - sm.ns); pb.pos[3 * v] = o[0]; pb.pos[3 * v + 1] = o[1]; pb.pos[3 * v + 2] = -1; }
      }
      continue;
    }
    if (!sm.az_ok) continue;
    const bool surf = i < sm.ns;
    const bool seeded = !sm.first_pass;
    const AzIndex ixq = az_index_of(sm, bv, surf);
    float4 qa = make_float4(0.f, 0.f, -1.f, 0.f);
    if (seeded) {  // certificates (lins_assoc_az.cuh: cert_check / cert_rejected): the stored answers still hold
      const float4 r1 = pb.qref[v], r2 = pb.qref2[v], ex = pb.qext[v];
      const unsigned nearbits = __float_as_uint(sm.nearf);
      const int w1s = pb.pos[3 * v], w2s = pb.pos[3 * v + 1], w3s = pb.pos[3 * v + 2];
      const int r1s = __float_as_int(ex.y), r2s = __float_as_int(ex.z), r3s = __float_as_int(ex.w);
      // every front-runner of the query in one batch of independent (predicated) loads; a slot is read only where the
      // sequential evaluation below could use it (the runner-up fields of a rejected search and the walk fields of a query
      // without a closest point are not maintained)
      const int ccr0 = pb.qccr[v];
      const bool walks = ccr0 >= 0;
      auto entry = [&](int slot, bool use) -> float4 {
        return use && slot >= 0 && slot < ixq.T ? ixq.pts[slot] : make_float4(0.f, 0.f, 0.f, 0.f);
      };
      const float4 tw1 = entry(w1s, true), tr1 = entry(r1s, w1s >= 0);
      const float4 tw2 = entry(w2s, walks), tr2 = entry(r2s, walks && w2s >= 0);
      const float4 tw3 = entry(w3s, walks && surf), tr3 = entry(r3s, walks && surf && w3s >= 0);
      const float moved1 = sqrtf(sqdist_f32(s.x, s.y, s.z, r1.x, r1.y, r1.z));
      const int c1 = w1s >= 0 ? cert_check<false>(tw1, tr1, s, r1s, r1.w, moved1, nearbits, 0)
                              : (cert_rejected(r1.w, moved1) ? kCertKeep : kCertFailSlack);
      const bool ok1 = c1 <= kCertSwap;
      ev = 1u | (1u << (ok1 ? 1 : c1)) | (c1 == kCertSwap ? 1u << 7 : 0u);
      // (a swap's write-back runs in P3, where a thread holds far fewer values than here)
      if (c1 == kCertSwap) { az_polar(s, qa); pb.qa[v] = qa; pb.qw[v] = make_int4(-4, 0, 0, 0); continue; }
      bool ok2 = false;
      int c2 = kCertKeep, c3 = kCertKeep;
      if (ok1 && walks) {  // (the walks' candidate sets are defined by the closest point: only meaningful while it stands)
        const int c0 = ccr0 & 0x00ffffff;
        const float moved2 = sqrtf(sqdist_f32(s.x, s.y, s.z, r2.x, r2.y, r2.z));
        c2 = w2s >= 0 ? cert_check<true>(tw2, tr2, s, r2s, r2.w, moved2, nearbits, c0) : (cert_rejected(r2.w, moved2) ? kCertKeep : kCertFailSlack);
        ok2 = c2 <= kCertSwap;
        if (ok2 && surf) {
          c3 = w3s >= 0 ? cert_check<true>(tw3, tr3, s, r3s, ex.x, moved2, nearbits, c0) : (cert_rejected(ex.x, moved2) ? kCertKeep : kCertFailSlack);
          ok2 = c3 <= kCertSwap;
        }
        ev |= (1u << 8) | (1u << (8 + (ok2 ? 1 : c2 <= kCertSwap ? c3 : c2))) |  // (the first that failed)
              (ok2 && (c2 == kCertSwap || c3 == kCertSwap) ? 1u << 15 : 0u);
      }
      if (ok1 && (ok2 || ccr0 < 0)) { pb.qw[v] = make_int4(-2, (c2 == kCertSwap ? 1 : 0) | (c3 == kCertSwap ? 2 : 0), 0, 0); continue; }
      if (ok1) { az_polar(s, qa); pb.qa[v] = qa; pb.qw[v] = make_int4(-3, 0, 0, 0); continue; }
    }
    const int w1 = az_prepare_nn(ixq, s, sm.nearf, seeded ? pb.pos[3 * v] : -1, (int)pb.qpt[v].w, qa);
    pb.qa[v] = qa;
    pb.qw[v] = make_int4(w1, 0, 0, 0);
    // (list order does not matter: every query's result goes to its own slot.)  Two lists share pb.wl: searches run by a
    // warp each from the front, searches run by a group of kGroupLanes lanes each from the back.  Groups serve the pass in
    // which (nearly) every query of a unit searches — its first — where throughput counts (measured: 1.5x faster there);
    // the handful of searches of a later pass are latency bound and finish sooner with a warp each.
    if (sm.first_pass && w1 >= 0 && (w1 & 0xffff) <= kThreadScanBins) pb.wl[NQ - 1 - atomicAdd(&cta.wl_tn[0], 1)] = v;
    else pb.wl[atomicAdd(&cta.wl_n[0], 1)] = v;
    if (bv.timers && w1 >= 0) atomicAdd(&cta.dbg[0], w1 & 0xffff);
    } while (false);
    if (bv.timers) count_cert_events(bv.timers, ev);
  }
  __syncthreads();
  LINS_TICK_PASS(3);

  if (cta.any_indexed) {
    // ---- A3/A4 fast path.  Scalar preparation (certificates, atan2f, asinf, bounds: P1 above, P3 below) runs one
    // THREAD per query so that all queries proceed in parallel; the memory scans (P2, P4) run one WARP per query.
    if (bv.timers && threadIdx.x == 0) {
      atomicAdd((unsigned long long*)&bv.timers[10], (unsigned long long)cta.wl_n[0]);
      atomicAdd((unsigned long long*)&bv.timers[12], (unsigned long long)cta.dbg[0]);
    }
    // result of a closest-point search -> the query's state (one thread)
    auto nn_finish = [&](int v, const AzIndex& ix, const float4 s, const Top3& top, int w1, float Bout) {
      const unsigned long long k1 = top.k1;
      const int p1 = top.p1;
      const float d1 = __uint_as_float((unsigned)(k1 >> 32));
      const Smem& sq = slots[slot_of(v, Q)];
      const bool acc1 = k1 != kKeyMax && p1 >= 0 && (double)d1 < sq.nearest_sq;
      // (diagnostics read what they need from shared memory, so that nothing extra stays live across the scan)
      if (bv.timers && !sq.first_pass && pb.pos[3 * v] >= 0 && acc1 && (p1 == pb.pos[3 * v] || p1 == __float_as_int(pb.qext[v].y)))
        atomicAdd((unsigned long long*)&bv.timers[kCertSlots + 6], 1ull);  // a failed certificate whose stored front-runners held the answer
      // accepted: what everything but the two front-runners exceeded; else the slack of "nothing within the gate"
      const float bound1 = w1 < 0 ? -1.f : acc1 ? cert_bound(top.d3, Bout) : rejected_slack((unsigned)(k1 >> 32), Bout, sq.gate);
      pb.qref[v] = make_float4(s.x, s.y, s.z, bound1);
      pb.qext[v].y = __int_as_float(acc1 ? top.p2 : -1);
      pb.pos[3 * v] = acc1 ? p1 : -1;
      pb.qccr[v] = acc1 ? ((slot_ring(ix.pts[p1].w) << 24) | (int)(unsigned)(k1 & 0xffffffffu)) : -1;
    };
    // P2, group-level list first: groups of kGroupLanes lanes pull queries (a warp whose groups find the list empty goes
    // straight to the warp-level list)
    constexpr int G = kGroupLanes;
    const int sub = lane & (G - 1), glead = lane & ~(G - 1);
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << glead);
    for (;;) {
      int k = 0;
      if (sub == 0) k = atomicAdd(&cta.wl_thead[0], 1);
      k = __shfl_sync(gmask, k, glead);
      if (k >= cta.wl_tn[0]) break;
      const int v = pb.wl[NQ - 1 - k];
      const int sl = slot_of(v, Q), i = v - sl * Q;
      const Smem& sm = slots[sl];
      const AzIndex ix = az_index_of(sm, bv, i < sm.ns);
      const float4 s = pb.sel[v];
      const int w1 = pb.qw[v].x;
      const float4 qag = pb.qa[v];
      const Top3 top = az_scan_nn_group<G>(ix, s, w1, qag.y, qag.w, sub, gmask);
      if (sub == 0) nn_finish(v, ix, s, top, w1, qag.w);
    }
    // P2: warps pull queries from the work list (the per-query cost is heavy-tailed; a static split leaves warps idle)
    for (;;) {
      int k = 0;
      if (lane == 0) k = atomicAdd(&cta.wl_head[0], 1);
      k = __shfl_sync(0xffffffffu, k, 0);
      if (k >= cta.wl_n[0]) break;
      const int v = pb.wl[k];
      const int sl = slot_of(v, Q), i = v - sl * Q;
      const Smem& sm = slots[sl];
      int w1 = pb.qw[v].x;
      Top3 top;
      top.init();
      const bool surf = i < sm.ns;
      const AzIndex ix = az_index_of(sm, bv, surf);
      const float4 s = pb.sel[v];
      float4 qa = pb.qa[v];
      if (w1 >= 0) {
        const int wp = sm.first_pass ? az_probe_window(ix, qa, w1) : -1;
        if (wp >= 0) {  // wide window (no usable previous answer): probe first, then search inside the implied window
          const Top3 pr = az_scan_nn(ix, s, wp, qa.y, sqrtf(widen(kProbeSq)));  // (a probe needs no exactness: anything it finds is an upper bound)
          if (pr.p1 >= 0) {
            w1 = az_nn_window(ix, az_seed_bound(ix, s, pr.p1, sm.nearf), qa);
            if (lane == 0) pb.qa[v] = qa;
          }
        }
        top = az_scan_nn(ix, s, w1, qa.y, qa.w);
      }
      if (lane == 0) nn_finish(v, ix, s, top, w1, qa.w);
    }
    __syncthreads();
    if (bv.timers && threadIdx.x == 0 && !cta.pass_first) {  // later passes by their number of closest-point searches
      const int n = cta.wl_n[0] + cta.wl_tn[0], b = n == 0 ? 0 : n <= 16 ? 1 : 2;
      atomicAdd((unsigned long long*)&bv.timers[kPassSlots + b], 1ull);
      atomicAdd((unsigned long long*)&bv.timers[kPassSlots + 3 + b], (unsigned long long)(clock64() - cta.tlast));
    }
    LINS_TICK_PASS(4);
    for (int v = threadIdx.x; v < NQ; v += kThreads) {  // P3
      const int sl = slot_of(v, Q), i = v - sl * Q;
      const Smem& sm = slots[sl];
      if (!sm.run || !sm.az_ok || i >= sm.ns + sm.nc || !sm.search) continue;
      const int2 lq = *reinterpret_cast<const int2*>(&pb.qw[v]);  // (level, walk swaps)
      const int lvl = lq.x;
      const bool surf = i < sm.ns;
      // swaps certified in P1: winner and runner-up change places, the IDs follow; the search position and bound stay
      auto swap_front = [&](int k, float* runner_up) {  // k = 0 closest point, 1 Ind2, 2 Ind3; returns the new winner's entry
        const int w = pb.pos[3 * v + k], r = __float_as_int(*runner_up);
        pb.pos[3 * v + k] = r;
        *runner_up = __int_as_float(w);
        return az_index_of(sm, bv, surf).pts[r].w;
      };
      if (lvl == -2) {
        if (lq.y) {
          int* const o = surf ? bv.ind_s + 3 * (size_t)(sm.qs0 + i) : bv.ind_c + 2 * (size_t)(sm.qc0 + i - sm.ns);
          if (lq.y & 1) o[1] = slot_index(swap_front(1, &pb.qext[v].z));
          if (lq.y & 2) o[2] = slot_index(swap_front(2, &pb.qext[v].w));
        }
        continue;
      }
      if (lvl == -4) {  // a new closest point: its walks are searched below (their candidate sets are defined by it)
        const float tw = swap_front(0, &pb.qext[v].y);
        pb.qccr[v] = (slot_ring(tw) << 24) | slot_index(tw);
      }
      const int ccr = pb.qccr[v];
      if (ccr < 0) {  // no closest point within the gate: nothing to walk
        pb.pos[3 * v + 1] = -1; pb.pos[3 * v + 2] = -1;
        pb.qw[v] = make_int4(-1, 0, 0, 0);
        if (surf) { int* o = bv.ind_s + 3 * (size_t)(sm.qs0 + i); o[0] = -1; o[1] = -1; o[2] = -1; }
        else { int* o = bv.ind_c + 2 * (size_t)(sm.qc0 + i - sm.ns); o[0] = -1; o[1] = -1; }
        continue;
      }
      int w2 = 0, w3 = 0;
      float B2 = 0.f, B3 = 0.f;
      const bool seeded = !sm.first_pass;
      const int sd2 = seeded ? pb.pos[3 * v + 1] : -1, sd3 = seeded ? pb.pos[3 * v + 2] : -1;
      const int c = ccr & 0x00ffffff, cr = (int)((unsigned)ccr >> 24);
      const AzIndex ix = az_index_of(sm, bv, surf);
      const int p1 = pb.pos[3 * v];
      if (surf) az_prepare_walk<true>(ix, pb.sel[v], pb.qa[v], p1, c, cr, sd2, sd3, min(sm.ns, sm.Ts), sm.nearf, w2, w3, B2, B3);
      else az_prepare_walk<false>(ix, pb.sel[v], pb.qa[v], p1, c, cr, sd2, sd3, min(sm.nc, sm.Tc), sm.nearf, w2, w3, B2, B3);
      pb.qw[v] = make_int4(lvl == -3 ? 2 : 1, w2, w3, ccr);  // (.x = 2: the walks' certificate failed; diagnostics only)
      reinterpret_cast<float2*>(pb.key)[v] = make_float2(B2, B3);
      if (sm.first_pass && (w2 & 0xffff) <= kThreadWalkBins && (w3 & 0xffff) <= kThreadWalkBins) pb.wl[NQ - 1 - atomicAdd(&cta.wl_tn[1], 1)] = v;
      else pb.wl[atomicAdd(&cta.wl_n[1], 1)] = v;
      if (bv.timers) atomicAdd(&cta.dbg[1], (w2 & 0xffff) + 4 * (w3 & 0xffff));
    }
    __syncthreads();
    if (bv.timers && threadIdx.x == 0) {
      atomicAdd((unsigned long long*)&bv.timers[11], (unsigned long long)cta.wl_n[1]);
      atomicAdd((unsigned long long*)&bv.timers[13], (unsigned long long)cta.dbg[1]);
    }
    // result of a query's walks -> its state + the correspondence IDs (one thread)
    auto walk_finish = [&](int v, const Smem& sm, int i, bool surf, const float4 s, int ccr, const WalkOut& wo) {
      float4 ex = pb.qext[v];  // (.y = the closest point's runner-up, written by P2 or kept from an earlier pass)
      if (bv.timers && pb.qw[v].x == 2) {  // did the stored front-runners hold every answer of the failed certificate?
        auto held = [](int w, int r, int now) { return w >= 0 ? now == w || now == r : now < 0; };
        if (held(pb.pos[3 * v + 1], __float_as_int(ex.z), wo.pos2) && (!surf || held(pb.pos[3 * v + 2], __float_as_int(ex.w), wo.pos3)))
          atomicAdd((unsigned long long*)&bv.timers[kCertSlots + 6], 1ull << 32);
      }
      pb.pos[3 * v + 1] = wo.pos2; pb.pos[3 * v + 2] = wo.pos3;
      pb.qref2[v] = make_float4(s.x, s.y, s.z, wo.bound2);
      ex.x = wo.bound3; ex.z = __int_as_float(wo.run2); ex.w = __int_as_float(wo.run3);
      pb.qext[v] = ex;
      const int i1 = ccr & 0x00ffffff;
      if (surf) { int* o = bv.ind_s + 3 * (size_t)(sm.qs0 + i); o[0] = i1; o[1] = wo.i2; o[2] = wo.i3; }
      else { int* o = bv.ind_c + 2 * (size_t)(sm.qc0 + i - sm.ns); o[0] = i1; o[1] = wo.i2; }
    };
    // P4, group-level list first.  :859 / :983 loop-bound quirk (+ OOB clamp): forward candidates count only below the
    // QUERY count
    for (;;) {
      int k = 0;
      if (sub == 0) k = atomicAdd(&cta.wl_thead[1], 1);
      k = __shfl_sync(gmask, k, glead);
      if (k >= cta.wl_tn[1]) break;
      const int v = pb.wl[NQ - 1 - k];
      const int sl = slot_of(v, Q), i = v - sl * Q;
      const Smem& sm = slots[sl];
      const int4 w = pb.qw[v];
      const bool surf = i < sm.ns;
      const float2 B = reinterpret_cast<const float2*>(pb.key)[v];
      const float4 s = pb.sel[v];
      const AzIndex ix = az_index_of(sm, bv, surf);
      const WalkOut wo = surf ? az_scan_walk_group<true, G>(ix, s, w.w, w.y, w.z, min(sm.ns, sm.Ts), sm.nearf, B.x, B.y, sub, gmask)
                              : az_scan_walk_group<false, G>(ix, s, w.w, w.y, w.z, min(sm.nc, sm.Tc), sm.nearf, B.x, B.y, sub, gmask);
      if (sub == 0) walk_finish(v, sm, i, surf, s, w.w, wo);
    }
    for (;;) {  // P4: same work-list scheme
      int k = 0;
      if (lane == 0) k = atomicAdd(&cta.wl_head[1], 1);
      k = __shfl_sync(0xffffffffu, k, 0);
      if (k >= cta.wl_n[1]) break;
      const int v = pb.wl[k];
      const int sl = slot_of(v, Q), i = v - sl * Q;
      const Smem& sm = slots[sl];
      const int4 w = pb.qw[v];
      const bool surf = i < sm.ns;
      const float2 B = reinterpret_cast<const float2*>(pb.key)[v];
      const int w2 = w.y, w3 = w.z;
      const float4 s = pb.sel[v];
      const AzIndex ix = az_index_of(sm, bv, surf);
      const WalkOut wo = surf ? az_scan_walk<true>(ix, s, w.w, w2, w3, min(sm.ns, sm.Ts), sm.nearf, B.x, B.y)
                              : az_scan_walk<false>(ix, s, w.w, w2, w3, min(sm.nc, sm.Tc), sm.nearf, B.x, B.y);
      if (lane == 0) walk_finish(v, sm, i, surf, s, w.w, wo);
    }
  }
  if (cta.any_legacy) {
    // ---- legacy: brute-force exact 1-NN + literal sequential walks, unit by unit ----------------------------------
    for (int sl = 0; sl < bv.nslots; ++sl) {
      const Smem& sm = slots[sl];
      if (!sm.run || sm.az_ok || !sm.search) continue;
      const bool sep = nn_separate(bv, sm.scan);
      const float4* __restrict__ nnS = sep ? bv.nn_s + bv.nn_s_off[sm.scan] : bv.ts + sm.ts0;
      const float4* __restrict__ nnC = sep ? bv.nn_c + bv.nn_c_off[sm.scan] : bv.tc + sm.tc0;
      const int TnS = sep ? bv.nn_s_off[sm.scan + 1] - bv.nn_s_off[sm.scan] : sm.Ts;
      const int TnC = sep ? bv.nn_c_off[sm.scan + 1] - bv.nn_c_off[sm.scan] : sm.Tc;
      if (sm.ns > 0 && TnS > 0) nn_brute(pb.sel + sl * Q, pb.key + sl * Q, sm.ns, nnS, TnS);
      if (sm.nc > 0 && TnC > 0) nn_brute(pb.sel + sl * Q + sm.ns, pb.key + sl * Q + sm.ns, sm.nc, nnC, TnC);
    }
    __syncthreads();
    for (int sl = 0; sl < bv.nslots; ++sl) {
      const Smem& sm = slots[sl];
      if (!sm.run || sm.az_ok || !sm.search) continue;
      const float4* __restrict__ tgtS = bv.ts + sm.ts0;
      const float4* __restrict__ tgtC = bv.tc + sm.tc0;
      const int fwdS = min(sm.ns, sm.Ts), fwdC = min(sm.nc, sm.Tc);
      for (int i = threadIdx.x; i < sm.ns + sm.nc; i += kThreads) {
        const int v = sl * Q + i;
        const bool surf = i < sm.ns;
        const unsigned long long k1 = pb.key[v];
        const float d1 = __uint_as_float((unsigned)(k1 >> 32));
        const int c = (int)(unsigned)(k1 & 0xffffffffu);
        const bool found = (k1 != kKeyMax) && ((double)d1 < sm.nearest_sq) && c < (surf ? sm.Ts : sm.Tc);
        int i1 = -1, i2 = -1, i3 = -1;
        if (found) {
          i1 = c;
          const float4 s = pb.sel[v];
          if (surf) walk_seq<true>(s, c, tgtS, sm.Ts, fwdS, sm.nearf, i2, i3);
          else walk_seq<false>(s, c, tgtC, sm.Tc, fwdC, sm.nearf, i2, i3);
        }
        pb.pos[3 * v] = i1; pb.pos[3 * v + 1] = i2; pb.pos[3 * v + 2] = i3;
        if (surf) { int* o = bv.ind_s + 3 * (size_t)(sm.qs0 + i); o[0] = i1; o[1] = i2; o[2] = i3; }
        else { int* o = bv.ind_c + 2 * (size_t)(sm.qc0 + i - sm.ns); o[0] = i1; o[1] = i2; }
      }
    }
  }
  __syncthreads();
  if (bv.timers && threadIdx.x == 0 && !cta.pass_first) {  // later passes by their number of walk searches
    const int n = cta.wl_n[1] + cta.wl_tn[1], b = n == 0 ? 0 : n <= 16 ? 1 : n <= 32 ? 2 : 3;
    atomicAdd((unsigned long long*)&bv.timers[kPassSlots + 6 + b], 1ull);
    atomicAdd((unsigned long long*)&bv.timers[kPassSlots + 10 + b], (unsigned long long)(clock64() - cta.tlast));
  }
  LINS_TICK_PASS(5);
  // the searches of this pass are over: reset the work lists for the next pass
  if (threadIdx.x == kThreads - 1) { cta.wl_n[0] = 0; cta.wl_n[1] = 0; cta.wl_tn[0] = 0; cta.wl_tn[1] = 0; cta.wl_head[0] = 0; cta.wl_head[1] = 0; cta.wl_thead[0] = 0; cta.wl_thead[1] = 0; cta.dbg[0] = 0; cta.dbg[1] = 0; }

  // ---- A5/A6 residuals + A7-A9 fold ------------------------------------------------------------------------------
  // tripod points: slots of the sorted copies after a fast-path search, otherwise original indices into the walk clouds.
  double* const fold_stage = cta.u.fold[warp];
  for (int v0 = warp * 32; v0 < NQ; v0 += kThreads) {
    const int sl = slot_of(v0, Q), i0 = v0 - sl * Q;
    const Smem& sm = slots[sl];
    const int ntot = sm.ns + sm.nc;
    if (!sm.run || i0 >= ntot) continue;  // (warp-uniform)
    const int v = v0 + lane, i = i0 + lane;
    const bool valid = i < ntot;
    const bool surf = i < sm.ns;
    const bool weighted = sm.weighted != 0;
    const bool by_slot = sm.search ? (sm.az_ok != 0) : (sm.pos_valid && sm.pos_is_slot);
    float4 coeff = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    bool ok = false;
    if (valid) {
      const int i1 = pb.pos[3 * v], i2 = pb.pos[3 * v + 1], i3 = pb.pos[3 * v + 2];
      s = pb.sel[v];
      if (surf) {
        if (i2 >= 0 && i3 >= 0 && i1 >= 0 && i1 < sm.Ts && i2 < sm.Ts && i3 < sm.Ts) {
          const float4* t = by_slot ? bv.az_s + sm.ts0 : bv.ts + sm.ts0;
          ok = plane_residual(s, t[i1], t[i2], t[i3], weighted, coeff);
        }
      } else {
        if (i2 >= 0 && i1 >= 0 && i1 < sm.Tc && i2 < sm.Tc) {
          const float4* t = by_slot ? bv.az_c + sm.tc0 : bv.tc + sm.tc0;
          ok = line_residual(s, t[i1], t[i2], weighted, coeff);
        }
      }
    }
    double g[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, r = 0.0;
    if (ok) {
      if (MODE == MODE_ICP_REDUCE) jacobian_row_icp(pb.qpt[v], coeff, sm.phi, sm.period, g, r);
      else jacobian_row(pb.qpt[v], coeff, sm.R, sm.lidar_scale, g, r);
    }
    const int vw = sl * pb.nvw + (i0 >> 5);
    warp_fold_mma(g, r, fold_stage, pb.wacc + vw * kNAcc);
    const unsigned mS = __ballot_sync(0xffffffffu, ok && surf), mC = __ballot_sync(0xffffffffu, ok && !surf);
    if (lane == kNAcc) pb.wcnt[vw * 2] = __popc(mS);
    else if (lane == kNAcc + 1) pb.wcnt[vw * 2 + 1] = __popc(mC);
    if (MODE == MODE_ASSOC && valid) {
      if (surf) {
        const size_t o = (size_t)(sm.qs0 + i);
        if (bv.sel_s) { bv.sel_s[3 * o] = s.x; bv.sel_s[3 * o + 1] = s.y; bv.sel_s[3 * o + 2] = s.z; }
        if (bv.coeff_s) { bv.coeff_s[4 * o] = coeff.x; bv.coeff_s[4 * o + 1] = coeff.y; bv.coeff_s[4 * o + 2] = coeff.z; bv.coeff_s[4 * o + 3] = coeff.w; }
        if (bv.mask_s) bv.mask_s[o] = ok ? 1 : 0;
      } else {
        const size_t o = (size_t)(sm.qc0 + i - sm.ns);
        if (bv.sel_c) { bv.sel_c[3 * o] = s.x; bv.sel_c[3 * o + 1] = s.y; bv.sel_c[3 * o + 2] = s.z; }
        if (bv.coeff_c) { bv.coeff_c[4 * o] = coeff.x; bv.coeff_c[4 * o + 1] = coeff.y; bv.coeff_c[4 * o + 2] = coeff.z; bv.coeff_c[4 * o + 3] = coeff.w; }
        if (bv.mask_c) bv.mask_c[o] = ok ? 1 : 0;
      }
    }
  }
  __syncthreads();
  LINS_TICK_PASS(6);
}

}  // namespace lins_dev
