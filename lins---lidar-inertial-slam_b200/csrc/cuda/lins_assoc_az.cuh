// Association through a (ring, azimuth-bin) index — the fast path of rows A3/A4 (exact 1-NN + ring walks,
// reference lins/include/StateEstimator.hpp:844-915 and :970-1029).
//
// Per scan, once: the target cloud (ring-sorted, as the reference's extractFeatures emits it, :727-826) is
// bucket-sorted on device by  ring * nb + azimuth_bin  into a packed copy (x, y, z, ring << 24 | original index) in
// global memory (served from L1 / L2: a unit's copy is ~80 KB and only the slices inside a search window are
// touched); the bucket table lives in shared memory (16-bit slots).  This replaces
// pcl::KdTreeFLANN::setInputCloud (:363-364, :1158-1159).
//
// Per query, per iteration, one warp:
//   every search is "the minimum of the exact f32 distance over a set of rings", and always comes with an upper
//   bound U on that minimum (the distance to the previous iteration's answer while it is still an admissible
//   candidate, else the 5 m gate NEAREST_FEATURE_SEARCH_SQ_DIST, which bounds every answer the reference can
//   accept).  A target whose azimuth differs from the query's by D is at least rho_q * sin(min(D, pi/2)) away
//   (rho_q = the query's distance from the z axis), so only the bins within
//        asin(1.002 * sqrt(U) / rho_q) + 1e-5 rad          (the whole ring if sqrt(U) >= rho_q)
//   of the query's azimuth can hold the minimum (or tie with it).  Those bins are one or two contiguous slices
//   of the sorted copy per ring.  Keys are (distance bits, order) u64 exactly as in the plain walk, so ties
//   resolve like the reference's "first strictly smaller wins" loops; the 1-NN key is (distance bits, original
//   index): lowest index among exact ties.
//
// Certificates.  Every search also returns its two front-runners (winner and runner-up slots) and a bound: the
// distance every OTHER candidate exceeded at the search position (the third best distance, or the distance bound of
// everything outside the window, whichever is smaller).  Later, one thread re-evaluates the two front-runners exactly;
// if the better of them (exact keys) is inside the gate and closer than bound - displacement (true distances change by
// at most the displacement), nothing else can have overtaken it: it is the answer — the stored winner, or the runner-up
// when the two swapped — and the search is skipped (cert_check).  A plain winner / runner-up margin cannot certify a
// query that sits almost midway between two neighbouring points of a ring — the common case; this can, on either side
// of the midpoint.  Three-way exact ties fail the test and are re-searched.  A search that found nothing within the gate keeps a plain slack
// (cert_rejected).  Windows are built for sqrt(U) + kCertMargin so the "outside" bound is not vacuous.  The closest
// point and the walks are certified separately (a new closest point always forces new walks).
#pragma once
#include "lins_kernels.cuh"

namespace lins_dev {

struct AzIndex {
  const float4* pts;      // sorted copy (global)
  const aztab_t* bstart;  // [nrings * nb + 1], shared
  const int (*elev)[2];   // per ring: [min, max] slope z / rho_xy of its targets (float_key), shared
  int nb, nrings, T;
};
// order-preserving float <-> int key (so that atomicMin / atomicMax on ints order floats)
__device__ __forceinline__ int float_key(float f) { const int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float key_float(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }
// "Elevation" of a point as the slope z / rho_xy of its ray in the (rho_xy, z) half plane (monotonic in the elevation angle;
// no atan2f).  rho_xy == 0 gives +-inf / NaN: az_build then marks the ring's band as unbounded.
__device__ __forceinline__ float slope_of(float x, float y, float z) {
  return __fdiv_rn(z, sqrtf(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))));
}
// Lower bound (m) on the distance from a query (rho_xy = rq, z = zq) to ANY point whose slope lies in the ring's band
// [lo, hi].  The 3-D distance is at least the distance in the (rho_xy, z) half plane; there a target of slope m lies on the
// ray t * (1, m), t >= 0, the distance from the query to a ray grows with the angle between them, and the distance to the
// ray at the band's nearer edge m* is at least the distance to its line, |zq - m* rq| / sqrt(1 + m*^2).  0.998 and 1e-4 m
// absorb the f32 rounding (slopes: 2 ulp -> < 2e-7 rad; the cancellation in zq - m rq: < 1e-5 m at 100 m).  An unbounded
// band (hi - lo not finite), an overflow or a NaN anywhere makes the comparison `bound > B` false: the ring is scanned.
__device__ __forceinline__ float ring_lower_bound(const AzIndex& ix, int r, float zq, float rq) {
  const float lo = key_float(ix.elev[r][0]), hi = key_float(ix.elev[r][1]);
  const float a = __fmaf_rn(lo, rq, -zq), b = __fmaf_rn(-hi, rq, zq);  // > 0: the query lies below / above the band
  const float m = a > b ? lo : hi;
  const float bound = fmaxf(a, b) * rsqrtf(__fmaf_rn(m, m, 1.f)) * 0.998f - 1.0e-4f;
  return hi - lo < 1.0e30f ? bound : -1.f;
}

__device__ __forceinline__ int az_bin(float x, float y, int nb) {
  const float a = atan2f(y, x);
  int b = (int)floorf((a + kPiF) * ((float)nb * (0.5f / kPiF)));
  return min(max(b, 0), nb - 1);
}
// bins per ring for a table of TAB entries
__device__ __forceinline__ int az_bins_for(int nrings, int tab) {
  int p2 = 1;
  while (p2 < nrings) p2 <<= 1;
  return tab / p2;
}

// Counting-sort counters / cursors, two 16-bit halves per 32-bit word (bucket b = half b & 1 of word b >> 1): every count
// and every cursor is at most T < 65536, so a half never carries into its neighbour.  Half the scratch of 32-bit counters
// keeps a CTA's shared memory under the 196 KB carve-out, which leaves the SM twice the L1 (see lins_kernels.cuh, CtaMem).
__device__ __forceinline__ int cnt16_add1(unsigned* cnt, int b) {  // atomic ++ of half b; returns its old value
  const int sh = (b & 1) * 16;
  return (int)((atomicAdd(&cnt[b >> 1], 1u << sh) >> sh) & 0xffffu);
}
// counting sort of `src` (ring-sorted, rings validated by check_ring_sorted, T < 65536) into dst; bucket starts ->
// table[0..TAB].  cnt (TAB / 2 + 1 packed words, cnt16_add1) and scan_tmp (kThreads ints) are CTA scratch.  Block-wide.
template <int TAB>
__device__ void az_build(const float4* __restrict__ src, int T, float4* dst, aztab_t* table, unsigned* cnt, int* scan_tmp, int nb, int (*elev)[2]) {
  unsigned short* cnt16 = reinterpret_cast<unsigned short*>(cnt);  // (plain reads / writes of the halves between barriers)
  for (int w = threadIdx.x; w <= TAB / 2; w += kThreads) cnt[w] = 0u;
  for (int r = threadIdx.x; r < kMaxRing; r += kThreads) { elev[r][0] = float_key(3.0e38f); elev[r][1] = float_key(-3.0e38f); }
  __syncthreads();
  for (int j = threadIdx.x; j < T; j += kThreads) {
    const float4 t = __ldg(&src[j]);
    cnt16_add1(cnt, (int)t.w * nb + az_bin(t.x, t.y, nb));
    const float e = slope_of(t.x, t.y, t.z);
    if (fabsf(e) < 1.0e30f) { const int k = float_key(e); atomicMin(&elev[(int)t.w][0], k); atomicMax(&elev[(int)t.w][1], k); }
    else { atomicMin(&elev[(int)t.w][0], float_key(-3.0e38f)); atomicMax(&elev[(int)t.w][1], float_key(3.0e38f)); }  // (on the z axis / NaN: never skip its ring)
  }
  __syncthreads();
  constexpr int PER = TAB / kThreads;
  static_assert(PER >= 1 && PER * kThreads == TAB, "table size must be a multiple of the block size");
  int loc[PER];
  int sum = 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) { loc[k] = cnt16[threadIdx.x * PER + k]; sum += loc[k]; }
  scan_tmp[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x < 32) {
    constexpr int PW = kThreads / 32;
    int part[PW];
    int s = 0;
#pragma unroll
    for (int k = 0; k < PW; ++k) { part[k] = scan_tmp[threadIdx.x * PW + k]; s += part[k]; }
    int incl = s;
#pragma unroll
    for (int m = 1; m < 32; m <<= 1) { const int o = __shfl_up_sync(0xffffffffu, incl, m); if ((int)threadIdx.x >= m) incl += o; }
    int run = incl - s;
#pragma unroll
    for (int k = 0; k < PW; ++k) { const int v = part[k]; scan_tmp[threadIdx.x * PW + k] = run; run += v; }
    if (threadIdx.x == 31) table[TAB] = (aztab_t)incl;
  }
  __syncthreads();
  {
    int run = scan_tmp[threadIdx.x];
#pragma unroll
    for (int k = 0; k < PER; ++k) { cnt16[threadIdx.x * PER + k] = (unsigned short)run; table[threadIdx.x * PER + k] = (aztab_t)run; run += loc[k]; }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < T; j += kThreads) {  // scatter; the counters are the cursors now
    const float4 t = __ldg(&src[j]);
    const int pos = cnt16_add1(cnt, (int)t.w * nb + az_bin(t.x, t.y, nb));
    dst[pos] = make_float4(t.x, t.y, t.z, __int_as_float(((int)t.w << 24) | j));  // ring (7 bits) | original index (24 bits)
  }
  __syncthreads();
}

// half-width (rad) of the azimuth window that can hold a target with squared distance <= U
__device__ __forceinline__ float az_halfwidth(float U, float rho) {
  const float r = sqrtf(U) * 1.002f + 1.0e-5f;
  if (!(r < rho)) return 4.0f;  // > pi: the whole ring
  return asinf(r / rho) + 1.0e-5f;
}
// bins [blo, blo + nbins) (mod nb) covering [aq - th, aq + th] plus one spare bin on each side
__device__ __forceinline__ void az_window(int nb, float aq, float th, int& blo, int& nbins) {
  const float inv_binw = (float)nb * (0.5f / kPiF);
  nbins = (int)(2.0f * th * inv_binw) + 3;
  if (!(th < kPiF) || nbins >= nb) { blo = 0; nbins = nb; return; }
  int b = (int)floorf((aq - th + kPiF) * inv_binw) - 1;
  b %= nb;
  if (b < 0) b += nb;
  blo = b;
}

__device__ __forceinline__ int slot_index(float w) { return __float_as_int(w) & 0x00ffffff; }
__device__ __forceinline__ int slot_ring(float w) { return (int)((unsigned)__float_as_int(w) >> 24); }
__device__ __forceinline__ int pack_window(int blo, int nbins) { return (blo << 16) | nbins; }
constexpr float kCertMargin = 0.1f;  // metres added to every search radius so that certificates have room
// bound used to build a window: (sqrt(U) + margin)^2
__device__ __forceinline__ float widen(float U) { const float r = sqrtf(U) + kCertMargin; return r * r; }
// slack (metres) of a search that found nothing within the gate: how far its best candidate (f32 squared-distance
// BITS, 0xffffffff = none) or everything not examined (Bout) lies beyond gate = sqrt(NEAREST_FEATURE_SEARCH_SQ_DIST).
// Negative = cannot be certified.
__device__ __forceinline__ float rejected_slack(unsigned best_bits, float Bout, float gate) {
  const float db = best_bits >= 0x7f800000u ? Bout : fminf(sqrtf(__uint_as_float(best_bits)), Bout);
  return db - gate * 1.00001f;
}

// ---- phase P1 (one THREAD per query): azimuth, range, bound and window of the closest-point search ------------
// qa = (azimuth, rho, -, outside bound B1); returns the packed window or -1 when the query cannot match anything
__device__ __forceinline__ void az_polar(const float4 s, float4& qa) {
  qa.x = atan2f(s.y, s.x);
  qa.y = sqrtf(__fadd_rn(__fmul_rn(s.x, s.x), __fmul_rn(s.y, s.y)));
}
// window of the closest-point search given an upper bound U1 on its answer (the gate, or the distance to any real
// target); qa.w <- distance bound of everything outside the window
__device__ __forceinline__ int az_nn_window(const AzIndex& ix, float U1, float4& qa) {
  const float Uw = widen(U1);
  int blo, nbins;
  az_window(ix.nb, qa.x, az_halfwidth(Uw, qa.y), blo, nbins);
  qa.w = nbins >= ix.nb ? 3.0e38f : sqrtf(Uw);
  return pack_window(blo, nbins);
}
__device__ __forceinline__ float az_seed_bound(const AzIndex& ix, const float4 s, int seed_slot, float U1) {
  if (seed_slot >= 0 && seed_slot < ix.T) {
    const float4 t = ix.pts[seed_slot];
    const float d = sqdist_f32(s.x, s.y, s.z, t.x, t.y, t.z);
    if (d < U1) U1 = d;
  }
  return U1;
}
__device__ __forceinline__ int az_bin_of_angle(float a, int nb) {
  const int b = (int)floorf((a + kPiF) * ((float)nb * (0.5f / kPiF)));
  return min(max(b, 0), nb - 1);
}
// Unseeded query (a unit's first pass): bound from a few real targets next to the query in the index — the buckets
// around the query's azimuth on the ring the query itself was measured on (ring_guess = int(intensity) of the raw query;
// the last scan has the same rings), then on the two adjacent rings when that found nothing within a metre.  Any real
// target's distance is a valid upper bound on the minimum, so this only narrows the window (exactness is untouched).
__device__ __forceinline__ float az_bucket_bound(const AzIndex& ix, const float4 s, float az, int ring_guess, float U1) {
  const int bq = az_bin_of_angle(az, ix.nb);
  const int r0 = min(max(ring_guess, 0), ix.nrings - 1);
#pragma unroll 1
  for (int k = 0; k < 3; ++k) {
    const int r = k == 0 ? r0 : (k == 1 ? r0 - 1 : r0 + 1);
    if (k == 1 && U1 < 1.0f) break;
    if (r < 0 || r >= ix.nrings) continue;
    const int base = r * ix.nb;
    int p = ix.bstart[base + max(bq - 1, 0)];
    const int pe = min((int)ix.bstart[base + min(bq + 2, ix.nb)], p + 4);
    for (; p < pe; ++p) U1 = az_seed_bound(ix, s, p, U1);
  }
  return U1;
}
__device__ __forceinline__ int az_prepare_nn(const AzIndex& ix, const float4 s, float nearf, int seed_slot, int ring_guess, float4& qa) {
  qa = make_float4(0.f, 0.f, -1.f, 0.f);
  if (!(s.x == s.x && s.y == s.y && s.z == s.z) || ix.T <= 0) return -1;
  az_polar(s, qa);
  // nothing beyond the gate can be accepted (StateEstimator.hpp:851)
  float U1 = az_seed_bound(ix, s, seed_slot, nearf);
  if (seed_slot < 0) U1 = az_bucket_bound(ix, s, qa.x, ring_guess, U1);
  return az_nn_window(ix, U1, qa);
}
// Probe radius: a search whose window (built from the gate, i.e. without a usable previous answer) is much wider
// than the window of this radius first scans the small window; the best candidate found there is a real target,
// so its distance is a valid upper bound and the exact search runs inside the (much smaller) window it implies.
constexpr float kProbeSq = 0.25f;  // (0.5 m)^2
__device__ __forceinline__ int az_probe_window(const AzIndex& ix, const float4 qa, int full_window) {
  int blo, nbins;
  az_window(ix.nb, qa.x, az_halfwidth(kProbeSq, qa.y), blo, nbins);
  return (full_window & 0xffff) > 2 * nbins + 4 ? pack_window(blo, nbins) : -1;
}

// ---- phase P2 (one WARP per query): exact 1-NN over all rings inside the window ---------------------------------
// LPR lanes share one ring; four candidates per lane are in flight per trip.  A lone warp runs these scans with
// nothing to hide latency behind, so the bookkeeping is branch-free straight-line code.
// The two smallest keys seen so far with their slots, and the distance bits of the third.  Certificates built on the
// third distance survive a near-tie between the two front-runners (the common reason an answer could not be certified:
// a query almost equidistant from two neighbouring points of a ring): those two are simply re-evaluated exactly.
struct Top3 {
  unsigned long long k1, k2;
  int p1, p2;
  unsigned d3;
  __device__ __forceinline__ void init() { k1 = kKeyMax; k2 = kKeyMax; p1 = -1; p2 = -1; d3 = 0xffffffffu; }
  __device__ __forceinline__ void insert(unsigned long long k, int p) {  // branch-free; kKeyMax changes nothing
    const bool lt1 = k < k1, lt2 = k < k2;
    d3 = lt2 ? (unsigned)(k2 >> 32) : min(d3, (unsigned)(k >> 32));
    k2 = lt1 ? k1 : (lt2 ? k : k2);
    p2 = lt1 ? p1 : (lt2 ? p : p2);
    k1 = lt1 ? k : k1;
    p1 = lt1 ? p : p1;
  }
};
__device__ __forceinline__ int warp_argmin_lane(unsigned long long k, unsigned long long& kmin) {
  const unsigned hi = (unsigned)(k >> 32), lo = (unsigned)(k & 0xffffffffu);
  const unsigned mhi = __reduce_min_sync(0xffffffffu, hi);
  const unsigned mlo = __reduce_min_sync(0xffffffffu, hi == mhi ? lo : 0xffffffffu);
  kmin = ((unsigned long long)mhi << 32) | mlo;
  return __ffs(__ballot_sync(0xffffffffu, hi == mhi && lo == mlo)) - 1;
}
// warp-wide top 3 of the lanes' Top3 (every lane receives the result)
__device__ __forceinline__ void warp_top3(Top3& t) {
  const int lane = threadIdx.x & 31;
  unsigned long long K1, K2;
  const int a = warp_argmin_lane(t.k1, K1);
  const int P1 = __shfl_sync(0xffffffffu, t.p1, a);
  const unsigned long long cand = lane == a ? t.k2 : t.k1;
  const int candp = lane == a ? t.p2 : t.p1;
  const int b = warp_argmin_lane(cand, K2);
  const int P2 = __shfl_sync(0xffffffffu, candp, b);
  // the best entry each lane has left after the two front-runners were taken
  unsigned rest;
  if (lane == a && lane == b) rest = t.d3;
  else if (lane == a || lane == b) rest = (unsigned)(t.k2 >> 32);
  else rest = (unsigned)(t.k1 >> 32);
  t.d3 = __reduce_min_sync(0xffffffffu, rest);
  t.k1 = K1; t.p1 = K1 == kKeyMax ? -1 : P1;
  t.k2 = K2; t.p2 = K2 == kKeyMax ? -1 : P2;
}
// distance (m) that every candidate other than the two front-runners exceeded at the search position
__device__ __forceinline__ float cert_bound(unsigned third_bits, float Bout) {
  return third_bits >= 0x7f800000u ? Bout : fminf(sqrtf(__uint_as_float(third_bits)), Bout);
}
__device__ __forceinline__ float4 ld_slot(const AzIndex& ix, int p) { return ix.pts[p]; }
template <int LPR>
__device__ __forceinline__ void az_scan_nn_slice(const AzIndex& ix, const float4 s, int p, int pe, Top3& top) {
  for (; p < pe; p += 4 * LPR) {
    unsigned long long k[4];
    int q[4];
    float4 tt[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) tt[u] = ld_slot(ix, p + u * LPR < pe ? p + u * LPR : p);  // four loads in flight
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int pu = p + u * LPR;
      const bool valid = pu < pe;
      const float4 t = tt[u];
      const unsigned d = __float_as_uint(sqdist_f32(s.x, s.y, s.z, t.x, t.y, t.z));
      k[u] = valid ? (((unsigned long long)d << 32) | (unsigned)slot_index(t.w)) : kKeyMax;  // (kKeyMax never wins and never lowers a runner-up)
      q[u] = pu;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) top.insert(k[u], q[u]);
  }
}
// Bout = the distance bound of everything outside the search (sqrt of the widened radius the window was built for): a ring
// whose elevation band is farther than that from the query cannot hold the minimum or tie with it, like a bin outside the
// azimuth window.
template <int LPR>
__device__ __forceinline__ Top3 az_scan_nn_t(const AzIndex& ix, const float4 s, int win, float rq, float Bout, long long* tm = nullptr) {
  const int lane = threadIdx.x & 31;
  const int blo = win >> 16, nbins = win & 0xffff;
  constexpr int RPP = 32 / LPR;
  const int sub = lane % LPR;
  Top3 top;
  top.init();
  const int e0 = min(blo + nbins, ix.nb), e1 = blo + nbins - ix.nb;
  int dbg_cand = 0;
  for (int rbase = 0; rbase < ix.nrings; rbase += RPP) {
    const int r = rbase + lane / LPR;
    if (r < ix.nrings && !(ring_lower_bound(ix, r, s.z, rq) > Bout)) {
      const int base = r * ix.nb;
      if (tm) { dbg_cand += max(0, (ix.bstart[base + e0] - ix.bstart[base + blo] - sub + LPR - 1) / LPR); if (e1 > 0) dbg_cand += max(0, (ix.bstart[base + e1] - ix.bstart[base] - sub + LPR - 1) / LPR); }
      az_scan_nn_slice<LPR>(ix, s, ix.bstart[base + blo] + sub, ix.bstart[base + e0], top);
      if (e1 > 0) az_scan_nn_slice<LPR>(ix, s, ix.bstart[base] + sub, ix.bstart[base + e1], top);
    }
  }
  if (tm) { tm[0] = clock64(); tm[2] = __reduce_max_sync(0xffffffffu, (unsigned)dbg_cand); tm[3] = __reduce_add_sync(0xffffffffu, (unsigned)dbg_cand); }
  warp_top3(top);
  if ((unsigned)(top.k1 >> 32) >= 0x7f800000u) { top.k1 = kKeyMax; top.p1 = -1; }  // only inf / NaN distances: nothing found
  if (tm) tm[1] = clock64();
  return top;
}
// -> the two nearest (key, slot) pairs and the third distance, over every ring inside the window
__device__ __forceinline__ Top3 az_scan_nn(const AzIndex& ix, const float4 s, int win, float rq, float Bout, long long* tm = nullptr) {
  if (ix.nrings <= 8) return az_scan_nn_t<4>(ix, s, win, rq, Bout, tm);
  if (ix.nrings <= 16) return az_scan_nn_t<2>(ix, s, win, rq, Bout, tm);
  return az_scan_nn_t<1>(ix, s, win, rq, Bout, tm);
}

// A GROUP of G lanes per query (G = 4: eight queries per warp): the same scans for small windows.  A warp per query
// spends most of its lanes on empty slices and its instructions on warp-wide bookkeeping when a window holds a few dozen
// candidates; with G lanes per query the rings are dealt round-robin to the lanes, every lane keeps its own Top3 and a
// log2(G)-step butterfly merges them.  Keys are unique ((distance, index) / (distance, visiting order)), so the two
// front-runners and the third distance of a set of candidates do not depend on who visits what in which order: results
// are identical to the warp scan by construction.
template <int G>
__device__ __forceinline__ void group_top3(Top3& t, unsigned gmask) {
#pragma unroll
  for (int m = 1; m < G; m <<= 1) {
    const unsigned long long ok1 = __shfl_xor_sync(gmask, t.k1, m), ok2 = __shfl_xor_sync(gmask, t.k2, m);
    const int op1 = __shfl_xor_sync(gmask, t.p1, m), op2 = __shfl_xor_sync(gmask, t.p2, m);
    const unsigned od3 = __shfl_xor_sync(gmask, t.d3, m);
    t.insert(ok1, op1);  // (the partner's candidates are disjoint from this lane's; kKeyMax entries change nothing)
    t.insert(ok2, op2);
    t.d3 = min(t.d3, od3);
  }
}
// one lane over the slots p, p + step, ... < pe (two loads in flight)
__device__ __forceinline__ void az_scan_slice_lane(const AzIndex& ix, const float4 s, int p, int pe, int step, Top3& top) {
  for (; p < pe; p += 2 * step) {
    const int p1 = p + step;
    const float4 t0 = ld_slot(ix, p), t1 = ld_slot(ix, p1 < pe ? p1 : p);
    const unsigned d0 = __float_as_uint(sqdist_f32(s.x, s.y, s.z, t0.x, t0.y, t0.z));
    const unsigned d1 = __float_as_uint(sqdist_f32(s.x, s.y, s.z, t1.x, t1.y, t1.z));
    top.insert(((unsigned long long)d0 << 32) | (unsigned)slot_index(t0.w), p);
    top.insert(p1 < pe ? (((unsigned long long)d1 << 32) | (unsigned)slot_index(t1.w)) : kKeyMax, p1);
  }
}
template <int G>
__device__ __forceinline__ Top3 az_scan_nn_group(const AzIndex& ix, const float4 s, int win, float rq, float Bout, int sub, unsigned gmask) {
  const int blo = win >> 16, nbins = win & 0xffff;
  const int e0 = min(blo + nbins, ix.nb), e1 = blo + nbins - ix.nb;
  Top3 top;
  top.init();
  for (int r = sub; r < ix.nrings; r += G) {  // rings dealt round-robin to the lanes of the group
    if (ring_lower_bound(ix, r, s.z, rq) > Bout) continue;  // (elevation band out of reach, see az_scan_nn_t)
    const int base = r * ix.nb;
    az_scan_slice_lane(ix, s, ix.bstart[base + blo], ix.bstart[base + e0], 1, top);
    if (e1 > 0) az_scan_slice_lane(ix, s, ix.bstart[base], ix.bstart[base + e1], 1, top);
  }
  group_top3<G>(top, gmask);
  if ((unsigned)(top.k1 >> 32) >= 0x7f800000u) { top.k1 = kKeyMax; top.p1 = -1; }  // only inf / NaN distances: nothing found
  return top;
}

// ---- phase P3 (one THREAD per query): bound + window the walks of a query whose closest point is (c, cr) -------
// w2 / w3 = windows of the Ind2 / Ind3 searches, B2 / B3 = distance bound of everything outside them
// bound from a candidate target while it is an admissible candidate of THIS search (CLS2: the Ind2 search)
template <bool SURF, bool CLS2>
__device__ __forceinline__ float seed_bound(const float4 t, bool valid, const float4 s, int c, int cr, int fwdBound, float U) {
  const int j = slot_index(t.w), r = slot_ring(t.w);
  const bool ring_ok = (SURF && CLS2) ? (r == cr) : (r != cr && r >= cr - 2 && r <= cr + 2);
  const float d = sqdist_f32(t.x, t.y, t.z, s.x, s.y, s.z);
  return (valid && ring_ok && j != c && (j < c || j < fwdBound) && d < U) ? d : U;
}
// Uinit = NEAREST_FEATURE_SEARCH_SQ_DIST: nothing beyond the gate is accepted
template <bool SURF>
__device__ __forceinline__ void az_prepare_walk(const AzIndex& ix, const float4 s, const float4 qa, int p1, int c, int cr, int seed2,
                                                int seed3, int fwdBound, float Uinit, int& w2, int& w3, float& B2, float& B3) {
  // Bounds from the previous answers and from the index neighbourhood of the closest point / of the query's azimuth on
  // the adjacent rings.  Each is used only while it is an admissible candidate of the search it bounds (seed_bound), so
  // the windows shrink (a unit's first pass has no previous answers: gate-wide windows otherwise) and exactness is
  // untouched.  The look-ups are independent: all loads of a batch are issued before the first is used (one L2 round
  // trip per batch instead of one per seed).
  auto fetch = [&](int seed, bool& valid) -> float4 {
    valid = seed >= 0 && seed < ix.T;
    return valid ? ix.pts[seed] : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  float U2 = Uinit, U3 = Uinit;
  {
    constexpr int NA = SURF ? 6 : 1;
    const int seeds[6] = {seed2, seed3, p1 - 2, p1 - 1, p1 + 1, p1 + 2};
    float4 t[NA];
    bool ok[NA];
#pragma unroll
    for (int k = 0; k < NA; ++k) t[k] = fetch(seeds[k], ok[k]);
    U2 = seed_bound<SURF, true>(t[0], ok[0], s, c, cr, fwdBound, U2);
    if (SURF) {
      U3 = seed_bound<SURF, false>(t[1 % NA], ok[1 % NA], s, c, cr, fwdBound, U3);
#pragma unroll
      for (int k = 2; k < NA; ++k) U2 = seed_bound<true, true>(t[k], ok[k], s, c, cr, fwdBound, U2);
    }
  }
  {
    const int bq = az_bin_of_angle(qa.x, ix.nb);
    float& U = SURF ? U3 : U2;
    float4 t[8];
    bool ok[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int r = cr + (k < 2 ? k - 2 : k - 1);
      const bool rok = r >= 0 && r < ix.nrings;
      const int slot = rok ? (int)ix.bstart[r * ix.nb + bq] : -1;
      t[2 * k] = fetch(slot, ok[2 * k]);
      t[2 * k + 1] = fetch(rok ? slot - 1 : -1, ok[2 * k + 1]);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) U = seed_bound<SURF, !SURF>(t[k], ok[k], s, c, cr, fwdBound, U);
  }
  int blo, nbins;
  const float Uw2 = widen(U2);
  az_window(ix.nb, qa.x, az_halfwidth(Uw2, qa.y), blo, nbins);
  w2 = pack_window(blo, nbins);
  B2 = nbins >= ix.nb ? 3.0e38f : sqrtf(Uw2);
  if (SURF) {
    const float Uw3 = widen(U3);
    az_window(ix.nb, qa.x, az_halfwidth(Uw3, qa.y), blo, nbins);
    w3 = pack_window(blo, nbins);
    B3 = nbins >= ix.nb ? 3.0e38f : sqrtf(Uw3);
  } else { w3 = w2; B3 = B2; }
}

// ---- phase P4 (one WARP per query): the ring walks inside their windows -------------------------------------------
// SURF: Ind2 over ring cr (window w2), Ind3 over rings cr-2, cr-1, cr+1, cr+2 (window w3).  Corner: Ind2 over rings
// cr-2, cr-1, cr+1, cr+2 (window w2).  Forward candidates (original index j > c) count only while j < fwdBound.
constexpr int kWalkInFlight = 4;
constexpr int kGroupWalkInFlight = 4;
struct WalkOut {  // per class: original index (-1 = none within the gate), slot, certificate bound, runner-up slot
  int i2, i3, pos2, pos3, run2, run3;
  float bound2, bound3;
};
template <bool SURF>
__device__ __forceinline__ WalkOut az_scan_walk(const AzIndex& ix, const float4 s, int ccr, int w2, int w3, int fwdBound, float nearf,
                                                float B2, float B3) {
  const int lane = threadIdx.x & 31;
  const int c = ccr & 0x00ffffff, cr = (int)((unsigned)ccr >> 24);
  // keys are NOT gated here: the minimum over the candidates is needed even when it lies beyond the gate (to certify
  // "still nothing within the gate"); the gate is applied to the reduced winner, which is equivalent to the
  // reference's `pointSqDis < minPointSqDis` starting from NEAREST_FEATURE_SEARCH_SQ_DIST.
  // a lane serves one ring, hence one class: it keeps a single Top3
  Top3 top;
  top.init();
  // lanes <-> rings.  SURF: the four adjacent rings (window w3, some 40 candidates each) get 7 lanes each, the closest
  // point's own ring (window w2, a handful) the last 4; corner: 8 lanes for each of the four adjacent rings.
  constexpr int LPR = SURF ? 7 : 8;
  const int q = lane / LPR;
  const bool own = SURF && q >= 4;
  const int r = own ? cr : cr + (q < 2 ? q - 2 : q - 1);
  const int sub = own ? lane - 4 * LPR : lane - q * LPR, step = own ? 4 : LPR;
  const bool cls2 = SURF ? own : true;
  if (r >= 0 && r < ix.nrings) {
    const int win = cls2 ? w2 : w3;
    const int blo = win >> 16, nbins = win & 0xffff, base = r * ix.nb;
    for (int seg = 0; seg < 2; ++seg) {
      int p, pe;
      if (seg == 0) { p = ix.bstart[base + blo]; pe = ix.bstart[base + min(blo + nbins, ix.nb)]; }
      else { const int e1 = blo + nbins - ix.nb; if (e1 <= 0) break; p = ix.bstart[base]; pe = ix.bstart[base + e1]; }
      for (p += sub; p < pe; p += kWalkInFlight * step) {  // kWalkInFlight candidates in flight per lane
        float4 tt[kWalkInFlight];
#pragma unroll
        for (int u = 0; u < kWalkInFlight; ++u) tt[u] = ld_slot(ix, p + step * u < pe ? p + step * u : p);
#pragma unroll
        for (int u = 0; u < kWalkInFlight; ++u) {
          const int pu = p + step * u;
          const float4 t = tt[u];
          const unsigned d = __float_as_uint(sqdist_f32(t.x, t.y, t.z, s.x, s.y, s.z));
          const int j = slot_index(t.w);
          const bool fwd = j > c;
          const bool adm = pu < pe && j != c && (!fwd || j < fwdBound);
          const unsigned long long k = adm ? (((unsigned long long)d << 32) | (fwd ? order_fwd(j) : order_bwd(j))) : kKeyMax;
          top.insert(k, pu);
        }
      }
    }
  }
  const float gate = sqrtf(nearf);
  const unsigned nearbits = __float_as_uint(nearf);
  const bool mine2 = cls2;
  Top3 neutral;
  neutral.init();
  WalkOut o;
  // accepted (within the gate): bound = distance everything but the two front-runners exceeded; otherwise the slack
  // of "still nothing within the gate" (rejected_slack)
  auto finish = [&](Top3 t, float Bout, int& idx, int& pos, int& run, float& bound) {
    warp_top3(t);
    const bool ok = (unsigned)(t.k1 >> 32) < nearbits && t.p1 >= 0;
    idx = ok ? order_decode((unsigned)(t.k1 & 0xffffffffu)) : -1;
    pos = ok ? t.p1 : -1;
    run = ok ? t.p2 : -1;
    bound = ok ? cert_bound(t.d3, Bout) : rejected_slack((unsigned)(t.k1 >> 32), Bout, gate);
  };
  finish(mine2 ? top : neutral, B2, o.i2, o.pos2, o.run2, o.bound2);
  if (SURF) finish(mine2 ? neutral : top, B3, o.i3, o.pos3, o.run3, o.bound3);
  else { o.i3 = -1; o.pos3 = -1; o.run3 = -1; o.bound3 = 0.f; }
  return o;
}

// the same walks by a group of G lanes (see az_scan_nn_group): the four adjacent rings are dealt to the lanes, the
// closest point's own ring (a handful of candidates) is strided over them
template <bool SURF, int G>
__device__ __forceinline__ WalkOut az_scan_walk_group(const AzIndex& ix, const float4 s, int ccr, int w2, int w3, int fwdBound, float nearf,
                                                      float B2, float B3, int sub, unsigned gmask) {
  const int c = ccr & 0x00ffffff, cr = (int)((unsigned)ccr >> 24);
  Top3 t2, t3;
  t2.init(); t3.init();
  auto scan_ring = [&](int r, int win, Top3& top, int start, int step) {
    const int blo = win >> 16, nbins = win & 0xffff, base = r * ix.nb;
    for (int seg = 0; seg < 2; ++seg) {
      int p, pe;
      if (seg == 0) { p = ix.bstart[base + blo]; pe = ix.bstart[base + min(blo + nbins, ix.nb)]; }
      else { const int e1 = blo + nbins - ix.nb; if (e1 <= 0) break; p = ix.bstart[base]; pe = ix.bstart[base + e1]; }
      for (p += start; p < pe; p += kGroupWalkInFlight * step) {
        float4 tt[kGroupWalkInFlight];
#pragma unroll
        for (int u = 0; u < kGroupWalkInFlight; ++u) tt[u] = ld_slot(ix, p + u * step < pe ? p + u * step : p);
#pragma unroll
        for (int u = 0; u < kGroupWalkInFlight; ++u) {
          const int pu = p + u * step;
          const float4 t = tt[u];
          const unsigned d = __float_as_uint(sqdist_f32(t.x, t.y, t.z, s.x, s.y, s.z));
          const int j = slot_index(t.w);
          const bool fwd = j > c;
          const bool adm = pu < pe && j != c && (!fwd || j < fwdBound);
          top.insert(adm ? (((unsigned long long)d << 32) | (fwd ? order_fwd(j) : order_bwd(j))) : kKeyMax, pu);
        }
      }
    }
  };
  if (SURF && cr < ix.nrings) scan_ring(cr, w2, t2, sub, G);
  for (int idx = sub; idx < 4; idx += G) {
    const int r = cr + (idx < 2 ? idx - 2 : idx - 1);
    if (r < 0 || r >= ix.nrings) continue;
    if (SURF) scan_ring(r, w3, t3, 0, 1); else scan_ring(r, w2, t2, 0, 1);
  }
  group_top3<G>(t2, gmask);
  if (SURF) group_top3<G>(t3, gmask);
  const float gate = sqrtf(nearf);
  const unsigned nearbits = __float_as_uint(nearf);
  WalkOut o;
  auto finish = [&](const Top3& t, float Bout, int& idx, int& pos, int& run, float& bound) {
    const bool ok = (unsigned)(t.k1 >> 32) < nearbits && t.p1 >= 0;
    idx = ok ? order_decode((unsigned)(t.k1 & 0xffffffffu)) : -1;
    pos = ok ? t.p1 : -1;
    run = ok ? t.p2 : -1;
    bound = ok ? cert_bound(t.d3, Bout) : rejected_slack((unsigned)(t.k1 >> 32), Bout, gate);
  };
  finish(t2, B2, o.i2, o.pos2, o.run2, o.bound2);
  if (SURF) finish(t3, B3, o.i3, o.pos3, o.run3, o.bound3);
  else { o.i3 = -1; o.pos3 = -1; o.run3 = -1; o.bound3 = 0.f; }
  return o;
}

// ---- certificates (phase P1, one THREAD per query) ------------------------------------------------------------------
// Of the two stored front-runners (winner w >= 0, runner-up r), re-evaluated exactly at the query's new position s, the
// one with the smaller key (exact keys, so ties fall like in a full search) is the answer of a search at s if it is
// closer than everything else can have become: bound - moved, where `bound` is what every other candidate exceeded at
// the search position and `moved` the displacement since (distances change by at most that much); 2e-4 m absorbs the
// f32 rounding of the distances involved.  Nothing else can then beat it or tie with it, whether it is the old winner
// or the runner-up: a query sliding along a ring past the midpoint of two neighbouring points swaps them and keeps its
// certificate.  That answer must also be inside the gate (an answer beyond it would mean "no match", which is searched).
// WALK: keys carry the visiting order relative to the closest point c instead of the original index.
// tw / tr = the winner's / runner-up's entry of the sorted copy, loaded by the caller (all of a query's front-runners are
// fetched in one batch: one L2 round trip instead of up to six dependent ones); r < 0 = no runner-up.
// Returns kCertKeep / kCertSwap (certified; on a swap the runner-up is the answer now) or the reason it failed.
enum : int { kCertKeep = 0, kCertSwap = 1, kCertFailRunnerUp = 2, kCertFailBound = 3, kCertFailGate = 4, kCertFailSlack = 5 };
template <bool WALK>
__device__ __forceinline__ int cert_check(const float4 tw, const float4 tr, const float4 s, int r, float bound, float moved, unsigned nearbits,
                                          int c) {
  auto key_of = [&](const float4 t) -> unsigned long long {
    const unsigned d = __float_as_uint(sqdist_f32(t.x, t.y, t.z, s.x, s.y, s.z));
    const int j = slot_index(t.w);
    const unsigned lo = WALK ? (j > c ? order_fwd(j) : order_bwd(j)) : (unsigned)j;
    return ((unsigned long long)d << 32) | lo;
  };
  const unsigned long long kw = key_of(tw), kr = r >= 0 ? key_of(tr) : kKeyMax;
  const bool swap = kr < kw;
  const unsigned dm = (unsigned)((swap ? kr : kw) >> 32);
  if (!(dm < nearbits)) return kCertFailGate;
  if (!(sqrtf(__uint_as_float(dm)) + moved + 2.0e-4f < bound)) return swap ? kCertFailRunnerUp : kCertFailBound;
  return swap ? kCertSwap : kCertKeep;
}
// a search that found nothing within the gate: stays that way while the query moved less than half the slack
__device__ __forceinline__ bool cert_rejected(float slack, float moved) { return slack > 0.f && 2.0f * moved + 2.0e-4f < slack; }

}  // namespace lins_dev
