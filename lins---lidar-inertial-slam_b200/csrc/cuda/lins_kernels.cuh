// Fused iterated-ESKF update kernel for sm_90a (H100): device functions shared by its phases.
//
// A CTA keeps up to kMaxSlots units resident ("slots"; a unit = query features of the new scan, target features of
// the last scan, prior) and runs the WHOLE performIESKF loop (reference lins/include/StateEstimator.hpp:465-600) for
// all of them in lockstep, phase by phase:
//   A2  transformToStart de-skew of every query               (:1066-1080)   f64 math, f32 store
//   A3/4 exact 1-NN + the +-2.5-ring index walks               (:844-915, :970-1029) f32, bit-exact indices
//   A5/6 point-to-plane / point-to-line residual + coeff       (:917-951, :1031-1060)
//   A7-9 Jacobian row (6 structural non-zeros) folded straight into the 18x18 information form
//        (21 + 6 + 1 scalars per scan; SURVEY.md §8 A9 form B) — H (Mx18) and S (MxM) are never formed
//   A10 boxMinus / gain solve / NaN + divergence tests / boxPlus / convergence (:548-580)
//   A11 Joseph covariance update at exit                        (:595-598)
// Why lockstep slots: the kernel's per-iteration code is ~100 KB of straight-line f64 / search code, far beyond the
// 32 KB instruction cache of an SM; a lone warp (the serial tail of an iteration, a late search) runs at the speed
// of instruction fetch from L2.  With several units per CTA every fetched instruction serves all of them: the
// thread-per-query phases cover the queries of every slot, the warp-per-search phases pull from one work list, and
// the serial tails of the slots run side by side on different warps.  CTAs pull units from a global counter as
// slots fall free, so iteration-count imbalance between units does not idle SMs.  All reductions use a fixed
// shuffle tree + fixed-order sums, so results are run-to-run deterministic (no floating-point atomics).
#pragma once
#include "../../../include/lins_gpu.h"
#include "lins_device_math.cuh"

namespace lins_dev {

constexpr int kThreads = 512;   // threads per CTA
constexpr int kMinCtas = 1;     // resident CTAs per SM the register budget is set for
constexpr int kWarps = kThreads / 32;
constexpr int kMaxSlots = 4;    // resident units per CTA (<= kWarps: warp w runs the serial tail of slot w)
constexpr int kMaxRing = 128;   // rings outside [0, kMaxRing) or unsorted clouds take the brute-force search + sequential walk
                                // ((ring << 24 | index) must stay non-negative: -1 is the "no closest point" sentinel)
constexpr int kNAcc = 28;       // 21 (sym 6x6) + 6 (g*r) + 1 (r*r)
constexpr int kNNChunk = 1024;  // targets per brute-force work item
constexpr int kAzTabS = 4096;   // (ring, azimuth bin) table entries, surf targets (see lins_assoc_az.cuh)
constexpr int kAzTabC = 1024;   // corner targets
constexpr float kPiF = 3.14159265358979f;
constexpr unsigned long long kKeyMax = 0xFFFFFFFFFFFFFFFFull;

enum KernelMode { MODE_IESKF = 0, MODE_ASSOC = 1, MODE_ICP_REDUCE = 2, MODE_JACOBIAN = 3 };

// one unit's estimator tuning (lins_slot_tuning without the IMU misalignment): NUM_ITER, ICP_FREQ (>= 1),
// NEAREST_FEATURE_SEARCH_SQ_DIST, LIDAR_STD, LIDAR_SCALE
struct UnitTuning {
  int num_iter, icp_freq;
  double nearest_sq, lidar_std, lidar_scale;
};

struct BatchView {
  int n_scans;
  const float4* qs; const int* qs_off;   // surf queries   (surfPointsFlat_)
  const float4* qc; const int* qc_off;   // corner queries (cornerPointsSharp_)
  const float4* ts; const int* ts_off;   // surf targets   (last surfPointsLessFlat_)
  const float4* tc; const int* tc_off;   // corner targets (last cornerPointsLessSharp_)
  // clouds the 1-NN index was built on where they differ from ts/tc: after a map refresh that failed the >=5 && >=20
  // guard (StateEstimator.hpp:1156-1157) scan_last_ advanced, the kd-trees did not.  Null (with nn_stale) = none.
  const float4* nn_s; const int* nn_s_off;
  const float4* nn_c; const int* nn_c_off;
  const unsigned char* nn_stale;         // per unit, set with nn_s: 1 = nn_s / nn_c hold its 1-NN clouds
  const double* state_in;                // n x 20 (19 used)
  const double* cov_in;                  // n x 324, column-major
  double* state_out;                     // n x 20
  double* cov_out;                       // n x 324, column-major
  lins_scan_result* results;             // n
  lins_report* reports;                  // n or null
  int* ind_s;                            // 3 per surf query   (pointSearchSurfInd1/2/3)
  int* ind_c;                            // 2 per corner query (pointSearchCornerInd1/2)
  float* sel_s; float* sel_c;            // optional dense traces (3 per query)
  float* coeff_s; float* coeff_c;        // optional (4 per query)
  unsigned char* mask_s; unsigned char* mask_c;  // optional
  double* accum;                         // n x 32 : 28 accumulators + m_surf + m_corner (modes 2,3)
  float4* az_s; float4* az_c;            // the (ring, azimuth)-sorted target copies built by the kernel (≙ the kd-trees),
                                         // same per-scan offsets as ts / tc; served from L1 / L2
  int* work_counter;
  long long* timers;                     // optional: per-phase SM cycles summed over CTAs (diagnostics), 64 slots
  int qtile;                             // per-slot capacity of the per-query arrays (>= the largest unit, multiple of 32)
  int nslots;                            // resident units per CTA
  const int* icp_done;                   // MODE_ICP_REDUCE: IcpState::done of unit 0, unit u's kIcpDoneStride ints further
                                         // (lins_icp_step.cuh); non-zero = that unit's Gauss-Newton loop has ended, skip it (or null)
  unsigned char* qscratch;               // per-CTA global scratch for the per-query arrays when they do not fit shared
  size_t qscratch_stride;                // memory (null: they live in shared memory)
  const double* unit_period;             // per unit: the SCAN_PERIOD of its de-skew (sequence mode's per-slot rigs); null =
                                         // every unit's is KParams::scan_period
  const UnitTuning* unit_tune;           // per unit: its estimator tuning (sequence mode's per-slot tuning); null = every
                                         // unit's is KParams'
};

// loop state of one unit's estimateTransform (lins_icp_step.cuh)
struct IcpState {
  double matP[36];
  int iters, converged, done, pad;
};
// BatchView::icp_done points at the `done` of unit 0's IcpState; unit u's is kIcpDoneStride ints further
constexpr int kIcpDoneStride = (int)(sizeof(IcpState) / sizeof(int));
static_assert(sizeof(IcpState) % sizeof(int) == 0, "IcpState stride");

struct KParams {
  int num_iter, icp_freq, force_all_iters, mode, iter0;
  double nearest_sq, lidar_std, lidar_scale, scan_period;
};

// unit `scan` searches a 1-NN cloud of its own (a stale index: brute-force 1-NN over it, then walks over the map)
__device__ __forceinline__ bool nn_separate(const BatchView& bv, int scan) {
  return bv.nn_s != nullptr && bv.nn_stale[scan] != 0;
}

__device__ __forceinline__ unsigned long long pack_key(float d, unsigned int lo) {
  return ((unsigned long long)__float_as_uint(d) << 32) | lo;
}
__device__ __forceinline__ unsigned long long shfl_xor_u64(unsigned long long v, int m) {
  return __shfl_xor_sync(0xffffffffu, v, m);
}
__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) {
    unsigned long long o = shfl_xor_u64(v, m);
    v = o < v ? o : v;
  }
  return v;
}

// shared-memory carve-up ---------------------------------------------------------------------------------
typedef unsigned short aztab_t;  // bucket tables hold slots of the sorted copies: the indexed path needs T < 65536

// one resident unit ("slot")
struct alignas(16) Smem {
  // iteration-invariant
  double prior[20];
  double Pc[18 * 6];    // P[:, c], c = {0,1,2,6,7,8}: the only part of the prior covariance an iteration reads
  // iterate
  double lin[20];
  double phi[3];        // Quat2axis(lin q)
  double R[9];          // toRotationMatrix(lin q)
  double Rinv[9];       // Rinvleft(-phi)
  double dvec[18];      // filterState (-) linState
  double acc[kNAcc + 4];
  double A6[36];
  double y6[6];
  double M6[36];        // A6 P_cc + sig2 I  (6x6 gain system, see form_M6)
  double X6[6];         // right-hand side / solution of the gain system
  double upd[18];
  double residualNorm;
  double period;        // SCAN_PERIOD of the unit's de-skew (transformToStart, the ICP fallback's rows)
  // the unit's tuning (BatchView::unit_tune or KParams): a pass mixes the queries of every resident unit, so each query
  // reads its own unit's gate, ICP_FREQ and LIDAR_SCALE here
  double nearest_sq;    // the 1-NN gate, compared in f64 ...
  double lidar_scale;
  double sig2;          // LIDAR_STD^2 of the gain
  float nearf;          // ... and in f32 by the windows, walks and certificates
  float gate;           // sqrtf(nearf)
  int num_iter, icp_freq;
  int search, weighted; // of the pass at `iter`: iter % ICP_FREQ == 0 (a closest-point search), iter >= ICP_FREQ (the
                        // residual's weight); set with iter, so a pass reads two flags instead of dividing per query
  int flags[4];         // 0 converged 1 diverged 2 has_nan 3 stop
  int cnt[2];
  // bookkeeping
  int scan;             // unit id, -1 = the slot is free
  int iter;             // index of the iteration being run (iterations completed so far)
  int fresh;            // just claimed: needs its prologue
  int run;              // takes part in the passes
  int finished;         // leaves after this pass (exit covariance + outputs)
  int first_pass;       // no previous answers to seed / certify from
  int pos_valid, pos_is_slot;  // pos[] holds this unit's correspondences; as slots of the sorted copies or original indices
  int qs0, ns, qc0, nc, ts0, Ts, tc0, Tc;
  int sortedS, sortedC;
  int az_ok;            // 1: both clouds ring-sorted + indexed (fast path); 0: brute-force 1-NN + sequential walks
  int nbS, nbC, nringsS, nringsC;
  aztab_t azTabS[kAzTabS + 2];  // (ring, azimuth bin) -> first slot of the sorted surf copy
  aztab_t azTabC[kAzTabC + 2];
  // per ring: [min, max] of the slope z / rho_xy (the tangent of the elevation angle) of its targets, as order-preserving int keys (see
  // lins_assoc_az.cuh: a ring whose elevation band is farther from the query's elevation than the search radius allows
  // is skipped by the closest-point scans)
  int elevS[kMaxRing][2], elevC[kMaxRing][2];
};

// per-CTA scratch
struct CtaMem {
  union {
    // counting-sort counters / cursors while a unit's index is built, 16 bits each (lins_assoc_az.cuh: cnt16_add1): 8 kB
    // instead of 16 kB brings the CTA (three slots of 320 queries) from 205 072 B to 196 880 B of shared memory, under the
    // 196 KB carve-out, so the SM keeps about 60 KB of L1 instead of 28 KB for the sorted target copies the searches and
    // the residuals read
    unsigned build_tab[kAzTabS / 2 + 1];
    struct { double P[324], X[324], U[108], V[108], X6[72]; } ex;  // exit covariance of one finished unit
    // the residual phase's tensor-core fold (warp_fold_mma): 8 staged rows of 8 doubles per warp, 16 x 512 B = 8192 B,
    // inside the 8196 B of build_tab, so the CTA does not grow.  Free then: the index build and the exit run outside passes.
    double fold[kWarps][64];
  } u;
  int scan_tmp[kThreads];
  int wl_n[2], wl_head[2];  // work lists of the closest-point / walk phases (entries, next entry to hand out)
  int wl_tn[2], wl_thead[2];  // ... and their group-level lists (filled from the back of the same array)
  int dbg[2];               // diagnostics (only touched when phase timers are enabled)
  int n_active, any_fresh, any_finished, any_legacy, any_indexed, exhausted, pass_first;
  unsigned long long mbar;
  unsigned int phase;
  long long tlast;
};
static_assert(sizeof(((CtaMem*)nullptr)->u.fold) <= sizeof(((CtaMem*)nullptr)->u.build_tab), "the fold stage must not grow the CTA");

// phase timers (thread 0 of each CTA; compiled in, enabled when bv.timers != nullptr)
#define LINS_TICK(k)                                                                   \
  do {                                                                                 \
    if (bv.timers && threadIdx.x == 0) {                                               \
      const long long _t = clock64();                                                  \
      atomicAdd((unsigned long long*)&bv.timers[k], (unsigned long long)(_t - cta.tlast)); \
      cta.tlast = _t;                                                                   \
    }                                                                                  \
  } while (0)
// a tick of the association pass: passes that contain a unit's first pass are clocked separately, in slot k + 32
// (cta.pass_first is read when the tick is taken, so no register is held across the pass for it)
#define LINS_TICK_PASS(k) LINS_TICK((k) + (cta.pass_first ? 32 : 0))

// ---------------------------------------------------------------------------------------------------------
// A2 transformToStart (StateEstimator.hpp:1066-1080) -------------------------------------------------------
__device__ __forceinline__ float4 transform_to_start(const float4 p, const Smem& sm, double scan_period) {
  float fi = p.w - (float)((int)p.w);
  double s = (1.f / scan_period) * fi;
  d3 v = mk3(s * sm.phi[0], s * sm.phi[1], s * sm.phi[2]);
  q4 r = axis2Quat(v);
  d3 P2 = mk3((double)p.x, (double)p.y, (double)p.z);
  d3 rp = qrot(r, P2);
  d3 t = mk3(s * sm.lin[0], s * sm.lin[1], s * sm.lin[2]);
  float4 o;
  o.x = (float)(rp.x + t.x); o.y = (float)(rp.y + t.y); o.z = (float)(rp.z + t.z); o.w = p.w;
  return o;
}

// Is the cloud ring-sorted with every ring in [0, kMaxRing)?  (what the reference's extractFeatures emits, :727-826; the
// (ring, azimuth) index requires it).  Block-wide; *sorted_flag is valid after the trailing barrier.
__device__ inline void check_ring_sorted(const float4* __restrict__ tgt, int T, int* sorted_flag) {
  if (threadIdx.x == 0) *sorted_flag = 1;
  __syncthreads();
  for (int j = threadIdx.x; j < T; j += kThreads) {
    const int rj = (int)__ldg(&tgt[j]).w;
    const int rp = j > 0 ? (int)__ldg(&tgt[j - 1]).w : -1;
    if (rj < 0 || rj >= kMaxRing || (j > 0 && rj < rp)) *sorted_flag = 0;
  }
  __syncthreads();
}

// A3/A4 exact brute-force 1-NN: every (32-query group, kNNChunk-target chunk) pair is one warp work item; all
// lanes of a warp read the same target (broadcast 16-B load), each lane keeps its own query's best.
__device__ inline void nn_brute(const float4* sel, unsigned long long* key, int nq, const float4* __restrict__ tgt, int T) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nqg = (nq + 31) >> 5, nch = (T + kNNChunk - 1) / kNNChunk;
  for (int item = warp; item < nqg * nch; item += kWarps) {
    const int qg = item % nqg, ch = item / nqg;
    const int qi = qg * 32 + lane;
    const bool valid = qi < nq;
    const float4 s = valid ? sel[qi] : make_float4(0.f, 0.f, 0.f, 0.f);
    const int j0 = ch * kNNChunk, j1 = min(T, j0 + kNNChunk);
    float best = __int_as_float(0x7f800000);
    int bi = -1;
#pragma unroll 4
    for (int j = j0; j < j1; ++j) {
      const float4 t = __ldg(&tgt[j]);
      const float d = sqdist_f32(s.x, s.y, s.z, t.x, t.y, t.z);
      if (d < best) { best = d; bi = j; }
    }
    if (valid && bi >= 0) atomicMin(&key[qi], pack_key(best, (unsigned)bi));
  }
}


// walk keys: high 32 = f32 distance bits, low 32 = visiting order (forward walk ascending j first, then the
// backward walk descending j) so that u64 min == "first strictly smaller wins" of the reference loops.
__device__ __forceinline__ unsigned int order_fwd(int j) { return (unsigned)j; }
__device__ __forceinline__ unsigned int order_bwd(int j) { return 0x80000000u | (unsigned)(0x7fffffff - j); }
__device__ __forceinline__ int order_decode(unsigned int o) { return (o & 0x80000000u) ? (0x7fffffff - (int)(o & 0x7fffffffu)) : (int)o; }

// Sequential walk, literal restatement (any ring order / values).  One thread.
template <bool SURF>
__device__ void walk_seq(const float4 s, int c, const float4* __restrict__ tgt, int T, int fwdBound, float nearf,
                         int& i2, int& i3) {
  const int cr = (int)__ldg(&tgt[c]).w;
  float m2 = nearf, m3 = nearf;
  i2 = -1; i3 = -1;
  for (int j = c + 1; j < fwdBound; ++j) {
    const float4 t = __ldg(&tgt[j]);
    const int rj = (int)t.w;
    if ((double)rj > (double)cr + 2.5) break;
    const float d = sqdist_f32(t.x, t.y, t.z, s.x, s.y, s.z);
    if (SURF) {
      if (rj <= cr) { if (d < m2) { m2 = d; i2 = j; } }
      else { if (d < m3) { m3 = d; i3 = j; } }
    } else {
      if (rj > cr) { if (d < m2) { m2 = d; i2 = j; } }
    }
  }
  for (int j = c - 1; j >= 0; --j) {
    const float4 t = __ldg(&tgt[j]);
    const int rj = (int)t.w;
    if ((double)rj < (double)cr - 2.5) break;
    const float d = sqdist_f32(t.x, t.y, t.z, s.x, s.y, s.z);
    if (SURF) {
      if (rj >= cr) { if (d < m2) { m2 = d; i2 = j; } }
      else { if (d < m3) { m3 = d; i3 = j; } }
    } else {
      if (rj < cr) { if (d < m2) { m2 = d; i2 = j; } }
    }
  }
}

// A5 plane residual (StateEstimator.hpp:917-951).  Returns accept mask; coeff = (s*jac, s*res).
__device__ __forceinline__ bool plane_residual(const float4 sel, const float4 t1, const float4 t2, const float4 t3,
                                               bool weighted, float4& coeff) {
  d3 P0 = mk3(sel.x, sel.y, sel.z), P1 = mk3(t1.x, t1.y, t1.z), P2 = mk3(t2.x, t2.y, t2.z), P3 = mk3(t3.x, t3.y, t3.z);
  d3 M = cross3(sub3(P1, P2), sub3(P1, P3));
  double r = dot3(sub3(P0, P1), M);
  double m = norm3(M);
  float res = (float)(r / m);
  d3 jac = div3(M, m);
  float s = 1.f;
  if (weighted) {
    float n2 = __fadd_rn(__fadd_rn(__fmul_rn(sel.x, sel.x), __fmul_rn(sel.y, sel.y)), __fmul_rn(sel.z, sel.z));
    float rt = sqrtf(sqrtf(n2));
    s = (float)(1.0 - 1.8 * (double)fabsf(res) / (double)rt);
  }
  if ((double)s > 0.1 && res != 0.f) {
    coeff.x = (float)((double)s * jac.x); coeff.y = (float)((double)s * jac.y); coeff.z = (float)((double)s * jac.z);
    coeff.w = __fmul_rn(s, res);
    return true;
  }
  return false;
}
// A6 line residual (StateEstimator.hpp:1031-1060)
__device__ __forceinline__ bool line_residual(const float4 sel, const float4 t1, const float4 t2, bool weighted,
                                              float4& coeff) {
  d3 P0 = mk3(sel.x, sel.y, sel.z), P1 = mk3(t1.x, t1.y, t1.z), P2 = mk3(t2.x, t2.y, t2.z);
  d3 P = cross3(sub3(P0, P1), sub3(P0, P2));
  float r = (float)norm3(P);
  float d12 = (float)norm3(sub3(P1, P2));
  float res = __fdiv_rn(r, d12);
  d3 a = sub3(P2, P1);
  d3 num = mk3(P.y * a.z + P.z * (-a.y), P.x * (-a.z) + P.z * a.x, P.x * a.y + P.y * (-a.x));
  double den = (double)__fmul_rn(d12, r);
  d3 jac = div3(num, den);
  float s = 1.f;
  if (weighted) s = (float)(1.0 - 1.8 * (double)fabsf(res));
  if ((double)s > 0.1 && res != 0.f) {
    coeff.x = (float)((double)s * jac.x); coeff.y = (float)((double)s * jac.y); coeff.z = (float)((double)s * jac.z);
    coeff.w = __fmul_rn(s, res);
    return true;
  }
  return false;
}

// A7-A9: the factored Jacobian row of one accepted measurement.
// g = [c ; P2 x (R^T c)]  (the Jacobian row is h = [c ; Rinv^T g_att], applied once per scan at solve time), r = residual
__device__ __forceinline__ void jacobian_row(const float4 kp, const float4 coeff, const double* R, double lidar_scale,
                                             double* g, double& r) {
  const double cx = coeff.x, cy = coeff.y, cz = coeff.z;
  r = lidar_scale * (double)coeff.w;
  const double ux = R[0] * cx + R[3] * cy + R[6] * cz;
  const double uy = R[1] * cx + R[4] * cy + R[7] * cz;
  const double uz = R[2] * cx + R[5] * cy + R[8] * cz;
  const double px = kp.x, py = kp.y, pz = kp.z;
  g[0] = cx; g[1] = cy; g[2] = cz;
  g[3] = py * uz - pz * uy; g[4] = pz * ux - px * uz; g[5] = px * uy - py * ux;
}
// ICP fallback variant (StateEstimator.hpp:1228-1258): interpolated rotation per point, rotation block first.
__device__ __forceinline__ void jacobian_row_icp(const float4 kp, const float4 coeff, const double* phi, double scan_period,
                                                 double* g, double& b) {
  float fi = kp.w - (float)((int)kp.w);
  double s = (1.f / scan_period) * fi;
  q4 rq = axis2Quat(mk3(s * phi[0], s * phi[1], s * phi[2]));
  m3 R = qtoR(rq);
  const double cx = coeff.x, cy = coeff.y, cz = coeff.z;
  b = -0.05 * (double)coeff.w;
  const double ux = R.m[0] * cx + R.m[3] * cy + R.m[6] * cz;
  const double uy = R.m[1] * cx + R.m[4] * cy + R.m[7] * cz;
  const double uz = R.m[2] * cx + R.m[5] * cy + R.m[8] * cz;
  const double px = kp.x, py = kp.y, pz = kp.z;
  g[0] = py * uz - pz * uy; g[1] = pz * ux - px * uz; g[2] = px * uy - py * ux;
  g[3] = cx; g[4] = cy; g[5] = cz;
}

__device__ __forceinline__ void dmma_8x8x4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// Warp fold of one row per lane into the 28 sums of the information form: entries 0..20 = upper triangle of g g^T
// (row-major), 21..26 = g r, 27 = r r.  They are entries of the 8 x 8 Gram matrix C = G^T G of the warp's 32 rows
// G = [g0..g5, r, 0], which eight FP64 tensor-core mma.sync m8n8k4 (four rows each) accumulate.  The A (8 x 4, row) and
// B (4 x 8, col) fragments of lane L are both G[4c + L % 4][L / 4], i.e. entries of other lanes' rows, so the rows pass
// through the warp's 512 B of shared memory `st`: four rounds of 8 rows (two MMAs each).  A staged row is four 16-B
// chunks, chunk k of row j at chunk 4 j + (k ^ (j >> 1)): the 8 writing lanes hit 8 different bank groups and the 32
// reads of an MMA one 256-B block.  Lane L writes C[L / 4][2 (L % 4) + {0, 1}] to dst[entry] where that is one of the
// 28 sums.  Fixed order => deterministic.  Lanes without a measurement pass g = 0, r = 0.
__device__ __forceinline__ void warp_fold_mma(const double* g, double r, double* st, double* dst) {
  const int lane = threadIdx.x & 31;
  const int wj = lane & 7, f = lane >> 2;
  double c0 = 0.0, c1 = 0.0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    __syncwarp();
    if ((lane >> 3) == q) {
      double2* row = reinterpret_cast<double2*>(st) + 4 * wj;
      const int sw = wj >> 1;
      row[0 ^ sw] = make_double2(g[0], g[1]); row[1 ^ sw] = make_double2(g[2], g[3]);
      row[2 ^ sw] = make_double2(g[4], g[5]); row[3 ^ sw] = make_double2(r, 0.0);
    }
    __syncwarp();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = 4 * h + (lane & 3);
      const double v = st[2 * (4 * j + ((f >> 1) ^ (j >> 1))) + (f & 1)];
      dmma_8x8x4(c0, c1, v, v);
    }
  }
  const int ci = f;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int cj = 2 * (lane & 3) + u;
    if (ci <= cj && cj <= 6) dst[cj < 6 ? ci * 6 - (ci * (ci - 1)) / 2 + (cj - ci) : (ci < 6 ? 21 + ci : 27)] = u ? c1 : c0;
  }
}

__device__ __forceinline__ int col6(int a) { return a < 3 ? a : a + 3; }  // {0,1,2,6,7,8}

// M = A6 P_cc + sig2 I6: the 6x6 system of the gain in push-through form.  With H = H6 E_c^T (only the 6
// structural columns c = {0,1,2,6,7,8} are non-zero) and R = sig2 I:
//   K = P H^T (H P H^T + R)^-1 = P[:,c] (A6 P[c,c] + sig2 I6)^-1 H6^T,   A6 = H6^T H6
// so  K (r + H d) = P[:,c] M^-1 (b6 + A6 d_c)  and nothing larger than 6x6 is ever factorised.
__device__ inline void form_M6(Smem& sm, double sig2, int idx, int stride) {
  for (int t = idx; t < 36; t += stride) {
    const int a = t / 6, c = t % 6;
    double s = 0;
    for (int k = 0; k < 6; ++k) s += sm.A6[a * 6 + k] * sm.Pc[col6(k) * 6 + c];
    if (a == c) s += sig2;
    sm.M6[t] = s;
  }
}

// linState (+) updateVec (KalmanFilter.hpp:71-81), thread 0
__device__ inline void box_plus(Smem& sm) {
  double* l = sm.lin; const double* u = sm.upd;
  for (int i = 0; i < 3; ++i) {
    l[0 + i] += u[0 + i]; l[3 + i] += u[3 + i]; l[10 + i] += u[9 + i]; l[13 + i] += u[12 + i]; l[16 + i] += u[15 + i];
  }
  q4 q; q.x = l[6]; q.y = l[7]; q.z = l[8]; q.w = l[9];
  q4 dq = axis2Quat(mk3(u[6], u[7], u[8]));
  q4 r = qnormalized(qmul(q, dq));
  l[6] = r.x; l[7] = r.y; l[8] = r.z; l[9] = r.w;
}


// ---------------------------------------------------------------------------------------------------------
// The serial tail of an iteration, executed by warp 0 alone between two block barriers.  Everything below is
// written so that the 32 lanes work on different entries of the same small formula in lockstep.

// N x N LU with partial pivoting, one COLUMN per lane held in registers: lanes [0, N) own the columns of S
// (row-major in shared memory), lanes [N, N + nrhs) the right-hand sides B (N x nrhs row-major, overwritten by
// the solution).  Pivot = first maximum of |column| from the diagonal down (what a sequential scan picks; a NaN
// on the diagonal poisons the step); one division per step; only the initial loads and the final stores touch
// shared memory.  nrhs <= 32 - N.
template <int N>
__device__ bool warp_lu_cols(const double* S, double* B, int nrhs) {
  const int lane = threadIdx.x & 31;
  const bool is_rhs = lane >= N && lane < N + nrhs;
  double c[N];
#pragma unroll
  for (int r = 0; r < N; ++r) c[r] = lane < N ? S[r * N + lane] : (is_rhs ? B[r * nrhs + (lane - N)] : 0.0);
  double dinv = 0.0;  // lane k keeps 1 / U[k][k]
  bool ok = true;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    int piv = k;
    double best = fabs(c[k]);
#pragma unroll
    for (int r = k + 1; r < N; ++r) {
      const double v = fabs(c[r]);
      if (v > best) { best = v; piv = r; }
    }
    piv = __shfl_sync(0xffffffffu, piv, k);
    best = __shfl_sync(0xffffffffu, best, k);
    if (!(best > 0.0)) { ok = false; break; }  // singular or NaN pivot (uniform: broadcast value)
#pragma unroll
    for (int r = k + 1; r < N; ++r)
      if (piv == r) { const double t = c[k]; c[k] = c[r]; c[r] = t; }
    const double inv = 1.0 / c[k];  // meaningful in lane k
    if (lane == k) dinv = inv;
#pragma unroll
    for (int r = k + 1; r < N; ++r) {
      const double f = __shfl_sync(0xffffffffu, c[r] * inv, k);
      if (f != 0.0 && lane > k) c[r] -= f * c[k];
    }
  }
  if (!ok) return false;
#pragma unroll
  for (int k = N - 1; k >= 0; --k) {
    double sacc = c[k];
#pragma unroll
    for (int m = k + 1; m < N; ++m) {
      const double u = __shfl_sync(0xffffffffu, c[k], m);  // U[k][m] lives in lane m
      sacc -= u * c[m];
    }
    const double inv = __shfl_sync(0xffffffffu, dinv, k);
    if (is_rhs) c[k] = sacc * inv;
  }
  if (is_rhs) {
#pragma unroll
    for (int r = 0; r < N; ++r) B[r * nrhs + (lane - N)] = c[r];
  }
  return true;
}

// sm.acc / sm.cnt = the sums of the per-warp partial folds of this pass (nvw of them), in warp order
__device__ __forceinline__ void finish_acc_warp0(Smem& sm, const double* wacc, const int* wcnt, int nvw) {
  const int lane = threadIdx.x & 31;
  if (lane < kNAcc) {
    double v = 0.0;
    for (int w = 0; w < nvw; ++w) v += wacc[w * kNAcc + lane];
    sm.acc[lane] = v;
  } else if (lane < kNAcc + 2) {
    const int k = lane - kNAcc;
    int a = 0;
    for (int w = 0; w < nvw; ++w) a += wcnt[w * 2 + k];
    sm.cnt[k] = a;
  }
  __syncwarp();
}

// A6 = T Ag T^T and y6 = T b with T = blockdiag(I3, Rinv^T), entry by entry with the structural zeros of T
// skipped (adding those zero products would not change a finite result).  Two lockstep rounds: the 27 entries
// that need arithmetic + 5 copies, then 4 copies + y6.
__device__ __forceinline__ void build_A6_warp0(Smem& sm) {
  const int lane = threadIdx.x & 31;
  auto Ag = [&](int i, int j) -> double {
    if (i > j) { const int tmp = i; i = j; j = tmp; }
    return sm.acc[i * 6 - (i * (i - 1)) / 2 + (j - i)];
  };
  auto entry = [&](int a, int c) -> double {
    if (a < 3 && c < 3) return Ag(a, c);
    if (a < 3) {  // Ag12 Rinv
      double u = 0;
      for (int j = 0; j < 3; ++j) u += Ag(a, 3 + j) * sm.Rinv[j * 3 + (c - 3)];
      return u;
    }
    if (c < 3) {  // Rinv^T Ag21
      double v = 0;
      for (int i = 0; i < 3; ++i) v += sm.Rinv[i * 3 + (a - 3)] * Ag(3 + i, c);
      return v;
    }
    double v = 0;  // Rinv^T Ag22 Rinv
    for (int i = 0; i < 3; ++i) {
      double u = 0;
      for (int j = 0; j < 3; ++j) u += Ag(3 + i, 3 + j) * sm.Rinv[j * 3 + (c - 3)];
      v += sm.Rinv[i * 3 + (a - 3)] * u;
    }
    return v;
  };
  // entry order: [3..5]x[3..5] (9), [0..2]x[3..5] (9), [3..5]x[0..2] (9), [0..2]x[0..2] (9)
  auto coords = [&](int e, int& a, int& c) {
    const int blk = e / 9, w = e % 9;
    a = w / 3 + ((blk == 0 || blk == 2) ? 3 : 0);
    c = w % 3 + ((blk == 0 || blk == 1) ? 3 : 0);
  };
  {
    int a, c;
    coords(lane, a, c);
    sm.A6[a * 6 + c] = entry(a, c);
  }
  if (lane < 4) {
    int a, c;
    coords(32 + lane, a, c);
    sm.A6[a * 6 + c] = entry(a, c);
  } else if (lane < 10) {
    const int a = lane - 4;
    double v = 0;
    if (a < 3) v = sm.acc[21 + a];
    else for (int i = 0; i < 3; ++i) v += sm.Rinv[i * 3 + (a - 3)] * sm.acc[24 + i];
    sm.y6[a] = v;  // b_h (A6 d_c is added by the caller)
  }
  __syncwarp();
}

// Start-of-iteration constants and filterState (-) linState in one lockstep pass: lane 0 derives phi, R, Rinv
// from the iterate, lane 1 the attitude part of boxMinus — both are Quat2axis of a quaternion, so the expensive
// part runs once for the two lanes.  (compute_iter_consts + box_minus, KalmanFilter.hpp:84-94.)
__device__ __forceinline__ void iter_consts_warp0(Smem& sm) {
  const int lane = threadIdx.x & 31;
  const double* f = sm.prior; const double* l = sm.lin;
  if (lane >= 2 && lane < 17) {  // the 15 vector-space components of boxMinus
    const int e = lane - 2, blk = e / 3, i = e % 3;
    const int so = blk == 0 ? 0 : blk == 1 ? 3 : 10 + 3 * (blk - 2);   // state offsets 0,3,10,13,16
    const int eo = blk == 0 ? 0 : blk == 1 ? 3 : 9 + 3 * (blk - 2);    // error-state offsets 0,3,9,12,15
    sm.dvec[eo + i] = f[so + i] - l[so + i];
  }
  if (lane < 2) {
    q4 ql; ql.x = l[6]; ql.y = l[7]; ql.z = l[8]; ql.w = l[9];
    q4 qf; qf.x = f[6]; qf.y = f[7]; qf.z = f[8]; qf.w = f[9];
    const q4 qd = qmul(qinverse(ql), qf);
    const q4 qin = lane == 0 ? ql : qd;
    const d3 ax = Quat2axis(qin);
    if (lane == 1) { sm.dvec[6] = ax.x; sm.dvec[7] = ax.y; sm.dvec[8] = ax.z; }
    else {
      sm.phi[0] = ax.x; sm.phi[1] = ax.y; sm.phi[2] = ax.z;
      const m3 R = qtoR(ql);
      const m3 Ri = Rinvleft(mk3(-ax.x, -ax.y, -ax.z));
      for (int i = 0; i < 9; ++i) { sm.R[i] = R.m[i]; sm.Rinv[i] = Ri.m[i]; }
    }
  }
  __syncwarp();
}

}  // namespace lins_dev
