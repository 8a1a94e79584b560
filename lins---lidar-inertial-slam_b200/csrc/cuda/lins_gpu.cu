// lins_gpu.cu — the fused IESKF kernel, its launch and the C-ABI around it (include/lins_gpu.h), sm_90a.  The batch upload
// is in lins_upload.cu, row F2 in lins_map.cu; the context they share in lins_ctx.hpp.
// Host side is plain C++ / CUDA runtime: no torch, no Eigen, no PCL in any signature.  There is NO CPU
// fallback: every entry point fails with LINS_E_NODEVICE / LINS_E_CUDA when the device path is unavailable.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <utility>

#include "lins_assoc.cuh"
#include "lins_ctx.hpp"
#include "lins_icp_step.cuh"

using namespace lins_dev;
using namespace lins_capi;

// lins_jacobian.cu
extern "C" int lins_jacobian_parts(int n_units, int sm_count);
extern "C" int lins_launch_jacobian_mma(const lins_dev::BatchView* bv, const lins_dev::KParams* kp, int n_units, int sm_count, int P, double* part_acc,
                                        int* part_cnt, cudaStream_t stream);

namespace {

// prologue of a freshly claimed unit: prior -> shared, the search index (≙ kdtree*->setInputCloud,
// StateEstimator.hpp:363-364 / :1158-1159) built on device, queries staged, first linearisation constants.  Block-wide.
template <int MODE>
__device__ void unit_prologue(CtaMem& cta, Smem& sm, const BatchView& bv, const KParams& kp, const PassBuffers& pb, int slot) {
  const int tid = threadIdx.x, warp = tid >> 5;
  const int scan = sm.scan;
  if (tid < 20) { const double v = tid < 19 ? bv.state_in[(size_t)scan * 20 + tid] : 0.0; sm.prior[tid] = v; sm.lin[tid] = v; }
  for (int e = tid; e < 108; e += kThreads) {  // P[:, c] (cov_in is column-major)
    const int a = e / 6, c = e % 6;
    sm.Pc[e] = bv.cov_in[(size_t)scan * 324 + col6(c) * 18 + a];
  }
  if (tid == 32) {
    sm.flags[0] = sm.flags[1] = sm.flags[2] = sm.flags[3] = 0; sm.residualNorm = 1e6;
    sm.cnt[0] = sm.cnt[1] = 0;
    sm.iter = MODE == MODE_IESKF ? 0 : kp.iter0;
    sm.fresh = 0; sm.finished = 0; sm.first_pass = 1; sm.pos_valid = 0; sm.pos_is_slot = 0;
    sm.run = 1;
    if (MODE == MODE_IESKF && kp.num_iter <= 0) { sm.run = 0; sm.finished = 1; cta.any_finished = 1; }
    sm.qs0 = bv.qs_off[scan]; sm.ns = bv.qs_off[scan + 1] - sm.qs0;
    sm.qc0 = bv.qc_off[scan]; sm.nc = bv.qc_off[scan + 1] - sm.qc0;
    sm.ts0 = bv.ts_off[scan]; sm.Ts = bv.ts_off[scan + 1] - sm.ts0;
    sm.tc0 = bv.tc_off[scan]; sm.Tc = bv.tc_off[scan + 1] - sm.tc0;
  }
  __syncthreads();
  check_ring_sorted(bv.ts + sm.ts0, sm.Ts, &sm.sortedS);
  check_ring_sorted(bv.tc + sm.tc0, sm.Tc, &sm.sortedC);
  if (tid == 0) {
    // slot payload = ring (7 bits) | index (24 bits); bucket tables hold 16-bit slots
    const bool ok = sm.sortedS && sm.sortedC && !nn_separate(bv, scan) && sm.Ts < 65536 && sm.Tc < 65536;
    sm.az_ok = ok ? 1 : 0;
    sm.nringsS = ok && sm.Ts > 0 ? (int)bv.ts[sm.ts0 + sm.Ts - 1].w + 1 : 0;  // ring-sorted: the last point has the largest ring
    sm.nringsC = ok && sm.Tc > 0 ? (int)bv.tc[sm.tc0 + sm.Tc - 1].w + 1 : 0;
    sm.nbS = az_bins_for(sm.nringsS, kAzTabS);
    sm.nbC = az_bins_for(sm.nringsC, kAzTabC);
  }
  __syncthreads();
  if (sm.az_ok) {
    az_build<kAzTabS>(bv.ts + sm.ts0, sm.Ts, bv.az_s + sm.ts0, sm.azTabS, cta.u.build_tab, cta.scan_tmp, sm.nbS, sm.elevS);
    az_build<kAzTabC>(bv.tc + sm.tc0, sm.Tc, bv.az_c + sm.tc0, sm.azTabC, cta.u.build_tab, cta.scan_tmp, sm.nbC, sm.elevC);
  }
  // queries: staged once per unit — 1-D TMA (cp.async.bulk + mbarrier) into shared memory, plain copies into the scratch
  float4* qdst = pb.qpt + (size_t)slot * bv.qtile;
  if (bv.qscratch == nullptr) {
    const uint32_t bytes = (uint32_t)(sm.ns + sm.nc) * 16u;
    if (bytes > 0) {
      if (tid == 0) {
        fence_proxy_async();
        mbar_expect_tx(&cta.mbar, bytes);
        if (sm.ns > 0) tma_load_1d(qdst, bv.qs + sm.qs0, (uint32_t)sm.ns * 16u, &cta.mbar);
        if (sm.nc > 0) tma_load_1d(qdst + sm.ns, bv.qc + sm.qc0, (uint32_t)sm.nc * 16u, &cta.mbar);
      }
      const unsigned int ph = cta.phase;  // one mbarrier phase per staged unit
      mbar_wait(&cta.mbar, ph & 1u);
      __syncthreads();
      if (tid == 0) cta.phase = ph + 1u;
    }
  } else {
    for (int i = tid; i < sm.ns + sm.nc; i += kThreads) qdst[i] = i < sm.ns ? __ldg(bv.qs + sm.qs0 + i) : __ldg(bv.qc + sm.qc0 + i - sm.ns);
  }
  if (warp == 0) iter_consts_warp0(sm);
  __syncthreads();
}

// The serial tail of one unit's iteration (StateEstimator.hpp:535-580), run by ONE warp: finish the reduction, 6x6 gain
// system, update, convergence logic, and the constants of the unit's NEXT iteration.  The tails of the resident units
// run side by side on different warps.
__device__ void unit_tail(CtaMem& cta, Smem& sm, const BatchView& bv, const KParams& kp, const PassBuffers& pb, int slot, double sig2) {
  const int lane = threadIdx.x & 31;
  const int iter = sm.iter;
  lins_report* rep = bv.reports ? bv.reports + sm.scan : nullptr;
  const int nq = sm.ns + sm.nc;
  finish_acc_warp0(sm, pb.wacc + (size_t)slot * pb.nvw * kNAcc, pb.wcnt + (size_t)slot * pb.nvw * 2, (nq + 31) >> 5);
  build_A6_warp0(sm);
  if (slot == 0) LINS_TICK(18);
  if (lane < 6) {  // y = b6 + A6 d_c on the 6 structural rows
    double y = sm.y6[lane];
    for (int c = 0; c < 6; ++c) y += sm.A6[lane * 6 + c] * sm.dvec[col6(c)];
    sm.X6[lane] = y;
  }
  form_M6(sm, sig2, lane, 32);
  __syncwarp();
  const bool ok = warp_lu_cols<6>(sm.M6, sm.X6, 1);  // z = M^-1 (b6 + A6 d_c)
  __syncwarp();
  if (slot == 0) LINS_TICK(19);
  double u = 0.0;
  if (lane < 18) {  // K (r + H d) = P[:,c] z
    double kx = 0;
    for (int c = 0; c < 6; ++c) kx += sm.Pc[lane * 6 + c] * sm.X6[c];
    u = ok ? (-kx + sm.dvec[lane]) : __longlong_as_double(0x7ff8000000000000ll);
  }
  const bool hasNaN = __ballot_sync(0xffffffffu, u != u) != 0u;  // :553-558
  if (u != u) u = 0.0;
  if (lane < 18) sm.upd[lane] = u;
  __syncwarp();
  double nrm = 0.0;  // lane 0: ||update||^2 (sequential order), lane 1: ||residual||^2
  if (lane == 0) for (int a = 0; a < 18; ++a) nrm += sm.upd[a] * sm.upd[a];
  if (lane == 1) nrm = sm.acc[27];
  nrm = sqrt(nrm);
  const double un = __shfl_sync(0xffffffffu, nrm, 0), rnorm = __shfl_sync(0xffffffffu, nrm, 1);
  if (slot == 0) LINS_TICK(21);
  if (lane == 0) {
    if (rep) {
      rep->m_surf[iter] = sm.cnt[0]; rep->m_corner[iter] = sm.cnt[1];
      rep->residual_norm[iter] = rnorm; rep->update_norm[iter] = un;
    }
    if (hasNaN) {  // :559-563
      sm.flags[2] = 1; sm.flags[1] = 1; sm.flags[3] = 1;
    } else if (rnorm > sm.residualNorm * 10) {  // :566-570
      sm.flags[1] = 1; sm.flags[3] = 1;
    } else {
      box_plus(sm);  // :573
      if (un <= 1e-2 && !kp.force_all_iters) { sm.flags[0] = 1; sm.flags[3] = 1; }  // :576-578
      sm.residualNorm = rnorm;
    }
    const bool search = (iter % kp.icp_freq) == 0;
    if (search) sm.pos_is_slot = sm.az_ok; else if (!sm.pos_valid) sm.pos_is_slot = 0;
    sm.pos_valid = 1;
    sm.first_pass = 0;
    sm.iter = iter + 1;
    if (sm.flags[3] || iter + 1 >= kp.num_iter) { sm.finished = 1; sm.run = 0; cta.any_finished = 1; }
  }
  __syncwarp();
  if (slot == 0) LINS_TICK(23);
  if (!sm.finished) iter_consts_warp0(sm);
  if (slot == 0) LINS_TICK(25);
}

// exit of one finished unit: covariance + outputs (StateEstimator.hpp:585-599).  Block-wide.
__device__ void unit_exit(CtaMem& cta, Smem& sm, const BatchView& bv, double sig2) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int scan = sm.scan, iters = sm.iter;
  const bool diverged = sm.flags[1] != 0;
  auto& ex = cta.u.ex;
  if (!diverged && iters > 0) {
    // Joseph form with the LAST iteration's K, H, R (:595-596), all through the 6x6 system:
    //   K H = U E_c^T,  U = P[:,c] M^-1 A6 ;   K R K^T = sig2 U V^T,  V = P[:,c] M^-1
    for (int e = tid; e < 324; e += kThreads) {
      const int r = e / 18, c = e % 18;
      ex.P[e] = bv.cov_in[(size_t)scan * 324 + c * 18 + r];
    }
    form_M6(sm, sig2, tid, kThreads);
    for (int e = tid; e < 72; e += kThreads) {  // right-hand sides [A6 | I6]
      const int a = e / 12, c = e % 12;
      ex.X6[e] = c < 6 ? sm.A6[a * 6 + c] : (a == c - 6 ? 1.0 : 0.0);
    }
    __syncthreads();
    if (warp == 0) {
      const bool ok = warp_lu_cols<6>(sm.M6, ex.X6, 12);
      if (!ok) for (int e = lane; e < 72; e += 32) ex.X6[e] = __longlong_as_double(0x7ff8000000000000ll);
    }
    __syncthreads();
    for (int t = tid; t < 216; t += kThreads) {
      const int which = t / 108, e = t % 108, a = e / 6, c = e % 6;
      double sacc = 0;
      for (int k = 0; k < 6; ++k) sacc += sm.Pc[a * 6 + k] * ex.X6[k * 12 + c + 6 * which];
      (which ? ex.V : ex.U)[e] = sacc;
    }
    __syncthreads();
    for (int e = tid; e < 324; e += kThreads) {  // X = (I - K H) P = P - U P[c,:]
      const int i = e / 18, j = e % 18;
      double sacc = ex.P[e];
      for (int c = 0; c < 6; ++c) sacc -= ex.U[i * 6 + c] * ex.P[col6(c) * 18 + j];
      ex.X[e] = sacc;
    }
    __syncthreads();
    for (int e = tid; e < 324; e += kThreads) {  // P <- X (I - K H)^T + sig2 U V^T
      const int i = e / 18, j = e % 18;
      double sacc = ex.X[e], t = 0;
      for (int c = 0; c < 6; ++c) { sacc -= ex.X[i * 18 + col6(c)] * ex.U[j * 6 + c]; t += ex.U[i * 6 + c] * ex.V[j * 6 + c]; }
      ex.P[e] = sacc + t * sig2;
    }
    __syncthreads();
  }
  // state_out / cov_out
  if (tid < 20) bv.state_out[(size_t)scan * 20 + tid] = diverged ? sm.prior[tid] : sm.lin[tid];
  for (int e = tid; e < 324; e += kThreads) {
    const int r = e / 18, c = e % 18;
    double v;
    if (diverged || iters == 0) v = bv.cov_in[(size_t)scan * 324 + c * 18 + r];
    else v = 0.5 * (ex.P[r * 18 + c] + ex.P[c * 18 + r]);  // enforceSymmetry (:597)
    bv.cov_out[(size_t)scan * 324 + c * 18 + r] = v;
  }
  if (tid == 0) {
    lins_scan_result& o = bv.results[scan];
    o.scan_id = scan;
    o.iters = (uint16_t)iters;
    o.flags = (uint16_t)((sm.flags[0] ? 1 : 0) | (sm.flags[1] ? 2 : 0) | (sm.flags[2] ? 4 : 0));
    const double* st = diverged ? sm.prior : sm.lin;
    o.pose[0] = st[0]; o.pose[1] = st[1]; o.pose[2] = st[2];
    o.pose[3] = st[6]; o.pose[4] = st[7]; o.pose[5] = st[8]; o.pose[6] = st[9];
    lins_report* rep = bv.reports ? bv.reports + scan : nullptr;
    if (rep) { rep->iters = iters; rep->converged = sm.flags[0]; rep->diverged = sm.flags[1]; rep->has_nan = sm.flags[2]; }
  }
  __syncthreads();  // (ex is reused by the next finished unit / the next prologue)
}

template <int MODE>
__global__ void __launch_bounds__(kThreads, kMinCtas) lins_ieskf_kernel(const __grid_constant__ BatchView bv,
                                                                     const __grid_constant__ KParams kp) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int S = bv.nslots;
  PassBuffers pb;
  const PassLayout lay = pass_layout(S, bv.qtile, &pb, smem_raw, bv.qscratch, blockIdx.x, bv.qscratch_stride);
  CtaMem& cta = *reinterpret_cast<CtaMem*>(smem_raw);
  Smem* slots = reinterpret_cast<Smem*>(smem_raw + lay.slots);
  const int tid = threadIdx.x, warp = tid >> 5;
  const double sig2 = kp.lidar_std * kp.lidar_std;

  if (tid == 0) {
    mbar_init(&cta.mbar, 1);
    cta.phase = 0;
    cta.wl_n[0] = 0; cta.wl_n[1] = 0; cta.wl_tn[0] = 0; cta.wl_tn[1] = 0; cta.wl_thead[0] = 0; cta.wl_thead[1] = 0; cta.wl_head[0] = 0; cta.wl_head[1] = 0; cta.dbg[0] = 0; cta.dbg[1] = 0;  // (reset after every pass)
    cta.exhausted = 0; cta.any_finished = 0;
    for (int s = 0; s < S; ++s) { slots[s].scan = -1; slots[s].fresh = 0; slots[s].run = 0; slots[s].finished = 0; }
    fence_mbar_init();
    cta.tlast = clock64();
  }
  __syncthreads();
  const long long t_cta0 = clock64();

  for (;;) {
    // ---- claim units for the free slots ------------------------------------------------------------------------------
    if (tid == 0) {
      int nact = 0, nfresh = 0;
      for (int s = 0; s < S; ++s) {
        Smem& sm = slots[s];
        if (MODE == MODE_ICP_REDUCE) {  // a unit whose Gauss-Newton loop has ended is passed over (the queued tail of its loop)
          while (sm.scan < 0 && !cta.exhausted) {
            const int u = atomicAdd(bv.work_counter, 1);
            if (u >= bv.n_scans) cta.exhausted = 1;
            else if (!bv.icp_done || !bv.icp_done[(size_t)u * kIcpDoneStride]) { sm.scan = u; sm.fresh = 1; }
          }
        } else if (sm.scan < 0 && !cta.exhausted) {
          const int u = atomicAdd(bv.work_counter, 1);
          if (u < bv.n_scans) { sm.scan = u; sm.fresh = 1; } else cta.exhausted = 1;
        }
        if (sm.scan >= 0) ++nact;
        if (sm.fresh) ++nfresh;
      }
      cta.n_active = nact; cta.any_fresh = nfresh;
      cta.pass_first = 0;
      if (bv.timers) {  // diagnostics: does this pass contain a unit's first pass (every query searches)?
        int nrun = 0;
        for (int s = 0; s < S; ++s) { if (slots[s].fresh || (slots[s].run && slots[s].first_pass)) cta.pass_first = 1; if (slots[s].scan >= 0) ++nrun; }
        atomicAdd((unsigned long long*)&bv.timers[cta.pass_first ? 62 : 30], 1ull);
        atomicAdd((unsigned long long*)&bv.timers[cta.pass_first ? 63 : 31], (unsigned long long)nrun);
      }
    }
    __syncthreads();
    if (cta.n_active == 0) {
      if (bv.timers && tid == 0) {  // busy time of this CTA: sum and max over CTAs give the tail imbalance
        const unsigned long long busy = (unsigned long long)(clock64() - t_cta0);
        atomicAdd((unsigned long long*)&bv.timers[26], busy);
        atomicMax((unsigned long long*)&bv.timers[27], busy);
      }
      break;
    }
    LINS_TICK(1);
    if (cta.any_fresh) {
      for (int s = 0; s < S; ++s)
        if (slots[s].fresh) unit_prologue<MODE>(cta, slots[s], bv, kp, pb, s);
      if (tid == 0) {
        int leg = 0, idx = 0;
        for (int s = 0; s < S; ++s) if (slots[s].scan >= 0) { if (slots[s].az_ok) idx = 1; else leg = 1; }
        cta.any_legacy = leg; cta.any_indexed = idx;
      }
      __syncthreads();
      LINS_TICK(0);
    }

    // ---- one pass of every resident unit (StateEstimator.hpp:475-581) -----------------------------------------------
    association_pass<MODE>(cta, slots, bv, kp, pb);
    if (MODE == MODE_IESKF) {
      if (warp < S && slots[warp].run) unit_tail(cta, slots[warp], bv, kp, pb, warp, sig2);
    } else {
      if (warp < S && slots[warp].run) {  // single-pass modes: the 28 sums + counts are the result
        Smem& sm = slots[warp];
        const int lane = tid & 31;
        const int scan = sm.scan;
        finish_acc_warp0(sm, pb.wacc + (size_t)warp * pb.nvw * kNAcc, pb.wcnt + (size_t)warp * pb.nvw * 2, (sm.ns + sm.nc + 31) >> 5);
        if (bv.accum) {
          if (lane < kNAcc) bv.accum[(size_t)scan * 32 + lane] = sm.acc[lane];
          if (lane == 28) bv.accum[(size_t)scan * 32 + 28] = (double)sm.cnt[0];
          if (lane == 29) bv.accum[(size_t)scan * 32 + 29] = (double)sm.cnt[1];
        }
        __syncwarp();
        if (lane == 0) { sm.scan = -1; sm.run = 0; }
      }
    }
    __syncthreads();
    LINS_TICK(8);
    if (MODE == MODE_IESKF && cta.any_finished) {
      for (int s = 0; s < S; ++s) {
        if (!slots[s].finished) continue;  // (uniform: shared flag)
        unit_exit(cta, slots[s], bv, sig2);
        if (tid == 0) { slots[s].scan = -1; slots[s].finished = 0; slots[s].run = 0; }
      }
      if (tid == 0) cta.any_finished = 0;
      __syncthreads();
      LINS_TICK(9);
    }
  }
}


// F1: transformToEnd (StateEstimator.hpp:1083-1101).  The per-scan constants (block-wide, into shared memory) and the
// per-point body, shared by the single-cloud kernel and the CSR kernel of sequence mode.
__device__ __forceinline__ void to_end_consts(const double* __restrict__ lin, double* sphi, double* srn, double* sq) {
  if (threadIdx.x == 0) {
    q4 q; q.x = lin[6]; q.y = lin[7]; q.z = lin[8]; q.w = lin[9];
    d3 phi = Quat2axis(q);
    sphi[0] = phi.x; sphi[1] = phi.y; sphi[2] = phi.z;
    srn[0] = lin[0]; srn[1] = lin[1]; srn[2] = lin[2];
    sq[0] = q.x; sq[1] = q.y; sq[2] = q.z; sq[3] = q.w;
  }
  __syncthreads();
}
__device__ __forceinline__ float4 to_end_point(float4 p, const double* sphi, const double* srn, const double* sq, double scan_period) {
  float fi = p.w - (float)((int)p.w);
  double s = (1.f / scan_period) * fi;
  q4 r = axis2Quat(mk3(s * sphi[0], s * sphi[1], s * sphi[2]));
  d3 P1 = add3(qrot(r, mk3(p.x, p.y, p.z)), mk3(s * srn[0], s * srn[1], s * srn[2]));
  q4 q; q.x = sq[0]; q.y = sq[1]; q.z = sq[2]; q.w = sq[3];
  d3 P2 = qrot(qinverse(q), sub3(P1, mk3(srn[0], srn[1], srn[2])));
  p.x = (float)P2.x; p.y = (float)P2.y; p.z = (float)P2.z;
  return p;
}

// CSR version: one block per unit u with run[u] != 0, its cloud pts[off[u], off[u+1]) with linState_ lin[20 u ..].
__global__ void lins_transform_to_end_csr_kernel(float4* __restrict__ pts, const int* __restrict__ off, const double* __restrict__ lin,
                                                 const unsigned char* __restrict__ run, double scan_period) {
  __shared__ double sphi[3], srn[3], sq[4];
  const int u = blockIdx.x;
  if (!run[u]) return;
  to_end_consts(lin + (size_t)u * 20, sphi, srn, sq);
  for (int i = off[u] + threadIdx.x; i < off[u + 1]; i += blockDim.x) pts[i] = to_end_point(pts[i], sphi, srn, sq, scan_period);
}

// in place on a packed cloud; out32 (optional) receives full PointXYZI records
__global__ void lins_transform_to_end_kernel(float4* __restrict__ pts, int n, const double* __restrict__ lin,
                                             double scan_period, lins_point* __restrict__ out32) {
  __shared__ double sphi[3], srn[3], sq[4];
  to_end_consts(lin, sphi, srn, sq);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = to_end_point(pts[i], sphi, srn, sq, scan_period);
  pts[i] = p;
  if (out32) {  // full pcl::PointXYZI records for a straight D2H into the caller's cloud
    float4* o = reinterpret_cast<float4*>(out32 + i);
    o[0] = make_float4(p.x, p.y, p.z, 1.0f);
    o[1] = make_float4(p.w, 0.f, 0.f, 0.f);
  }
}

// ---------------------------------------------------------------------------------------------------------
// host-side helpers
// ---------------------------------------------------------------------------------------------------------
KParams make_kparams(const lins_params& p, int mode, int iter0) {
  KParams k;
  k.num_iter = p.num_iter; k.icp_freq = p.icp_freq < 1 ? 1 : p.icp_freq; k.force_all_iters = p.force_all_iters;
  k.mode = mode; k.iter0 = iter0;
  k.nearest_sq = p.nearest_feature_search_sq_dist; k.lidar_std = p.lidar_std; k.lidar_scale = p.lidar_scale;
  k.scan_period = p.scan_period;
  return k;
}

int validate_params(const lins_params* p) {
  if (!p) return LINS_E_INVALID;
  if (p->num_iter < 0 || p->num_iter > LINS_MAX_ITER) return LINS_E_INVALID;
  if (p->icp_freq < 1) return LINS_E_INVALID;
  if (!(p->scan_period > 0)) return LINS_E_INVALID;
  return LINS_OK;
}

template <int MODE>
int launch_mode(lins_ctx* ctx, Resident& r, const BatchView& bv_in, const KParams& kp) {
  BatchView bv = bv_in;
  // resident units per CTA: as many as fit shared memory (per-query arrays of every slot + fixed part), but no more
  // than the batch can fill on every SM
  const int limit = ctx->max_smem_optin;
  int want = std::min(kMaxSlots, std::max(1, (bv.n_scans + ctx->sm_count - 1) / ctx->sm_count));
  if (ctx->force_slots > 0) want = std::min(kMaxSlots, ctx->force_slots);
  int S = want;
  PassLayout lay = pass_layout(S, bv.qtile);
  while (S > 1 && (int)(lay.fixed_bytes + lay.query_bytes) > limit) lay = pass_layout(--S, bv.qtile);
  size_t smem = lay.fixed_bytes + lay.query_bytes;
  bv.qscratch = nullptr; bv.qscratch_stride = 0;
  if ((int)smem > limit) {  // even one unit's per-query arrays exceed shared memory: keep them in a per-CTA global scratch
    smem = lay.fixed_bytes;
    if ((int)smem > limit) return fail(ctx, LINS_E_TOOBIG, "unit too large for the fused kernel");
    bv.qscratch_stride = lay.query_bytes;
  }
  bv.nslots = S;
  CK(cudaFuncSetAttribute(lins_ieskf_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lins_ieskf_kernel<MODE>, kThreads, smem));
  if (per_sm < 1) per_sm = 1;
  int grid = std::min((bv.n_scans + S - 1) / S, ctx->sm_count * per_sm);
  if (grid < 1) grid = 1;
  if (bv.qscratch_stride) {
    CK(r.qscratch.reserve(bv.qscratch_stride * (size_t)grid));
    bv.qscratch = r.qscratch.p;
  }
  if (ctx->verbose) std::fprintf(stderr, "[lins_gpu] mode %d: %d threads, %zu B shared, %d CTA/SM, grid %d, slots %d qtile %d%s\n", MODE, kThreads, smem, per_sm, grid, S, bv.qtile, bv.qscratch ? " (per-query arrays in global scratch)" : "");
  CK(cudaMemsetAsync(bv.work_counter, 0, sizeof(int), ctx->stream));
  lins_ieskf_kernel<MODE><<<grid, kThreads, smem, ctx->stream>>>(bv, kp);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return LINS_OK;
}

int launch(lins_ctx* ctx, Resident& r, const BatchView& bv, const KParams& kp) {
  switch (kp.mode) {
    case MODE_IESKF: return launch_mode<MODE_IESKF>(ctx, r, bv, kp);
    case MODE_ASSOC: return launch_mode<MODE_ASSOC>(ctx, r, bv, kp);
    case MODE_ICP_REDUCE: return launch_mode<MODE_ICP_REDUCE>(ctx, r, bv, kp);
  }
  return fail(ctx, LINS_E_INVALID, "bad kernel mode");
}

int choose_qtile(int max_q) {
  int q = ((max_q + 31) / 32) * 32;
  if (q < 32) q = 32;
  return q;
}

BatchView view_of(const Resident& r, bool reports, bool trace) {
  BatchView bv;
  std::memset(&bv, 0, sizeof(bv));
  bv.n_scans = r.n;
  bv.qs = r.qs.p; bv.qs_off = r.qs_off.p; bv.qc = r.qc.p; bv.qc_off = r.qc_off.p;
  bv.ts = r.ts.p; bv.ts_off = r.ts_off.p; bv.tc = r.tc.p; bv.tc_off = r.tc_off.p;
  bv.state_in = r.state_in.p; bv.cov_in = r.cov_in.p; bv.state_out = r.state_out.p; bv.cov_out = r.cov_out.p;
  bv.results = r.results.p; bv.reports = reports ? r.reports.p : nullptr;
  bv.ind_s = r.ind_s.p; bv.ind_c = r.ind_c.p;
  bv.az_s = r.az_s.p; bv.az_c = r.az_c.p;
  if (trace) {
    bv.sel_s = r.sel_s.p; bv.sel_c = r.sel_c.p; bv.coeff_s = r.coeff_s.p; bv.coeff_c = r.coeff_c.p;
    bv.mask_s = r.mask_s.p; bv.mask_c = r.mask_c.p;
  }
  bv.accum = r.accum.p;
  bv.work_counter = r.counter.p;
  bv.qtile = choose_qtile(r.max_q);
  return bv;
}

// Upload the queries + prior of ONE scan into ctx->single and point its targets at the resident map.
int stage_single(lins_ctx* ctx, const lins_point* surf_flat, int ns, const lins_point* corner_sharp, int nc,
                 const double* state_in, const double* cov_in, bool trace) {
  if (ctx->map_ns < 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_set_map has not been called");
  if (check_cloud(ctx, surf_flat, ns, "bad surf_flat cloud") != LINS_OK || check_cloud(ctx, corner_sharp, nc, "bad corner_sharp cloud") != LINS_OK)
    return LINS_E_INVALID;
  Resident& r = ctx->single;
  r.n = 1; r.nqs = ns; r.nqc = nc; r.max_q = ns + nc;
  CK(r.qs.reserve(ns + 1)); CK(r.qc.reserve(nc + 1));
  CK(r.qs_off.reserve(2)); CK(r.qc_off.reserve(2));
  CK(r.state_in.reserve(20)); CK(r.cov_in.reserve(324));
  CK(r.h_pts.reserve((size_t)ns + nc + 1)); CK(r.h_off.reserve(4)); CK(r.h_state.reserve(20)); CK(r.h_cov.reserve(324));
  pack_into(r.h_pts.p, surf_flat, ns);
  pack_into(r.h_pts.p + ns, corner_sharp, nc);
  r.h_off.p[0] = 0; r.h_off.p[1] = ns; r.h_off.p[2] = 0; r.h_off.p[3] = nc;
  pad_states(r.h_state.p, state_in, 1);
  if (cov_in) std::memcpy(r.h_cov.p, cov_in, sizeof(double) * 324); else std::memset(r.h_cov.p, 0, sizeof(double) * 324);
  if (ns) CK(cudaMemcpyAsync(r.qs.p, r.h_pts.p, sizeof(float4) * ns, cudaMemcpyHostToDevice, ctx->stream));
  if (nc) CK(cudaMemcpyAsync(r.qc.p, r.h_pts.p + ns, sizeof(float4) * nc, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(r.qs_off.p, r.h_off.p, sizeof(int) * 2, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(r.qc_off.p, r.h_off.p + 2, sizeof(int) * 2, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(r.state_in.p, r.h_state.p, sizeof(double) * 20, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(r.cov_in.p, r.h_cov.p, sizeof(double) * 324, cudaMemcpyHostToDevice, ctx->stream));
  r.nts = (size_t)std::max(std::max(ctx->map_ns, ctx->tree_ns), 0);
  r.ntc = (size_t)std::max(std::max(ctx->map_nc, ctx->tree_nc), 0);
  return reserve_outputs(ctx, r, true, trace);
}

BatchView single_view(lins_ctx* ctx, bool trace) {
  BatchView bv = view_of(ctx->single, true, trace);
  bv.ts = ctx->map_s.p; bv.ts_off = ctx->map_off.p + 0;
  bv.tc = ctx->map_c.p; bv.tc_off = ctx->map_off.p + 2;
  if (!ctx->tree_is_map) {
    bv.nn_s = ctx->tree_s.p; bv.nn_s_off = ctx->map_off.p + 4;
    bv.nn_c = ctx->tree_c.p; bv.nn_c_off = ctx->map_off.p + 6;
  }
  return bv;
}

int upload_map_offsets(lins_ctx* ctx) {
  CK(ctx->map_off.reserve(8));
  int h[8] = {0, ctx->map_ns, 0, ctx->map_nc, 0, ctx->tree_ns, 0, ctx->tree_nc};
  // (h is pageable stack memory: cudaMemcpyAsync returns once it has been copied to the driver's staging buffer)
  CK(cudaMemcpyAsync(ctx->map_off.p, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
  return LINS_OK;
}

// r's outputs into the caller's arrays (each may be null; states as ABI rows) through r's pinned staging: one synchronisation
int download_outputs(lins_ctx* ctx, Resident& r, double* state_out, double* cov_out, lins_scan_result* results, lins_report* reports) {
  const size_t n = r.n;
  if (state_out) { CK(r.h_state_out.reserve(n * 20)); CK(cudaMemcpyAsync(r.h_state_out.p, r.state_out.p, sizeof(double) * 20 * n, cudaMemcpyDeviceToHost, ctx->stream)); }
  if (cov_out) { CK(r.h_cov_out.reserve(n * 324)); CK(cudaMemcpyAsync(r.h_cov_out.p, r.cov_out.p, sizeof(double) * 324 * n, cudaMemcpyDeviceToHost, ctx->stream)); }
  if (results) { CK(r.h_results.reserve(n)); CK(cudaMemcpyAsync(r.h_results.p, r.results.p, sizeof(lins_scan_result) * n, cudaMemcpyDeviceToHost, ctx->stream)); }
  if (reports) { CK(r.h_reports.reserve(n)); CK(cudaMemcpyAsync(r.h_reports.p, r.reports.p, sizeof(lins_report) * n, cudaMemcpyDeviceToHost, ctx->stream)); }
  CK(cudaStreamSynchronize(ctx->stream));
  if (state_out) strip_states(state_out, r.h_state_out.p, n);
  if (cov_out) std::memcpy(cov_out, r.h_cov_out.p, sizeof(double) * 324 * n);
  if (results) std::memcpy(results, r.h_results.p, sizeof(lins_scan_result) * n);
  if (reports) std::memcpy(reports, r.h_reports.p, sizeof(lins_report) * n);
  return LINS_OK;
}

// the correspondence IDs of r's last IESKF / association (each destination may be null); one stream synchronisation
int download_indices(lins_ctx* ctx, const Resident& r, int32_t* surf_ind, int32_t* corner_ind) {
  CK(cudaSetDevice(ctx->device));
  CK(d2h(ctx, surf_ind, r.ind_s.p, sizeof(int32_t) * 3 * r.nqs));
  CK(d2h(ctx, corner_ind, r.ind_c.p, sizeof(int32_t) * 2 * r.nqc));
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}

}  // namespace

// ---- what sequence mode (lins_seq.cu) runs of this unit: lins_ctx.hpp declares these ------------------------------------
namespace lins_capi {

int fused_ieskf_launch(lins_ctx* ctx, Resident& r, const BatchView& bv) {
  return launch(ctx, r, bv, make_kparams(ctx->prm, MODE_IESKF, 0));
}

int fused_qtile(int max_q) { return choose_qtile(max_q); }

size_t icp_state_bytes() { return sizeof(IcpState); }

// the Gauss-Newton loop of estimateTransform on the bv.n_scans units of bv, whose queries, maps and poses (pose: 20 doubles
// per unit, the linearisation point) are on the device: every iteration is one reduction launch over all units
// (MODE_ICP_REDUCE) + one step launch with a block per unit that updates the unit's pose.  icp holds one IcpState per unit,
// set by the caller: zero = run, done = 1 = skip.  Once a unit's step sets `done`, the remaining queued launches pass it
// over.  No synchronisation.
int icp_loop(lins_ctx* ctx, Resident& r, BatchView bv, double* pose, IcpState* icp) {
  bv.state_in = pose;
  bv.icp_done = &icp->done;
  for (int iter = 0; iter < ctx->prm.num_iter; ++iter) {
    const int rc = launch(ctx, r, bv, make_kparams(ctx->prm, MODE_ICP_REDUCE, iter));
    if (rc != LINS_OK) return rc;
    lins_icp_step_kernel<<<bv.n_scans, 32, 0, ctx->stream>>>(bv.accum, pose, icp, iter);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  return LINS_OK;
}

int transform_to_end_csr(lins_ctx* ctx, float4* pts, const int* off, int n_units, const double* lin, const unsigned char* run) {
  if (n_units <= 0) return LINS_OK;
  lins_transform_to_end_csr_kernel<<<n_units, 256, 0, ctx->stream>>>(pts, off, lin, run, ctx->prm.scan_period);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return LINS_OK;
}

}  // namespace lins_capi

// =========================================================================================================
// C-ABI
// =========================================================================================================
extern "C" {

int lins_gpu_abi_version(void) { return 1; }

int lins_gpu_create(const lins_params* params, int device, void* stream, lins_ctx** out) {
  if (!out) return LINS_E_INVALID;
  *out = nullptr;
  if (validate_params(params) != LINS_OK) return LINS_E_INVALID;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return LINS_E_NODEVICE;
  if (cudaSetDevice(device) != cudaSuccess) return LINS_E_NODEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return LINS_E_NODEVICE;
  if (prop.major != 9) return LINS_E_NODEVICE;  // the fatbin holds sm_90a code only
  lins_ctx* ctx = new (std::nothrow) lins_ctx();
  if (!ctx) return LINS_E_INVALID;
  ctx->device = device;
  ctx->prm = *params;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  ctx->verbose = std::getenv("LINS_VERBOSE") != nullptr;
  if (const char* e = std::getenv("LINS_SLOTS")) ctx->force_slots = std::atoi(e);
  if (stream) { ctx->stream = (cudaStream_t)stream; ctx->own_stream = false; }
  else {
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return LINS_E_CUDA; }
    ctx->own_stream = true;
  }
  *out = ctx;
  return LINS_OK;
}

void lins_gpu_destroy(lins_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->tmp_ev) cudaEventDestroy(ctx->tmp_ev);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;  // (frees every buffer)
}

const char* lins_gpu_last_error(const lins_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

int lins_gpu_set_params(lins_ctx* ctx, const lins_params* params) {
  if (!ctx) return LINS_E_INVALID;
  if (validate_params(params) != LINS_OK) return fail(ctx, LINS_E_INVALID, "bad params");
  ctx->prm = *params;
  return LINS_OK;
}

int64_t lins_gpu_launch_count(const lins_ctx* ctx) { return ctx ? ctx->launches : 0; }

int lins_gpu_set_map(lins_ctx* ctx, const lins_point* surf, int ns, const lins_point* corner, int nc) {
  if (!ctx) return LINS_E_INVALID;
  if (check_cloud(ctx, surf, ns, "bad surf map cloud") != LINS_OK || check_cloud(ctx, corner, nc, "bad corner map cloud") != LINS_OK)
    return LINS_E_INVALID;
  CK(cudaSetDevice(ctx->device));
  const int rc = upload2(ctx, ctx->map_s, surf, ns, ctx->map_c, corner, nc);
  if (rc != LINS_OK) return rc;
  ctx->map_ns = ns; ctx->map_nc = nc; ctx->tree_ns = ns; ctx->tree_nc = nc; ctx->tree_is_map = true;
  return upload_map_offsets(ctx);
}

int lins_gpu_ieskf(lins_ctx* ctx, const lins_point* surf_flat, int ns, const lins_point* corner_sharp, int nc,
                   const double* state_in, const double* cov_in, double* state_out, double* cov_out, lins_report* rep) {
  if (!ctx) return LINS_E_INVALID;
  if (!state_in || !cov_in) return fail(ctx, LINS_E_INVALID, "null prior");
  CK(cudaSetDevice(ctx->device));
  int rc = stage_single(ctx, surf_flat, ns, corner_sharp, nc, state_in, cov_in, false);
  if (rc != LINS_OK) return rc;
  Resident& r = ctx->single;
  BatchView bv = single_view(ctx, false);
  CK(cudaMemsetAsync(r.reports.p, 0, sizeof(lins_report), ctx->stream));
  rc = launch(ctx, r, bv, make_kparams(ctx->prm, MODE_IESKF, 0));
  if (rc != LINS_OK) return rc;
  return download_outputs(ctx, r, state_out, cov_out, nullptr, rep);
}

int lins_gpu_download_indices(lins_ctx* ctx, int32_t* surf_ind, int32_t* corner_ind) {
  if (!ctx) return LINS_E_INVALID;
  if (ctx->single.n != 1 || !ctx->single.ind_s.p) return fail(ctx, LINS_E_INVALID, "no single-scan call has run");
  return download_indices(ctx, ctx->single, surf_ind, corner_ind);
}

int lins_gpu_associate(lins_ctx* ctx, const lins_point* surf_flat, int ns, const lins_point* corner_sharp, int nc,
                       const double* lin_state, int iter, int32_t* surf_ind, int32_t* corner_ind, float* surf_coeff,
                       float* corner_coeff, uint8_t* surf_mask, uint8_t* corner_mask, float* surf_sel, float* corner_sel) {
  if (!ctx) return LINS_E_INVALID;
  if (!lin_state || iter < 0) return fail(ctx, LINS_E_INVALID, "bad lin_state / iter");
  CK(cudaSetDevice(ctx->device));
  // pointSearch*Ind persist on device between calls (buffers are only re-allocated when they must grow)
  int rc = stage_single(ctx, surf_flat, ns, corner_sharp, nc, lin_state, nullptr, true);
  if (rc != LINS_OK) return rc;
  Resident& r = ctx->single;
  BatchView bv = single_view(ctx, true);
  rc = launch(ctx, r, bv, make_kparams(ctx->prm, MODE_ASSOC, iter));
  if (rc != LINS_OK) return rc;
  CK(d2h(ctx, surf_ind, r.ind_s.p, sizeof(int) * 3 * ns));
  CK(d2h(ctx, corner_ind, r.ind_c.p, sizeof(int) * 2 * nc));
  CK(d2h(ctx, surf_coeff, r.coeff_s.p, sizeof(float) * 4 * ns));
  CK(d2h(ctx, corner_coeff, r.coeff_c.p, sizeof(float) * 4 * nc));
  CK(d2h(ctx, surf_mask, r.mask_s.p, ns));
  CK(d2h(ctx, corner_mask, r.mask_c.p, nc));
  CK(d2h(ctx, surf_sel, r.sel_s.p, sizeof(float) * 3 * ns));
  CK(d2h(ctx, corner_sel, r.sel_c.p, sizeof(float) * 3 * nc));
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}


// ---- batched mode (lins_gpu_batch_upload: lins_upload.cu) -------------------------------------------------
int lins_gpu_batch_run(lins_ctx* ctx) {
  if (!ctx) return LINS_E_INVALID;
  Resident& r = ctx->batch;
  if (r.n <= 0) return fail(ctx, LINS_E_INVALID, "no resident batch");
  CK(cudaSetDevice(ctx->device));
  BatchView bv = view_of(r, true, false);
  if (ctx->timers_on) {
    CK(r.timers.reserve(64));
    CK(cudaMemsetAsync(r.timers.p, 0, sizeof(long long) * 64, ctx->stream));
    bv.timers = r.timers.p;
  }
  return launch(ctx, r, bv, make_kparams(ctx->prm, MODE_IESKF, 0));
}

int lins_gpu_batch_download(lins_ctx* ctx, double* state_out, double* cov_out, lins_scan_result* results,
                            lins_report* reports) {
  if (!ctx) return LINS_E_INVALID;
  if (ctx->batch.n <= 0) return fail(ctx, LINS_E_INVALID, "no resident batch");
  CK(cudaSetDevice(ctx->device));
  return download_outputs(ctx, ctx->batch, state_out, cov_out, results, reports);
}

int lins_gpu_batch_download_indices(lins_ctx* ctx, int32_t* surf_ind, int32_t* corner_ind) {
  if (!ctx) return LINS_E_INVALID;
  if (ctx->batch.n <= 0) return fail(ctx, LINS_E_INVALID, "no resident batch");
  return download_indices(ctx, ctx->batch, surf_ind, corner_ind);
}

int lins_gpu_ieskf_batch(lins_ctx* ctx, const lins_batch_desc* batch, double* state_out, double* cov_out,
                         lins_scan_result* results) {
  int rc = lins_gpu_batch_upload(ctx, batch);
  if (rc != LINS_OK) return rc;
  if (batch->n_scans == 0) return LINS_OK;
  rc = lins_gpu_batch_run(ctx);
  if (rc != LINS_OK) return rc;
  return lins_gpu_batch_download(ctx, state_out, cov_out, results, nullptr);
}

int lins_gpu_batch_results_device(lins_ctx* ctx, void** dev_ptr, int* n_scans) {
  if (!ctx || !dev_ptr) return LINS_E_INVALID;
  *dev_ptr = ctx->batch.results.p;
  if (n_scans) *n_scans = ctx->batch.n;
  return LINS_OK;
}

// Diagnostics: enable per-phase cycle counters for lins_gpu_batch_run (enable != 0), and/or read the 32
// counters of the last run (out may be NULL).  Slot meaning: see LINS_TICK sites in lins_gpu.cu / lins_kernels.cuh.
int lins_gpu_debug_phase_cycles(lins_ctx* ctx, int enable, long long* out) {
  if (!ctx) return LINS_E_INVALID;
  CK(cudaSetDevice(ctx->device));
  if (out) {
    if (!ctx->batch.timers.p) return fail(ctx, LINS_E_INVALID, "timers were not enabled for the last run");
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaMemcpy(out, ctx->batch.timers.p, sizeof(long long) * 64, cudaMemcpyDeviceToHost));
  }
  ctx->timers_on = enable != 0;
  return LINS_OK;
}


int lins_gpu_host_register(void* ptr, size_t bytes) {
  if (!ptr || bytes == 0) return LINS_E_INVALID;
  const cudaError_t e = cudaHostRegister(ptr, bytes, cudaHostRegisterPortable);
  if (e != cudaSuccess) { cudaGetLastError(); return e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? LINS_E_NODEVICE : LINS_E_CUDA; }
  return LINS_OK;
}
int lins_gpu_host_unregister(void* ptr) {
  if (!ptr) return LINS_E_INVALID;
  const cudaError_t e = cudaHostUnregister(ptr);
  if (e != cudaSuccess) { cudaGetLastError(); return LINS_E_CUDA; }
  return LINS_OK;
}

int lins_gpu_sync(lins_ctx* ctx) {
  if (!ctx) return LINS_E_INVALID;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}


int lins_gpu_batch_jacobian_pass(lins_ctx* ctx, double* accum_out) {
  if (!ctx) return LINS_E_INVALID;
  Resident& r = ctx->batch;
  if (r.n <= 0) return fail(ctx, LINS_E_INVALID, "no resident batch");
  CK(cudaSetDevice(ctx->device));
  BatchView bv = view_of(r, false, false);
  bv.state_in = r.state_out.p;  // linearise at the updated state; IDs = the last iteration's
  KParams kp = make_kparams(ctx->prm, MODE_JACOBIAN, 1);
  // lins_jacobian.cu: FP64 tensor-core fold, multiply-add contraction
  const int P = lins_jacobian_parts(r.n, ctx->sm_count);
  if (P > 1) { CK(r.jac_part.reserve((size_t)r.n * P * 32)); CK(r.jac_cnt.reserve((size_t)r.n)); }
  const int e = lins_launch_jacobian_mma(&bv, &kp, r.n, ctx->sm_count, P, r.jac_part.p, r.jac_cnt.p, ctx->stream);
  if (e != 0) return fail(ctx, LINS_E_CUDA, "jacobian kernel launch", (cudaError_t)e);
  CK(cudaGetLastError());
  ctx->launches += 1;
  if (accum_out) {
    // the device rows are 32 doubles apart; the caller's are the 30 the header documents
    CK(r.h_accum.reserve((size_t)r.n * 32));
    CK(cudaMemcpy2DAsync(r.h_accum.p, sizeof(double) * 30, r.accum.p, sizeof(double) * 32, sizeof(double) * 30, (size_t)r.n,
                         cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::memcpy(accum_out, r.h_accum.p, sizeof(double) * 30 * (size_t)r.n);
  }
  return LINS_OK;
}

// ≙ estimateTransform (StateEstimator.hpp:1163-1196): the association + J^T J / J^T b reduction of every
// Gauss-Newton step runs on device (MODE_ICP_REDUCE), and so do the 6x6 solve / degeneracy projection / pose update of
// calculateTransformation (:1260-1320): lins_icp_step.cuh.
int lins_gpu_estimate_transform(lins_ctx* ctx, const lins_point* surf_flat, int ns, const lins_point* corner_sharp,
                                int nc, double* pose_io, int* iters_out, int* converged_out) {
  if (!ctx) return LINS_E_INVALID;
  if (!pose_io) return fail(ctx, LINS_E_INVALID, "null pose");
  CK(cudaSetDevice(ctx->device));
  // queries + initial pose are staged ONCE, then the loop runs on the device (icp_loop).  One D2H + one synchronisation
  // at the end.
  double lin[19] = {};
  pose_to_state(pose_io, lin);
  int rc = stage_single(ctx, surf_flat, ns, corner_sharp, nc, lin, nullptr, false);
  if (rc != LINS_OK) return rc;
  Resident& r = ctx->single;
  CK(r.icp.reserve(1)); CK(r.h_icp.reserve(1)); CK(r.h_state_out.reserve(20));
  CK(cudaMemsetAsync(r.icp.p, 0, sizeof(IcpState), ctx->stream));
  rc = icp_loop(ctx, r, single_view(ctx, false), r.state_in.p, r.icp.p);
  if (rc != LINS_OK) return rc;
  CK(cudaMemcpyAsync(r.h_state_out.p, r.state_in.p, sizeof(double) * 20, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(r.h_icp.p, r.icp.p, sizeof(IcpState), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  state_to_pose(r.h_state_out.p, pose_io);
  if (iters_out) *iters_out = r.h_icp.p->iters;
  if (converged_out) *converged_out = r.h_icp.p->converged;
  return LINS_OK;
}

// ≙ updatePointCloud (StateEstimator.hpp:1116-1161), XYZ part: transformToEnd on the device, then the map swap + the
// guarded index refresh.  The clouds stay on the device as the next map; copying them back is optional (the reference
// transforms scan_new_'s clouds in place because the mapping node consumes them) and, when asked for, is one D2H of
// full PointXYZI records straight into the caller's clouds — one stream synchronisation per call, none without read-back.
int lins_gpu_update_map_ex(lins_ctx* ctx, const lins_point* surf, int ns, const lins_point* corner, int nc, const double* lin_state,
                           lins_point* surf_out, lins_point* corner_out, int* map_replaced) {
  if (!ctx) return LINS_E_INVALID;
  if (check_cloud(ctx, surf, ns, "bad update_map surf cloud") != LINS_OK || check_cloud(ctx, corner, nc, "bad update_map corner cloud") != LINS_OK)
    return LINS_E_INVALID;
  CK(cudaSetDevice(ctx->device));
  const double* lin_dev = nullptr;
  if (!lin_state) {  // the posterior the last lins_gpu_ieskf left on the device (linState_ of a run that did not diverge)
    if (ctx->single.n != 1 || !ctx->single.state_out.p) return fail(ctx, LINS_E_INVALID, "no device-resident state: call lins_gpu_ieskf first or pass lin_state");
    lin_dev = ctx->single.state_out.p;
  }
  const bool rebuild = nc >= 5 && ns >= 20;  // :1156-1157
  const bool want_out = (ns > 0 && surf_out) || (nc > 0 && corner_out);
  // every allocation first: the context is only changed once nothing can fail any more
  const bool keep_tree = !rebuild && ctx->tree_is_map;  // keep the old map alive as the 1-NN cloud if the guard fails
  Buf<float4>& dst_s = keep_tree ? ctx->tree_s : ctx->map_s;  // (after the swap below these are the new map buffers)
  Buf<float4>& dst_c = keep_tree ? ctx->tree_c : ctx->map_c;
  int rc = upload2_reserve(ctx, dst_s, ns, dst_c, nc);  // (waits until the H2D of a previous call has read the staging)
  if (rc != LINS_OK) return rc;
  CK(ctx->map_s.reserve(1)); CK(ctx->map_c.reserve(1)); CK(ctx->tree_s.reserve(1)); CK(ctx->tree_c.reserve(1));
  CK(ctx->tmp_lin.reserve(20));
  if (want_out) CK(ctx->tmp_out.reserve((size_t)ns + nc + 1));
  if (keep_tree) {
    std::swap(ctx->tree_s, ctx->map_s); std::swap(ctx->tree_c, ctx->map_c);
    ctx->tree_ns = std::max(ctx->map_ns, 0); ctx->tree_nc = std::max(ctx->map_nc, 0);
    ctx->tree_is_map = false;
  }
  if (lin_state) {
    double lin[20];
    pad_states(lin, lin_state, 1);
    CK(cudaMemcpyAsync(ctx->tmp_lin.p, lin, sizeof(lin), cudaMemcpyHostToDevice, ctx->stream));  // (pageable source: staged before the call returns)
    lin_dev = ctx->tmp_lin.p;
  }
  rc = upload2_queue(ctx, ctx->map_s, surf, ns, ctx->map_c, corner, nc);
  if (rc != LINS_OK) return rc;
  lins_point* o_s = surf_out && ns ? ctx->tmp_out.p : nullptr;
  lins_point* o_c = corner_out && nc ? ctx->tmp_out.p + ns : nullptr;
  if (ns) { lins_transform_to_end_kernel<<<(ns + 255) / 256, 256, 0, ctx->stream>>>(ctx->map_s.p, ns, lin_dev, ctx->prm.scan_period, o_s); ctx->launches += 1; }
  if (nc) { lins_transform_to_end_kernel<<<(nc + 255) / 256, 256, 0, ctx->stream>>>(ctx->map_c.p, nc, lin_dev, ctx->prm.scan_period, o_c); ctx->launches += 1; }
  CK(cudaGetLastError());
  ctx->map_ns = ns; ctx->map_nc = nc;
  if (rebuild) { ctx->tree_is_map = true; ctx->tree_ns = ns; ctx->tree_nc = nc; }
  if (map_replaced) *map_replaced = rebuild ? 1 : 0;
  rc = upload_map_offsets(ctx);
  if (rc != LINS_OK) return rc;
  if (want_out) {  // full records through pinned staging (a D2H into pageable memory is staged chunk by chunk by the driver)
    CK(ctx->h_out.reserve((size_t)ns + nc + 1));
    if (o_s) CK(cudaMemcpyAsync(ctx->h_out.p, o_s, sizeof(lins_point) * ns, cudaMemcpyDeviceToHost, ctx->stream));
    if (o_c) CK(cudaMemcpyAsync(ctx->h_out.p + ns, o_c, sizeof(lins_point) * nc, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (o_s) std::memcpy(surf_out, ctx->h_out.p, sizeof(lins_point) * ns);
    if (o_c) std::memcpy(corner_out, ctx->h_out.p + ns, sizeof(lins_point) * nc);
  }
  return LINS_OK;
}

int lins_gpu_update_map(lins_ctx* ctx, lins_point* surf, int ns, lins_point* corner, int nc, const double* lin_state,
                        int* map_replaced) {
  if (!ctx) return LINS_E_INVALID;
  if (!lin_state) return fail(ctx, LINS_E_INVALID, "bad update_map args");
  return lins_gpu_update_map_ex(ctx, surf, ns, corner, nc, lin_state, surf, corner, map_replaced);
}

}  // extern "C"
