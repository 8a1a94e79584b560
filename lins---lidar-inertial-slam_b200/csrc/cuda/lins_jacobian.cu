// lins_jacobian.cu — the split "Jacobian kernel" (SURVEY.md §8(d) unit U1; rows A5-A9 form B GIVEN the correspondence IDs):
// per unit, stream the queries (16 B) and their IDs (12 / 8 B) coalesced, gather the 3 / 2 matched targets (16 B each),
// recompute de-skew, residual, robust weight and the factored Jacobian row g = [c ; P2 x (R^T c)] with residual r, and
// reduce  sum g g^T (21), sum g r (6), sum r r (1)  per unit (reference lins/include/StateEstimator.hpp:499-546 with the
// M x M products folded into the 6 x 6 information form).  This is the kernel whose achieved HBM bandwidth the north_star
// asks about; the product path is the fused kernel in lins_gpu.cu, which never calls this one.
//
// Its own translation unit because it is tolerance-checked (tests/test_gpu_jacobian.py: each sum within a few f64 ulps of
// its condition scale of an exact-sum reference), not bit-checked, and is built for speed:
//   * compiled WITH multiply-add contraction (lins_gpu.cu is -fmad=false for the bit-exact association); the per-unit
//     constants of the de-skew (|phi|, phi / |phi|) are hoisted and sin / cos of the small half angle come from their
//     Taylor polynomials (|x| < 1/8: remainder < 1e-19) — differences to the fused kernel's values are a few f64 ulps;
//   * the 28 sums are a Gram matrix G^T G of the warp's 32 rows G = [g0..g5, r, 0]: every lane stages its row in
//     shared memory and eight FP64 tensor-core MMAs (mma.sync m8n8k4, one per four queries) accumulate the 8 x 8 result
//     in two registers per lane — instead of 28 products and a 31-step shuffle tree per trip.  Fixed order, so the
//     sums are run-to-run deterministic;
//   * one warp per unit in a two-deep software pipeline: while trip k is computed, the gathers of trip k + 1 and the
//     query / ID loads of trip k + 2 are in flight (a unit's ~16 trips are a serial chain: its memory latency, not the
//     SM's issue rate, is what one warp per unit has to hide).
#include "lins_kernels.cuh"

namespace lins_dev {

constexpr int kJacWarps = 8;            // warps per CTA
constexpr int kJacRow = 12;             // doubles per staged row (8 used): 96-B stride -> conflict-free 8-B reads
// resident CTAs per SM the register budget is set for.  Measured on an H100 SXM (400 W limit; 5000 units, 408 MB working
// set): 1 98 us, 2 (128 registers, no spills, 16 warps per SM) 76.6 us, 3 (80 registers) 101 us
constexpr int kJacMinCtas = 2;

// sin / cos of a small angle (|x| < 0.125) to better than one ulp
__device__ __forceinline__ void sincos_small(double x, double& sn, double& cs) {
  const double x2 = x * x;
  sn = x * (1.0 + x2 * (-1.0 / 6 + x2 * (1.0 / 120 + x2 * (-1.0 / 5040 + x2 * (1.0 / 362880 + x2 * (-1.0 / 39916800))))));
  cs = 1.0 + x2 * (-0.5 + x2 * (1.0 / 24 + x2 * (-1.0 / 720 + x2 * (1.0 / 40320 + x2 * (-1.0 / 3628800 + x2 * (1.0 / 479001600))))));
}

// P = parts a unit is cut into (trips dealt round-robin to P warps): with one warp per unit and only a few units per warp the
// grid's last round is nearly empty; cutting units keeps every warp busy to the end.  The parts' sums meet in part_acc and
// the warp that arrives last adds them in part order (deterministic).
__global__ void __launch_bounds__(kJacWarps * 32, kJacMinCtas) lins_jacobian_mma_kernel(const __grid_constant__ BatchView bv,
                                                                                             const __grid_constant__ KParams kp, int P,
                                                                                             double* __restrict__ part_acc, int* __restrict__ part_cnt) {
  __shared__ __align__(16) double stage[kJacWarps][32 * kJacRow];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* my = stage[warp];
  const int warps_per_grid = gridDim.x * kJacWarps;
  const double inv_period = 1.f / kp.scan_period;
  const bool weighted = kp.iter0 >= kp.icp_freq;
  for (int item = blockIdx.x * kJacWarps + warp; item < bv.n_scans * P; item += warps_per_grid) {
    const int scan = item / P, part = item - scan * P;
    // per-unit constants (every lane computes the same values)
    const double* st = bv.state_in + (size_t)scan * 20;
    const double rn0 = st[0], rn1 = st[1], rn2 = st[2];
    q4 q; q.x = st[6]; q.y = st[7]; q.z = st[8]; q.w = st[9];
    const d3 phi = Quat2axis(q);
    const double th0 = norm3(phi);
    const double ith0 = th0 > 0.0 ? 1.0 / th0 : 0.0;
    const d3 ax = mk3(phi.x * ith0, phi.y * ith0, phi.z * ith0);
    const m3 R = qtoR(q);
    const int qs0 = bv.qs_off[scan], ns = bv.qs_off[scan + 1] - qs0;
    const int qc0 = bv.qc_off[scan], nc = bv.qc_off[scan + 1] - qc0;
    const float4* __restrict__ tgtS = bv.ts + bv.ts_off[scan];
    const float4* __restrict__ tgtC = bv.tc + bv.tc_off[scan];
    const int Ts = bv.ts_off[scan + 1] - bv.ts_off[scan], Tc = bv.tc_off[scan + 1] - bv.tc_off[scan];
    double c0 = 0.0, c1 = 0.0;  // this lane's two entries of the 8 x 8 Gram matrix
    int cs = 0, cc = 0;
    auto fetch = [&](int i, float4& p, int& i1, int& i2, int& i3) {
      p = make_float4(0.f, 0.f, 0.f, 0.f); i1 = -1; i2 = -1; i3 = -1;
      if (i < ns) {
        p = __ldg(bv.qs + qs0 + i);
        const int* id = bv.ind_s + 3 * (size_t)(qs0 + i);
        i1 = __ldg(id); i2 = __ldg(id + 1); i3 = __ldg(id + 2);
      } else if (i < ns + nc) {
        p = __ldg(bv.qc + qc0 + (i - ns));
        const int* id = bv.ind_c + 2 * (size_t)(qc0 + (i - ns));
        i1 = __ldg(id); i2 = __ldg(id + 1);
      }
    };
    // two-deep software pipeline: while trip k is computed, the gathers of trip k + 1 and the streaming loads (query, IDs)
    // of trip k + 2 are in flight
    auto gather = [&](int i, int i1, int i2, int i3, float4& t1, float4& t2, float4& t3) -> bool {
      t1 = make_float4(0.f, 0.f, 0.f, 0.f); t2 = t1; t3 = t1;
      if (i < ns) {
        if (i2 >= 0 && i3 >= 0 && i1 >= 0 && i1 < Ts && i2 < Ts && i3 < Ts) { t1 = __ldg(&tgtS[i1]); t2 = __ldg(&tgtS[i2]); t3 = __ldg(&tgtS[i3]); return true; }
      } else if (i < ns + nc) {
        if (i2 >= 0 && i1 >= 0 && i1 < Tc && i2 < Tc) { t1 = __ldg(&tgtC[i1]); t2 = __ldg(&tgtC[i2]); return true; }
      }
      return false;
    };
    float4 pc, pn; int n1, n2, n3;       // the next trip's query; the query + IDs of the trip after it
    float4 t1, t2, t3;                   // the next trip's targets
    bool have;
    {
      int a1, a2, a3;
      fetch(part * 32 + lane, pc, a1, a2, a3);
      have = gather(part * 32 + lane, a1, a2, a3, t1, t2, t3);
      fetch((part + P) * 32 + lane, pn, n1, n2, n3);
    }
    const int stride = 32 * P;
    for (int i0 = part * 32; i0 < ns + nc; i0 += stride) {
      const int i = i0 + lane;
      const float4 p = pc;
      const bool surf = i < ns;
      const float4 u1 = t1, u2 = t2, u3 = t3;
      const bool chave = have;
      // next trip: its gathers now (IDs arrived during the previous trip); the trip after: its streaming loads
      have = gather(i + stride, n1, n2, n3, t1, t2, t3);
      pc = pn;
      fetch(i + 2 * stride, pn, n1, n2, n3);
      double g[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, r = 0.0;
      bool ok = false;
      if (chave) {
        // A2 de-skew (transformToStart, StateEstimator.hpp:1066-1080): rotation by s * phi about the unit's fixed axis
        const float fi = p.w - (float)((int)p.w);
        const double s = inv_period * fi;
        const double half = 0.5 * (s * th0);
        // (s = 0 or phi = 0 give sin = 0, cos = 1: the identity, like the reference's theta < 1e-10 shortcut)
        q4 rq;
        {
          double sn, csn;
          if (fabs(half) < 0.125) sincos_small(half, sn, csn); else sincos(half, &sn, &csn);
          rq.w = csn; rq.x = ax.x * sn; rq.y = ax.y * sn; rq.z = ax.z * sn;
        }
        const d3 rp = qrot(rq, mk3(p.x, p.y, p.z));
        float4 sel;
        sel.x = (float)(rp.x + s * rn0); sel.y = (float)(rp.y + s * rn1); sel.z = (float)(rp.z + s * rn2); sel.w = p.w;
        float4 coeff = make_float4(0.f, 0.f, 0.f, 0.f);
        ok = surf ? plane_residual(sel, u1, u2, u3, weighted, coeff) : line_residual(sel, u1, u2, weighted, coeff);
        if (ok) jacobian_row(p, coeff, R.m, kp.lidar_scale, g, r);
      }
      // stage the row [g0..g5, r, 0] and fold the warp's 32 rows: C += G^T G, four queries per MMA.
      // A (8 x 4, row) and B (4 x 8, col) fragments of lane L are both G[4c + L % 4][L / 4].
      __syncwarp();
      double2* row = reinterpret_cast<double2*>(my + lane * kJacRow);
      row[0] = make_double2(g[0], g[1]); row[1] = make_double2(g[2], g[3]); row[2] = make_double2(g[4], g[5]); row[3] = make_double2(r, 0.0);
      __syncwarp();
      const double* col = my + (lane & 3) * kJacRow + (lane >> 2);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const double v = col[c * 4 * kJacRow];
        dmma_8x8x4(c0, c1, v, v);
      }
      cs += __popc(__ballot_sync(0xffffffffu, ok && surf));
      cc += __popc(__ballot_sync(0xffffffffu, ok && !surf));
    }
    // C[i][j] with i = lane / 4, j = 2 * (lane % 4) + {0, 1}: upper triangle of the 6 x 6 block -> entries 0..20 (row-major),
    // column 6 -> g r (21..26) and r r (27)
    double* dst = P == 1 ? bv.accum + (size_t)scan * 32 : part_acc + ((size_t)scan * P + part) * 32;
    const int ci = lane >> 2;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int cj = 2 * (lane & 3) + u;
      const double v = u ? c1 : c0;
      if (ci <= cj && cj <= 6) {
        int e;
        if (cj < 6) e = ci * 6 - (ci * (ci - 1)) / 2 + (cj - ci);
        else e = ci < 6 ? 21 + ci : 27;
        dst[e] = v;
      }
    }
    if (lane == 28) dst[28] = (double)cs;
    if (lane == 29) dst[29] = (double)cc;
    if (P > 1) {
      __threadfence();
      __syncwarp();
      int old = 0;
      if (lane == 0) old = atomicAdd(&part_cnt[scan], 1);
      old = __shfl_sync(0xffffffffu, old, 0);
      if (old == P - 1) {  // every part of this unit has arrived: add them in part order
        __threadfence();
        if (lane < 30) {
          double v = 0.0;
          for (int p = 0; p < P; ++p) v += __ldcg(part_acc + ((size_t)scan * P + p) * 32 + lane);
          bv.accum[(size_t)scan * 32 + lane] = v;
        }
      }
    }
  }
}

}  // namespace lins_dev

// launched from lins_gpu.cu (lins_gpu_batch_jacobian_pass)
// parts per unit.  The kernel is bound by its scattered 32-B sector gathers, not by the emptiness of the grid's last round,
// and cutting units only adds per-unit set-up and spoils locality.  One part unless the batch cannot even fill the resident warps.
extern "C" int lins_jacobian_parts(int n_units, int sm_count) {
  using namespace lins_dev;
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lins_jacobian_mma_kernel, kJacWarps * 32, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  const long warps = (long)sm_count * per_sm * kJacWarps;
  const long P = n_units > 0 && n_units < warps / 2 ? warps / n_units : 1;
  return (int)(P < 1 ? 1 : (P > 4 ? 4 : P));
}
extern "C" int lins_launch_jacobian_mma(const lins_dev::BatchView* bv, const lins_dev::KParams* kp, int n_units, int sm_count, int P, double* part_acc,
                                        int* part_cnt, cudaStream_t stream) {
  using namespace lins_dev;
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lins_jacobian_mma_kernel, kJacWarps * 32, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  long items = (long)n_units * P;
  int grid = (int)((items + kJacWarps - 1) / kJacWarps);
  if (grid > sm_count * per_sm) grid = sm_count * per_sm;
  if (grid < 1) grid = 1;
  if (P > 1 && cudaMemsetAsync(part_cnt, 0, sizeof(int) * (size_t)n_units, stream) != cudaSuccess) return (int)cudaGetLastError();
  lins_jacobian_mma_kernel<<<grid, kJacWarps * 32, 0, stream>>>(*bv, *kp, P, part_acc, part_cnt);
  return (int)cudaGetLastError();
}
