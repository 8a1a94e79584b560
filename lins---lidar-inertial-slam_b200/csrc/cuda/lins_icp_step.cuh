// The 6-DoF Gauss-Newton step of the ICP fallback on the device (row A12: calculateTransformation, reference
// lins/include/StateEstimator.hpp:1260-1320): x = (J^T J).colPivHouseholderQr().solve(J^T b), the eigenvalue-10 degeneracy
// projection of iteration 0 (matP), pose update q <- (q * rpy2Quat(x[0:3])).normalized(), t += x[3:6], and the
// 0.1 deg / 0.1 cm exit.  One thread: the work is a few hundred flops on a 6 x 6 system, once per iteration; what matters
// is that the pose, matP and the exit flag never leave the device, so lins_gpu_estimate_transform queues every iteration
// up front and synchronises once.  Same algorithms, in the same order, as csrc/host/small_linalg.hpp (which the host
// shim still uses elsewhere): Householder QR with column pivoting and Eigen's rank rule, cyclic Jacobi, Gauss-Jordan.
#pragma once
#include "lins_device_math.cuh"
#include "lins_kernels.cuh"  // IcpState

namespace lins_dev {

__device__ inline void icp_qr_solve6(double A[6][6], double b[6], double x[6]) {
  int perm[6];
  for (int i = 0; i < 6; ++i) perm[i] = i;
  double maxpiv = 0.0;
  for (int k = 0; k < 6; ++k) {
    int best = k;
    double bestn = -1.0;
    for (int j = k; j < 6; ++j) {
      double s = 0;
      for (int i = k; i < 6; ++i) s += A[i][j] * A[i][j];
      if (s > bestn) { bestn = s; best = j; }
    }
    if (best != k) {
      for (int i = 0; i < 6; ++i) { const double t = A[i][k]; A[i][k] = A[i][best]; A[i][best] = t; }
      const int t = perm[k]; perm[k] = perm[best]; perm[best] = t;
    }
    const double nrm = sqrt(bestn > 0 ? bestn : 0.0);
    if (nrm == 0.0) continue;
    const double alpha = A[k][k] > 0 ? -nrm : nrm;
    double v[6] = {0, 0, 0, 0, 0, 0};
    for (int i = k; i < 6; ++i) v[i] = A[i][k];
    v[k] -= alpha;
    double vv = 0;
    for (int i = k; i < 6; ++i) vv += v[i] * v[i];
    if (vv > 0) {
      for (int j = k; j < 6; ++j) {
        double d = 0;
        for (int i = k; i < 6; ++i) d += v[i] * A[i][j];
        d *= 2.0 / vv;
        for (int i = k; i < 6; ++i) A[i][j] -= d * v[i];
      }
      double d = 0;
      for (int i = k; i < 6; ++i) d += v[i] * b[i];
      d *= 2.0 / vv;
      for (int i = k; i < 6; ++i) b[i] -= d * v[i];
    }
    maxpiv = fmax(maxpiv, fabs(A[k][k]));
  }
  const double thr = 2.220446049250313e-16 * 6 * maxpiv;
  int rank = 0;
  while (rank < 6 && fabs(A[rank][rank]) > thr) ++rank;
  double y[6] = {0, 0, 0, 0, 0, 0};
  for (int k = rank - 1; k >= 0; --k) {
    double s = b[k];
    for (int j = k + 1; j < rank; ++j) s -= A[k][j] * y[j];
    y[k] = s / A[k][k];
  }
  for (int k = 0; k < 6; ++k) x[k] = 0.0;
  for (int k = 0; k < 6; ++k) x[perm[k]] = y[k];
}

// eigenvalues ascending, eigenvector k = column k of V, largest-magnitude component positive
__device__ inline void icp_sym_eigen6(double A[6][6], double evals[6], double V[6][6], double Vs[6][6]) {
  for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0;
    for (int i = 0; i < 6; ++i) for (int j = i + 1; j < 6; ++j) off += A[i][j] * A[i][j];
    if (off < 1e-300) break;
    for (int p = 0; p < 5; ++p)
      for (int q = p + 1; q < 6; ++q) {
        if (A[p][q] == 0.0) continue;
        const double tau = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (tau >= 0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
        const double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
        for (int k = 0; k < 6; ++k) { const double x = A[k][p], y = A[k][q]; A[k][p] = c * x - s * y; A[k][q] = s * x + c * y; }
        for (int k = 0; k < 6; ++k) { const double x = A[p][k], y = A[q][k]; A[p][k] = c * x - s * y; A[q][k] = s * x + c * y; }
        for (int k = 0; k < 6; ++k) { const double x = V[k][p], y = V[k][q]; V[k][p] = c * x - s * y; V[k][q] = s * x + c * y; }
      }
  }
  int ord[6];
  for (int i = 0; i < 6; ++i) ord[i] = i;
  for (int i = 1; i < 6; ++i) {
    const int o = ord[i];
    int j = i - 1;
    while (j >= 0 && A[ord[j]][ord[j]] > A[o][o]) { ord[j + 1] = ord[j]; --j; }
    ord[j + 1] = o;
  }
  for (int k = 0; k < 6; ++k) {
    evals[k] = A[ord[k]][ord[k]];
    int big = 0;
    for (int i = 1; i < 6; ++i) if (fabs(V[i][ord[k]]) > fabs(V[big][ord[k]])) big = i;
    const double sg = V[big][ord[k]] < 0 ? -1.0 : 1.0;
    for (int i = 0; i < 6; ++i) Vs[i][k] = sg * V[i][ord[k]];
  }
  for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) V[i][j] = Vs[i][j];
}

__device__ inline bool icp_inverse6(double A[6][6], double inv[6][6]) {
  for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) inv[i][j] = i == j ? 1.0 : 0.0;
  for (int k = 0; k < 6; ++k) {
    int piv = k;
    for (int i = k + 1; i < 6; ++i) if (fabs(A[i][k]) > fabs(A[piv][k])) piv = i;
    if (A[piv][k] == 0.0 || A[piv][k] != A[piv][k]) return false;
    if (piv != k) for (int j = 0; j < 6; ++j) { double t = A[piv][j]; A[piv][j] = A[k][j]; A[k][j] = t; t = inv[piv][j]; inv[piv][j] = inv[k][j]; inv[k][j] = t; }
    const double d = 1.0 / A[k][k];
    for (int j = 0; j < 6; ++j) { A[k][j] *= d; inv[k][j] *= d; }
    for (int i = 0; i < 6; ++i) {
      if (i == k) continue;
      const double f = A[i][k];
      if (f == 0.0) continue;
      for (int j = 0; j < 6; ++j) { A[i][j] -= f * A[k][j]; inv[i][j] -= f * inv[k][j]; }
    }
  }
  return true;
}

// One 32-thread block per unit u = blockIdx.x, thread 0 working.  accum + 32 u: the 28 sums + counts of one MODE_ICP_REDUCE
// pass (entries 0..20 = upper triangle of J^T J, 21..26 = J^T b, 28 / 29 = matched surfs / corners); state + 20 u: the
// 20-double pose block the next pass linearises at (t at 0..2, q xyzw at 6..9); st + u: the unit's loop state.  The loop
// ends at the unit's own NUM_ITER, tune[u].num_iter (null tune: num_iter): the step of its last iteration sets done, and a
// unit whose cap the launch is past (NUM_ITER 0, where its caller did not start it done) is done without an iteration.
__global__ void lins_icp_step_kernel(const double* __restrict__ accum, double* __restrict__ state, IcpState* __restrict__ st, int iter,
                                     const UnitTuning* __restrict__ tune, int num_iter) {
  const int u = blockIdx.x;
  accum += (size_t)u * 32;
  state += (size_t)u * 20;
  st += u;
  if (threadIdx.x != 0 || st->done) return;
  const int cap = tune ? tune[u].num_iter : num_iter;
  if (iter >= cap) { st->done = 1; return; }
  st->iters = iter + 1;
  if (iter + 1 >= cap) st->done = 1;  // (the loop's last iteration: converged or not, nothing reads the unit again)
  const double* a = accum;
  if (a[28] < 10) return;  // "Insufficient matched surfs..." (:1175-1178)
  if (a[29] < 5) return;   // "Insufficient matched corners..." (:1181-1184)
  // (every matrix lives in shared memory: plain dynamically indexed loads / stores, no register-promoted local arrays)
  __shared__ double JTJ[6][6], Aw[6][6], Ev[6][6], V2[6][6], Vc[6][6], Vinv[6][6], Vscr[6][6];
  __shared__ double JTb[6], x[6], bw[6], E[6];
  int k = 0;
  for (int i = 0; i < 6; ++i) for (int j = i; j < 6; ++j) { JTJ[i][j] = a[k]; JTJ[j][i] = a[k]; ++k; }
  for (int i = 0; i < 6; ++i) JTb[i] = a[21 + i];
  for (int i = 0; i < 6; ++i) { bw[i] = JTb[i]; for (int j = 0; j < 6; ++j) Aw[i][j] = JTJ[i][j]; }
  icp_qr_solve6(Aw, bw, x);
  bool degenerate = false;
  if (iter == 0) {  // :1269-1296
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) Aw[i][j] = JTJ[i][j];
    icp_sym_eigen6(Aw, E, Ev, Vscr);
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) { V2[i][j] = Ev[i][j]; Vc[i][j] = Ev[i][j]; }
    for (int i = 0; i < 6; ++i) {
      if (E[i] < 10.) { for (int j = 0; j < 6; ++j) V2[i][j] = 0; degenerate = true; }
      else break;
    }
    if (!icp_inverse6(Vc, Vinv)) for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) Vinv[i][j] = __longlong_as_double(0x7ff8000000000000ll);
    for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) { double s = 0; for (int m = 0; m < 6; ++m) s += Vinv[i][m] * V2[m][j]; st->matP[i * 6 + j] = s; }
    st->pad = degenerate ? 1 : 0;
  }
  // (the reference's isDegenerate is a local of calculateTransformation: true only in the iteration that computed matP)
  if (degenerate) {
    double x2[6];
    for (int i = 0; i < 6; ++i) x2[i] = x[i];
    for (int i = 0; i < 6; ++i) { double s = 0; for (int j = 0; j < 6; ++j) s += st->matP[i * 6 + j] * x2[j]; x[i] = s; }
  }
  // q <- (q * rpy2Quat(x[0:3])).normalized(), t += x[3:6]   (math_utils.h:131-149)
  const double hy = x[2] * 0.5, hp = x[1] * 0.5, hr = x[0] * 0.5;
  const double cy = cos(hy), sy = sin(hy), cp = cos(hp), sp = sin(hp), cr = cos(hr), sr = sin(hr);
  q4 dq; dq.w = cr * cp * cy + sr * sp * sy; dq.x = sr * cp * cy - cr * sp * sy; dq.y = cr * sp * cy + sr * cp * sy; dq.z = cr * cp * sy - sr * sp * cy;
  q4 q; q.x = state[6]; q.y = state[7]; q.z = state[8]; q.w = state[9];
  q = qnormalized(qmul(q, dq));
  state[6] = q.x; state[7] = q.y; state[8] = q.z; state[9] = q.w;
  state[0] += x[3]; state[1] += x[4]; state[2] += x[5];
  const double r2d = 180.0 / 3.14159265358979323846;
  const double dR = sqrt((x[0] * r2d) * (x[0] * r2d) + ((x[1] * r2d) * (x[1] * r2d) + (x[2] * r2d) * (x[2] * r2d)));
  const double dT = sqrt((100 * x[3]) * (100 * x[3]) + ((100 * x[4]) * (100 * x[4]) + (100 * x[5]) * (100 * x[5])));
  if (dR < 0.1 && dT < 0.1) { st->converged = 1; st->done = 1; }
}

}  // namespace lins_dev
