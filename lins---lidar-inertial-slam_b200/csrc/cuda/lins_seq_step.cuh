// lins_seq_step.cuh — the per-sequence filter algebra of sequence mode (include/lins_gpu.h: lins_gpu_seq_*), as
// __host__ __device__ code so that the device kernels of lins_seq.cu and a g++ test compile the same source.
//
// Every function follows the host code it replaces operation for operation (same operand order, same zero
// initialisations, same skipped zero products), so that a build without multiply-add contraction (nvcc -fmad=false;
// g++ on x86-64 without -mfma) reproduces it bit for bit up to the libm of sin / cos / asin / atan2:
//   predict            csrc/host/kalman_filter.hpp StatePredictor::predict   (KalmanFilter.hpp:125-186)
//   reset(1)           csrc/host/kalman_filter.hpp StatePredictor::reset     (KalmanFilter.hpp:320-353)
//   integrate          csrc/host/state_estimator.hpp integrateTransformation (StateEstimator.hpp:608-617)
//   roll / pitch       calculateRPfromGravity + correctRollPitch            (StateEstimator.hpp:427-431, :602-605)
// States are the C-ABI's 19 doubles: rn[0..2] vn[3..5] q(x,y,z,w)[6..9] ba[10..12] bw[13..15] gn[16..18]; covariances
// 18x18 column-major.  Vectors are math_utils.hpp's V3D, quaternions its Q4D, matrices its row-major M3D.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define LSQ_HD __host__ __device__ __forceinline__
#else
#define LSQ_HD inline
#endif

namespace lins_seq {

constexpr double kG0 = 9.81;  // parameters.h:62
constexpr int kPos = 0, kVel = 3, kAtt = 6, kAcc = 9, kGyr = 12, kGra = 15;  // error-state (covariance) blocks
constexpr int sRn = 0, sVn = 3, sBa = 10, sBw = 13, sGn = 16;                // the 19-double state layout

struct V3 { double d[3]; };
struct Q4 { double x, y, z, w; };
struct M3 { double a[9]; };  // row-major

LSQ_HD V3 v3(double x, double y, double z) { V3 r; r.d[0] = x; r.d[1] = y; r.d[2] = z; return r; }
LSQ_HD V3 vadd(V3 a, V3 b) { for (int i = 0; i < 3; ++i) a.d[i] += b.d[i]; return a; }
LSQ_HD V3 vsub(V3 a, V3 b) { for (int i = 0; i < 3; ++i) a.d[i] -= b.d[i]; return a; }
LSQ_HD V3 vscl(double s, V3 a) { for (int i = 0; i < 3; ++i) a.d[i] *= s; return a; }
LSQ_HD V3 vdiv(V3 a, double s) { for (int i = 0; i < 3; ++i) a.d[i] /= s; return a; }
LSQ_HD double vnorm(V3 a) { return sqrt(a.d[0] * a.d[0] + a.d[1] * a.d[1] + a.d[2] * a.d[2]); }
LSQ_HD V3 vcross(V3 a, V3 b) {
  return v3(a.d[1] * b.d[2] - a.d[2] * b.d[1], a.d[2] * b.d[0] - a.d[0] * b.d[2], a.d[0] * b.d[1] - a.d[1] * b.d[0]);
}
LSQ_HD Q4 q4(double w, double x, double y, double z) { Q4 q; q.w = w; q.x = x; q.y = y; q.z = z; return q; }
LSQ_HD Q4 qident() { return q4(1.0, 0.0, 0.0, 0.0); }
LSQ_HD Q4 qmul(Q4 a, Q4 b) {
  return q4(a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x);
}
LSQ_HD double qsqnorm(Q4 q) { return q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w; }
LSQ_HD Q4 qnormalized(Q4 q) { const double n = sqrt(qsqnorm(q)); return q4(q.w / n, q.x / n, q.y / n, q.z / n); }
LSQ_HD Q4 qinverse(Q4 q) { const double n = qsqnorm(q); return q4(q.w / n, -q.x / n, -q.y / n, -q.z / n); }
LSQ_HD V3 qrot(Q4 q, V3 v) {
  const V3 qv = v3(q.x, q.y, q.z);
  const V3 t = vscl(2.0, vcross(qv, v));
  return vadd(vadd(v, vscl(q.w, t)), vcross(qv, t));
}
LSQ_HD M3 qtoR(Q4 q) {
  const double x2 = q.x + q.x, y2 = q.y + q.y, z2 = q.z + q.z;
  const double wx = x2 * q.w, wy = y2 * q.w, wz = z2 * q.w;
  const double xx = x2 * q.x, xy = y2 * q.x, xz = z2 * q.x, yy = y2 * q.y, yz = z2 * q.y, zz = z2 * q.z;
  M3 r;
  r.a[0] = 1 - (yy + zz); r.a[1] = xy - wz;       r.a[2] = xz + wy;
  r.a[3] = xy + wz;       r.a[4] = 1 - (xx + zz); r.a[5] = yz - wx;
  r.a[6] = xz - wy;       r.a[7] = yz + wx;       r.a[8] = 1 - (xx + yy);
  return r;
}
LSQ_HD M3 mmul(const M3& x, const M3& y) {
  M3 r;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += x.a[3 * i + k] * y.a[3 * k + j]; r.a[3 * i + j] = s; }
  return r;
}
LSQ_HD M3 mneg(M3 m) { for (int i = 0; i < 9; ++i) m.a[i] = -m.a[i]; return m; }
LSQ_HD M3 skew(V3 q) {
  M3 a;
  for (int i = 0; i < 9; ++i) a.a[i] = 0;
  a.a[1] = -q.d[2]; a.a[2] = q.d[1];
  a.a[3] = q.d[2];  a.a[5] = -q.d[0];
  a.a[6] = -q.d[1]; a.a[7] = q.d[0];
  return a;
}
LSQ_HD Q4 axis2Quat(V3 vec) {
  const double theta = vnorm(vec);
  if (theta < 1e-10) return qident();
  const V3 ax = vdiv(vec, theta);
  const double m = sin(theta / 2.0);
  return q4(cos(theta / 2.0), ax.d[0] * m, ax.d[1] * m, ax.d[2] * m);
}
LSQ_HD int sign(double x) { return x >= 0 ? 1 : -1; }
LSQ_HD Q4 rpy2Quat(V3 rpy) {
  const double hy = rpy.d[2] * 0.5, hp = rpy.d[1] * 0.5, hr = rpy.d[0] * 0.5;
  const double cy = cos(hy), sy = sin(hy), cp = cos(hp), sp = sin(hp), cr = cos(hr), sr = sin(hr);
  return q4(cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy);
}
LSQ_HD V3 Q2rpy(Q4 q) {
  const M3 R = qtoR(q);
  V3 rpy;
  rpy.d[1] = atan2(-R.a[6], sqrt(R.a[7] * R.a[7] + R.a[8] * R.a[8]));
  rpy.d[0] = atan2(R.a[7] / cos(rpy.d[1]), R.a[8] / cos(rpy.d[1]));
  rpy.d[2] = atan2(R.a[3] / cos(rpy.d[1]), R.a[0] / cos(rpy.d[1]));
  return rpy;
}

// ---- the C-ABI state layout ---------------------------------------------------------------------------------------
LSQ_HD V3 ld3(const double* s, int o) { return v3(s[o], s[o + 1], s[o + 2]); }
LSQ_HD void st3(double* s, int o, V3 v) { s[o] = v.d[0]; s[o + 1] = v.d[1]; s[o + 2] = v.d[2]; }
LSQ_HD Q4 ldq(const double* s) { return q4(s[9], s[6], s[7], s[8]); }
LSQ_HD void stq(double* s, Q4 q) { s[6] = q.x; s[7] = q.y; s[8] = q.z; s[9] = q.w; }

// The filter constants the device chain needs.  noise = StatePredictor::noise_ (setNoise); pos_var / att_var = the
// diagonals reset(1) installs: sq(init_pos_std) and pow(deg2rad(init_att_std), 2), computed on the host once.
struct Consts {
  double noise[4];
  double pos_var[3], att_var[3];
};

// ---- predict (kalman_filter.hpp:98-170) ----------------------------------------------------------------------------
// The state part of one predict call: updates s (rn, vn, q) and returns R = toRotationMatrix of the new q plus the two
// non-trivial Ft blocks va = -(R skew(acc - ba)) and aa = -skew(gyr - bw).
struct PredictBlocks { M3 R, va, aa; };
LSQ_HD PredictBlocks predict_state(double* s, const double* acc_last, const double* gyr_last, double dt, const double* acc,
                                   const double* gyr) {
  const V3 rn = ld3(s, sRn), vn = ld3(s, sVn), ba = ld3(s, sBa), bw = ld3(s, sBw), gn = ld3(s, sGn);
  const V3 a0 = ld3(acc_last, 0), g0 = ld3(gyr_last, 0), a1 = ld3(acc, 0), g1 = ld3(gyr, 0);
  Q4 q = ldq(s);
  const V3 un_acc_0 = vadd(qrot(q, vsub(a0, ba)), gn);
  const V3 un_gyr = vsub(vscl(0.5, vadd(g0, g1)), bw);
  const Q4 dq = axis2Quat(vscl(dt, un_gyr));
  q = qnormalized(qmul(q, dq));
  const V3 un_acc_1 = vadd(qrot(q, vsub(a1, ba)), gn);
  const V3 un_acc = vscl(0.5, vadd(un_acc_0, un_acc_1));
  st3(s, sRn, vadd(vadd(rn, vscl(dt, vn)), vscl(0.5 * dt * dt, un_acc)));
  st3(s, sVn, vadd(vn, vscl(dt, un_acc)));
  stq(s, q);
  PredictBlocks b;
  b.R = qtoR(q);
  b.va = mneg(mmul(b.R, skew(vsub(a1, ba))));
  b.aa = mneg(skew(vsub(g1, bw)));
  return b;
}
// Ft (18x18, row-major, every other entry +0): entry e = 18 i + j
LSQ_HD double ft_entry(const PredictBlocks& b, int i, int j) {
  const int bi = i / 3, bj = j / 3, r = i % 3, c = j % 3;
  if (bi == 0 && bj == 1 && r == c) return 1.0;
  if (bi == 1 && bj == 5 && r == c) return 1.0;
  if (bi == 2 && bj == 4 && r == c) return -1.0;
  if (bi == 1 && bj == 2) return b.va.a[3 * r + c];
  if (bi == 1 && bj == 3) return -b.R.a[3 * r + c];
  if (bi == 2 && bj == 2) return b.aa.a[3 * r + c];
  return 0.0;
}
// F = I + Ft dt + 0.5 (Ft Ft) dt^2, entry (i, j); Ft row-major
LSQ_HD double f_entry(const double* Ft, int i, int j, double dt) {
  double ff = 0.0;
  for (int k = 0; k < 18; ++k) {
    const double f = Ft[i * 18 + k];
    if (f == 0.0) continue;
    ff += f * Ft[k * 18 + j];
  }
  return (i == j ? 1.0 : 0.0) + Ft[i * 18 + j] * dt + 0.5 * ff * dt * dt;
}
// Q = Gt noise Gt^T, entry (i, j)
LSQ_HD double q_entry(const PredictBlocks& b, const double* noise, int i, int j, double dt) {
  const double dt2 = dt * dt;
  if (i / 3 == 1 && j / 3 == 1) {
    const int r = i % 3, c = j % 3;
    double s = 0;
    for (int k = 0; k < 3; ++k) s += b.R.a[3 * r + k] * b.R.a[3 * c + k];
    return s * noise[0] * dt2;
  }
  if (i != j) return 0.0;
  if (i / 3 == 2) return noise[1] * dt2;
  if (i / 3 == 3) return noise[2] * dt2;
  if (i / 3 == 4) return noise[3] * dt2;
  return 0.0;
}
// (F P)(i, j), F row-major, P column-major
LSQ_HD double fp_entry(const double* F, const double* P, int i, int j) {
  double s = 0.0;
  for (int k = 0; k < 18; ++k) {
    const double f = F[i * 18 + k];
    if (f == 0.0) continue;
    s += f * P[j * 18 + k];
  }
  return s;
}
// (F P F^T + Q)(i, j), FP row-major
LSQ_HD double fpft_entry(const double* FP, const double* F, double q, int i, int j) {
  double s = 0;
  for (int k = 0; k < 18; ++k) s += FP[i * 18 + k] * F[j * 18 + k];
  return s + q;
}

// One predict call on the host (the g++ test; the device runs the same phases across a warp).  s: 19 doubles, P: 324.
inline void predict_host(double* s, double* P, double* acc_last, double* gyr_last, const double* noise, double dt, const double* acc,
                         const double* gyr) {
  const PredictBlocks b = predict_state(s, acc_last, gyr_last, dt, acc, gyr);
  double Ft[324], F[324], FP[324], P2[324];
  for (int e = 0; e < 324; ++e) Ft[e] = ft_entry(b, e / 18, e % 18);
  for (int e = 0; e < 324; ++e) F[e] = f_entry(Ft, e / 18, e % 18, dt);
  for (int e = 0; e < 324; ++e) FP[e] = fp_entry(F, P, e / 18, e % 18);
  for (int e = 0; e < 324; ++e) P2[e] = fpft_entry(FP, F, q_entry(b, noise, e / 18, e % 18, dt), e / 18, e % 18);
  for (int e = 0; e < 324; ++e) { const int i = e / 18, j = e % 18; P[j * 18 + i] = 0.5 * (P2[i * 18 + j] + P2[j * 18 + i]); }
  for (int k = 0; k < 3; ++k) { acc_last[k] = acc[k]; gyr_last[k] = gyr[k]; }
}

// ---- reset(1) (kalman_filter.hpp:226-248) ---------------------------------------------------------------------------
LSQ_HD M3 block3(const double* P, int r0, int c0) {
  M3 m;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) m.a[3 * i + j] = P[(c0 + j) * 18 + r0 + i];
  return m;
}
LSQ_HD void set_block3(double* P, int r0, int c0, const M3& m) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) P[(c0 + j) * 18 + r0 + i] = m.a[3 * i + j];
}
LSQ_HD void reset1(double* s, double* P, const Consts& k) {
  const M3 vel_cov = block3(P, kVel, kVel), acc_cov = block3(P, kAcc, kAcc), gyr_cov = block3(P, kGyr, kGyr), gra_cov = block3(P, kGra, kGra);
  Q4 q = ldq(s);
  const M3 Rinv = qtoR(qinverse(q)), R = qtoR(q);
  for (int e = 0; e < 324; ++e) P[e] = 0.0;
  for (int i = 0; i < 3; ++i) { P[(kPos + i) * 18 + kPos + i] = k.pos_var[i]; P[(kAtt + i) * 18 + kAtt + i] = k.att_var[i]; }
  set_block3(P, kVel, kVel, mmul(mmul(Rinv, vel_cov), R));
  set_block3(P, kAcc, kAcc, acc_cov);
  set_block3(P, kGyr, kGyr, gyr_cov);
  set_block3(P, kGra, kGra, mmul(mmul(Rinv, gra_cov), R));
  st3(s, sRn, v3(0.0, 0.0, 0.0));
  st3(s, sVn, qrot(qinverse(q), ld3(s, sVn)));
  q = qident();
  stq(s, q);
  V3 gn = qrot(qinverse(q), ld3(s, sGn));
  const double n = vnorm(gn);
  st3(s, sGn, vdiv(vscl(9.81, gn), n));
}

// ---- integrateTransformation + the roll / pitch correction (state_estimator.hpp:205-209, :253-271) ------------------
// g: globalState_ (19), f: filter_->state_ before reset(1)
LSQ_HD void integrate(double* g, const double* f) {
  const Q4 fq = ldq(f);
  Q4 gq = ldq(g);
  st3(g, sRn, vadd(qrot(gq, ld3(f, sRn)), ld3(g, sRn)));
  gq = qmul(gq, fq);
  stq(g, gq);
  st3(g, sVn, qrot(qmul(gq, qinverse(fq)), ld3(f, sVn)));
  for (int i = 0; i < 3; ++i) { g[sBa + i] = f[sBa + i]; g[sBw + i] = f[sBw + i]; }
  st3(g, sGn, qrot(gq, ld3(f, sGn)));
}
// fs: filter_->state_ after reset(1)
LSQ_HD void correct_roll_pitch(double* g, const double* fs) {
  const V3 fb = ld3(fs, sGn);
  const double pitch = -sign(fb.d[2]) * asin(fb.d[0] / kG0);
  const double roll = sign(fb.d[2]) * asin(fb.d[1] / kG0);
  const V3 rpy = Q2rpy(ldq(g));
  stq(g, rpy2Quat(v3(roll, pitch, rpy.d[2])));
}

// ---- sequence initialisation: processFirstScan / processSecondScan (state_estimator.hpp:186-220) ---------------------
// The constants they read.  var = the diagonal initializeCovariance installs (kalman_filter.hpp:197-209), in error-state
// order: sq(init_pos_std), sq(init_vel_std), pow(deg2rad(init_att_std), 2), sq(init_acc_std), sq(init_gyr_std), 0.01 —
// computed on the host once, like Consts; ba / bw = init_ba / init_bw.
struct InitConsts {
  double var[18];
  double ba[3], bw[3];
};

// The pre-integration between the first and the second scan (state_estimator.hpp:41-62): 20 doubles per sequence,
// acc_0[0..2] gyr_0[3..5] delta_p[6..8] delta_v[9..11] delta_q(x,y,z,w)[12..15] sum_dt[16]; linearized_ba / bg are init_ba /
// init_bw.
constexpr int pAcc = 0, pGyr = 3, pDp = 6, pDv = 9, pDq = 12, pSum = 16;
LSQ_HD Q4 ldq_at(const double* s, int o) { return q4(s[o + 3], s[o], s[o + 1], s[o + 2]); }
LSQ_HD void stq_at(double* s, int o, Q4 q) { s[o] = q.x; s[o + 1] = q.y; s[o + 2] = q.z; s[o + 3] = q.w; }

// IntegrationBase(acc0, gyr0, ba, bg): delta_p = delta_v = 0, delta_q = identity, sum_dt = 0
LSQ_HD void preint_begin(double* pre, const double* imu) {
  for (int i = 0; i < 20; ++i) pre[i] = 0.0;
  for (int i = 0; i < 3; ++i) { pre[pAcc + i] = imu[i]; pre[pGyr + i] = imu[3 + i]; }
  stq_at(pre, pDq, qident());
}
// IntegrationBase::propagate
LSQ_HD void preint_propagate(double* pre, const InitConsts& k, double dt, const double* acc, const double* gyr) {
  const V3 ba = ld3(k.ba, 0), bg = ld3(k.bw, 0), a0 = ld3(pre, pAcc), g0 = ld3(pre, pGyr), a1 = ld3(acc, 0), g1 = ld3(gyr, 0);
  const V3 dp = ld3(pre, pDp), dv = ld3(pre, pDv);
  const Q4 dq = ldq_at(pre, pDq);
  const V3 un_acc_0 = qrot(dq, vsub(a0, ba));
  const V3 un_gyr = vsub(vscl(0.5, vadd(g0, g1)), bg);
  const Q4 rq = qmul(dq, q4(1.0, un_gyr.d[0] * dt / 2, un_gyr.d[1] * dt / 2, un_gyr.d[2] * dt / 2));
  const V3 un_acc_1 = qrot(rq, vsub(a1, ba));
  const V3 un_acc = vscl(0.5, vadd(un_acc_0, un_acc_1));
  st3(pre, pDp, vadd(vadd(dp, vscl(dt, dv)), vscl(0.5 * dt * dt, un_acc)));
  st3(pre, pDv, vadd(dv, vscl(dt, un_acc)));
  stq_at(pre, pDq, qnormalized(rq));
  pre[pSum] += dt;
  st3(pre, pAcc, a1);
  st3(pre, pGyr, g1);
}

// GlobalState::setIdentity (19 doubles + the device's pad)
LSQ_HD void state_identity(double* s) {
  for (int i = 0; i < 20; ++i) s[i] = 0.0;
  stq(s, qident());
  s[sGn + 2] = -kG0;
}
// GlobalState(rn, vn, qbn, ba, bw)
LSQ_HD void state_set(double* s, V3 rn, V3 vn, Q4 q, V3 ba, V3 bw) {
  state_identity(s);
  st3(s, sRn, rn); st3(s, sVn, vn); stq(s, q); st3(s, sBa, ba); st3(s, sBw, bw);
}
// StatePredictor::initializeCovariance (P column-major; only the diagonal is non-zero)
LSQ_HD void initialize_covariance(double* P, const InitConsts& k) {
  for (int e = 0; e < 324; ++e) P[e] = 0.0;
  for (int i = 0; i < 18; ++i) P[i * 18 + i] = k.var[i];
}

// What a newly constructed StateEstimator holds: globalState_ and the filter state identity, initializeCovariance
LSQ_HD void fresh_slot(double* glob, double* filt, double* P, const InitConsts& k) {
  state_identity(glob);
  state_identity(filt);
  initialize_covariance(P, k);
}

// processFirstScan once its gate has passed: linState_ identity, a new pre-integration from the scan's IMU sample, and
// filter_->initialization(time, 0, 0, 0, 0, acc, gyr).  imu: acc (3) + gyr (3) of the scan; imu_last: acc_last / gyr_last.
LSQ_HD void first_scan(double* filt, double* P, double* lin, double* pre, double* imu_last, const double* imu, const InitConsts& k) {
  const V3 z = v3(0.0, 0.0, 0.0);
  state_identity(lin);
  preint_begin(pre, imu);
  state_set(filt, z, z, rpy2Quat(v3(0.0, 0.0, 0.0)), z, z);
  for (int i = 0; i < 6; ++i) imu_last[i] = imu[i];
  initialize_covariance(P, k);
}

// processSecondScan, before estimateTransform: the ICP's start pose pl = delta_p + 0.5 sum_dt^2 gn (linState_.gn_ is
// the identity's), ql = delta_q, as the 20-double pose block the ICP linearises at (t at 0..2, q at 6..9, the rest 0)
LSQ_HD void second_scan_start(const double* pre, double* pose) {
  const double sum_dt = pre[pSum];
  const V3 gn = v3(0.0, 0.0, -kG0);
  for (int i = 0; i < 20; ++i) pose[i] = 0.0;
  st3(pose, sRn, vadd(ld3(pre, pDp), vscl(0.5 * sum_dt * sum_dt, gn)));
  stq(pose, ldq_at(pre, pDq));
}

// processSecondScan after estimateTransform (pose: its result): linState_ = (t, q) over the identity,
// estimateInitialState (v = p / sum_dt: no guard, like the reference), filter_->initialization(time, pl, v1, ba0, bw0, acc,
// gyr), calculateRPfromGravity(acc - ba0) and the hand-over to globalState_.
LSQ_HD void second_scan(double* glob, double* filt, double* P, double* lin, double* imu_last, const double* pre, const double* pose,
                        const double* imu, const InitConsts& k) {
  const V3 pl = ld3(pose, sRn);
  const Q4 ql = ldq(pose);
  state_identity(lin);
  st3(lin, sRn, pl);
  stq(lin, ql);
  const V3 v1 = vdiv(pl, pre[pSum]);
  const V3 ba0 = ld3(k.ba, 0), bw0 = ld3(k.bw, 0);
  state_set(filt, pl, v1, rpy2Quat(v3(0.0, 0.0, 0.0)), ba0, bw0);
  for (int i = 0; i < 6; ++i) imu_last[i] = imu[i];
  initialize_covariance(P, k);
  const V3 f = vsub(ld3(imu, 0), ba0);
  const double pitch = -sign(f.d[2]) * asin(f.d[0] / kG0);
  const double roll = sign(f.d[2]) * asin(f.d[1] / kG0);
  state_set(glob, pl, v1, rpy2Quat(v3(roll, pitch, 0.0)), ba0, bw0);
}

}  // namespace lins_seq
