// global_state_yzx.hpp — globalStateYZX_ of StateEstimator::updatePointCloud (StateEstimator.hpp:1116-1161), the pose
// LinsFusion::publishTopics hands the mapping node:
//   rn_yzx  = Q_xyz_to_yzx * rn
//   qbn_yzx = Q_xyz_to_yzx * qbn * Q_xyz_to_yzx.inverse()
// in f64, each operation in the order of the Eigen expressions as math_utils.hpp restates them (Q4D operator*, the
// quaternion-vector product v + w t + q.vec x t with t = 2 q.vec x v, inverse() = conjugate / squaredNorm).  One copy,
// called by the shim's updatePointCloud and by sequence mode's publish step (lins_seq.cu), so the two are the same
// arithmetic.  PRODUCT code: no dependency, host only.
#ifndef LINS_HOST_GLOBAL_STATE_YZX_HPP_
#define LINS_HOST_GLOBAL_STATE_YZX_HPP_

namespace lins {

// Q_xyz_to_yzx = R2Quat(R_yzx_to_xyz^T) (StateEstimator.hpp:217-220), x y z w: Shepperd's method on that permutation
// matrix takes its trace-0 branch with i = 0 and every step exact
constexpr double kQxyzToYzx[4] = {0.5, 0.5, 0.5, -0.5};

namespace detail {
// a * b, both x y z w (math_utils.hpp: operator*(Q4D, Q4D))
inline void quat_mul(const double* a, const double* b, double* o) {
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  const double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
inline void cross3(const double* a, const double* b, double* o) {
  const double x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  o[0] = x; o[1] = y; o[2] = z;
}
}  // namespace detail

// rn (3), qbn (x y z w) -> pos (3), quat (x y z w) of globalStateYZX_ (outputs may not alias inputs)
inline void global_state_yzx(const double* rn, const double* qbn, double* pos, double* quat) {
  const double* Q = kQxyzToYzx;
  // Q * rn: t = 2.0 * cross(q.vec, v); v + q.w * t + cross(q.vec, t)
  double t[3], c[3];
  detail::cross3(Q, rn, t);
  for (int i = 0; i < 3; ++i) t[i] *= 2.0;
  detail::cross3(Q, t, c);
  for (int i = 0; i < 3; ++i) pos[i] = (rn[i] + t[i] * Q[3]) + c[i];
  // Q * qbn * Q.inverse(), left to right
  const double n = Q[0] * Q[0] + Q[1] * Q[1] + Q[2] * Q[2] + Q[3] * Q[3];
  const double qi[4] = {-Q[0] / n, -Q[1] / n, -Q[2] / n, Q[3] / n};
  double m[4];
  detail::quat_mul(Q, qbn, m);
  detail::quat_mul(m, qi, quat);
}

}  // namespace lins

#endif  // LINS_HOST_GLOBAL_STATE_YZX_HPP_
