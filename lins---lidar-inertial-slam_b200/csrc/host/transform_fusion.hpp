// transform_fusion.hpp — the LOAM pose algebra the mapping node and transform_fusion_node share, and the fusion node's
// output (transform_fusion_node.cpp, /integrated_to_init): every scan's odometry corrected by the mapping node's latest
// scan-to-map result.
//   - tf_get_rpy / tf_set_rpy: tf's Matrix3x3::getRPY and Quaternion::setRPY (= createQuaternionMsgFromRollPitchYaw), f64;
//   - odometry_transform: laserOdometryHandler's transformSum (lidar_mapping_node.cpp:711-724, transform_fusion_node.cpp
//     :217-231, the same conversion);
//   - transform_associate_to_map: transformAssociateToMap (lidar_mapping_node.cpp:411-536, transform_fusion_node.cpp
//     :91-215, the same algebra) in f32 with the f32 overloads of cos / sin / asin / atan2 (DESIGN.md §4.4);
//   - published_pair: what odomAftMappedHandler (:256-277) receives from publishTF (lidar_mapping_node.cpp:737-777);
//   - transform_fusion: laserOdometryHandler of transform_fusion_node (:217-254).
// One copy, called by the mapper's host cycle (lins_mapper.cu) and by the fusion entries (lins_mappers.cu, lins_seq.cu);
// the CPU suite compiles it with g++.  Built without multiply-add contraction (g++ does not contract on x86-64 without
// -mfma).  PRODUCT code: no dependency, host only.
#ifndef LINS_HOST_TRANSFORM_FUSION_HPP_
#define LINS_HOST_TRANSFORM_FUSION_HPP_

#include <cmath>

namespace lins_tf {

// tf::Matrix3x3(q).getRPY(roll, pitch, yaw) (tf/LinearMath/Matrix3x3.h: setRotation, getEulerYPR with solution 1)
inline void tf_get_rpy(double qx, double qy, double qz, double qw, double& roll, double& pitch, double& yaw) {
  const double d = qx * qx + qy * qy + qz * qz + qw * qw;
  const double s = 2.0 / d;
  const double xs = qx * s, ys = qy * s, zs = qz * s;
  const double wx = qw * xs, wy = qw * ys, wz = qw * zs;
  const double xx = qx * xs, xy = qx * ys, xz = qx * zs;
  const double yy = qy * ys, yz = qy * zs, zz = qz * zs;
  const double m00 = 1.0 - (yy + zz), m10 = xy + wz, m20 = xz - wy, m21 = yz + wx, m22 = 1.0 - (xx + yy);
  if (std::fabs(m20) >= 1) {
    yaw = 0;
    const double delta = std::atan2(m21, m22);
    if (m20 < 0) { pitch = M_PI / 2.0; roll = delta; }
    else { pitch = -M_PI / 2.0; roll = delta; }
  } else {
    pitch = -std::asin(m20);
    roll = std::atan2(m21 / std::cos(pitch), m22 / std::cos(pitch));
    yaw = std::atan2(m10 / std::cos(pitch), m00 / std::cos(pitch));
  }
}

// tf::Quaternion::setRPY(roll, pitch, yaw) -> q (x, y, z, w).  createQuaternionMsgFromRollPitchYaw copies it unchanged
// (quaternionTFToMsg normalises only beyond |length2 - 1| > 0.1, which setRPY's output never reaches).
inline void tf_set_rpy(double roll, double pitch, double yaw, double q[4]) {
  const double halfYaw = yaw * 0.5, halfPitch = pitch * 0.5, halfRoll = roll * 0.5;
  const double cosYaw = std::cos(halfYaw), sinYaw = std::sin(halfYaw);
  const double cosPitch = std::cos(halfPitch), sinPitch = std::sin(halfPitch);
  const double cosRoll = std::cos(halfRoll), sinRoll = std::sin(halfRoll);
  q[0] = sinRoll * cosPitch * cosYaw - cosRoll * sinPitch * sinYaw;
  q[1] = cosRoll * sinPitch * cosYaw + sinRoll * cosPitch * sinYaw;
  q[2] = cosRoll * cosPitch * sinYaw - sinRoll * sinPitch * cosYaw;
  q[3] = cosRoll * cosPitch * cosYaw + sinRoll * sinPitch * sinYaw;
}

// a LOAM transform (rx, ry, rz, tx, ty, tz) from a pose message whose orientation is quat (x, y, z, w): getRPY of the
// shuffled quaternion (z, -x, -y, w), then (-pitch, -yaw, roll), stored to f32
inline void odometry_transform(const double quat[4], const double pos[3], float T[6]) {
  double roll, pitch, yaw;
  tf_get_rpy(quat[2], -quat[0], -quat[1], quat[3], roll, pitch, yaw);
  T[0] = -pitch; T[1] = -yaw; T[2] = roll;
  T[3] = pos[0]; T[4] = pos[1]; T[5] = pos[2];
}

// the orientation a LOAM node publishes for a transform's angles: (-q.y, -q.z, q.x, q.w) of setRPY(T[2], -T[0], -T[1])
inline void published_quat(const float T[6], double quat[4]) {
  double q[4];
  tf_set_rpy(T[2], -T[0], -T[1], q);
  quat[0] = -q[1]; quat[1] = -q[2]; quat[2] = q[0]; quat[3] = q[3];
}

// transformAssociateToMap: Incre[3..5] and Tobe from Sum (the odometry), Bef (the odometry of the last transformUpdate)
// and Aft (the mapped pose of that update).  Incre[0..2] are not written.
inline void transform_associate_to_map(const float Sum[6], const float Bef[6], const float Aft[6], float Inc[6], float T[6]) {
  using std::cos; using std::sin;
  float x1 = cos(Sum[1]) * (Bef[3] - Sum[3]) - sin(Sum[1]) * (Bef[5] - Sum[5]);
  float y1 = Bef[4] - Sum[4];
  float z1 = sin(Sum[1]) * (Bef[3] - Sum[3]) + cos(Sum[1]) * (Bef[5] - Sum[5]);
  float x2 = x1;
  float y2 = cos(Sum[0]) * y1 + sin(Sum[0]) * z1;
  float z2 = -sin(Sum[0]) * y1 + cos(Sum[0]) * z1;
  Inc[3] = cos(Sum[2]) * x2 + sin(Sum[2]) * y2;
  Inc[4] = -sin(Sum[2]) * x2 + cos(Sum[2]) * y2;
  Inc[5] = z2;
  const float sbcx = sin(Sum[0]), cbcx = cos(Sum[0]), sbcy = sin(Sum[1]), cbcy = cos(Sum[1]), sbcz = sin(Sum[2]), cbcz = cos(Sum[2]);
  const float sblx = sin(Bef[0]), cblx = cos(Bef[0]), sbly = sin(Bef[1]), cbly = cos(Bef[1]), sblz = sin(Bef[2]), cblz = cos(Bef[2]);
  const float salx = sin(Aft[0]), calx = cos(Aft[0]), saly = sin(Aft[1]), caly = cos(Aft[1]), salz = sin(Aft[2]), calz = cos(Aft[2]);
  const float srx = -sbcx * (salx * sblx + calx * cblx * salz * sblz + calx * calz * cblx * cblz) -
                    cbcx * sbcy * (calx * calz * (cbly * sblz - cblz * sblx * sbly) - calx * salz * (cbly * cblz + sblx * sbly * sblz) + cblx * salx * sbly) -
                    cbcx * cbcy * (calx * salz * (cblz * sbly - cbly * sblx * sblz) - calx * calz * (sbly * sblz + cbly * cblz * sblx) + cblx * cbly * salx);
  T[0] = -std::asin(srx);
  const float srycrx = sbcx * (cblx * cblz * (caly * salz - calz * salx * saly) - cblx * sblz * (caly * calz + salx * saly * salz) + calx * saly * sblx) -
                       cbcx * cbcy * ((caly * calz + salx * saly * salz) * (cblz * sbly - cbly * sblx * sblz) +
                                      (caly * salz - calz * salx * saly) * (sbly * sblz + cbly * cblz * sblx) - calx * cblx * cbly * saly) +
                       cbcx * sbcy * ((caly * calz + salx * saly * salz) * (cbly * cblz + sblx * sbly * sblz) +
                                      (caly * salz - calz * salx * saly) * (cbly * sblz - cblz * sblx * sbly) + calx * cblx * saly * sbly);
  const float crycrx = sbcx * (cblx * sblz * (calz * saly - caly * salx * salz) - cblx * cblz * (saly * salz + caly * calz * salx) + calx * caly * sblx) +
                       cbcx * cbcy * ((saly * salz + caly * calz * salx) * (sbly * sblz + cbly * cblz * sblx) +
                                      (calz * saly - caly * salx * salz) * (cblz * sbly - cbly * sblx * sblz) + calx * caly * cblx * cbly) -
                       cbcx * sbcy * ((saly * salz + caly * calz * salx) * (cbly * sblz - cblz * sblx * sbly) +
                                      (calz * saly - caly * salx * salz) * (cbly * cblz + sblx * sbly * sblz) - calx * caly * cblx * sbly);
  T[1] = std::atan2(srycrx / cos(T[0]), crycrx / cos(T[0]));
  const float srzcrx = (cbcz * sbcy - cbcy * sbcx * sbcz) * (calx * salz * (cblz * sbly - cbly * sblx * sblz) - calx * calz * (sbly * sblz + cbly * cblz * sblx) + cblx * cbly * salx) -
                       (cbcy * cbcz + sbcx * sbcy * sbcz) * (calx * calz * (cbly * sblz - cblz * sblx * sbly) - calx * salz * (cbly * cblz + sblx * sbly * sblz) + cblx * salx * sbly) +
                       cbcx * sbcz * (salx * sblx + calx * cblx * salz * sblz + calx * calz * cblx * cblz);
  const float crzcrx = (cbcy * sbcz - cbcz * sbcx * sbcy) * (calx * calz * (cbly * sblz - cblz * sblx * sbly) - calx * salz * (cbly * cblz + sblx * sbly * sblz) + cblx * salx * sbly) -
                       (sbcy * sbcz + cbcy * cbcz * sbcx) * (calx * salz * (cblz * sbly - cbly * sblx * sblz) - calx * calz * (sbly * sblz + cbly * cblz * sblx) + cblx * cbly * salx) +
                       cbcx * cbcz * (salx * sblx + calx * cblx * salz * sblz + calx * calz * cblx * cblz);
  T[2] = std::atan2(srzcrx / cos(T[0]), crzcrx / cos(T[0]));
  x1 = cos(T[2]) * Inc[3] - sin(T[2]) * Inc[4];
  y1 = sin(T[2]) * Inc[3] + cos(T[2]) * Inc[4];
  z1 = Inc[5];
  x2 = x1;
  y2 = cos(T[0]) * y1 - sin(T[0]) * z1;
  z2 = sin(T[0]) * y1 + cos(T[0]) * z1;
  T[3] = Aft[3] - (cos(T[1]) * x2 + sin(T[1]) * z2);
  T[4] = Aft[4] - y2;
  T[5] = Aft[5] - (-sin(T[1]) * x2 + cos(T[1]) * z2);
}

// publishTF -> odomAftMappedHandler: the (transformAftMapped, transformBefMapped) pair the fusion node holds after the
// mapping node published aft / bef.  Every NaN becomes 0 (publishTF :738-750; here on the published copy only: the
// mapping node's own members keep theirs, DESIGN.md §4.9); the angles of aft go through the published orientation and
// getRPY of its shuffle in f64 and are stored to f32 (they wrap into the Euler ranges); the positions and bef go through
// the message's f64 fields unchanged.
inline void published_pair(const float aft[6], const float bef[6], float aft_out[6], float bef_out[6]) {
  float a[6];
  for (int i = 0; i < 6; ++i) {
    a[i] = std::isnan(aft[i]) ? 0.0f : aft[i];
    bef_out[i] = std::isnan(bef[i]) ? 0.0f : bef[i];
  }
  double q[4];
  published_quat(a, q);
  const double pos[3] = {a[3], a[4], a[5]};
  odometry_transform(q, pos, aft_out);
}

// transform_fusion_node's laserOdometryHandler for one odometry message (orientation quat x y z w, position pos):
// transformSum from the message, transformAssociateToMap against the fusion node's pair, and the published pose
// (/integrated_to_init): T = transformMapped, pos_out = T[3..5], quat_out = the orientation published for T.  published:
// the mapping node has published (aft, bef) (it has run a processed cycle); before that the fusion node's pair is the
// zeros it was constructed with, and aft / bef are not read.
inline void transform_fusion(const double quat[4], const double pos[3], bool published, const float aft[6], const float bef[6],
                             float T[6], double pos_out[3], double quat_out[4]) {
  float Sum[6], Aft[6] = {0, 0, 0, 0, 0, 0}, Bef[6] = {0, 0, 0, 0, 0, 0}, Inc[6];
  if (published) published_pair(aft, bef, Aft, Bef);
  odometry_transform(quat, pos, Sum);
  transform_associate_to_map(Sum, Bef, Aft, Inc, T);
  for (int i = 0; i < 3; ++i) pos_out[i] = T[3 + i];
  published_quat(T, quat_out);
}

}  // namespace lins_tf

#endif  // LINS_HOST_TRANSFORM_FUSION_HPP_
