// lins_projection.cuh — the per-pixel arithmetic of image projection (lins/src/image_projection_node.cpp:191-415:
// findStartEndAngle, projectPointCloud, groundRemoval's angle test, labelComponents' edge test) as __host__ __device__
// code.  lins_projection.cu runs it on the device; g++ compiles the same header next to csrc/host/image_projection.hpp so a
// CPU test checks it bit for bit (tests/test_projection_cpu.py).  The contract is the host restatement, expression by
// expression: `std::atan2(float, float) * 180` is a float product and only `/ M_PI` is double.  Plain IEEE arithmetic:
// the device unit is built with -fmad=false, and g++ on x86-64 without -mfma does not contract either.
//
// The transcendentals are glibc's atan2f (lins_features.cuh restates it; equal on normal inputs, an ulp apart at worst
// with a subnormal x) and sqrtf (correctly rounded on both sides).  The edge test's sinf / cosf of the two angular
// resolutions are constants of a lidar model: the host computes them with libm and passes them in.
#pragma once
#include "lins_features.cuh"

namespace lins_proj {

using lins_feat::atan2f_fdlibm;

// findStartEndAngle (:191-203) of a scan with n >= 2 points: p0 = point 0, pl = point n - 1, pl2x = point n - 2's x (the
// reference's [size - 2].x slip).  ori = startOrientation, endOrientation, orientationDiff (cloud_info's floats).
LINS_FHD void start_end_angle(float p0x, float p0y, float ply, float pl2x, float ori[3]) {
  const float start = -atan2f_fdlibm(p0y, p0x);
  float end = (float)(-atan2f_fdlibm(ply, pl2x) + 2 * M_PI);
  if (end - start > 3 * M_PI) end = (float)(end - 2 * M_PI);
  else if (end - start < M_PI) end = (float)(end + 2 * M_PI);
  ori[0] = start;
  ori[1] = end;
  ori[2] = end - start;
}

// projectPointCloud (:205-243) for one point: its pixel, or false where the reference skips it (outside the fan,
// colD < 0, or past the wrap).  A NaN point fails !(rowF >= 0).  colD >= 2 * scan_num is skipped before the conversion
// to an integer: the reference's (long) of such a value is still >= scan_num after the wrap (or LONG_MIN, < 0).
LINS_FHD bool project(float x, float y, float z, int line_num, int scan_num, float ang_res_x, float ang_res_y, float ang_bottom,
                      int& row, int& col) {
  const float verticalAngle = (float)(atan2f_fdlibm(z, sqrtf(x * x + y * y)) * 180 / M_PI);
  const float rowF = (verticalAngle + ang_bottom) / ang_res_y;
  if (!(rowF >= 0) || rowF >= (float)line_num) return false;
  const float horizonAngle = (float)(atan2f_fdlibm(x, y) * 180 / M_PI);
  const double colD = -round((horizonAngle - 90.0) / ang_res_x) + scan_num / 2;
  if (colD < 0 || colD >= 2.0 * scan_num) return false;
  long c = (long)colD;
  if (c >= scan_num) c -= scan_num;
  row = (int)rowF;
  col = (int)c;
  return true;
}

// the range image's value of a point (:231)
LINS_FHD float point_range(float x, float y, float z) { return sqrtf(x * x + y * y + z * z); }

// the intensity fullCloud carries (:234): row + col / 10000, the sum in double, rounded once
LINS_FHD float pixel_intensity(int row, int col) { return (float)((float)row + (float)col / 10000.0); }

// groundRemoval's test of a vertical pixel pair (:262-274): lower point l, upper point u, sensorMountAngle 0
LINS_FHD bool ground_pair(float lx, float ly, float lz, float ux, float uy, float uz) {
  const float diffX = ux - lx, diffY = uy - ly, diffZ = uz - lz;
  const float angle = (float)(atan2f_fdlibm(diffZ, sqrtf(diffX * diffX + diffY * diffY)) * 180 / M_PI);
  return fabsf(angle - 0.0f) <= 10;
}

// labelComponents' segmentAlphaX / Y (:350-351): the angular resolution in radians, stored as float
LINS_FHD float segment_alpha(float ang_res) { return (float)(ang_res / 180.0 * M_PI); }

// labelComponents' edge test (:384-391) from a pixel of range r_from to a neighbour of range r_this, with sin_a / cos_a =
// sinf / cosf of the direction's segment_alpha.  std::max / std::min of floats.
LINS_FHD bool edge(float r_from, float r_this, float sin_a, float cos_a) {
  const float d1 = r_from < r_this ? r_this : r_from;
  const float d2 = r_this < r_from ? r_this : r_from;
  return atan2f_fdlibm(d2 * sin_a, d1 - d2 * cos_a) > 1.0472f;
}

}  // namespace lins_proj
