// lins_features.cuh — the per-point arithmetic of StateEstimator's feature extraction (lins/include/StateEstimator.hpp:
// rotatePoint :1104-1114, undistortPcl :619-654, calculateSmoothness :656-678, markOccludedPoints :680-713) and the voxel
// key of the per-ring pcl::VoxelGrid (:822-825), as __host__ __device__ code.  lins_features.cu runs it on the device; g++
// compiles the same header next to csrc/host/feature_extraction.hpp so a CPU test checks it bit for bit (tests/
// test_features_cpu.py).  Plain IEEE arithmetic only: the device unit is built with -fmad=false, and g++ on x86-64 without
// -mfma does not contract either.
//
// The one transcendental is the float atan2 of undistortPcl: `std::atan2(point.y, point.x)` of two floats resolves to the
// float overload, glibc's atan2f.  Up to glibc 2.40 that is the fdlibm float algorithm (not correctly rounded: it differs
// from the f64 atan2 rounded to float on about one input in six), so atan2f_fdlibm below restates that algorithm in float
// arithmetic.  It equals glibc 2.39's atan2f on all normal inputs (5e7 random pairs, tests/test_features_cpu.py checks
// a sample); with a subnormal x the two can differ by an ulp.  A glibc with a correctly rounded atan2f (2.41+) would
// need the f64 atan2 rounded to float instead.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define LINS_FHD __host__ __device__ __forceinline__
#else
#define LINS_FHD inline
#endif

namespace lins_feat {

// the largest ring span (endRingIndex - startRingIndex) the on-chip sorts take; include/lins_gpu.h LINS_FEAT_RING_CAP
constexpr int kRingCap = 2048;
constexpr int kMaxLines = 128;

LINS_FHD uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
LINS_FHD float bitsf(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

// fdlibm s_atanf.c (Sun Microsystems, freely redistributable): atan(x) in float by argument reduction to one of four
// breakpoints and an 11-term odd polynomial
LINS_FHD float atanf_fdlibm(float x) {
  const float atanhi[4] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f, 1.5707962513e+00f};
  const float atanlo[4] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f, 7.5497894159e-08f};
  const float aT[11] = {3.3333334327e-01f, -2.0000000298e-01f, 1.4285714924e-01f, -1.1111110449e-01f,
                        9.0908870101e-02f, -7.6918758452e-02f, 6.6610731184e-02f, -5.8335702866e-02f,
                        4.9768779427e-02f, -3.6531571299e-02f, 1.6285819933e-02f};
  const int32_t hx = (int32_t)fbits(x), ix = hx & 0x7fffffff;
  int id;
  if (ix >= 0x50800000) {  // |x| >= 2^34
    if (ix > 0x7f800000) return x + x;
    return hx > 0 ? atanhi[3] + atanlo[3] : -atanhi[3] - atanlo[3];
  }
  if (ix < 0x3ee00000) {  // |x| < 0.4375
    if (ix < 0x31000000) return x;
    id = -1;
  } else {
    x = fabsf(x);
    if (ix < 0x3f980000) {
      if (ix < 0x3f300000) { id = 0; x = (2.0f * x - 1.0f) / (2.0f + x); }
      else { id = 1; x = (x - 1.0f) / (x + 1.0f); }
    } else if (ix < 0x401c0000) { id = 2; x = (x - 1.5f) / (1.0f + 1.5f * x); }
    else { id = 3; x = -1.0f / x; }
  }
  float z = x * x;
  const float w = z * z;
  const float s1 = z * (aT[0] + w * (aT[2] + w * (aT[4] + w * (aT[6] + w * (aT[8] + w * aT[10])))));
  const float s2 = w * (aT[1] + w * (aT[3] + w * (aT[5] + w * (aT[7] + w * aT[9]))));
  if (id < 0) return x - x * (s1 + s2);
  z = atanhi[id] - ((x * (s1 + s2) - atanlo[id]) - x);
  return hx < 0 ? -z : z;
}

// fdlibm e_atan2f.c with the large-ratio cut-offs glibc 2.39 uses
LINS_FHD float atan2f_fdlibm(float y, float x) {
  const float tiny = 1.0e-30f, pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f,
              pi_lo = -8.7422776573e-08f;
  const int32_t hx = (int32_t)fbits(x), ix = hx & 0x7fffffff, hy = (int32_t)fbits(y), iy = hy & 0x7fffffff;
  if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;
  if (hx == 0x3f800000) return atanf_fdlibm(y);
  const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
  if (iy == 0) {
    if (m < 2) return y;
    return m == 2 ? pi + tiny : -pi - tiny;
  }
  if (ix == 0) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  if (ix == 0x7f800000) {
    if (iy == 0x7f800000) {
      switch (m) { case 0: return pi_o_4 + tiny; case 1: return -pi_o_4 - tiny; case 2: return 3.0f * pi_o_4 + tiny; default: return -3.0f * pi_o_4 - tiny; }
    }
    switch (m) { case 0: return 0.0f; case 1: return -0.0f; case 2: return pi + tiny; default: return -pi - tiny; }
  }
  if (iy == 0x7f800000) return hy < 0 ? -pi_o_2 - tiny : pi_o_2 + tiny;
  const int k = (iy - ix) >> 23;
  float z;
  if (k > 24) z = pi_o_2 + 0.5f * pi_lo;
  else if (hx < 0 && k < -26) z = 0.0f;
  else z = atanf_fdlibm(fabsf(y / x));
  switch (m) {
    case 0: return z;
    case 1: return bitsf(fbits(z) ^ 0x80000000u);
    case 2: return pi - (z - pi_lo);
    default: return (z - pi_lo) - pi;
  }
}

// rotatePoint (:1104-1114): c / s = cos / sin of deg2rad(IMU_LIDAR_EXTRINSIC_ANGLE), computed once with libm
LINS_FHD void rotate_xy(double c, double s, float x, float y, float& ox, float& oy) {
  const double px = x, py = y;
  ox = (float)(c * px - s * py);
  oy = (float)(s * px + c * py);
}

// undistortPcl's orientation of a (rotated) point before the halfPassed switch: the not-passed branch, and whether it
// flips halfPassed (:641-645).  The point where it flips still takes this branch.
LINS_FHD double ori_not_passed(float x, float y, float start, bool& flips) {
  double ori = -atan2f_fdlibm(y, x);
  if (ori < start - M_PI / 2) ori += 2 * M_PI;
  else if (ori > start + M_PI * 3 / 2) ori -= 2 * M_PI;
  flips = ori - start > M_PI;
  return ori;
}
// the branch of every point after the one that flipped (:646-650)
LINS_FHD double ori_passed(float x, float y, float end) {
  double ori = -atan2f_fdlibm(y, x);
  ori += 2 * M_PI;
  if (ori < end - M_PI * 3 / 2) ori += 2 * M_PI;
  else if (ori > end + M_PI / 2) ori -= 2 * M_PI;
  return ori;
}
// intensity = int(ring) + SCAN_PERIOD * relTime (:651-652), rounded to f32 once
LINS_FHD float stamp(float intensity, double ori, float start, float diff, double scan_period) {
  const double relTime = (ori - start) / diff;
  return (float)(int(intensity) + scan_period * relTime);
}

// calculateSmoothness (:660-664): float sums left to right (R[i] * 10 a float product), squared in double.  R points at
// range[i - 5].
LINS_FHD double curvature(const float* R) {
  const float d = R[0] + R[1] + R[2] + R[3] + R[4] - R[5] * 10 + R[6] + R[7] + R[8] + R[9] + R[10];
  return (double)d * d;
}

// markOccludedPoints (:684-711) for point i (5 <= i < n - 6): bit 0 marks [i - 5, i], bit 1 marks [i + 1, i + 6], bit 2
// marks i.  R and C point at range[i - 1] and col_ind[i - 1].
LINS_FHD int occlusion_marks(const float* R, const uint32_t* C) {
  const float depth1 = R[1], depth2 = R[2];
  const int columnDiff = abs(int(C[2] - C[1]));
  int marks = 0;
  if (columnDiff < 10) {
    if (depth1 - depth2 > 0.3) marks |= 1;
    else if (depth2 - depth1 > 0.3) marks |= 2;
  }
  const float diff1 = fabsf(R[0] - R[1]), diff2 = fabsf(R[2] - R[1]);
  if (diff1 > 0.02 * R[1] && diff2 > 0.02 * R[1]) marks |= 4;
  return marks;
}

// sextant j of a ring (:724-726), in 64-bit integers (int32 products of large indices overflow)
LINS_FHD void sextant(int64_t s, int64_t e, int j, int64_t& sp, int64_t& ep) {
  const int64_t a = s * (6 - j) + e * j, b = s * (5 - j) + e * (j + 1);
  // C++ integer division truncates toward zero
  sp = a / 6;
  ep = b / 6 - 1;
}

// pcl::VoxelGrid: inverse leaf (1.0f / leaf in f32, as setLeafSize takes it), the box bounds, and a point's voxel index.
// The leaf defaults to the 0.2 m of feature extraction; the mapping node's filters pass 0.2 / 0.4.
LINS_FHD float voxel_inv(float leaf = 0.2f) { return 1.0f / leaf; }
LINS_FHD int voxel_bound(float v, float inv = voxel_inv()) { return (int)floorf(v * inv); }
LINS_FHD uint32_t voxel_key(float x, float y, float z, const int min_b[3], const int mul[3], float inv = voxel_inv()) {
  const int i0 = (int)(floorf(x * inv) - (float)min_b[0]);
  const int i1 = (int)(floorf(y * inv) - (float)min_b[1]);
  const int i2 = (int)(floorf(z * inv) - (float)min_b[2]);
  return (uint32_t)(i0 * mul[0] + i1 * mul[1] + i2 * mul[2]);
}

}  // namespace lins_feat
