// lins_cloud2.cuh — the per-field conversion and the layout check of sensor_msgs/PointCloud2 decoding (pcl::fromROSMsg
// <pcl::PointXYZI>, image_projection_node.cpp:172-177), shared by the device decode (lins_cloud2.cu) and the host.  No
// CUDA types outside __CUDA_ARCH__ blocks: tests/test_cloud2_cpu.py compiles this header with g++ and checks it against
// csrc/host/rosbag_reader.hpp (read_scalar, decode_pointcloud2).  DESIGN.md §4.8.
#pragma once
#include <cstdint>
#include <cstring>

#include "../../../include/lins_gpu.h"

#ifdef __CUDACC__
#define LINS_C2_HD __host__ __device__ __forceinline__
#else
#define LINS_C2_HD inline
#endif

namespace lins_cloud2 {

// bytes of a sensor_msgs/PointField datatype (1 INT8, 2 UINT8, 3 INT16, 4 UINT16, 5 INT32, 6 UINT32, 7 FLOAT32,
// 8 FLOAT64; anything else 0)
LINS_C2_HD uint32_t type_size(uint32_t dt) { return dt == 8 ? 8u : dt >= 5 && dt <= 7 ? 4u : dt >= 3 && dt <= 4 ? 2u : dt >= 1 && dt <= 2 ? 1u : 0u; }

// A field's little-endian bits (the low type_size(dt) bytes of b) -> (float)read_scalar(p, dt): the integers and the
// double are rounded once, to nearest even (int32 / uint32 above 2^24, doubles); a float keeps its bits, so -0.0, inf
// and NaN stay what they are (the host's float -> double -> float may quiet a signalling NaN: NaN either way).
LINS_C2_HD float to_float(uint64_t b, uint32_t dt) {
  const uint32_t lo = (uint32_t)b;
  switch (dt) {
    case 1: return (float)(int8_t)(uint8_t)lo;  // (exact)
    case 2: return (float)(uint8_t)lo;
    case 3: return (float)(int16_t)(uint16_t)lo;
    case 4: return (float)(uint16_t)lo;
#ifdef __CUDA_ARCH__
    case 5: return __int2float_rn((int)lo);
    case 6: return __uint2float_rn(lo);
    case 7: return __uint_as_float(lo);
    case 8: return __double2float_rn(__longlong_as_double((long long)b));
#else
    case 5: { int32_t v; std::memcpy(&v, &lo, 4); return (float)(double)v; }
    case 6: return (float)(double)lo;
    case 7: { float v; std::memcpy(&v, &lo, 4); return v; }
    case 8: { double v; std::memcpy(&v, &b, 8); return (float)v; }
#endif
  }
  return 0.f;
}

// the little-endian bits of the size-byte field at p (host; the device assembles them from aligned words)
inline uint64_t load_host(const uint8_t* p, uint32_t size) {
  uint64_t b = 0;
  for (uint32_t k = 0; k < size; ++k) b |= (uint64_t)p[k] << (8 * k);
  return b;
}

// nullptr when decode_pointcloud2 (csrc/host/rosbag_reader.hpp) accepts a message of layout l whose data field is len
// bytes long, else the reason it does not.  Every extent in 128-bit arithmetic: no product of two u32 wraps.
inline const char* check_layout(const lins_cloud2_layout& l, int64_t len) {
  if (l.is_bigendian) return "big-endian PointCloud2 data";
  for (int k = 0; k < 4; ++k) {
    const uint32_t dt = l.datatype[k];
    if (k == 3 && dt == 0) continue;  // no intensity field
    if (dt == 0) return "PointCloud2 without an x, y or z field";
    if (dt > 8) return "PointField datatype outside 1..8";
    if ((uint64_t)l.offset[k] + type_size(dt) > (uint64_t)l.point_step) return "PointField past point_step";
  }
  if ((uint64_t)l.width * l.height == 0) return nullptr;
  const unsigned __int128 end = (unsigned __int128)(l.height - 1) * l.row_step + (unsigned __int128)(l.width - 1) * l.point_step + l.point_step;
  if (len < 0 || end > (unsigned __int128)(uint64_t)len) return "PointCloud2 point past the message's data";
  return nullptr;
}

}  // namespace lins_cloud2
