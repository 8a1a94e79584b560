// lins_mapper_tf.cuh — the key-frame store's transform (transformPointCloud :624-652 with the constants of
// updateTransformPointCloudSinCos :609-622), shared by the units that fill the store and those that read a key frame's
// map-frame clouds from its body-frame ones: lins_mapper.cu (a step's saved and corrected key frames), lins_checkpoint.cu
// (a loaded slot's device store rebuilt from its body-frame clouds) and lins_loops.cu (the history sub-maps and global
// maps gathered from the host store).  All three are built with -fmad=false, so a point's transform is the same bits in
// each: the invariant c = T(b, pose) that the device store, the loads and the gathers rely on.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

#include "lins_ctx.hpp"

namespace lins_capi {

struct TfConsts { float cr, sr, cp, sp, cy, sy, tx, ty, tz; };

// updateTransformPointCloudSinCos of a key pose: libm's f32 sin / cos of the f32 fields (host)
inline TfConsts tf_consts(const MapperKeyPose& k) {
  TfConsts c;
  c.cr = std::cos(k.roll); c.sr = std::sin(k.roll); c.cp = std::cos(k.pitch); c.sp = std::sin(k.pitch);
  c.cy = std::cos(k.yaw); c.sy = std::sin(k.yaw); c.tx = k.x; c.ty = k.y; c.tz = k.z;
  return c;
}

// one point of transformPointCloud
__device__ __forceinline__ float4 tf_point(const TfConsts& c, const float4 p) {
  const float x1 = c.cy * p.x - c.sy * p.y;
  const float y1 = c.sy * p.x + c.cy * p.y;
  const float z1 = p.z;
  const float x2 = x1;
  const float y2 = c.cr * y1 - c.sr * z1;
  const float z2 = c.sr * y1 + c.cr * z1;
  return make_float4(c.cp * x2 + c.sp * z2 + c.tx, y2 + c.ty, -c.sp * x2 + c.cp * z2 + c.tz, p.w);
}

}  // namespace lins_capi
