// lins_map_types.cuh — the records row F2's kernels (lins_map.cuh) share with host code that launches none of them
// (lins_mappers.cu): no kernels here, so any translation unit may include it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lins_map {

struct PassConsts {
  float cRoll, sRoll, cPitch, sPitch, cYaw, sYaw, tX, tY, tZ;  // updatePointAssociateToMapSinCos :579-592
  float srx, crx, sry, cry, srz, crz;                          // LMOptimization :1527-1532
};

struct GridIndex {
  const float4* pts;      // map points bucket-sorted: (x, y, z, original index as int bits)
  const int* start;       // [n_buckets + 1]
  unsigned mask;          // n_buckets - 1 (power of two)
  float ox, oy, oz;       // grid origin
};
// one slot of a many-slot scan-to-map queue (lins_gpu_mappers_step): maps and queries k = 0 corner, 1 surf
struct MapSlot {
  GridIndex g[2];         // its grids: the shared bucket arrays from bucket0[k] on
  const float4* map[2];   // map clouds (capacities cap[k]; the first *n_map[k] points are real)
  const float4* q[2];     // query clouds (capacities nq[k]; NaN past the real points)
  const int* n_map[2];
  int cap[2], nq[2];
  int blk[2], nblk[2];    // its fit blocks in the corner / surf launch
  int bucket0[2], m0[2];  // first bucket; first point in the grid build's numbering (slot-major, corner then surf)
  float T[6];             // transformTobeMapped at the start
  int run;                // 0: the loop starts done (no map)
};

// state of one scan2MapOptimization call on the device
struct MapLoopState {
  float T[6];            // transformTobeMapped
  float matP[36];
  int isDegenerate, done, iters, converged;
  int n_sel[10];  // (LINS_MAP_MAX_ITER)
  float delta_r[10], delta_t[10];
};

}  // namespace lins_map
