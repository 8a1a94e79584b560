// global_map.hpp — the key-frame selection of the mapping node's publishGlobalMap (lidar_mapping_node.cpp:976-1031):
// steps 1-3 of DESIGN.md §4.15 on a node's key poses (lins_loops.cu gathers and down-samples the named key frames).
// Plain C++ with no CUDA, so the CPU suite compiles it with g++ (tests/test_globalmap_cpu.py).  f32 arithmetic as the
// reference types it, without contraction (g++ does not contract on x86-64 without -mfma; nvcc's host pass neither).
#pragma once
#include <algorithm>
#include <cassert>
#include <climits>
#include <cmath>
#include <cstdint>
#include <utility>
#include <vector>

namespace lins_gm {

constexpr float kRadiusSq = 500.0f * 500.0f;  // globalMapVisualizationSearchRadius (parameters.h:101), compared squared
constexpr float kPoseLeaf = 1.0f;             // downSizeFilterGlobalMapKeyPoses (:1003)

// globalMapKeyPoses: the key poses within the radius of cur (KdTreeFLANN::radiusSearch, max_nn = 0), as loop_candidate
// compares: the f32 squared distance ((dx^2 + dy^2) + dz^2) strictly below 500^2.  A non-finite pose, which
// setInputCloud drops, fails the test.  Ascending key index.
template <typename Pose>
std::vector<int32_t> select_key_poses(const std::vector<Pose>& poses, const float cur[3]) {
  std::vector<int32_t> sel;
  for (int32_t i = 0; i < (int32_t)poses.size(); ++i) {
    const Pose& q = poses[i];
    const float ex = q.x - cur[0], ey = q.y - cur[1], ez = q.z - cur[2];
    const float d2 = ex * ex + ey * ey + ez * ez;
    if (d2 < kRadiusSq) sel.push_back(i);
  }
  return sel;
}

// globalMapKeyPosesDS: pcl::VoxelGrid at 1 m of the selected poses (x, y, z, intensity = key index), and of each voxel,
// in ascending voxel index, (int) of its intensity centroid: the f32 sum of the indices in input order over the f32
// count, truncated.  That may name a key frame outside the voxel, and two voxels may name the same key frame.  Only the
// intensities are read, so the x, y, z centroids are not formed.  The box's bounds are the f32 floors of min * inv and
// max * inv as feature_extraction.hpp's VoxelGrid computes them; in a 500 m ball their differences are exact and at
// most 1001, so the box has at most 1002^3 < INT32_MAX voxels.
template <typename Pose>
std::vector<int32_t> key_poses_ds(const std::vector<Pose>& poses, const std::vector<int32_t>& sel) {
  std::vector<int32_t> ids;
  if (sel.empty()) return ids;
  const float inv = 1.0f / kPoseLeaf;  // (lins_feat::voxel_inv)
  float lo[3], hi[3];
  for (int k = 0; k < 3; ++k) { lo[k] = INFINITY; hi[k] = -INFINITY; }
  auto xyz = [&](int32_t i, int k) { return k == 0 ? poses[i].x : k == 1 ? poses[i].y : poses[i].z; };
  for (int32_t i : sel)
    for (int k = 0; k < 3; ++k) { lo[k] = std::min(lo[k], xyz(i, k)); hi[k] = std::max(hi[k], xyz(i, k)); }
  long long mul[3];
  for (int k = 0; k < 3; ++k) { lo[k] = std::floor(lo[k] * inv); hi[k] = std::floor(hi[k] * inv); }
  const long long div[3] = {(long long)(hi[0] - lo[0]) + 1, (long long)(hi[1] - lo[1]) + 1, (long long)(hi[2] - lo[2]) + 1};
  assert(div[0] <= 1002 && div[1] <= 1002 && div[2] <= 1002);
  assert(div[0] * div[1] * div[2] <= (long long)INT_MAX);
  mul[0] = 1; mul[1] = div[0]; mul[2] = div[0] * div[1];
  std::vector<std::pair<long long, int32_t>> key(sel.size());  // (voxel, key index), sorted stably: input order per voxel
  for (size_t j = 0; j < sel.size(); ++j) {
    long long v = 0;
    for (int k = 0; k < 3; ++k) v += (long long)(std::floor(xyz(sel[j], k) * inv) - lo[k]) * mul[k];
    key[j] = {v, sel[j]};
  }
  std::stable_sort(key.begin(), key.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  for (size_t j = 0; j < key.size();) {
    float sum = 0.f;
    size_t e = j;
    for (; e < key.size() && key[e].first == key[j].first; ++e) sum += (float)key[e].second;
    const int32_t id = (int32_t)(sum / (float)(e - j));
    // the sum is of non-negative values; the mean of c distinct indices lies (c - 1) / 2 or more below the largest, and
    // the sum's f32 error moves the mean by less than mean * c * 2^-24: below 2^22 key poses the id stays in range
    assert(id >= 0 && id < (int32_t)poses.size());
    ids.push_back(id);
    j = e;
  }
  return ids;
}

}  // namespace lins_gm
