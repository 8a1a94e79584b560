// lins_mapper.cu — the mapping node (lidar_mapping_node.cpp run() :1806-1855, without loop closure) whose cycle
// lins_mappers.cu runs for one or many drives: a node's host logic, its key-frame store's transform, and the device
// pcl::VoxelGrid the cycle runs (also behind lins_gpu_voxel_grid).
//
// Host, per node (MapperNode): transformAssociateToMap (csrc/host/transform_fusion.hpp, which the fusion shares), the
// fused pose of an odometry message against the node's state, the window's deque of key-frame ids, transformUpdate with
// the IMU ring, the 0.3 m key-frame test, the pose's round trip through gtsam's Rot3 and the loop-candidate search, in the
// reference's f32 / f64 types (no multiply-add contraction: this unit is built with -fmad=false and g++ does not
// contract on x86-64 without -mfma).  Device: the key-frame store, each key frame's DS clouds transformed into the map
// frame once, at save time, with its PointTypePose (one launch for the key frames a step saves); on a slot with loop
// closure the same launch writes the body-frame clouds into the host store through their mapped addresses.
//
// VoxelGrid (csrc/host/feature_extraction.hpp restates PCL's applyFilter), on one or many clouds (segments) in one pass:
// each segment's finite points' min / max (ordered-integer atomics: min / max are exact in any order), its min_b =
// floor(min * inv) as int64, the key floor(p * inv) - (float)min_b per axis (vg_key), a stable CUB radix
// sort of (key, index) — with more than one segment of ((segment, key), index) on 32 + ceil(log2 segments) bits, so
// the segments stay in their input ranges — and one centroid per voxel, its points summed in f32 in input order (the
// sort is stable), output in ascending key order at the segment's own offset.  Non-finite points and every point of a
// segment whose div_x * div_y * div_z exceeds INT32_MAX get the key 0xffffffff, which no voxel can have, and are
// dropped; each output has room for its segment's points and is NaN past the voxel count.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>

#include "../host/transform_fusion.hpp"
#include "lins_ctx.hpp"
#include "lins_features.cuh"
#include "lins_mapper_tf.cuh"

using namespace lins_capi;

namespace {

constexpr unsigned kInvalidKey = 0xffffffffu;
constexpr int kVgThreads = 256;

__device__ __forceinline__ unsigned f2ord(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }
__device__ __forceinline__ bool finite3(const float4 p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

// the segments of one VoxelGrid call: off (n + 1) and out (n) on the device; n == 1 needs neither (out is a kernel argument)
struct VgSegs { const int* off; float4* const* out; int n; };
__device__ __forceinline__ int seg_of(const VgSegs& sg, int i) {  // the segment of input point i
  if (sg.n == 1) return 0;
  int lo = 0, hi = sg.n - 1;
  while (lo < hi) { const int m = (lo + hi + 1) >> 1; if (__ldg(&sg.off[m]) <= i) lo = m; else hi = m - 1; }
  return lo;
}
__device__ __forceinline__ void vg_flush(VgInfo* info, const unsigned e[6]) {
  for (int k = 0; k < 3; ++k) { atomicMin(&info->enc[k], e[k]); atomicMax(&info->enc[3 + k], e[3 + k]); }
}
// 32-bit keys: one segment; 64-bit keys: (segment, voxel key)
template <typename Key> __device__ __forceinline__ Key make_key(int sgi, unsigned k) {
  if constexpr (sizeof(Key) == 8) return ((Key)sgi << 32) | k;
  else return k;
}
template <typename Key> __device__ __forceinline__ int key_seg(Key k) {
  if constexpr (sizeof(Key) == 8) return (int)(k >> 32);
  else return 0;
}
template <typename Key> __device__ __forceinline__ unsigned key_low(Key k) { return (unsigned)k; }

// per segment: the finite points' min / max.  Each warp scans one contiguous run of points, its lanes interleaved
// (coalesced loads); a lane looks its segment up only when it passes the end of the last one, and accumulates while the
// segment stays the same.  A warp whose lanes all end in one segment reduces before its one set of atomics.
__global__ void __launch_bounds__(kVgThreads) lins_vg_bounds_kernel(const float4* __restrict__ p, int n, VgSegs sg, VgInfo* __restrict__ info) {
  unsigned e[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
  int cur = -1, seg_end = 0;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5, warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long per = ((n + n_warps - 1) / n_warps + 31) & ~31ll;
  const int i1 = (int)min((long long)n, (warp + 1) * per);
  for (int i = (int)min((long long)n, warp * per) + (threadIdx.x & 31); i < i1; i += 32) {
    const float4 q = p[i];
    if (!finite3(q)) continue;
    if (i >= seg_end) {
      const int sgi = seg_of(sg, i);
      seg_end = sg.n == 1 ? n : __ldg(&sg.off[sgi + 1]);
      if (sgi != cur) {
        if (cur >= 0) vg_flush(info + cur, e);
        cur = sgi;
        for (int k = 0; k < 3; ++k) { e[k] = 0xffffffffu; e[3 + k] = 0u; }
      }
    }
    const unsigned a[3] = {f2ord(q.x), f2ord(q.y), f2ord(q.z)};
    for (int k = 0; k < 3; ++k) { e[k] = min(e[k], a[k]); e[3 + k] = max(e[3 + k], a[k]); }
  }
  const int c0 = __reduce_max_sync(0xffffffffu, cur);
  if (__all_sync(0xffffffffu, cur == c0 || cur < 0)) {
    for (int off = 16; off > 0; off >>= 1)
      for (int k = 0; k < 6; ++k) {
        const unsigned o = __shfl_xor_sync(0xffffffffu, e[k], off);
        e[k] = k < 3 ? min(e[k], o) : max(e[k], o);
      }
    if ((threadIdx.x & 31) == 0 && c0 >= 0) vg_flush(info + c0, e);
  } else if (cur >= 0) {
    vg_flush(info + cur, e);
  }
}

// getMinMax3D -> min_b, div_b, divb_mul (feature_extraction.hpp VoxelGrid::filter), one thread per segment.  The bounds
// are int64 of the f32 floors: an int cast clamps beyond 2^31 voxels from the origin, and a box there would get div = 1
// on that axis and merge distinct voxels.  A floor at or beyond 2^62 in magnitude (an overflow of min / max * inv to
// inf included) has no exact int64 difference and makes the segment toobig.
__global__ void lins_vg_box_kernel(VgInfo* __restrict__ infos, int n_seg) {
  const int sgi = blockIdx.x * blockDim.x + threadIdx.x;
  if (sgi >= n_seg) return;
  VgInfo& v = infos[sgi];
  v.any = v.enc[0] != 0xffffffffu;
  v.toobig = 0;
  if (!v.any) return;
  long long div[3];
  for (int k = 0; k < 3; ++k) {
    const float lo = floorf(ord2f(v.enc[k]) * v.inv), hi = floorf(ord2f(v.enc[3 + k]) * v.inv);
    if (!(fabsf(lo) < 0x1p62f && fabsf(hi) < 0x1p62f)) { v.toobig = 1; return; }
    v.base[k] = lo;
    div[k] = (long long)hi - (long long)lo + 1;
  }
  v.toobig = (double)div[0] * (double)div[1] * (double)div[2] > (double)INT_MAX;  // (exact below 2^53; no overflow)
  v.mul[0] = 1; v.mul[1] = (int)div[0]; v.mul[2] = v.toobig ? 0 : (int)(div[0] * div[1]);
}

// a point's voxel key (feature_extraction.hpp: (int)(floor(p * inv) - (float)min_b) per axis): the f32 differences to
// the box's f32 floor as int64, combined in 64 bits.  In a box of at most INT32_MAX voxels a difference rounds to at
// most 2^31, and the key stays below 0xffffffff.
__device__ __forceinline__ unsigned vg_key(const float4 q, const VgInfo& v) {
  const long long i0 = (long long)(floorf(q.x * v.inv) - v.base[0]);
  const long long i1 = (long long)(floorf(q.y * v.inv) - v.base[1]);
  const long long i2 = (long long)(floorf(q.z * v.inv) - v.base[2]);
  return (unsigned)(i0 + i1 * v.mul[1] + i2 * v.mul[2]);
}

// the keys, and NaN in every output record (the centroids then overwrite a segment's first `count`)
template <typename Key>
__global__ void __launch_bounds__(kVgThreads) lins_vg_key_kernel(const float4* __restrict__ p, int n, VgSegs sg, const VgInfo* __restrict__ info,
                                                                 float4* __restrict__ out, Key* __restrict__ key, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int sgi = seg_of(sg, i);
  const VgInfo& v = info[sgi];
  const float4 q = p[i];
  key[i] = make_key<Key>(sgi, v.any && !v.toobig && finite3(q) ? vg_key(q, v) : kInvalidKey);
  idx[i] = i;
  const float nan = __int_as_float(0xffffffff);
  if (sg.n == 1) out[i] = make_float4(nan, nan, nan, nan);
  else sg.out[sgi][i - __ldg(&sg.off[sgi])] = make_float4(nan, nan, nan, nan);
}

template <typename Key>
__global__ void __launch_bounds__(kVgThreads) lins_vg_head_kernel(const Key* __restrict__ key, int n, int* __restrict__ head) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  head[i] = key_low(key[i]) != kInvalidKey && (i == 0 || key[i] != key[i - 1]);
}

// one thread per voxel head: the f32 sums of its points in sorted (= input) order, divided by the count.  The sort keeps
// each segment in its input range, so a segment's voxel ids count from the inclusive scan just before that range.
template <typename Key>
__global__ void __launch_bounds__(kVgThreads) lins_vg_centroid_kernel(const Key* __restrict__ key, const int* __restrict__ idx,
                                                                      const int* __restrict__ vid, int n, VgSegs sg, const float4* __restrict__ p,
                                                                      float4* __restrict__ out, VgInfo* __restrict__ info) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Key k = key[i];
  if (key_low(k) == kInvalidKey) return;
  const int sgi = key_seg(k);
  const int b0 = sg.n == 1 ? 0 : __ldg(&sg.off[sgi]), b1 = sg.n == 1 ? n : __ldg(&sg.off[sgi + 1]);
  const int base = b0 > 0 ? vid[b0 - 1] : 0;
  if (i + 1 == b1 || key_low(key[i + 1]) == kInvalidKey) info[sgi].count = vid[i] - base;
  if (i > 0 && key[i - 1] == k) return;
  float cx = 0.f, cy = 0.f, cz = 0.f, ci = 0.f;
  int j = i;
  for (; j < n && key[j] == k; ++j) {
    const float4 q = p[idx[j]];
    cx += q.x; cy += q.y; cz += q.z; ci += q.w;
  }
  const float c = (float)(j - i);
  float4* o = sg.n == 1 ? out : sg.out[sgi];
  o[vid[i] - base - 1] = make_float4(cx / c, cy / c, cz / c, ci / c);
}

// transformPointCloud (:624-652) with the constants of updateTransformPointCloudSinCos (:609-622), one block per job
struct TfJob { const float4* in; float4* out; int n, pad; TfConsts c; };
__global__ void __launch_bounds__(256) lins_mapper_transform_kernel(const TfJob* __restrict__ jobs) {
  const TfJob& jb = jobs[blockIdx.x];
  const TfConsts c = jb.c;
  for (int i = threadIdx.x; i < jb.n; i += blockDim.x) jb.out[i] = tf_point(c, jb.in[i]);
}

int ceil_log2(int n) { int b = 0; while ((1 << b) < n) ++b; return b; }

template <typename Key>
int vg_queue(lins_ctx* ctx, VgScratch& w, Key* const k[2], const float4* in, int n, const VgSegs& sg, float4* out, VgInfo* info) {
  const int blocks = (n + kVgThreads - 1) / kVgThreads;
  lins_vg_bounds_kernel<<<std::min(blocks, 8 * ctx->sm_count), kVgThreads, 0, ctx->stream>>>(in, n, sg, info);
  lins_vg_box_kernel<<<(sg.n + 127) / 128, 128, 0, ctx->stream>>>(info, sg.n);
  lins_vg_key_kernel<Key><<<blocks, kVgThreads, 0, ctx->stream>>>(in, n, sg, info, out, k[0], w.idx[0].p);
  CK(cudaGetLastError());
  size_t bytes = w.temp.cap;
  CK(cub::DeviceRadixSort::SortPairs(w.temp.p, bytes, k[0], k[1], w.idx[0].p, w.idx[1].p, n, 0, 32 + ceil_log2(sg.n), ctx->stream));
  lins_vg_head_kernel<Key><<<blocks, kVgThreads, 0, ctx->stream>>>(k[1], n, w.head.p);
  bytes = w.temp.cap;
  CK(cub::DeviceScan::InclusiveSum(w.temp.p, bytes, w.head.p, w.vid.p, n, ctx->stream));
  lins_vg_centroid_kernel<Key><<<blocks, kVgThreads, 0, ctx->stream>>>(k[1], w.idx[1].p, w.vid.p, n, sg, in, out, info);
  CK(cudaGetLastError());
  ctx->launches += 7;
  return LINS_OK;
}

}  // namespace

namespace lins_capi {

int voxel_grid_reserve(lins_ctx* ctx, VgScratch& w, int n, int n_seg) {
  if (n <= 0) return LINS_OK;
  CK(w.idx[0].grow((size_t)n)); CK(w.idx[1].grow((size_t)n)); CK(w.head.grow((size_t)n)); CK(w.vid.grow((size_t)n));
  size_t b_sort = 0, b_scan = 0;
  const int bits = 32 + ceil_log2(n_seg);
  if (n_seg == 1) {
    CK(w.key[0].grow((size_t)n)); CK(w.key[1].grow((size_t)n));
    CK(cub::DeviceRadixSort::SortPairs(nullptr, b_sort, w.key[0].p, w.key[1].p, w.idx[0].p, w.idx[1].p, n, 0, bits, ctx->stream));
  } else {
    CK(w.key64[0].grow((size_t)n)); CK(w.key64[1].grow((size_t)n));
    CK(cub::DeviceRadixSort::SortPairs(nullptr, b_sort, w.key64[0].p, w.key64[1].p, w.idx[0].p, w.idx[1].p, n, 0, bits, ctx->stream));
  }
  CK(cub::DeviceScan::InclusiveSum(nullptr, b_scan, w.head.p, w.vid.p, n, ctx->stream));
  CK(w.temp.grow(std::max(b_sort, b_scan) + 16));
  return LINS_OK;
}

int voxel_grid_queue(lins_ctx* ctx, VgScratch& w, const float4* in, int n_seg, const int* h_off, const int* d_off, const float* leaf,
                     float4* out, float4* const* d_out, VgInfo* h_init, VgInfo* info) {
  // (pinned staging: a pageable H2D could complete before the copy engine reads it; the callers rewrite it only after
  // the cycle's read-back)
  for (int k = 0; k < n_seg; ++k) {
    VgInfo& v = h_init[k];
    std::memset(&v, 0, sizeof(v));
    for (int a = 0; a < 3; ++a) { v.enc[a] = 0xffffffffu; v.enc[3 + a] = 0u; }
    v.inv = lins_feat::voxel_inv(leaf[k]);
  }
  CK(cudaMemcpyAsync(info, h_init, sizeof(VgInfo) * n_seg, cudaMemcpyHostToDevice, ctx->stream));
  const int n = h_off[n_seg];
  if (n <= 0) return LINS_OK;
  const int rc = voxel_grid_reserve(ctx, w, n, n_seg);
  if (rc != LINS_OK) return rc;
  if (n_seg == 1) {
    unsigned* const k[2] = {w.key[0].p, w.key[1].p};
    return vg_queue(ctx, w, k, in, n, VgSegs{nullptr, nullptr, 1}, out, info);
  }
  unsigned long long* const k[2] = {w.key64[0].p, w.key64[1].p};
  return vg_queue(ctx, w, k, in, n, VgSegs{d_off, d_out, n_seg}, nullptr, info);
}

int keyframes_queue(lins_ctx* ctx, const KfSave* saves, int n, Buf<unsigned char>& dev, Buf<unsigned char, kPinned>& host) {
  std::vector<TfJob> jobs;
  for (int i = 0; i < n; ++i) {
    const KfSave& sv = saves[i];
    const TfConsts c = tf_consts(sv.kp);
    const TfConsts id = {1.f, 0.f, 1.f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f};  // (the identity: the bits T(b, pose) is built on)
    float4* body = sv.body;
    for (int a = 0; a < 3; ++a) {
      CK(sv.kf->c[a].grow((size_t)sv.kf->n[a] + 1));
      if (sv.kf->n[a]) jobs.push_back(TfJob{sv.ds[a], sv.kf->c[a].p, sv.kf->n[a], 0, c});
      if (sv.kf->n[a] && body) jobs.push_back(TfJob{sv.ds[a], body, sv.kf->n[a], 0, id});
      if (body) body += sv.kf->n[a];
    }
  }
  if (jobs.empty()) return LINS_OK;
  const size_t bytes = sizeof(TfJob) * jobs.size();
  CK(dev.reserve(bytes)); CK(host.reserve(bytes));
  std::memcpy(host.p, jobs.data(), bytes);
  CK(cudaMemcpyAsync(dev.p, host.p, bytes, cudaMemcpyHostToDevice, ctx->stream));
  lins_mapper_transform_kernel<<<(int)jobs.size(), 256, 0, ctx->stream>>>(reinterpret_cast<const TfJob*>(dev.p));
  CK(cudaGetLastError());
  ctx->launches += 1;
  return LINS_OK;
}

}  // namespace lins_capi

namespace {

// ---- host scalar code, typed as the reference types it ---------------------------------------------------------------
using lins_pg::rot3_rzryrx;
using lins_pg::rot3_xyz;

// transformUpdate (:538-577)
void transform_update(MapperScalars& s, double timeLaserOdometry, double SCAN_PERIOD) {
  float* T = s.transformTobeMapped;
  if (s.imuPointerLast >= 0) {
    float imuRollLast = 0, imuPitchLast = 0;
    while (s.imuPointerFront != s.imuPointerLast) {
      if (timeLaserOdometry + SCAN_PERIOD < s.imuTime[s.imuPointerFront]) break;
      s.imuPointerFront = (s.imuPointerFront + 1) % LINS_MAPPER_IMU_QUEUE;
    }
    const int f = s.imuPointerFront;
    if (timeLaserOdometry + SCAN_PERIOD > s.imuTime[f]) {
      imuRollLast = s.imuRoll[f];
      imuPitchLast = s.imuPitch[f];
    } else {
      const int b = (f + LINS_MAPPER_IMU_QUEUE - 1) % LINS_MAPPER_IMU_QUEUE;
      const float ratioFront = (timeLaserOdometry + SCAN_PERIOD - s.imuTime[b]) / (s.imuTime[f] - s.imuTime[b]);
      const float ratioBack = (s.imuTime[f] - timeLaserOdometry - SCAN_PERIOD) / (s.imuTime[f] - s.imuTime[b]);
      imuRollLast = s.imuRoll[f] * ratioFront + s.imuRoll[b] * ratioBack;
      imuPitchLast = s.imuPitch[f] * ratioFront + s.imuPitch[b] * ratioBack;
    }
    T[0] = 0.998 * T[0] + 0.002 * imuPitchLast;
    T[2] = 0.998 * T[2] + 0.002 * imuRollLast;
  }
  for (int i = 0; i < 6; i++) {
    s.transformBefMapped[i] = s.transformSum[i];
    s.transformAftMapped[i] = T[i];
  }
}

}  // namespace

namespace lins_capi {

MapperKeyFrame& store_keyframe(MapperNode& M, int id, const int n[3]) {
  auto it = M.slot_of.find(id);
  int s;
  if (it != M.slot_of.end()) s = it->second;
  else if (!M.free_slots.empty()) { s = M.free_slots.back(); M.free_slots.pop_back(); }
  else { s = (int)M.slots.size(); M.slots.emplace_back(); }
  M.slot_of[id] = s;
  MapperKeyFrame& f = M.slots[s];
  std::copy(n, n + 3, f.n);
  return f;
}

// the non-empty copies of a batch through the gather list, at entries base.. (two batches of one cycle do not overlap)
int queue_copies(lins_ctx* ctx, CopyList& l, std::vector<DevCopy> v, int base) {
  v.erase(std::remove_if(v.begin(), v.end(), [](const DevCopy& c) { return c.n <= 0; }), v.end());
  const int rc = l.stage(ctx, v.data(), (int)v.size(), base);
  return rc != LINS_OK ? rc : l.launch(ctx, base, (int)v.size());
}

void mapper_node_reset(MapperNode& m, lins_arena::Arena& store) {
  m.s = MapperScalars();
  m.stepped = false;
  m.loops = MapperLoops();
  m.gm = MapperGlobalMap();  // (frees the last global map's cloud)
  m.poses.clear();
  for (auto& kv : m.slot_of) m.free_slots.push_back(kv.second);
  m.slot_of.clear();
  store.give_back(m.held);
  m.host.clear();
  m.last = MapperLast();
}

void mapper_node_imu(MapperScalars& s, const double* time, const double* roll, const double* pitch, int n) {
  for (int i = 0; i < n; ++i) {  // imuHandler :731-734
    s.imuPointerLast = (s.imuPointerLast + 1) % LINS_MAPPER_IMU_QUEUE;
    s.imuTime[s.imuPointerLast] = time[i];
    s.imuRoll[s.imuPointerLast] = (float)roll[i];
    s.imuPitch[s.imuPointerLast] = (float)pitch[i];
  }
}

bool mapper_cycle_begin(const MapperNode& m, MapperScalars& s, double timeLaserOdometry, const double quat[4], const double pos[3], lins_mapper_report& r) {
  std::memset(&r, 0, sizeof(r));
  r.loop_candidate = -1;
  {  // laserOdometryHandler :713-722
    lins_tf::odometry_transform(quat, pos, s.transformSum);
  }
  if (!(timeLaserOdometry - s.timeLastProcessing >= 0.3)) {  // :1821 (the odometry still replaces transformSum)
    r.skipped_interval = 1;
    r.n_keyframes = (int)m.poses.size();
    r.window_len = (int)s.window.size();
    for (int i = 0; i < 6; ++i) { r.transform_guess[i] = s.transformTobeMapped[i]; r.transform_aft_mapped[i] = s.transformAftMapped[i]; }
    return false;
  }
  s.timeLastProcessing = timeLaserOdometry;
  lins_tf::transform_associate_to_map(s.transformSum, s.transformBefMapped, s.transformAftMapped, s.transformIncre, s.transformTobeMapped);
  for (int i = 0; i < 6; ++i) r.transform_guess[i] = s.transformTobeMapped[i];
  // extractSurroundingKeyFrames :1201-1246 (the deque of ids)
  const int numPoses = (int)m.poses.size();
  if (numPoses > 0) {
    if ((int)s.window.size() < LINS_MAPPER_WINDOW) {
      s.window.clear();
      for (int i = numPoses - 1; i >= 0; --i) {
        s.window.push_front(i);
        if ((int)s.window.size() >= LINS_MAPPER_WINDOW) break;
      }
    } else if (s.latestFrameID != numPoses - 1) {
      s.window.pop_front();
      s.latestFrameID = numPoses - 1;
      s.window.push_back(s.latestFrameID);
    }
  }
  return true;
}

void mapper_node_fuse(const MapperNode& m, double time, const double quat[4], const double pos[3], lins_fused_pose& out) {
  // every processed cycle ends with a key pose (the first one always saves), so a node without key poses has not
  // published; the pair it holds then is the fusion node's initial zeros, not yet round-tripped through publishTF
  std::memset(&out, 0, sizeof(out));
  out.time = time;
  lins_tf::transform_fusion(quat, pos, !m.poses.empty(), m.s.transformAftMapped, m.s.transformBefMapped, out.transform_mapped, out.pos, out.quat);
  out.valid = 1;
}

void mapper_window_sizes(const MapperNode& m, const MapperScalars& s, int& n_corner, int& n_surf) {
  n_corner = n_surf = 0;
  for (int id : s.window) {
    const MapperKeyFrame& kf = m.slots[m.slot_of.at(id)];
    n_corner += kf.n[0]; n_surf += kf.n[1] + kf.n[2];
  }
}

void mapper_cycle_end(MapperNode& M, MapperScalars& s, double timeLaserOdometry, double scan_period, const int cnt[6], const lins_map::MapLoopState* st,
                      lins_mapper_report& r, KfSave* save, bool* saved) {
  // (without key poses the reference returns before the filters and keeps the previous sizes, which are 0 then)
  const int nmc = cnt[0], nms = cnt[1], ndc = cnt[2], nds = cnt[3], ndo = cnt[4], ndt = cnt[5];
  if (st) {
    map_loop_report(*st, s.transformTobeMapped, &r.map);
    transform_update(s, timeLaserOdometry, scan_period);
  } else {
    r.map.skipped = 1;
  }
  *saved = false;
  // saveKeyFramesAndFactor :1654-1765
  const float cur[3] = {s.transformAftMapped[3], s.transformAftMapped[4], s.transformAftMapped[5]};  // currentRobotPosPoint
  bool save_kf = true;
  {
    const float dx = s.previousRobotPos[0] - cur[0], dy = s.previousRobotPos[1] - cur[1], dz = s.previousRobotPos[2] - cur[2];
    if (std::sqrt(dx * dx + dy * dy + dz * dz) < 0.3) save_kf = false;
  }
  if (save_kf || M.poses.empty()) {
    for (int k = 0; k < 3; ++k) s.previousRobotPos[k] = cur[k];
    // the pose inserted into iSAM2, and its estimate: without a loop factor the pose itself (DESIGN.md §4.9), else the
    // solve of the slot's graph (§4.14)
    const float* P = M.poses.empty() ? s.transformTobeMapped : s.transformAftMapped;
    double R[3][3], xyz[3];
    rot3_rzryrx(P[2], P[0], P[1], R);
    double t[3] = {P[5], P[3], P[4]};  // Point3(x = T[5], y = T[3], z = T[4])
    if (M.loops.enabled) mapper_loops_save(M, s, R, t);
    if (M.poses.empty()) for (int i = 0; i < 6; ++i) s.transformLast[i] = s.transformTobeMapped[i];
    rot3_xyz(R, xyz);  // roll() = xyz[0], pitch() = xyz[1], yaw() = xyz[2]
    MapperKeyPose kp;
    kp.x = (float)t[1]; kp.y = (float)t[2]; kp.z = (float)t[0];
    kp.roll = (float)xyz[1]; kp.pitch = (float)xyz[2]; kp.yaw = (float)xyz[0];
    kp.time = timeLaserOdometry;
    const int id = (int)M.poses.size();
    M.poses.push_back(kp);
    if (M.poses.size() > 1) {
      s.transformAftMapped[0] = (float)xyz[1]; s.transformAftMapped[1] = (float)xyz[2]; s.transformAftMapped[2] = (float)xyz[0];
      s.transformAftMapped[3] = (float)t[1]; s.transformAftMapped[4] = (float)t[2]; s.transformAftMapped[5] = (float)t[0];
      for (int i = 0; i < 6; ++i) { s.transformLast[i] = s.transformAftMapped[i]; s.transformTobeMapped[i] = s.transformAftMapped[i]; }
    }
    // the key frame's clouds, in the map frame once (its pose changes only in correctPoses)
    const int n[3] = {ndc, nds, ndo};
    save->kf = &store_keyframe(M, id, n);
    save->kp = kp;
    *saved = true;
    r.keyframe_saved = 1;
    r.loop_candidate = loop_candidate(M, cur, timeLaserOdometry);
    // the device store keeps the window and the newest key frame: nothing else can enter a later window (a slot with
    // loop closure keeps every key frame in its host store, for the history sub-maps and the global map)
    for (auto it = M.slot_of.begin(); it != M.slot_of.end();) {
      const int kid = it->first;
      if (kid != id && std::find(s.window.begin(), s.window.end(), kid) == s.window.end()) { M.free_slots.push_back(it->second); it = M.slot_of.erase(it); }
      else ++it;
    }
  }
  M.s = s;
  M.last.valid = true;
  for (int k = 0; k < 6; ++k) M.last.n[k] = cnt[k];
  r.processed = 1;
  r.n_map_corner_ds = nmc; r.n_map_surf_ds = nms;
  r.n_corner_ds = ndc; r.n_surf_ds = nds; r.n_outlier_ds = ndo; r.n_surf_total_ds = ndt;
  r.n_keyframes = (int)M.poses.size();
  r.window_len = (int)s.window.size();
  for (int i = 0; i < 6; ++i) r.transform_aft_mapped[i] = s.transformAftMapped[i];
  M.loops.rebuild = false;
  if (M.loops.enabled) {
    std::memcpy(M.loops.cur, cur, sizeof(cur));
    if (M.loops.closed) mapper_correct_poses(M);  // correctPoses :1767-1795 (after the report: window_len is this cycle's)
  }
}

// detectLoopClosure's candidate (:1050-1064): radius 5 m around currentRobotPosPoint, nearest first, |dt| > 30 s
int loop_candidate(const MapperNode& M, const float cur[3], double time) {
  int id = -1;
  float best = 0.f;
  for (int i = 0; i < (int)M.poses.size(); ++i) {
    const MapperKeyPose& q = M.poses[i];
    const float ex = q.x - cur[0], ey = q.y - cur[1], ez = q.z - cur[2];
    const float d2 = ex * ex + ey * ey + ez * ez;
    if (!(d2 < 25.0f) || !(std::fabs(q.time - time) > 30.0)) continue;
    if (id < 0 || d2 < best) { id = i; best = d2; }
  }
  return id;
}

int mapper_node_download(lins_ctx* ctx, const MapperNode& M, const float4* const src[6], double* key_poses, int32_t* window, float* const dst[6]) {
  if (key_poses)
    for (size_t i = 0; i < M.poses.size(); ++i) {
      const MapperKeyPose& k = M.poses[i];
      const double v[7] = {k.x, k.y, k.z, k.roll, k.pitch, k.yaw, k.time};
      std::memcpy(key_poses + 7 * i, v, sizeof(v));
    }
  if (window) { int i = 0; for (int id : M.s.window) window[i++] = id; }
  for (int k = 0; k < 6 && M.last.valid; ++k) CK(d2h(ctx, dst[k], src[k], sizeof(float4) * M.last.n[k]));
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}

}  // namespace lins_capi

extern "C" {

int lins_gpu_voxel_grid(lins_ctx* ctx, const lins_point* in, int n, float leaf, float* out, int* n_out) {
  if (!ctx) return LINS_E_INVALID;
  if (check_cloud(ctx, in, n, "bad VoxelGrid input cloud") != LINS_OK || check_cloud(ctx, out, n, "bad VoxelGrid output cloud") != LINS_OK)
    return LINS_E_INVALID;
  if (!n_out || !(leaf > 0.f) || !std::isfinite(leaf)) return fail(ctx, LINS_E_INVALID, "bad VoxelGrid n_out / leaf");
  CK(cudaSetDevice(ctx->device));
  VoxelGridState& v = ctx->vg;
  CK(v.in.reserve((size_t)n + 1)); CK(v.out.reserve((size_t)n + 1)); CK(v.h_in.reserve((size_t)n + 1));
  CK(v.info.reserve(1)); CK(v.h_info.reserve(1));
  pack_into(v.h_in.p, in, n);
  if (n) CK(cudaMemcpyAsync(v.in.p, v.h_in.p, sizeof(float4) * n, cudaMemcpyHostToDevice, ctx->stream));
  const int off[2] = {0, n};
  const int rc = voxel_grid_queue(ctx, v.w, v.in.p, 1, off, nullptr, &leaf, v.out.p, nullptr, v.h_info.p, v.info.p);
  if (rc != LINS_OK) return rc;
  CK(cudaMemcpyAsync(v.h_info.p, v.info.p, sizeof(VgInfo), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (v.h_info.p->toobig) return fail(ctx, LINS_E_TOOBIG, "VoxelGrid: the leaf is too small for the cloud's extent (div_x * div_y * div_z > INT32_MAX)");
  const int c = n > 0 ? v.h_info.p->count : 0;
  CK(d2h(ctx, out, v.out.p, sizeof(float4) * c));
  CK(cudaStreamSynchronize(ctx->stream));
  *n_out = c;
  return LINS_OK;
}

}  // extern "C"
