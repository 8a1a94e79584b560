// lins_loops.cu — the mapping node's loop closure (lidar_mapping_node.cpp loopClosureThread :1033-1041,
// detectLoopClosure :1043-1112, performLoopClosure :1114-1186, correctPoses :1767-1795) for the enabled slots of a
// lockstep run (the single mapper is a run of one slot).
//
// Host, per slot (DESIGN.md §4.14): the key-pose graph (csrc/host/pose_graph.hpp) a key-frame save extends and, once it
// holds a loop factor, solves; correctPoses; the candidate (lins_mapper.cu's loop_candidate) and the loop factor from
// ICP's result (pcl's getTranslationAndEulerAngles / getTransformation in f32, gtsam's Pose3 in f64).
//
// Device, one pass over every slot with a candidate (one synchronisation): one gather of the sources (the latest key
// frame's corner + surf cloud in the map frame, from the device store) and the history clouds (key frames closest +- 25,
// corner + surf, read from the host store over the host link and transformed by their key poses on the way), one
// segmented VoxelGrid (0.4 m, a segment per slot), then up to 100 queued ICP iterations, each one exhaustive 1-NN
// launch over every active slot's source points and one launch of a CTA per slot that reduces the correspondences in a
// fixed order, solves the rigid transform (Horn's quaternion form of the Umeyama / SVD optimum), applies PCL's
// DefaultConvergenceCriteria and sets the slot's done flag; then the fitness pass and one read-back.  A 1-NN block
// covers source points of one slot only and every sum runs in a fixed order, so each slot's result is that of a run
// of one slot.
//
// The global map (publishGlobalMap :976-1031, DESIGN.md §4.15) of the same enabled slots reuses the gather and
// segmented VoxelGrid of the history sub-maps (gather_voxel_grid) on the key frames csrc/host/global_map.hpp selects.
// A key frame's map-frame cloud is T(b, key pose) of its host-store body cloud b: the bits the device store holds for
// the key frames it keeps (every save and correctPoses writes them so, and a load rebuilds them so).
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../host/global_map.hpp"
#include "lins_ctx.hpp"
#include "lins_mapper_tf.cuh"

using namespace lins_capi;

namespace {

constexpr int kNnThreads = 128;
constexpr int kNnTile = 1024;      // target points per shared-memory tile (16 KB)
constexpr int kRedThreads = 256;
constexpr int kRedSums = 18;       // count, sum s (3), sum t (3), sum s t^T (9), sum of distances, source points
constexpr int kIcpIters = 100;     // setMaximumIterations (:1129)
constexpr float kMaxCorrSq = 100.f * 100.f;  // setMaxCorrespondenceDistance (:1128), compared squared
constexpr int kHistory = 25;       // historyKeyframeSearchNum (parameters.h:99)
constexpr float kFitness = 0.3f;   // historyKeyframeFitnessScore (parameters.h:100)

// (int)intensity >= 0 (:1080): x86's truncation gives INT_MIN for NaN and for values outside the int range
__device__ __forceinline__ bool keep_point(float w) { return w > -1.f && w < 2147483648.f; }

// pt' = T pt of PCL's transformCloud on a 3 x 4 f32 matrix, rows summed left to right (no contraction)
__device__ __forceinline__ float4 xf(const float* T, float4 p) {
  float4 o;
  o.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], p.x), __fmul_rn(T[1], p.y)), __fmul_rn(T[2], p.z)), T[3]);
  o.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], p.x), __fmul_rn(T[5], p.y)), __fmul_rn(T[6], p.z)), T[7]);
  o.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], p.x), __fmul_rn(T[9], p.y)), __fmul_rn(T[10], p.z)), T[11]);
  o.w = p.w;
  return o;
}

// the exact 1-NN of every source point of the block's slot over the slot's whole target (FLANN's L2 on x, y, z:
// ((dx^2 + dy^2) + dz^2) in f32; ties to the lower target index).  fit = 0: an ICP iteration on the running source,
// first moved by the slot's last increment; fit = 1: getFitnessScore's pass on the source under the final transform.
__global__ void __launch_bounds__(kNnThreads) lins_loop_nn_kernel(const LoopSlot* __restrict__ slots, const int2* __restrict__ blk,
                                                                  const LoopIcpState* __restrict__ st, int fit) {
  __shared__ float4 tile[kNnTile];
  const int2 b = blk[blockIdx.x];
  const LoopSlot sl = slots[b.x];
  const LoopIcpState& S = st[b.x];
  if (!fit && S.done) return;
  const int i = b.y + threadIdx.x;
  const bool valid = i < sl.n_src;
  float4 p = make_float4(0.f, 0.f, 0.f, -2.f);
  if (valid) {
    if (fit) {
      p = xf(S.fin, sl.src0[i]);
    } else {
      p = sl.src[i];
      if (S.iters > 0) { p = xf(S.inc, p); sl.src[i] = p; }
    }
  }
  const bool keep = valid && keep_point(p.w);
  const int n_t = *sl.n_tgt;
  float best = FLT_MAX;
  int bi = -1;
  for (int t0 = 0; t0 < n_t; t0 += kNnTile) {
    const int nt = min(kNnTile, n_t - t0);
    __syncthreads();
    for (int j = threadIdx.x; j < nt; j += kNnThreads) tile[j] = sl.tgt[t0 + j];
    __syncthreads();
    if (!keep) continue;
    for (int j = 0; j < nt; ++j) {
      const float4 q = tile[j];
      const float dx = __fsub_rn(q.x, p.x), dy = __fsub_rn(q.y, p.y), dz = __fsub_rn(q.z, p.z);
      const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
      if (d < best) { best = d; bi = t0 + j; }
    }
  }
  if (valid) { sl.corr[i] = keep ? bi : -2; sl.dist[i] = best; }
}

// the symmetric 4 x 4 eigenvector of the largest eigenvalue (cyclic Jacobi, f64)
__device__ void max_eigvec4(double A[4][4], double q[4]) {
  double V[4][4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) V[i][j] = i == j;
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0, diag = 0;
    for (int i = 0; i < 4; ++i) {
      diag += A[i][i] * A[i][i];
      for (int j = i + 1; j < 4; ++j) off += A[i][j] * A[i][j];
    }
    if (!(off > 1e-32 * diag)) break;
    for (int p = 0; p < 3; ++p)
      for (int r = p + 1; r < 4; ++r) {
        if (A[p][r] == 0.0) continue;
        const double th = (A[r][r] - A[p][p]) / (2.0 * A[p][r]);
        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 4; ++k) {  // A <- A J
          const double akp = A[k][p], akr = A[k][r];
          A[k][p] = c * akp - s * akr; A[k][r] = s * akp + c * akr;
        }
        for (int k = 0; k < 4; ++k) {  // A <- J^T A
          const double apk = A[p][k], ark = A[r][k];
          A[p][k] = c * apk - s * ark; A[r][k] = s * apk + c * ark;
        }
        for (int k = 0; k < 4; ++k) {
          const double vkp = V[k][p], vkr = V[k][r];
          V[k][p] = c * vkp - s * vkr; V[k][r] = s * vkp + c * vkr;
        }
      }
  }
  int m = 0;
  for (int i = 1; i < 4; ++i) if (A[i][i] > A[m][m]) m = i;
  for (int i = 0; i < 4; ++i) q[i] = V[i][m];
}

// one CTA per slot: the fixed-order sums of the slot's correspondences (fit = 0) or 1-NN distances (fit = 1), then on
// thread 0 the iteration's transform, final = T final and the convergence test, or the fitness score
__global__ void __launch_bounds__(kRedThreads) lins_loop_icp_kernel(const LoopSlot* __restrict__ slots, LoopIcpState* __restrict__ st, int fit) {
  __shared__ double red[kRedSums][kRedThreads];
  const LoopSlot sl = slots[blockIdx.x];
  LoopIcpState& S = st[blockIdx.x];
  if (!fit && S.done) return;
  double a[kRedSums];
  for (int k = 0; k < kRedSums; ++k) a[k] = 0.0;
  for (int i = threadIdx.x; i < sl.n_src; i += kRedThreads) {
    const int c = sl.corr[i];
    if (c == -2) continue;  // dropped by the intensity filter
    a[17] += 1.0;
    const float d = sl.dist[i];
    if (fit) {
      if (c >= 0) { a[0] += 1.0; a[16] += (double)d; }
      continue;
    }
    if (c < 0 || d > kMaxCorrSq) continue;
    const float4 p = sl.src[i], q = sl.tgt[c];
    const double s3[3] = {p.x, p.y, p.z}, t3[3] = {q.x, q.y, q.z};
    a[0] += 1.0;
    for (int k = 0; k < 3; ++k) { a[1 + k] += s3[k]; a[4 + k] += t3[k]; }
    for (int r = 0; r < 3; ++r)
      for (int k = 0; k < 3; ++k) a[7 + 3 * r + k] += s3[r] * t3[k];
    a[16] += (double)d;
  }
  for (int k = 0; k < kRedSums; ++k) red[k][threadIdx.x] = a[k];
  __syncthreads();
  for (int w = kRedThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int k = 0; k < kRedSums; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  double v[kRedSums];
  for (int k = 0; k < kRedSums; ++k) v[k] = red[k][0];
  const double n = v[0];
  S.n_src = (int)v[17];
  if (fit) {  // getFitnessScore (max range DBL_MAX)
    S.n_fit = (int)n;
    S.fitness = n > 0 ? v[16] / n : DBL_MAX;
    return;
  }
  if (S.iters == 0) S.n_corr0 = (int)n;
  if (n < 3) { S.converged = 0; S.done = 1; return; }  // "Not enough correspondences found"
  // Umeyama without scale: the rotation maximising trace(R^T H), H = sum (s - ms)(t - mt)^T, by Horn's quaternion
  const double ms[3] = {v[1] / n, v[2] / n, v[3] / n}, mt[3] = {v[4] / n, v[5] / n, v[6] / n};
  double H[3][3];
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) H[r][k] = v[7 + 3 * r + k] - n * ms[r] * mt[k];
  const double Sxx = H[0][0], Sxy = H[0][1], Sxz = H[0][2], Syx = H[1][0], Syy = H[1][1], Syz = H[1][2], Szx = H[2][0], Szy = H[2][1], Szz = H[2][2];
  double N[4][4] = {{Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx},
                    {Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz},
                    {Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy},
                    {Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz}};
  double q[4];
  max_eigvec4(N, q);
  const double w = q[0], x = q[1], y = q[2], z = q[3], qn = w * w + x * x + y * y + z * z;
  const double R[3][3] = {{(w * w + x * x - y * y - z * z) / qn, 2 * (x * y - w * z) / qn, 2 * (x * z + w * y) / qn},
                          {2 * (x * y + w * z) / qn, (w * w - x * x + y * y - z * z) / qn, 2 * (y * z - w * x) / qn},
                          {2 * (x * z - w * y) / qn, 2 * (y * z + w * x) / qn, (w * w - x * x - y * y + z * z) / qn}};
  float T[12];
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) T[4 * r + k] = (float)R[r][k];
    T[4 * r + 3] = (float)(mt[r] - (R[r][0] * ms[0] + R[r][1] * ms[1] + R[r][2] * ms[2]));
  }
  float F[12];  // final_transformation_ = transformation_ * final_transformation_ (f32, row 3 = 0 0 0 1)
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 4; ++k) {
      float s = __fadd_rn(__fadd_rn(__fmul_rn(T[4 * r], S.fin[k]), __fmul_rn(T[4 * r + 1], S.fin[4 + k])), __fmul_rn(T[4 * r + 2], S.fin[8 + k]));
      if (k == 3) s = __fadd_rn(s, T[4 * r + 3]);
      F[4 * r + k] = s;
    }
  for (int k = 0; k < 12; ++k) { S.inc[k] = T[k]; S.fin[k] = F[k]; }
  S.iters += 1;
  // DefaultConvergenceCriteria::hasConverged, in its order (rotation threshold 0.99999 as PCL 1.7 leaves it; 1.8 and
  // later set 1 - transformation epsilon: DESIGN.md §4.14).  The step above is f64 where PCL's is f32 (a precision choice)
  bool conv = false;
  if (S.iters >= kIcpIters) {
    conv = true;
  } else {
    const double cos_angle = 0.5 * (double)(__fsub_rn(__fadd_rn(__fadd_rn(T[0], T[5]), T[10]), 1.f));
    const float tsq = __fadd_rn(__fadd_rn(__fmul_rn(T[3], T[3]), __fmul_rn(T[7], T[7])), __fmul_rn(T[11], T[11]));
    if (cos_angle >= 0.99999 && (double)tsq <= 1e-6) {
      conv = true;
    } else {
      const double mse = v[16] / n;
      if (fabs(mse - S.prev_mse) < 1e-12 || fabs(mse - S.prev_mse) / S.prev_mse < 1e-6) conv = true;
      else S.prev_mse = mse;
    }
  }
  if (conv) { S.converged = 1; S.done = 1; }
}

// one copy of the gather in front of a segmented VoxelGrid: n records from src (device memory, or the host store's
// mapped memory) to dst, through tf_point(c) when tf != 0 (a host-store body cloud into the map frame)
struct GatherJob { const float4* src; float4* dst; int n, tf; TfConsts c; };

// one block per job; each source record is read once
__global__ void __launch_bounds__(256) lins_loop_gather_kernel(const GatherJob* __restrict__ jobs) {
  const GatherJob& jb = jobs[blockIdx.x];
  const TfConsts c = jb.c;
  if (jb.tf)
    for (int i = threadIdx.x; i < jb.n; i += blockDim.x) jb.dst[i] = tf_point(c, jb.src[i]);
  else
    for (int i = threadIdx.x; i < jb.n; i += blockDim.x) jb.dst[i] = jb.src[i];
}

// the gather jobs of a host-store key frame's clouds a (0 corner, 1 surf, 2 outlier) for a < n_clouds, each transformed
// by the key pose, appended to v (dst is set by gather_voxel_grid)
void host_kf_jobs(const MapperNode& m, int id, int n_clouds, std::vector<GatherJob>& v) {
  const HostKeyFrame& h = m.host[id];
  const TfConsts c = tf_consts(m.poses[id]);
  const float4* p = h.p;
  for (int a = 0; a < n_clouds; ++a) { v.push_back(GatherJob{p, nullptr, h.n[a], 1, c}); p += h.n[a]; }
}

// pcl::getTransformation(x, y, z, roll, pitch, yaw) as a 3 x 4 f32 matrix
void pcl_transformation(float x, float y, float z, float roll, float pitch, float yaw, float t[12]) {
  const float A = std::cos(yaw), B = std::sin(yaw), C = std::cos(pitch), D = std::sin(pitch), E = std::cos(roll), F = std::sin(roll);
  const float DE = D * E, DF = D * F;
  const float m[12] = {A * C, A * DF - B * E, B * F + A * DE, x, B * C, A * E + B * DF, B * DE - A * F, y, -D, C * F, C * E, z};
  std::memcpy(t, m, sizeof(m));
}
// pcl::getTranslationAndEulerAngles of a 3 x 4 f32 matrix: x, y, z, roll, pitch, yaw
void pcl_euler(const float t[12], float o[6]) {
  o[0] = t[3]; o[1] = t[7]; o[2] = t[11];
  o[3] = std::atan2(t[9], t[10]);
  o[4] = std::asin(-t[8]);
  o[5] = std::atan2(t[4], t[0]);
}
// Affine3f a * b on 3 x 4 matrices
void affine_mul(const float a[12], const float b[12], float c[12]) {
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 4; ++k) {
      float s = a[4 * r] * b[k] + a[4 * r + 1] * b[4 + k] + a[4 * r + 2] * b[8 + k];
      if (k == 3) s += a[4 * r + 3];
      c[4 * r + k] = s;
    }
}
lins_pg::Pose3 pose3(double roll, double pitch, double yaw, double x, double y, double z) {  // Pose3(Rot3::RzRyRx(r, p, y), Point3)
  lins_pg::Pose3 p;
  lins_pg::rot3_rzryrx(roll, pitch, yaw, p.R);
  p.t[0] = x; p.t[1] = y; p.t[2] = z;
  return p;
}
// a key pose's fields from an estimate (saveKeyFramesAndFactor :1721-1733, correctPoses :1775-1790)
void key_pose_from(const lins_pg::Pose3& e, MapperKeyPose& k) {
  double xyz[3];
  lins_pg::rot3_xyz(e.R, xyz);
  k.x = (float)e.t[1]; k.y = (float)e.t[2]; k.z = (float)e.t[0];
  k.roll = (float)xyz[1]; k.pitch = (float)xyz[2]; k.yaw = (float)xyz[0];
}

const lins_pg::Vec6 kOdomVar = {1e-6, 1e-6, 1e-6, 1e-8, 1e-8, 1e-6};  // priorNoise / odometryNoise (:382-385)

// every buffer gather_voxel_grid uses for n points in n_seg segments and n_jobs gather jobs (grow-only)
int gather_voxel_grid_reserve(lins_ctx* ctx, MappersState& ms, int n, int n_seg, size_t n_jobs) {
  LoopPass& lp = ms.lp;
  int rc;
  if ((rc = voxel_grid_reserve(ctx, ms.vg, n, n_seg)) != LINS_OK) return rc;
  CK(lp.tin.grow((size_t)n + 1)); CK(lp.tgt.grow((size_t)n + 1));
  CK(lp.info.reserve(n_seg)); CK(lp.h_info.reserve(n_seg)); CK(lp.h_init.reserve(n_seg));
  CK(lp.off.reserve(n_seg + 1)); CK(lp.h_off.reserve(n_seg + 1)); CK(lp.out.reserve(n_seg)); CK(lp.h_out.reserve(n_seg));
  CK(lp.jobs.reserve(sizeof(GatherJob) * (n_jobs + 1))); CK(lp.h_jobs.reserve(sizeof(GatherJob) * (n_jobs + 1)));
  return LINS_OK;
}

// The history sub-maps of close_loops and the global map: segment p of one segmented 0.4 m VoxelGrid is the
// concatenation of the clouds lists[p] (host-store key frames, transformed on the way).  One gather launch (the
// caller's jobs first, with their own destinations) into ms.lp.tin at toff[p] (lists.size() + 1 offsets, filled
// here), then the VoxelGrid into ms.lp.tgt at the same offsets, its records at ms.lp.info for the caller to read back.
// Every buffer is reserved before anything is queued.  The pinned job table is rewritten only after the caller's
// synchronisation of the previous call (each caller reads its results back before it gathers again).
int gather_voxel_grid(lins_ctx* ctx, MappersState& ms, const std::vector<std::vector<GatherJob>>& lists, std::vector<GatherJob> jobs,
                      std::vector<int>& toff) {
  LoopPass& lp = ms.lp;
  const int A = (int)lists.size();
  toff.assign(A + 1, 0);
  for (int p = 0; p < A; ++p) {
    int n = 0;
    for (const GatherJob& c : lists[p]) n += c.n;
    toff[p + 1] = toff[p] + n;
  }
  const int nt = toff[A];
  size_t n_jobs = jobs.size();
  for (const auto& l : lists) n_jobs += l.size();
  int rc;
  if ((rc = gather_voxel_grid_reserve(ctx, ms, nt, A, n_jobs)) != LINS_OK) return rc;
  for (int p = 0; p < A; ++p) {
    float4* o = lp.tin.p + toff[p];
    for (GatherJob c : lists[p]) { c.dst = o; jobs.push_back(c); o += c.n; }
  }
  jobs.erase(std::remove_if(jobs.begin(), jobs.end(), [](const GatherJob& c) { return c.n <= 0; }), jobs.end());
  if (!jobs.empty()) {
    const size_t bytes = sizeof(GatherJob) * jobs.size();
    std::memcpy(lp.h_jobs.p, jobs.data(), bytes);
    CK(cudaMemcpyAsync(lp.jobs.p, lp.h_jobs.p, bytes, cudaMemcpyHostToDevice, ctx->stream));
    lins_loop_gather_kernel<<<(unsigned)jobs.size(), 256, 0, ctx->stream>>>(reinterpret_cast<const GatherJob*>(lp.jobs.p));
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  std::vector<float> leaf(A, 0.4f);
  for (int p = 0; p < A; ++p) { lp.h_off.p[p] = toff[p]; lp.h_out.p[p] = lp.tgt.p + toff[p]; }
  lp.h_off.p[A] = nt;
  CK(cudaMemcpyAsync(lp.off.p, lp.h_off.p, sizeof(int) * (A + 1), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(lp.out.p, lp.h_out.p, sizeof(float4*) * A, cudaMemcpyHostToDevice, ctx->stream));
  return voxel_grid_queue(ctx, ms.vg, lp.tin.p, A, toff.data(), lp.off.p, leaf.data(), lp.tgt.p, lp.out.p, lp.h_init.p, lp.info.p);
}

}  // namespace

namespace lins_capi {

// saveKeyFramesAndFactor's graph (:1673-1719) on an enabled node before key pose n = m.poses.size() is stored: the
// prior (n = 0) or the chain factor from transformLast, the inserted pose (R, t), and latestEstimate back in (R, t): the inserted pose itself without a loop factor, else the solve of the whole graph
void mapper_loops_save(MapperNode& m, const MapperScalars& s, double R[3][3], double t[3]) {
  MapperLoops& L = m.loops;
  lins_pg::Pose3 ins;
  std::memcpy(ins.R, R, sizeof(ins.R));
  std::memcpy(ins.t, t, sizeof(ins.t));
  const int n = (int)m.poses.size();
  if (n == 0) {
    L.graph.assign(1, lins_pg::Factor{0, -1, ins, kOdomVar});
    L.est.clear();
  } else {
    const float* T = s.transformLast;
    const lins_pg::Pose3 from = pose3(T[2], T[0], T[1], T[5], T[3], T[4]);
    L.graph.push_back(lins_pg::Factor{n - 1, n, lins_pg::between(from, ins), kOdomVar});
  }
  L.est.push_back(ins);
  if (L.n_loop == 0) return;
  lins_pg::solve(L.graph, L.est);
  std::memcpy(R, L.est.back().R, sizeof(ins.R));
  std::memcpy(t, L.est.back().t, sizeof(ins.t));
}

// correctPoses (:1767-1795): every key pose from the estimate of the last save, and the window cleared, so that the next
// processed cycle takes extractSurroundingKeyFrames' rebuild branch (rebuild: the step re-transforms the stored clouds)
void mapper_correct_poses(MapperNode& m) {
  for (size_t i = 0; i < m.loops.est.size() && i < m.poses.size(); ++i) key_pose_from(m.loops.est[i], m.poses[i]);
  m.s.window.clear();
  m.loops.closed = false;
  m.loops.rebuild = true;
}

int mappers_close_loops(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, lins_loop_report* reps) {
  const int M = ms.n;
  for (int s = 0; s < M; ++s)
    if (mask[s] && !ms.node[s].loops.enabled) return fail(ctx, LINS_E_INVALID, "lins_gpu_mappers_close_loops: a masked slot does not have loop closure enabled");
  CK(cudaSetDevice(ctx->device));
  std::vector<lins_loop_report> rr(M);
  std::vector<int> act;  // slots with a candidate
  for (int s = 0; s < M; ++s) {
    if (!mask[s]) continue;
    lins_loop_report& r = rr[s];
    std::memset(&r, 0, sizeof(r));
    r.closest_history_frame_id = r.latest_frame_id = -1;
    const MapperNode& m = ms.node[s];
    if (m.poses.empty()) continue;  // :1115
    const int c = loop_candidate(m, m.loops.cur, m.loops.time);
    if (c < 0) continue;
    r.closest_history_frame_id = c;
    r.latest_frame_id = (int)m.poses.size() - 1;
    act.push_back(s);
  }
  const int A = (int)act.size();
  auto finish = [&]() {
    if (reps) for (int s = 0; s < M; ++s) if (mask[s]) reps[s] = rr[s];
    return LINS_OK;
  };
  if (A == 0) return finish();

  // the sources (latest corner, surf) and history clouds (closest +- 25: corner, surf per key frame)
  LoopPass& lp = ms.lp;
  std::vector<int> soff(A + 1, 0);
  std::vector<std::vector<GatherJob>> hist(A);
  auto kf = [&](const MapperNode& m, int id) -> const MapperKeyFrame& { return m.slots[m.slot_of.at(id)]; };
  for (int p = 0; p < A; ++p) {
    const MapperNode& m = ms.node[act[p]];
    const int latest = rr[act[p]].latest_frame_id, closest = rr[act[p]].closest_history_frame_id;
    soff[p + 1] = soff[p] + kf(m, latest).n[0] + kf(m, latest).n[1];
    for (int j = std::max(0, closest - kHistory); j <= std::min(latest, closest + kHistory); ++j) host_kf_jobs(m, j, 2, hist[p]);
  }
  const int ns = soff[A];
  std::vector<int2> blocks;
  for (int p = 0; p < A; ++p)
    for (int i = 0; i < soff[p + 1] - soff[p]; i += kNnThreads) blocks.push_back(make_int2(p, i));
  const int nb = (int)blocks.size();
  // every buffer first (a growth frees memory queued work may still read; gather_voxel_grid reserves its own before it
  // queues anything)
  int rc;
  CK(lp.src0.grow((size_t)ns + 1)); CK(lp.src.grow((size_t)ns + 1));
  CK(lp.corr.grow((size_t)ns + 1)); CK(lp.dist.grow((size_t)ns + 1));
  CK(lp.slot.reserve(A)); CK(lp.h_slot.reserve(A)); CK(lp.st.reserve(A)); CK(lp.h_st.reserve(A));
  CK(lp.blk.reserve(std::max(nb, 1))); CK(lp.h_blk.reserve(std::max(nb, 1)));
  std::vector<GatherJob> copies;  // the sources, from the device store (the newest key frame stays there)
  for (int p = 0; p < A; ++p) {
    const MapperNode& m = ms.node[act[p]];
    const int latest = rr[act[p]].latest_frame_id;
    float4* o = lp.src0.p + soff[p];
    for (int a = 0; a < 2; ++a) { copies.push_back(GatherJob{kf(m, latest).c[a].p, o, kf(m, latest).n[a], 0, TfConsts{}}); o += kf(m, latest).n[a]; }
  }
  // nearHistorySurfKeyFrameCloudDS: one segmented VoxelGrid, a segment per slot, gathered with the sources
  std::vector<int> toff;
  if ((rc = gather_voxel_grid(ctx, ms, hist, std::move(copies), toff)) != LINS_OK) return rc;
  if (ns) CK(cudaMemcpyAsync(lp.src.p, lp.src0.p, sizeof(float4) * ns, cudaMemcpyDeviceToDevice, ctx->stream));
  // the ICP: the slot table, the block table and the initial states (identity, prev MSE DBL_MAX)
  for (int p = 0; p < A; ++p) {
    lp.h_slot.p[p] = LoopSlot{lp.src0.p + soff[p], lp.src.p + soff[p], lp.tgt.p + toff[p], &lp.info.p[p].count, lp.corr.p + soff[p], lp.dist.p + soff[p],
                              soff[p + 1] - soff[p], 0};
    LoopIcpState& S = lp.h_st.p[p];
    std::memset(&S, 0, sizeof(S));
    S.fin[0] = S.fin[5] = S.fin[10] = 1.f;
    S.prev_mse = DBL_MAX;
  }
  std::copy(blocks.begin(), blocks.end(), lp.h_blk.p);
  CK(cudaMemcpyAsync(lp.slot.p, lp.h_slot.p, sizeof(LoopSlot) * A, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(lp.st.p, lp.h_st.p, sizeof(LoopIcpState) * A, cudaMemcpyHostToDevice, ctx->stream));
  if (nb) CK(cudaMemcpyAsync(lp.blk.p, lp.h_blk.p, sizeof(int2) * nb, cudaMemcpyHostToDevice, ctx->stream));
  for (int it = 0; it <= kIcpIters; ++it) {  // kIcpIters iterations, then the fitness pass
    const int fit = it == kIcpIters;
    if (nb) lins_loop_nn_kernel<<<nb, kNnThreads, 0, ctx->stream>>>(lp.slot.p, lp.blk.p, lp.st.p, fit);
    lins_loop_icp_kernel<<<A, kRedThreads, 0, ctx->stream>>>(lp.slot.p, lp.st.p, fit);
    ctx->launches += nb ? 2 : 1;
  }
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(lp.h_st.p, lp.st.p, sizeof(LoopIcpState) * A, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(lp.h_info.p, lp.info.p, sizeof(VgInfo) * A, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));  // the call's one read-back
  for (int p = 0; p < A; ++p)
    if (lp.h_info.p[p].toobig) return fail(ctx, LINS_E_TOOBIG, "VoxelGrid: the leaf is too small for the history cloud's extent");

  // the reports, and on acceptance the loop factor (:1156-1185)
  for (int p = 0; p < A; ++p) {
    const int s = act[p];
    MapperNode& m = ms.node[s];
    const LoopIcpState& S = lp.h_st.p[p];
    lins_loop_report& r = rr[s];
    r.n_source = S.n_src;
    r.n_history_ds = lp.h_info.p[p].count;
    r.icp_iters = S.iters;
    r.n_corr0 = S.n_corr0;
    r.converged = S.converged;
    r.fitness = S.fitness;
    for (int k = 0; k < 12; ++k) r.final_transform[k] = S.fin[k];
    r.final_transform[15] = 1.f;
    r.accepted = S.converged && !(S.fitness > (double)kFitness);
    if (!r.accepted) continue;
    float cam[6], tw[12], cl[12], tc[12], o[6];
    pcl_euler(S.fin, cam);  // x, y, z, roll, pitch, yaw of correctionCameraFrame
    pcl_transformation(cam[2], cam[0], cam[1], cam[5], cam[3], cam[4], cl);  // correctionLidarFrame
    const MapperKeyPose& kl = m.poses[r.latest_frame_id];
    pcl_transformation(kl.z, kl.x, kl.y, kl.yaw, kl.roll, kl.pitch, tw);  // pclPointToAffine3fCameraToLidar
    affine_mul(cl, tw, tc);
    pcl_euler(tc, o);
    const lins_pg::Pose3 from = pose3(o[3], o[4], o[5], o[0], o[1], o[2]);
    const MapperKeyPose& kc = m.poses[r.closest_history_frame_id];
    const lins_pg::Pose3 to = pose3(kc.yaw, kc.roll, kc.pitch, kc.z, kc.x, kc.y);  // pclPointTogtsamPose3
    const lins_pg::Pose3 z = lins_pg::between(from, to);
    const double noise = (double)(float)S.fitness;
    m.loops.graph.push_back(lins_pg::Factor{r.latest_frame_id, r.closest_history_frame_id, z, {noise, noise, noise, noise, noise, noise}});
    m.loops.n_loop += 1;
    m.loops.closed = true;
    double xyz[3];
    lins_pg::rot3_xyz(z.R, xyz);
    const double f[6] = {z.t[0], z.t[1], z.t[2], xyz[0], xyz[1], xyz[2]};
    std::memcpy(r.factor, f, sizeof(f));
    r.noise = noise;
  }
  return finish();
}

// publishGlobalMap (:976-1031) of the masked slots (DESIGN.md §4.15): the key-frame selection on the host
// (csrc/host/global_map.hpp), then the named key frames' map-frame clouds (T(b, pose) of their host-store clouds, the
// bits the device store holds for its key frames) gathered and down-sampled in passes of up to
// LINS_GLOBAL_MAP_PASS_POINTS points, a segment per slot, one synchronisation per pass.  Each result is copied into a
// buffer of the slot's own; nothing else of the node changes.
int mappers_global_map(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, lins_global_map_report* reps) {
  const int M = ms.n;
  for (int s = 0; s < M; ++s)
    if (mask[s] && !ms.node[s].loops.enabled)
      return fail(ctx, LINS_E_INVALID, "lins_gpu_mappers_global_map: a masked slot does not have loop closure enabled");
  CK(cudaSetDevice(ctx->device));
  struct Job { int s; lins_global_map_report rep; std::vector<int32_t> keys; std::vector<GatherJob> clouds; };
  std::vector<Job> jobs;
  for (int s = 0; s < M; ++s) {
    if (!mask[s]) continue;
    const MapperNode& m = ms.node[s];
    Job j{s, {}, {}, {}};
    const std::vector<int32_t> sel = lins_gm::select_key_poses(m.poses, m.loops.cur);  // (none without key poses)
    j.keys = lins_gm::key_poses_ds(m.poses, sel);
    long long n = 0;
    for (int32_t id : j.keys) {
      host_kf_jobs(m, id, 3, j.clouds);
      for (int a = 0; a < 3; ++a) n += m.host[id].n[a];
    }
    if (n > INT_MAX) return fail(ctx, LINS_E_TOOBIG, "lins_gpu_mappers_global_map: a slot's key-frame clouds exceed INT32_MAX points");
    j.rep.n_key_poses = (int32_t)sel.size();
    j.rep.n_key_frames = (int32_t)j.keys.size();
    j.rep.n_points = n;
    jobs.push_back(std::move(j));
  }
  // the passes over the jobs with points, in slot order: a pass takes slots while its points stay within the budget
  std::vector<std::pair<size_t, size_t>> passes;  // [first, last) job
  long long in_pass = 0;
  for (size_t k = 0; k < jobs.size(); ++k) {
    const long long n = jobs[k].rep.n_points;
    if (n == 0) continue;
    if (passes.empty() || in_pass + n > LINS_GLOBAL_MAP_PASS_POINTS) {  // (a slot above the budget runs alone)
      passes.push_back({k, k});
      in_pass = 0;
    }
    passes.back().second = k + 1;
    in_pass += n;
  }
  // every pass's buffers first: a pass's result copies read them while the next pass is queued
  for (const auto& ps : passes) {
    int n = 0, segs = 0;
    size_t n_copies = 0;
    for (size_t k = ps.first; k < ps.second; ++k)
      if (jobs[k].rep.n_points) { n += (int)jobs[k].rep.n_points; segs += 1; n_copies += jobs[k].clouds.size(); }
    const int rc = gather_voxel_grid_reserve(ctx, ms, n, segs, n_copies);
    if (rc != LINS_OK) return rc;
  }
  std::vector<Buf<float4>> cloud(jobs.size());
  LoopPass& lp = ms.lp;
  for (const auto& ps : passes) {
    std::vector<size_t> seg;
    std::vector<std::vector<GatherJob>> lists;
    for (size_t k = ps.first; k < ps.second; ++k)
      if (jobs[k].rep.n_points) { seg.push_back(k); lists.push_back(jobs[k].clouds); }
    std::vector<int> toff;
    int rc;
    if ((rc = gather_voxel_grid(ctx, ms, lists, {}, toff)) != LINS_OK) return rc;
    CK(cudaMemcpyAsync(lp.h_info.p, lp.info.p, sizeof(VgInfo) * seg.size(), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));  // the pass's one read-back
    for (size_t p = 0; p < seg.size(); ++p) {
      lins_global_map_report& r = jobs[seg[p]].rep;
      const VgInfo& v = lp.h_info.p[p];
      // PCL 1.7's VoxelGrid publishes its input when the leaf is too small (output = *input_): the concatenation
      r.unfiltered = v.toobig;
      r.n_map = v.toobig ? (int32_t)r.n_points : v.count;
      CK(cloud[seg[p]].reserve((size_t)r.n_map));
      if (r.n_map)
        CK(cudaMemcpyAsync(cloud[seg[p]].p, (v.toobig ? lp.tin.p : lp.tgt.p) + toff[p], sizeof(float4) * r.n_map, cudaMemcpyDeviceToDevice,
                           ctx->stream));
    }
  }
  if (!passes.empty()) CK(cudaStreamSynchronize(ctx->stream));  // the results' copies
  for (size_t k = 0; k < jobs.size(); ++k) {
    MapperGlobalMap& g = ms.node[jobs[k].s].gm;
    g.valid = true;
    g.rep = jobs[k].rep;
    g.keys = std::move(jobs[k].keys);
    g.cloud = std::move(cloud[k]);
    if (reps) reps[jobs[k].s] = g.rep;
  }
  return LINS_OK;
}

}  // namespace lins_capi
