// lins_features.cu — StateEstimator's feature extraction on the device (lins/include/StateEstimator.hpp:619-827:
// undistortPcl, calculateSmoothness, markOccludedPoints, extractFeatures with the per-ring pcl::VoxelGrid, leaf 0.2 m),
// for a batch of segmented scans: lins_gpu_extract_features.  The contract is the host restatement
// csrc/host/feature_extraction.hpp, bit for bit (fresh per-scan arrays, suppression that stops at the cloud's start), apart
// from the order between equal curvatures (DESIGN.md §4.6).  Built with -fmad=false.
//
// One CTA per scan.  The per-point stages run over the scan's points in parallel: halfPassed is a prefix property, so
// the point where it flips is the smallest index whose not-passed orientation exceeds start + pi (a block minimum).  The
// rings and their sextants then run in order, as the reference does, because suppression may cross from one sextant or
// ring into the next: each sextant's [sp, ep) is sorted by (curvature, position) with a block radix sort (stable), and
// warp 0 runs the greedy corner and flat picks 32 candidates at a time (ballot, then the first hit in loop order).  The
// ring's less-flat candidates are voxel-filtered by the whole block: stable radix sort by voxel index, one thread per
// occupied voxel sums its points in input order.
#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>
#include <cstring>
#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>
#include <vector>

#include "lins_ctx.hpp"
#include "lins_features.cuh"

using namespace lins_capi;

namespace {

constexpr int kThreads = 256;
constexpr int kSextantItems = 2;                        // 512 sort slots >= the longest sextant of a kRingCap ring (342)
constexpr int kVoxelItems = lins_feat::kRingCap / kThreads;  // 2048 slots: a ring's less-flat candidates
static_assert(kThreads * kSextantItems >= lins_feat::kRingCap / 6 + 2, "sextant sort capacity");

struct FeatArgs {
  int line_num;
  const float4* pts;  const int* off;
  const int* count; int count_stride;  // scan i: [off[i], off[i] + count[count_stride * i]); null: [off[i], off[i + 1])
  const unsigned char* ground; const unsigned* col; const float* range;
  const int* ring;    // n x 2 x line_num: startRingIndex, endRingIndex
  const float* ori;   // n x 3: startOrientation, endOrientation, orientationDiff
  const FeatConsts* k;  // n: each scan's constants
  float4* und;        // de-skewed cloud, at the input offsets
  float4* out[4];     // surf_flat, corner_sharp, surf_less_flat, corner_less_sharp, at the input offsets
  int* counts;        // n x 5: the four counts, then the scan's status (FEAT_*)
  double* curv; int* sind; unsigned char* picked; signed char* label;  // per-point scratch at the input offsets
};
enum { FEAT_OK = 0, FEAT_INVALID = 1, FEAT_TOOBIG = 2 };

// the +-5 neighbour suppression (:764-777 / :796-811).  Visited entries carry ind 0 or 5 <= ind < n - 5, so only the
// cloud's start can stop it.
__device__ void suppress(const unsigned* C, unsigned char* picked, int ind) {
  picked[ind] = 1;
  for (int l = 1; l <= 5; l++) {
    if (abs(int(C[ind + l] - C[ind + l - 1])) > 10) break;
    picked[ind + l] = 1;
  }
  for (int l = -1; l >= -5; l--) {
    if (ind + l < 0) break;
    if (abs(int(C[ind + l] - C[ind + l + 1])) > 10) break;
    picked[ind + l] = 1;
  }
}

__global__ void __launch_bounds__(kThreads) lins_features_kernel(const FeatArgs a) {
  using SextantSort = cub::BlockRadixSort<unsigned long long, kThreads, kSextantItems, int>;
  using VoxelSort = cub::BlockRadixSort<unsigned, kThreads, kVoxelItems, int>;
  using Scan = cub::BlockScan<int, kThreads>;
  __shared__ union {
    typename SextantSort::TempStorage ss;
    typename VoxelSort::TempStorage vs;
    typename Scan::TempStorage sc;
  } tmp;
  __shared__ int s_cand[lins_feat::kRingCap];   // the ring's less-flat candidates (point indices, ascending)
  __shared__ unsigned s_key[lins_feat::kRingCap];  // their sorted voxel keys
  __shared__ int s_pos[lins_feat::kRingCap];    // ... and candidate positions
  __shared__ int s_ind[kThreads * kSextantItems + 1];  // the sextant's entries [sp, ep] after the sort
  __shared__ float s_red[kThreads / 32][6];
  __shared__ int s_box[6];                      // min_b (3), mul (3)
  __shared__ int s_half, s_bad, s_m, s_cnt[4];

  const int sc = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int base = a.off[sc], np = a.count ? a.count[(size_t)a.count_stride * sc] : a.off[sc + 1] - base;
  const int L = a.line_num;
  const int* rs = a.ring + (size_t)sc * 2 * L;
  const int* re = rs + L;
  const float start = a.ori[3 * sc], end = a.ori[3 * sc + 1], diff = a.ori[3 * sc + 2];
  const FeatConsts kc = a.k[sc];
  const float4* P = a.pts + base;
  const float* R = a.range + base;
  const unsigned* C = a.col + base;
  const unsigned char* G = a.ground + base;
  float4* U = a.und + base;
  double* curv = a.curv + base;
  int* sind = a.sind + base;
  unsigned char* picked = a.picked + base;
  signed char* label = a.label + base;
  if (tid == 0) { s_bad = 0; s_half = np; s_m = 0; for (int c = 0; c < 4; ++c) s_cnt[c] = 0; }
  __syncthreads();

  // ---- validation: visited sextants inside the cloud, ring spans within the sort capacity, finite input --------------
  for (int i = tid; i < L; i += kThreads) {
    bool visited = false;
    for (int j = 0; j < 6; ++j) {
      int64_t sp, ep;
      lins_feat::sextant(rs[i], re[i], j, sp, ep);
      if (sp >= ep) continue;
      visited = true;
      if (sp < 0 || ep > np - 1) atomicOr(&s_bad, FEAT_INVALID);
    }
    if (visited && (int64_t)re[i] - rs[i] > lins_feat::kRingCap) atomicOr(&s_bad, FEAT_TOOBIG);
  }
  if (tid == 0) {
    if (!(isfinite(start) && isfinite(end) && isfinite(diff))) atomicOr(&s_bad, FEAT_INVALID);
    // the visited ranges of the rings follow each other without overlap (abutting is fine): then every output cloud is
    // at most as long as the scan
    int64_t prev = -1;
    for (int i = 0; i < L; ++i) {
      int64_t lo = INT64_MAX, hi = -1;
      for (int j = 0; j < 6; ++j) {
        int64_t sp, ep;
        lins_feat::sextant(rs[i], re[i], j, sp, ep);
        if (sp < ep) { lo = min(lo, sp); hi = max(hi, ep); }
      }
      if (hi < 0) continue;
      if (lo <= prev) atomicOr(&s_bad, FEAT_INVALID);
      prev = hi;
    }
  }
  for (int i = tid; i < np; i += kThreads) {
    const float4 p = P[i];
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && isfinite(p.w) && isfinite(R[i]))) atomicOr(&s_bad, FEAT_INVALID);
  }
  __syncthreads();
  if (s_bad) {
    if (tid == 0) {
      for (int c = 0; c < 4; ++c) a.counts[5 * sc + c] = 0;
      a.counts[5 * sc + 4] = (s_bad & FEAT_INVALID) ? FEAT_INVALID : FEAT_TOOBIG;
    }
    return;
  }

  // ---- undistortPcl: where halfPassed flips, then every point's stamp ---------------------------------------------------
  for (int i = tid; i < np; i += kThreads) {
    const float4 p = P[i];
    float x, y;
    lins_feat::rotate_xy(kc.c, kc.s, p.x, p.y, x, y);
    bool flips;
    lins_feat::ori_not_passed(x, y, start, flips);
    if (flips) atomicMin(&s_half, i);
  }
  __syncthreads();
  const int half = s_half;
  for (int i = tid; i < np; i += kThreads) {
    const float4 p = P[i];
    float x, y;
    lins_feat::rotate_xy(kc.c, kc.s, p.x, p.y, x, y);
    bool flips;
    const double ori = i <= half ? lins_feat::ori_not_passed(x, y, start, flips) : lins_feat::ori_passed(x, y, end);
    U[i] = make_float4(x, y, p.z, lins_feat::stamp(p.w, ori, start, diff, kc.scan_period));
    // calculateSmoothness on [5, n - 5); elsewhere the fresh arrays' defaults (curvature 0, entry (0, ind 0))
    const bool inner = i >= 5 && i < np - 5;
    curv[i] = inner ? lins_feat::curvature(R + i - 5) : 0.0;
    sind[i] = inner ? i : 0;
    picked[i] = 0;
    label[i] = 0;
  }
  __syncthreads();
  // markOccludedPoints: its marks only ever set flags
  for (int i = 5 + tid; i < np - 6; i += kThreads) {
    const int m = lins_feat::occlusion_marks(R + i - 1, C + i - 1);
    if (m & 1) for (int k = -5; k <= 0; ++k) picked[i + k] = 1;
    if (m & 2) for (int k = 1; k <= 6; ++k) picked[i + k] = 1;
    if (m & 4) picked[i] = 1;
  }
  __syncthreads();

  // ---- extractFeatures: rings and sextants in order ---------------------------------------------------------------------
  float4* out_sf = a.out[0] + base;
  float4* out_cs = a.out[1] + base;
  float4* out_slf = a.out[2] + base;
  float4* out_cls = a.out[3] + base;
  for (int ring = 0; ring < L; ++ring) {
    for (int j = 0; j < 6; ++j) {
      int64_t sp64, ep64;
      lins_feat::sextant(rs[ring], re[ring], j, sp64, ep64);
      if (sp64 >= ep64) continue;
      const int sp = (int)sp64, ep = (int)ep64, len = ep - sp;
      // std::sort of [sp, ep) by curvature; equal curvatures keep their positions (stable radix sort)
      unsigned long long keys[kSextantItems];
      int vals[kSextantItems];
      for (int q = 0; q < kSextantItems; ++q) {
        const int p = tid * kSextantItems + q;
        if (p < len) {
          const int ind = sind[sp + p];
          const double v = curv[ind];
          memcpy(&keys[q], &v, 8);  // (curvatures are squares: >= 0, so their bits sort as unsigned integers)
          vals[q] = ind;
        } else {
          keys[q] = ~0ull;
          vals[q] = 0;
        }
      }
      SextantSort(tmp.ss).Sort(keys, vals);
      for (int q = 0; q < kSextantItems; ++q) {
        const int p = tid * kSextantItems + q;
        if (p < len) { s_ind[p] = vals[q]; sind[sp + p] = vals[q]; }
      }
      if (tid == 0) s_ind[len] = sind[ep];  // entry ep is visited but not sorted
      __syncthreads();
      if (warp == 0) {
        const unsigned FULL = 0xffffffffu;
        // corner pick: from ep down, at most 20, the first 2 sharp
        int largest = 0;
        for (int k = ep; k >= sp;) {
          const int kk = k - lane;
          int ind = 0;
          bool ok = false;
          if (kk >= sp) { ind = s_ind[kk - sp]; ok = picked[ind] == 0 && curv[ind] > kc.edge && G[ind] == 0; }
          const unsigned b = __ballot_sync(FULL, ok);
          if (!b) { k -= 32; continue; }
          const int l = __ffs(b) - 1;
          const int pind = __shfl_sync(FULL, ind, l);
          if (++largest > 20) break;
          if (lane == 0) {
            const float4 pt = U[pind];
            if (largest <= 2) { label[pind] = 2; out_cs[s_cnt[1]++] = pt; }
            else label[pind] = 1;
            out_cls[s_cnt[3]++] = pt;
            suppress(C, picked, pind);
          }
          __syncwarp();
          k -= l + 1;
        }
        // flat pick: from sp up; the 4th is pushed but neither marked nor suppressed
        int smallest = 0;
        for (int k = sp; k <= ep;) {
          const int kk = k + lane;
          int ind = 0;
          bool ok = false;
          if (kk <= ep) { ind = s_ind[kk - sp]; ok = picked[ind] == 0 && curv[ind] < kc.surf && G[ind] == 1; }
          const unsigned b = __ballot_sync(FULL, ok);
          if (!b) { k += 32; continue; }
          const int l = __ffs(b) - 1;
          const int pind = __shfl_sync(FULL, ind, l);
          ++smallest;
          if (lane == 0) {
            label[pind] = -1;
            out_sf[s_cnt[0]++] = U[pind];
            if (smallest < 4) suppress(C, picked, pind);
          }
          __syncwarp();
          if (smallest >= 4) break;
          k += l + 1;
        }
        // surfPointsLessFlatScan: label <= 0, by point index
        int m = s_m;
        for (int k0 = sp; k0 <= ep; k0 += 32) {
          const int k = k0 + lane;
          const bool ok = k <= ep && label[k] <= 0;
          const unsigned b = __ballot_sync(FULL, ok);
          if (ok) s_cand[m + __popc(b & ((1u << lane) - 1))] = k;
          m += __popc(b);
        }
        if (lane == 0) s_m = m;
      }
      __syncthreads();
    }

    // ---- the ring's VoxelGrid ----------------------------------------------------------------------------------------
    const int m = s_m;
    if (m == 0) continue;  // (uniform: s_m is read after a barrier)
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int t = tid; t < m; t += kThreads) {
      const float4 p = U[s_cand[t]];
      mn[0] = fminf(mn[0], p.x); mn[1] = fminf(mn[1], p.y); mn[2] = fminf(mn[2], p.z);
      mx[0] = fmaxf(mx[0], p.x); mx[1] = fmaxf(mx[1], p.y); mx[2] = fmaxf(mx[2], p.z);
    }
    for (int o = 16; o; o >>= 1)
      for (int d = 0; d < 3; ++d) {
        mn[d] = fminf(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
        mx[d] = fmaxf(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
      }
    if (lane == 0) for (int d = 0; d < 3; ++d) { s_red[warp][d] = mn[d]; s_red[warp][3 + d] = mx[d]; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kThreads / 32; ++w)
        for (int d = 0; d < 3; ++d) { mn[d] = fminf(mn[d], s_red[w][d]); mx[d] = fmaxf(mx[d], s_red[w][3 + d]); }
      int div[3];
      for (int d = 0; d < 3; ++d) {
        s_box[d] = lins_feat::voxel_bound(mn[d]);
        div[d] = lins_feat::voxel_bound(mx[d]) - s_box[d] + 1;
      }
      s_box[3] = 1; s_box[4] = div[0]; s_box[5] = div[0] * div[1];
    }
    __syncthreads();
    const int min_b[3] = {s_box[0], s_box[1], s_box[2]}, mul[3] = {s_box[3], s_box[4], s_box[5]};
    unsigned vk[kVoxelItems];
    int vp[kVoxelItems];
    for (int q = 0; q < kVoxelItems; ++q) {
      const int p = tid * kVoxelItems + q;
      vp[q] = p;
      if (p < m) { const float4 pt = U[s_cand[p]]; vk[q] = lins_feat::voxel_key(pt.x, pt.y, pt.z, min_b, mul); }
      else vk[q] = 0xffffffffu;  // (after every candidate: the sort is stable and these come last in the input)
    }
    VoxelSort(tmp.vs).Sort(vk, vp);
    for (int q = 0; q < kVoxelItems; ++q) { s_key[tid * kVoxelItems + q] = vk[q]; s_pos[tid * kVoxelItems + q] = vp[q]; }
    __syncthreads();
    int heads = 0;
    for (int q = 0; q < kVoxelItems; ++q) {
      const int p = tid * kVoxelItems + q;
      heads += p < m && (p == 0 || s_key[p] != s_key[p - 1]);
    }
    int rank, total;
    Scan(tmp.sc).ExclusiveSum(heads, rank, total);
    const int obase = s_cnt[2];
    for (int q = 0; q < kVoxelItems; ++q) {
      const int p = tid * kVoxelItems + q;
      if (!(p < m && (p == 0 || s_key[p] != s_key[p - 1]))) continue;
      float cx = 0, cy = 0, cz = 0, ci = 0;
      int e = p;
      for (; e < m && s_key[e] == s_key[p]; ++e) {
        const float4 pt = U[s_cand[s_pos[e]]];
        cx += pt.x; cy += pt.y; cz += pt.z; ci += pt.w;
      }
      const float cnt = (float)(e - p);
      out_slf[obase + rank++] = make_float4(cx / cnt, cy / cnt, cz / cnt, ci / cnt);
    }
    __syncthreads();
    if (tid == 0) { s_cnt[2] += total; s_m = 0; }
    __syncthreads();
  }
  if (tid == 0) {
    for (int c = 0; c < 4; ++c) a.counts[5 * sc + c] = s_cnt[c];
    a.counts[5 * sc + 4] = FEAT_OK;
  }
}

}  // namespace

namespace lins_capi {

// features_run: validate the descriptor on the host (offsets, arrays, line_num), upload it, then features_launch.
// features_launch: extract on the device and read the counts back (one D2H and one stream synchronisation).  The device
// checks what needs the points (finite input, sextants inside the cloud, ring spans) and reports it in the same
// read-back.  On return f.h_counts holds n x 5 (counts, status) and the clouds are in f.out / f.und at the input offsets.
// lins_gpu_seq_step_raw calls features_launch on the projection's output where it lies (ctx->proj, raw offsets).
FeatConsts feat_consts(const lins_feature_params& fp, double scan_period) {
  FeatConsts k;
  const double y = fp.imu_lidar_extrinsic_angle * M_PI / 180.0;  // math_utils::deg2rad
  k.c = std::cos(y); k.s = std::sin(y);
  k.edge = fp.edge_threshold; k.surf = fp.surf_threshold; k.scan_period = scan_period;
  return k;
}

int features_run(lins_ctx* ctx, const lins_feature_params* fp, const lins_pcl_desc* d, const double* period) {
  if (!fp || !d || d->n_scans < 0) return fail(ctx, LINS_E_INVALID, "bad feature extraction arguments");
  if (d->line_num < 1 || d->line_num > lins_feat::kMaxLines) return fail(ctx, LINS_E_INVALID, "line_num outside 1..128");
  const int n = d->n_scans, L = d->line_num;
  int rc = check_csr(ctx, d->cloud_off, n, d->cloud, "bad cloud offsets / cloud");
  if (rc != LINS_OK) return rc;
  const int total = d->cloud_off[n];
  if (total > 0 && (!d->ground_flag || !d->col_ind || !d->range)) return fail(ctx, LINS_E_INVALID, "null per-point array");
  if (n > 0 && (!d->start_ring_index || !d->end_ring_index || !d->orientation)) return fail(ctx, LINS_E_INVALID, "null cloud_info array");
  if (d->point_format != LINS_POINTS_XYZI32 && d->point_format != LINS_POINTS_PACKED16) return fail(ctx, LINS_E_INVALID, "bad point_format");
  CK(cudaSetDevice(ctx->device));
  FeatState& f = ctx->feat;
  std::vector<int32_t> zeros(n + 1, 0);
  const lins_point* pts[4] = {d->cloud, nullptr, nullptr, nullptr};
  const int32_t* offs[4] = {d->cloud_off, zeros.data(), zeros.data(), zeros.data()};
  rc = upload_clouds(ctx, f.up, n, pts, offs, d->point_format);  // (synchronises the stream first)
  if (rc != LINS_OK) return rc;
  std::vector<FeatConsts> k(n);
  for (int i = 0; i < n; ++i) k[i] = feat_consts(*fp, period ? period[i] : ctx->prm.scan_period);
  if (n == 0) return features_launch(ctx, k.data(), FeatInputs());
  const size_t N = (size_t)total + 1;
  CK(f.ground.reserve(N)); CK(f.col.reserve(N)); CK(f.range.reserve(N)); CK(f.ring.reserve(2 * (size_t)n * L)); CK(f.ori.reserve(3 * (size_t)n));
  f.h_ring.resize(2 * (size_t)n * L);
  for (int i = 0; i < n; ++i) {
    std::memcpy(&f.h_ring[(size_t)i * 2 * L], d->start_ring_index + (size_t)i * L, sizeof(int32_t) * L);
    std::memcpy(&f.h_ring[(size_t)i * 2 * L + L], d->end_ring_index + (size_t)i * L, sizeof(int32_t) * L);
  }
  if (total) {
    CK(cudaMemcpyAsync(f.ground.p, d->ground_flag, total, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(f.col.p, d->col_ind, sizeof(uint32_t) * total, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(f.range.p, d->range, sizeof(float) * total, cudaMemcpyHostToDevice, ctx->stream));
  }
  CK(cudaMemcpyAsync(f.ring.p, f.h_ring.data(), sizeof(int) * f.h_ring.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(f.ori.p, d->orientation, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, ctx->stream));
  FeatInputs in;
  in.n = n; in.line_num = L; in.total = total;
  in.pts = f.up.qs.p; in.off = f.up.qs_off.p;
  in.ground = f.ground.p; in.col = f.col.p; in.range = f.range.p; in.ring = f.ring.p; in.ori = f.ori.p;
  return features_launch(ctx, k.data(), in);
}

int features_launch(lins_ctx* ctx, const FeatConsts* k, const FeatInputs& in) {
  FeatState& f = ctx->feat;
  const int n = in.n;
  CK(f.h_counts.reserve(5 * (size_t)n + 1));
  if (n == 0) return LINS_OK;
  const size_t N = (size_t)in.total + 1;
  CK(f.und.reserve(N)); for (auto& o : f.out) CK(o.reserve(N));
  CK(f.consts.reserve(n)); CK(f.h_consts.reserve(n));
  CK(f.counts.reserve(5 * (size_t)n)); CK(f.curv.reserve(N)); CK(f.sind.reserve(N)); CK(f.picked.reserve(N)); CK(f.label.reserve(N));
  FeatArgs a;
  a.line_num = in.line_num;
  a.pts = in.pts; a.off = in.off; a.count = in.count; a.count_stride = in.count_stride;
  a.ground = in.ground; a.col = in.col; a.range = in.range; a.ring = in.ring; a.ori = in.ori;
  std::memcpy(f.h_consts.p, k, sizeof(FeatConsts) * n);  // (the last extraction ended with a synchronisation)
  CK(cudaMemcpyAsync(f.consts.p, f.h_consts.p, sizeof(FeatConsts) * n, cudaMemcpyHostToDevice, ctx->stream));
  a.k = f.consts.p;
  a.und = f.und.p;
  for (int k = 0; k < 4; ++k) a.out[k] = f.out[k].p;
  a.counts = f.counts.p;
  a.curv = f.curv.p; a.sind = f.sind.p; a.picked = f.picked.p; a.label = reinterpret_cast<signed char*>(f.label.p);
  CK(f.ev.start(ctx->stream));
  lins_features_kernel<<<n, kThreads, 0, ctx->stream>>>(a);
  CK(cudaGetLastError());
  ctx->launches += 1;
  CK(f.ev.stop(ctx->stream));
  CK(cudaMemcpyAsync(f.h_counts.p, f.counts.p, sizeof(int) * 5 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < n; ++i) {
    const int st = f.h_counts.p[5 * i + 4];
    if (st == FEAT_INVALID) return fail(ctx, LINS_E_INVALID, "invalid segmented scan (non-finite point / range / orientation, or a sextant outside the cloud)");
    if (st == FEAT_TOOBIG) return fail(ctx, LINS_E_TOOBIG, "a ring span exceeds LINS_FEAT_RING_CAP");
  }
  return LINS_OK;
}

}  // namespace lins_capi

extern "C" {

int lins_gpu_extract_features(lins_ctx* ctx, const lins_feature_params* fp, const lins_pcl_desc* d, lins_point* surf_flat,
                              lins_point* corner_sharp, lins_point* surf_less_flat, lins_point* corner_less_sharp,
                              lins_point* undist, int32_t* counts) {
  if (!ctx) return LINS_E_INVALID;
  if (!counts) return fail(ctx, LINS_E_INVALID, "null counts");
  if (d && d->n_scans > 0 && d->cloud_off && d->cloud_off[d->n_scans] > 0 && (!surf_flat || !corner_sharp || !surf_less_flat || !corner_less_sharp))
    return fail(ctx, LINS_E_INVALID, "null output cloud");
  const int rc = features_run(ctx, fp, d);
  if (rc != LINS_OK) return rc;
  const int n = d->n_scans;
  if (n == 0) return LINS_OK;
  FeatState& f = ctx->feat;
  const int total = d->cloud_off[n];
  lins_point* dst[5] = {surf_flat, corner_sharp, surf_less_flat, corner_less_sharp, undist};
  Buf<float4>* src[5] = {&f.out[0], &f.out[1], &f.out[2], &f.out[3], &f.und};
  std::vector<float4> h((size_t)total);
  for (int k = 0; k < 5; ++k) {
    if (!dst[k] || total == 0) continue;
    CK(cudaMemcpy(h.data(), src[k]->p, sizeof(float4) * total, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) {
      const int o = d->cloud_off[i], cnt = k < 4 ? f.h_counts.p[5 * i + k] : d->cloud_off[i + 1] - o;
      for (int t = o; t < o + cnt; ++t) {
        const float4 p = h[t];
        if (d->point_format == LINS_POINTS_PACKED16) reinterpret_cast<float4*>(dst[k])[t] = p;
        else dst[k][t] = unpack_point(p);
      }
    }
  }
  for (int i = 0; i < n; ++i) for (int k = 0; k < 4; ++k) counts[4 * i + k] = f.h_counts.p[5 * i + k];
  return LINS_OK;
}

int lins_gpu_extract_ms(lins_ctx* ctx, float* ms) {
  if (!ctx) return LINS_E_INVALID;
  return event_ms(ctx, ctx->feat.ev, ms, "no extraction has run");
}

}  // extern "C"
