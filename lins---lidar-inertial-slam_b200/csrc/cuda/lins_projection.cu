// lins_projection.cu — image projection on the device (lins/src/image_projection_node.cpp:191-415: findStartEndAngle,
// projectPointCloud, groundRemoval, cloudSegmentation with labelComponents) for a batch of raw sweeps:
// lins_gpu_project_scans.  The contract is the host restatement csrc/host/image_projection.hpp, bit for bit, run on a
// fresh ImageProjection per scan.  Built with -fmad=false.  DESIGN.md §4.7.
//
// One CTA per scan at a time (a grid of as many CTAs as fit, each looping over scans), with the range image in global
// scratch of its own (L2 / HBM: a 64 x 1024 image's labels alone exceed shared memory).  The stages:
//  - projection: every point does an atomicMax of its index into its pixel, so the last point of a pixel wins, as the
//    reference's overwrite does; range and fullCloud are then gathered from the winner;
//  - ground removal: one thread per column walks the rows in order (iteration i may overwrite the 1 of iteration i - 1);
//  - segmentation: labelComponents' neighbours are directed (std::pair<uint8_t, uint8_t> offsets: right with the wrap
//    S-1 -> 0, 255 columns right or column 0 past the end, down; "up" is always out of range).  The component of a pixel
//    is the smallest raster index among the unblocked pixels that reach it over qualifying edges (DESIGN.md §4.7), so
//    labels are propagated to that fixpoint: a segmented prefix minimum along each row's runs of right edges, and pushes
//    along the jump, wrap and down edges, until a round changes nothing;
//  - feasibility from per-owner counts and row extents (the seed's own row is not counted), then cloudSegmentation's
//    compaction in raster order with a block scan.
// lins_gpu_seq_step_raw runs the kernel with drop_nonfinite: copyPointCloud's pcl::removeNaNFromPointCloud
// (image_projection_node.cpp:172-177) without a compaction pass.  A non-finite point is never projected, and
// findStartEndAngle reads the first, last and second-to-last finite points; the removal keeps the order, so the highest
// index of a pixel is still the point the filtered sweep's overwrite would leave.  A scan whose present flag is 0 is
// projected as an empty sweep.
// Each scan reads its lidar model from a device-resident table (lins_gpu_project_scans_mixed and the _mixed step
// entries; the single-model entries pass a table of one), so sweeps of different sensors share a call.  Ring indices use
// the table's largest line_num as their stride; a scan's rings past its own line_num are written as 0.
#include <cuda_runtime.h>

#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <cub/block/block_scan.cuh>
#include <vector>

#include "lins_ctx.hpp"
#include "lins_projection.cuh"

using namespace lins_capi;

namespace {

constexpr int kThreads = 512;
constexpr int kBlocked = INT_MAX;  // the label of a ground or empty pixel (labelMat == -1)
constexpr int kMidRow = 1 << 30;   // (owner counts stay below 2^18 = 128 x 2048)
enum : unsigned char { E_RIGHT = 1, E_JUMP = 2, E_DOWN = 4, FEASIBLE = 0x80 };

struct ProjArgs {
  int n;
  int L_max;                     // the ring stride: the largest line_num in the table
  size_t P_max;                  // the per-CTA scratch stride: the largest line_num x scan_num in the table
  const ProjModel* models;       // the model table (device)
  const int* model_of;           // n: each scan's entry in models, or null = every scan uses models[0]
  const float4* pts; const int* off;
  const unsigned char* present;  // n, or null = all (lins_gpu_seq_step_raw)
  int drop_nonfinite;            // copyPointCloud's NaN removal (lins_gpu_seq_step_raw)
  // per-CTA scratch, P_max entries each
  int* idx; float* rng; signed char* gnd; int* lab; unsigned char* edg; int* cnt; int* rlo; int* rhi;
  // outputs at the raw offsets
  float4* seg; unsigned char* ground; unsigned* col; float* range; float4* outl;
  int* ring;    // n x 2 x L_max: startRingIndex, endRingIndex; a scan's rings past its own line_num are 0
  float* ori;   // n x 3
  int* counts;  // n x 2: segmented, outlier
};

__device__ __forceinline__ bool push_label(int* lab, int t, int v) {
  return lab[t] > v && atomicMin(&lab[t], v) > v;
}

// pcl::removeNaNFromPointCloud keeps a point iff its x, y and z are finite
__device__ __forceinline__ bool finite_xyz(const float4& q) { return isfinite(q.x) && isfinite(q.y) && isfinite(q.z); }

__global__ void __launch_bounds__(kThreads) lins_projection_kernel(const ProjArgs a) {
  using Scan = cub::BlockScan<unsigned long long, kThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_fin[3];  // drop_nonfinite: the first, last and second-to-last finite point (-1: none)
  __shared__ ProjModel s_m; // the current scan's model
  const unsigned FULL = 0xffffffffu;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t so = (size_t)blockIdx.x * a.P_max;
  int* idx = a.idx + so;
  float* rng = a.rng + so;
  signed char* gnd = a.gnd + so;
  int* lab = a.lab + so;
  unsigned char* edg = a.edg + so;
  int* cnt = a.cnt + so;  // per owner: member count, | kMidRow once a pushed member lies strictly between rlo and rhi
  int* rlo = a.rlo + so;  // per owner: the lowest / highest row of its pushed (non-seed) members
  int* rhi = a.rhi + so;
  auto blocked = [&](int p) { return gnd[p] == 1 || rng[p] == FLT_MAX; };

  for (int sc = blockIdx.x; sc < a.n; sc += gridDim.x) {
    if (tid == 0) s_m = a.models[a.model_of ? a.model_of[sc] : 0];
    __syncthreads();  // (the previous scan's last reads of s_m are behind its final barrier)
    const int L = s_m.L, S = s_m.S, P = L * S;
    const int base = a.off[sc], np = a.present && !a.present[sc] ? 0 : a.off[sc + 1] - base;
    const float4* pt = a.pts + base;
    for (int p = tid; p < P; p += kThreads) {
      idx[p] = -1; gnd[p] = 0; cnt[p] = 0; rlo[p] = INT_MAX; rhi[p] = -1;
    }
    if (a.drop_nonfinite) {  // the filtered sweep's ends: warp 0 from the front, warp 1 from the back, 32 points a round
      if (warp == 0) {
        int f = -1;
        for (int i0 = 0; i0 < np && f < 0; i0 += 32) {
          const unsigned b = __ballot_sync(FULL, i0 + lane < np && finite_xyz(pt[i0 + lane]));
          if (b) f = i0 + __ffs(b) - 1;
        }
        if (lane == 0) s_fin[0] = f;
      } else if (warp == 1) {
        int l1 = -1, l2 = -1;
        for (int i0 = np - 1; i0 >= 0 && l2 < 0; i0 -= 32) {
          unsigned b = __ballot_sync(FULL, i0 - lane >= 0 && finite_xyz(pt[i0 - lane]));
          for (; b && l2 < 0; b &= b - 1) {
            const int k = i0 - (__ffs(b) - 1);
            if (l1 < 0) l1 = k; else l2 = k;
          }
        }
        if (lane == 0) { s_fin[1] = l1; s_fin[2] = l2; }
      }
      __syncthreads();
    }
    if (tid == 0) {  // findStartEndAngle; a scan of fewer than 2 (finite) points keeps a fresh cloud_info's zeros
      float o[3] = {0.f, 0.f, 0.f};
      if (a.drop_nonfinite) {
        if (s_fin[2] >= 0) lins_proj::start_end_angle(pt[s_fin[0]].x, pt[s_fin[0]].y, pt[s_fin[1]].y, pt[s_fin[2]].x, o);
      } else if (np >= 2) {
        lins_proj::start_end_angle(pt[0].x, pt[0].y, pt[np - 1].y, pt[np - 2].x, o);
      }
      for (int k = 0; k < 3; ++k) a.ori[3 * sc + k] = o[k];
    }
    __syncthreads();

    // ---- projectPointCloud: the highest point index of a pixel wins ---------------------------------------------------
    for (int i = tid; i < np; i += kThreads) {
      const float4 q = pt[i];
      int r, c;
      if ((!a.drop_nonfinite || finite_xyz(q)) && lins_proj::project(q.x, q.y, q.z, L, S, s_m.res_x, s_m.res_y, s_m.bottom, r, c))
        atomicMax(&idx[r * S + c], i);
    }
    __syncthreads();
    for (int p = tid; p < P; p += kThreads) {
      const int k = idx[p];
      rng[p] = k < 0 ? FLT_MAX : lins_proj::point_range(pt[k].x, pt[k].y, pt[k].z);
    }
    // ---- groundRemoval: each column's rows in order ------------------------------------------------------------------
    for (int j = tid; j < S; j += kThreads)
      for (int i = 0; i < s_m.gsi; ++i) {
        const int lo = idx[i * S + j], up = idx[(i + 1) * S + j];
        if (lo < 0 || up < 0) { gnd[i * S + j] = -1; continue; }
        const float4 l = pt[lo], u = pt[up];
        if (lins_proj::ground_pair(l.x, l.y, l.z, u.x, u.y, u.z)) { gnd[i * S + j] = 1; gnd[(i + 1) * S + j] = 1; }
      }
    __syncthreads();

    // ---- labelComponents: initial labels and the qualifying out-edges -------------------------------------------------
    for (int p = tid; p < P; p += kThreads) {
      const int r = p / S, c = p - r * S;
      const bool blk = blocked(p);
      lab[p] = blk ? kBlocked : p;
      unsigned char e = 0;
      if (!blk) {
        const float rp = rng[p];
        const int t1 = r * S + (c + 1 < S ? c + 1 : 0), t2 = r * S + (c + 255 < S ? c + 255 : 0);
        if (!blocked(t1) && lins_proj::edge(rp, rng[t1], s_m.sin_x, s_m.cos_x)) e |= E_RIGHT;
        if (!blocked(t2) && lins_proj::edge(rp, rng[t2], s_m.sin_x, s_m.cos_x)) e |= E_JUMP;
        if (r + 1 < L && !blocked(p + S) && lins_proj::edge(rp, rng[p + S], s_m.sin_y, s_m.cos_y)) e |= E_DOWN;
      }
      edg[p] = e;
    }
    __syncthreads();
    // min-label propagation to the fixpoint (labels only decrease)
    for (;;) {
      int changed = 0;
      for (int p = tid; p < P; p += kThreads) {
        const int r = p / S, c = p - r * S;
        const unsigned char m = edg[p] & (E_JUMP | E_DOWN | (c == S - 1 ? E_RIGHT : 0));
        if (!m) continue;
        const int v = lab[p];
        if ((m & E_RIGHT) && push_label(lab, r * S, v)) changed = 1;
        if ((m & E_JUMP) && push_label(lab, r * S + (c + 255 < S ? c + 255 : 0), v)) changed = 1;
        if ((m & E_DOWN) && push_label(lab, p + S, v)) changed = 1;
      }
      __syncthreads();
      // the right edges inside each row: a segmented inclusive prefix minimum (a segment starts where the edge from the
      // left neighbour does not qualify), one warp per row, 32 columns at a time with the carry of the previous chunk
      for (int r = warp; r < L; r += kThreads / 32) {
        int carry = kBlocked;
        for (int c0 = 0; c0 < S; c0 += 32) {
          const int c = c0 + lane, p = r * S + c;
          const int old = c < S ? lab[p] : kBlocked;
          int v = old;
          int head = !(c < S && c > 0 && (edg[p - 1] & E_RIGHT));
          for (int d = 1; d < 32; d <<= 1) {
            const int ov = __shfl_up_sync(FULL, v, d), oh = __shfl_up_sync(FULL, head, d);
            if (lane >= d && !head) { v = min(v, ov); head = oh; }
          }
          if (!head) v = min(v, carry);
          if (c < S && v < old) { lab[p] = v; changed = 1; }
          carry = __shfl_sync(FULL, v, 31);
        }
      }
      if (!__syncthreads_or(changed)) break;
    }

    // ---- feasibility: size >= 30, or >= 5 with >= 3 rows among the pushed (non-seed) members.  The pushed members
    // span >= 3 distinct rows exactly when one of them lies strictly between their lowest and highest row.
    for (int p = tid; p < P; p += kThreads) {
      const int o = lab[p];
      if (o == kBlocked) continue;
      atomicAdd(&cnt[o], 1);
      if (o != p) { const int r = p / S; atomicMin(&rlo[o], r); atomicMax(&rhi[o], r); }
    }
    __syncthreads();
    for (int p = tid; p < P; p += kThreads) {
      const int o = lab[p];
      if (o == kBlocked || o == p) continue;
      const int r = p / S;
      if (r > rlo[o] && r < rhi[o]) atomicOr(&cnt[o], kMidRow);
    }
    __syncthreads();
    for (int p = tid; p < P; p += kThreads) {
      if (lab[p] != p) continue;
      const int size = cnt[p] & ~kMidRow;
      if (size >= 30 || (size >= 5 && (cnt[p] & kMidRow))) edg[p] |= FEASIBLE;
    }
    __syncthreads();

    // ---- cloudSegmentation's compaction in raster order ----------------------------------------------------------------
    const int LM = a.L_max;
    int* ring = a.ring + (size_t)sc * 2 * LM;  // start: ring[0 .. L), end: ring[LM .. LM + L)
    for (int r = L + tid; r < LM; r += kThreads) { ring[r] = 0; ring[LM + r] = 0; }  // (the buffer is reused)
    int n_seg = 0, n_out = 0;
    for (int q0 = 0; q0 < P; q0 += kThreads) {
      const int p = q0 + tid;
      bool s = false, o = false;
      int r = 0, c = 0;
      if (p < P) {
        r = p / S; c = p - r * S;
        const int ow = lab[p];
        if (gnd[p] == 1) {
          s = c % 5 == 0 || c <= 5 || c >= S - 5;  // the ground thinning
        } else if (ow != kBlocked) {
          const bool feasible = edg[ow] & FEASIBLE;
          s = feasible;
          o = !feasible && r > s_m.gsi && c % 5 == 0;  // label 999999
        }
      }
      unsigned long long pre, tot;
      Scan(tmp).ExclusiveSum((unsigned long long)s | ((unsigned long long)o << 32), pre, tot);
      const int ps = n_seg + (int)(pre & 0xffffffffu), po = n_out + (int)(pre >> 32);
      if (s || o) {
        const float4 q = pt[idx[p]];
        const float4 full = make_float4(q.x, q.y, q.z, lins_proj::pixel_intensity(r, c));
        if (s) {
          a.seg[base + ps] = full;
          a.ground[base + ps] = gnd[p] == 1;
          a.col[base + ps] = (unsigned)c;
          a.range[base + ps] = rng[p];
        } else {
          a.outl[base + po] = full;
        }
      }
      if (p < P && c == 0) {
        ring[r] = ps - 1 + 5;
        if (r > 0) ring[LM + r - 1] = ps - 1 - 5;
      }
      n_seg += (int)(tot & 0xffffffffu);
      n_out += (int)(tot >> 32);
      __syncthreads();  // (tmp is reused)
    }
    if (tid == 0) {
      ring[LM + L - 1] = n_seg - 1 - 5;
      a.counts[2 * sc] = n_seg;
      a.counts[2 * sc + 1] = n_out;
    }
    __syncthreads();  // the scratch is reset for the next scan
  }
}

// lins_gpu_project_scans' read-back: each scan's used prefixes of the clouds at the raw offsets -> dense offsets (one CTA
// per scan)
struct PackArgs {
  int n;
  const int* off; const int* doff; const int* counts;  // raw offsets (n + 1); dense offsets: segmented, outlier (2 x (n + 1))
  const float4* seg; const float4* outl; const unsigned char* ground; const unsigned* col; const float* range;
  float4* dseg; float4* doutl; unsigned char* dground; unsigned* dcol; float* drange;
};

__global__ void lins_projection_pack_kernel(const PackArgs a) {
  const int sc = blockIdx.x, o = a.off[sc], ns = a.counts[2 * sc], no = a.counts[2 * sc + 1];
  const int ds = a.doff[sc], dq = a.doff[a.n + 1 + sc];
  for (int t = threadIdx.x; t < ns; t += blockDim.x) {
    a.dseg[ds + t] = a.seg[o + t]; a.dground[ds + t] = a.ground[o + t]; a.dcol[ds + t] = a.col[o + t]; a.drange[ds + t] = a.range[o + t];
  }
  for (int t = threadIdx.x; t < no; t += blockDim.x) a.doutl[dq + t] = a.outl[o + t];
}

}  // namespace

namespace lins_capi {

int check_model(lins_ctx* ctx, const lins_lidar_model* m) {
  if (!m) return fail(ctx, LINS_E_INVALID, "null lidar model");
  if (m->line_num < 1 || m->line_num > lins_feat::kMaxLines) return fail(ctx, LINS_E_INVALID, "line_num outside 1..128");
  if (m->scan_num < 2 || m->scan_num > LINS_FEAT_RING_CAP) return fail(ctx, LINS_E_INVALID, "scan_num outside 2..LINS_FEAT_RING_CAP");
  if (!(std::isfinite(m->ang_res_x) && m->ang_res_x > 0 && std::isfinite(m->ang_res_y) && m->ang_res_y > 0))
    return fail(ctx, LINS_E_INVALID, "angular resolutions must be finite and positive");
  if (!std::isfinite(m->ang_bottom)) return fail(ctx, LINS_E_INVALID, "ang_bottom must be finite");
  if (m->ground_scan_ind < 0 || m->ground_scan_ind > m->line_num - 1) return fail(ctx, LINS_E_INVALID, "ground_scan_ind outside 0..line_num-1");
  return LINS_OK;
}

int check_models(lins_ctx* ctx, const lins_lidar_models* t) {
  if (!t) return fail(ctx, LINS_E_INVALID, "null lidar model table");
  if (t->n_models < 1) return fail(ctx, LINS_E_INVALID, "n_models < 1");
  if (!t->models) return fail(ctx, LINS_E_INVALID, "null lidar model");
  for (int i = 0; i < t->n_models; ++i) {
    const int rc = check_model(ctx, &t->models[i]);
    if (rc != LINS_OK) return rc;
  }
  if (!t->model_of && t->n_models > 1) return fail(ctx, LINS_E_INVALID, "null model_of with more than one lidar model");
  return LINS_OK;
}

int check_model_of(lins_ctx* ctx, const lins_lidar_models* t, int n) {
  if (t->model_of)
    for (int i = 0; i < n; ++i)
      if (t->model_of[i] < 0 || t->model_of[i] >= t->n_models) return fail(ctx, LINS_E_INVALID, "model_of entry outside 0..n_models-1");
  return LINS_OK;
}

int max_line_num(const lins_lidar_models* t) {
  int L = 0;
  for (int i = 0; i < t->n_models; ++i) L = std::max(L, (int)t->models[i].line_num);
  return L;
}

// Validate the model table and the descriptor on the host, upload the sweeps and queue the projection kernel (no
// synchronisation).  Afterwards ctx->proj holds the projected clouds at the raw offsets, n x 2 x L_max ring indices (L_max
// = max_line_num(t)), n x 3 orientations and n x 2 counts, all on the device.  drop_nonfinite / present: see ProjArgs.
int projection_run(lins_ctx* ctx, const lins_lidar_models* t, const lins_raw_desc* d, bool drop_nonfinite, const uint8_t* present) {
  int rc = check_models(ctx, t);
  if (rc != LINS_OK) return rc;
  if (!d || d->n_scans < 0) return fail(ctx, LINS_E_INVALID, "bad raw sweep descriptor");
  const int n = d->n_scans;
  if (!d->cloud_off) return fail(ctx, LINS_E_INVALID, "null cloud offsets");
  rc = check_model_of(ctx, t, n);
  if (rc != LINS_OK) return rc;
  CK(cudaSetDevice(ctx->device));
  ProjState& pr = ctx->proj;
  std::vector<int32_t> zeros(n + 1, 0);
  const lins_point* pts[4] = {d->cloud, nullptr, nullptr, nullptr};
  const int32_t* offs[4] = {d->cloud_off, zeros.data(), zeros.data(), zeros.data()};
  rc = upload_clouds(ctx, pr.up, n, pts, offs, d->point_format);  // (validates the offsets and the format; synchronises first)
  if (rc != LINS_OK) return rc;
  if (n == 0) return LINS_OK;
  return projection_launch(ctx, t, n, (size_t)d->cloud_off[n], drop_nonfinite, present);
}

int projection_launch(lins_ctx* ctx, const lins_lidar_models* t, int n, size_t total, bool drop_nonfinite, const uint8_t* present) {
  ProjState& pr = ctx->proj;
  const int nm = t->n_models, L_max = max_line_num(t);
  size_t P_max = 0;
  for (int i = 0; i < nm; ++i) P_max = std::max(P_max, (size_t)t->models[i].line_num * t->models[i].scan_num);
  const size_t N = total + 1;
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lins_projection_kernel, kThreads, 0));
  const int grid = std::max(1, std::min(n, per_sm * ctx->sm_count));
  const size_t G = (size_t)grid * P_max;
  CK(pr.idx.reserve(G)); CK(pr.rng.reserve(G)); CK(pr.gnd.reserve(G)); CK(pr.lab.reserve(G)); CK(pr.edg.reserve(G));
  CK(pr.cnt.reserve(G)); CK(pr.rlo.reserve(G)); CK(pr.rhi.reserve(G));
  CK(pr.seg.reserve(N)); CK(pr.outl.reserve(N)); CK(pr.ground.reserve(N)); CK(pr.col.reserve(N)); CK(pr.range.reserve(N));
  CK(pr.ring.reserve(2 * (size_t)n * L_max)); CK(pr.ori.reserve(3 * (size_t)n)); CK(pr.counts.reserve(2 * (size_t)n));
  // (the upload synchronised the stream: the staging is free)
  CK(pr.models.reserve(nm)); CK(pr.h_models.reserve(nm));
  for (int i = 0; i < nm; ++i) {
    const lins_lidar_model& m = t->models[i];
    ProjModel& q = pr.h_models.p[i];
    q.L = m.line_num; q.S = m.scan_num; q.gsi = m.ground_scan_ind;
    q.res_x = m.ang_res_x; q.res_y = m.ang_res_y; q.bottom = m.ang_bottom;
    const float ax = lins_proj::segment_alpha(m.ang_res_x), ay = lins_proj::segment_alpha(m.ang_res_y);
    q.sin_x = std::sin(ax); q.cos_x = std::cos(ax); q.sin_y = std::sin(ay); q.cos_y = std::cos(ay);  // (float overloads: sinf / cosf)
  }
  CK(cudaMemcpyAsync(pr.models.p, pr.h_models.p, sizeof(ProjModel) * nm, cudaMemcpyHostToDevice, ctx->stream));
  if (t->model_of) {
    CK(pr.model_of.reserve(n)); CK(pr.h_model_of.reserve(n));
    std::memcpy(pr.h_model_of.p, t->model_of, sizeof(int32_t) * n);
    CK(cudaMemcpyAsync(pr.model_of.p, pr.h_model_of.p, sizeof(int32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (present) {
    CK(pr.present.reserve(n)); CK(pr.h_present.reserve(n));
    std::memcpy(pr.h_present.p, present, n);
    CK(cudaMemcpyAsync(pr.present.p, pr.h_present.p, n, cudaMemcpyHostToDevice, ctx->stream));
  }
  ProjArgs a;
  a.n = n; a.L_max = L_max; a.P_max = P_max;
  a.models = pr.models.p; a.model_of = t->model_of ? pr.model_of.p : nullptr;
  a.present = present ? pr.present.p : nullptr;
  a.drop_nonfinite = drop_nonfinite;
  a.pts = pr.up.qs.p; a.off = pr.up.qs_off.p;
  a.idx = pr.idx.p; a.rng = pr.rng.p; a.gnd = reinterpret_cast<signed char*>(pr.gnd.p); a.lab = pr.lab.p; a.edg = pr.edg.p;
  a.cnt = pr.cnt.p; a.rlo = pr.rlo.p; a.rhi = pr.rhi.p;
  a.seg = pr.seg.p; a.ground = pr.ground.p; a.col = pr.col.p; a.range = pr.range.p; a.outl = pr.outl.p;
  a.ring = pr.ring.p; a.ori = pr.ori.p; a.counts = pr.counts.p;
  CK(pr.ev.start(ctx->stream));
  lins_projection_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
  CK(cudaGetLastError());
  ctx->launches += 1;
  CK(pr.ev.stop(ctx->stream));
  return LINS_OK;
}

}  // namespace lins_capi

extern "C" {

int lins_gpu_project_scans_mixed(lins_ctx* ctx, const lins_lidar_models* t, const lins_raw_desc* d, lins_point* seg, uint8_t* ground_flag,
                                 uint32_t* col_ind, float* range, lins_point* outlier, int32_t* start_ring, int32_t* end_ring, float* ori,
                                 int32_t* counts) {
  if (!ctx) return LINS_E_INVALID;
  if (d && d->n_scans > 0) {
    if (!start_ring || !end_ring || !ori || !counts) return fail(ctx, LINS_E_INVALID, "null cloud_info output");
    if (d->cloud_off && d->cloud_off[d->n_scans] > 0 && (!seg || !ground_flag || !col_ind || !range || !outlier))
      return fail(ctx, LINS_E_INVALID, "null output cloud");
  }
  const int rc = projection_run(ctx, t, d, false, nullptr);
  if (rc != LINS_OK) return rc;
  const int n = d->n_scans;
  if (n == 0) return LINS_OK;
  ProjState& pr = ctx->proj;
  const int L = max_line_num(t);
  // the counts first (one synchronisation), then only the clouds' used prefixes: packed to dense offsets on the device
  // and read back through pinned staging (a second synchronisation)
  CK(pr.h_counts.reserve(2 * (size_t)n)); CK(pr.h_ring.reserve(2 * (size_t)n * L)); CK(pr.h_ori.reserve(3 * (size_t)n));
  CK(pr.h_doff.reserve(2 * (size_t)(n + 1)));
  CK(cudaMemcpyAsync(pr.h_counts.p, pr.counts.p, sizeof(int) * 2 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(pr.h_ring.p, pr.ring.p, sizeof(int) * 2 * (size_t)n * L, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(pr.h_ori.p, pr.ori.p, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  int* doff = pr.h_doff.p;  // dense offsets: segmented (n + 1), outlier (n + 1)
  doff[0] = doff[n + 1] = 0;
  for (int i = 0; i < n; ++i) {
    doff[i + 1] = doff[i] + pr.h_counts.p[2 * i];
    doff[n + 2 + i] = doff[n + 1 + i] + pr.h_counts.p[2 * i + 1];
  }
  const int ts = doff[n], to = doff[2 * n + 1];
  CK(pr.dseg.reserve((size_t)ts + 1)); CK(pr.dground.reserve((size_t)ts + 1)); CK(pr.dcol.reserve((size_t)ts + 1));
  CK(pr.drange.reserve((size_t)ts + 1)); CK(pr.doutl.reserve((size_t)to + 1)); CK(pr.doff.reserve(2 * (size_t)(n + 1)));
  CK(pr.h_seg.reserve((size_t)ts + 1)); CK(pr.h_ground.reserve((size_t)ts + 1)); CK(pr.h_col.reserve((size_t)ts + 1));
  CK(pr.h_range.reserve((size_t)ts + 1)); CK(pr.h_outl.reserve((size_t)to + 1));
  CK(cudaMemcpyAsync(pr.doff.p, doff, sizeof(int) * 2 * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
  if (ts + to > 0) {
    PackArgs k;
    k.n = n; k.off = pr.up.qs_off.p; k.doff = pr.doff.p; k.counts = pr.counts.p;
    k.seg = pr.seg.p; k.outl = pr.outl.p; k.ground = pr.ground.p; k.col = pr.col.p; k.range = pr.range.p;
    k.dseg = pr.dseg.p; k.doutl = pr.doutl.p; k.dground = pr.dground.p; k.dcol = pr.dcol.p; k.drange = pr.drange.p;
    lins_projection_pack_kernel<<<n, 256, 0, ctx->stream>>>(k);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  if (ts) {
    CK(cudaMemcpyAsync(pr.h_seg.p, pr.dseg.p, sizeof(float4) * ts, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(pr.h_ground.p, pr.dground.p, ts, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(pr.h_col.p, pr.dcol.p, sizeof(uint32_t) * ts, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(pr.h_range.p, pr.drange.p, sizeof(float) * ts, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (to) CK(cudaMemcpyAsync(pr.h_outl.p, pr.doutl.p, sizeof(float4) * to, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  const bool p16 = d->point_format == LINS_POINTS_PACKED16;
  auto put = [&](lins_point* dst, int t, const float4& p) {
    if (p16) reinterpret_cast<float4*>(dst)[t] = p;
    else dst[t] = unpack_point(p);
  };
  for (int i = 0; i < n; ++i) {
    const int o = d->cloud_off[i], ns = pr.h_counts.p[2 * i], no = pr.h_counts.p[2 * i + 1], ds = doff[i], dq = doff[n + 1 + i];
    for (int t = 0; t < ns; ++t) {
      put(seg, o + t, pr.h_seg.p[ds + t]);
      ground_flag[o + t] = pr.h_ground.p[ds + t]; col_ind[o + t] = pr.h_col.p[ds + t]; range[o + t] = pr.h_range.p[ds + t];
    }
    for (int t = 0; t < no; ++t) put(outlier, o + t, pr.h_outl.p[dq + t]);
    std::memcpy(start_ring + (size_t)i * L, pr.h_ring.p + (size_t)i * 2 * L, sizeof(int32_t) * L);
    std::memcpy(end_ring + (size_t)i * L, pr.h_ring.p + (size_t)i * 2 * L + L, sizeof(int32_t) * L);
    for (int k = 0; k < 3; ++k) ori[3 * i + k] = pr.h_ori.p[3 * i + k];
    counts[2 * i] = ns;
    counts[2 * i + 1] = no;
  }
  return LINS_OK;
}

int lins_gpu_project_scans(lins_ctx* ctx, const lins_lidar_model* m, const lins_raw_desc* d, lins_point* seg, uint8_t* ground_flag,
                           uint32_t* col_ind, float* range, lins_point* outlier, int32_t* start_ring, int32_t* end_ring, float* ori,
                           int32_t* counts) {
  const lins_lidar_models t = {1, m, nullptr};
  return lins_gpu_project_scans_mixed(ctx, &t, d, seg, ground_flag, col_ind, range, outlier, start_ring, end_ring, ori, counts);
}

int lins_gpu_project_ms(lins_ctx* ctx, float* ms) {
  if (!ctx) return LINS_E_INVALID;
  return event_ms(ctx, ctx->proj.ev, ms, "no projection has run");
}

}  // extern "C"
