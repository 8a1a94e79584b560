// lins_map.cu — host side of row F2 (SURVEY.md §8(f)): the mapping node's scan-to-map refinement, whose kernels are in
// lins_map.cuh.  One driver over a table of slots (ScanToMap): the host fills the table, then queues the grid build and
// the loop.  The mapping nodes run a slot each; lins_gpu_map_set / scan2map / map_associate run the one slot of ctx->mp.
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>

#include "lins_ctx.hpp"
#include "lins_map.cuh"

using namespace lins_capi;

// ---- row F2: the mapping node's scan-to-map refinement (lidar_mapping_node.cpp:1635-1652) --------------------------------
namespace {

lins_map::PassConsts host_pass_consts(const float* T) {  // libm sin / cos in f32, like the reference (:579-592, :1527-1532)
  lins_map::PassConsts pc;
  pc.cRoll = std::cos(T[0]); pc.sRoll = std::sin(T[0]); pc.cPitch = std::cos(T[1]); pc.sPitch = std::sin(T[1]);
  pc.cYaw = std::cos(T[2]); pc.sYaw = std::sin(T[2]); pc.tX = T[3]; pc.tY = T[4]; pc.tZ = T[5];
  pc.srx = std::sin(T[0]); pc.crx = std::cos(T[0]); pc.sry = std::sin(T[1]); pc.cry = std::cos(T[1]);
  pc.srz = std::sin(T[2]); pc.crz = std::cos(T[2]);
  return pc;
}

// which 5-NN search map_associate's pass uses: the hashed grid (exact for every point that can be accepted) or the
// brute-force slices (exact for every point, the default).  LINS_MAP_KNN=grid|brute overrides it; the loop always
// searches the grid.
bool map_use_grid() {
  const char* e = std::getenv("LINS_MAP_KNN");  // (read per call: tests flip it between calls)
  return e && std::strcmp(e, "grid") == 0;
}

// the grid origin of a host cloud: its finite minimum (cells are addressed by hash: the extent does not matter)
void map_grid_origin(const lins_point* host_pts, int n, lins_map::GridIndex& g) {
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f};
  for (int i = 0; i < n; ++i) {
    const float v[3] = {host_pts[i].x, host_pts[i].y, host_pts[i].z};
    for (int k = 0; k < 3; ++k) if (v[k] == v[k] && std::fabs(v[k]) < 1.0e30f && v[k] < mn[k]) mn[k] = v[k];
  }
  for (int k = 0; k < 3; ++k) mn[k] = mn[k] < 3.0e38f ? mn[k] : 0.f;
  g.ox = mn[0]; g.oy = mn[1]; g.oz = mn[2];
}

// the 5-NN of kind k (0 corner, 1 surf) through every slot's grid, for the table's fit blocks
void queue_knn_grid(lins_ctx* ctx, const ScanToMap& sm, int k, const lins_map::MapLoopState* st) {
  using namespace lins_map;
  lins_map_knn_grid_kernel<<<sm.blocks[k] * kFitThreads / kGridKnnWarps, kGridKnnWarps * 32, 0, ctx->stream>>>(
      sm.blocks[k] * kFitThreads, sm.consts.p, st, sm.part_d.p, sm.part_i.p, sm.mslot.p, sm.n_slots, sm.blk_slot.p + (k ? sm.blocks[0] : 0), k);
}

// the fits and block partials of kind k over n_slices partial lists per row, with dense outputs where non-null
void queue_fit(lins_ctx* ctx, const ScanToMap& sm, int k, int n_slices, const lins_map::MapLoopState* st, int32_t* knn, float* coeff,
               uint8_t* mask) {
  using namespace lins_map;
  const size_t b0 = k ? sm.blocks[0] : 0;
  auto* fit = k ? lins_map_fit_kernel<false> : lins_map_fit_kernel<true>;
  fit<<<sm.blocks[k], kFitThreads, 0, ctx->stream>>>(n_slices, sm.part_d.p, sm.part_i.p, sm.consts.p, st, knn, coeff, mask,
                                                     sm.partial.p + b0 * (kRowAcc + 1), sm.mslot.p, sm.n_slots, sm.blk_slot.p + b0);
}

}  // namespace

// the start of every slot's loop (n slots): its loop state takes the start transform and a cleared report (matP /
// isDegenerate persist), and scan2MapOptimization's gate (:1636) on the device-resident map sizes marks a slot done
// before its first pass when its map fails, or when it has none (run = 0)
__global__ void lins_map_gate_kernel(lins_map::MapLoopState* __restrict__ st, const lins_map::MapSlot* __restrict__ sl, int n) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const lins_map::MapSlot& v = sl[s];
  lins_map::MapLoopState& m = st[s];
  for (int i = 0; i < 6; ++i) m.T[i] = v.T[i];
  m.done = m.iters = m.converged = 0;
  for (int i = 0; i < LINS_MAP_MAX_ITER; ++i) { m.n_sel[i] = 0; m.delta_r[i] = 0.f; m.delta_t[i] = 0.f; }
  if (!v.run) { m.done = 1; return; }
  if (!(*v.n_map[0] > 10 && *v.n_map[1] > 100)) m.done = 1;
}

namespace lins_capi {

int map_fill_table(lins_ctx* ctx, ScanToMap& sm, int n_slots) {
  using namespace lins_map;
  MapSlot* h = sm.h_mslot.p;
  // per slot: each map's bucket count from its capacity, fit blocks that start with the slot's queries
  int nb_tot = 0, pts = 0, blocks[2] = {0, 0};
  std::vector<int> blk_slot[2];
  for (int s = 0; s < n_slots; ++s) {
    MapSlot& v = h[s];
    for (int k = 0; k < 2; ++k) {
      unsigned nb = v.run ? 4096 : 1;  // (a slot that does not run searches nothing)
      while (v.run && nb < 2u * (unsigned)v.cap[k] && nb < (1u << 24)) nb <<= 1;
      v.g[k].mask = nb - 1;
      v.bucket0[k] = nb_tot; nb_tot += (int)nb;
      v.m0[k] = pts; pts += v.cap[k];
      v.blk[k] = blocks[k];
      v.nblk[k] = v.run ? (v.nq[k] + kFitThreads - 1) / kFitThreads : 0;
      blocks[k] += v.nblk[k];
      blk_slot[k].insert(blk_slot[k].end(), v.nblk[k], s);
    }
  }
  size_t scan_bytes = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, sm.count.p, sm.grid_start.p, nb_tot + 1, ctx->stream));
  CK(sm.scan_temp.grow(scan_bytes + 16));
  CK(sm.grid_start.grow((size_t)nb_tot + 2)); CK(sm.count.grow((size_t)nb_tot + 2)); CK(sm.cursor.grow((size_t)nb_tot + 2));
  CK(sm.sorted.grow((size_t)pts + 1));
  const size_t rows = (size_t)std::max(blocks[0], blocks[1]) * kFitThreads;
  CK(sm.part_d.grow(5 * rows + 1)); CK(sm.part_i.grow(5 * rows + 1));
  CK(sm.partial.grow((size_t)(blocks[0] + blocks[1] + 1) * (kRowAcc + 1)));
  CK(sm.blk_slot.grow((size_t)blocks[0] + blocks[1] + 1)); CK(sm.h_blk_slot.grow((size_t)blocks[0] + blocks[1] + 1));
  CK(sm.consts.grow(n_slots)); CK(sm.h_consts.grow(n_slots)); CK(sm.mslot.grow(n_slots));
  for (int s = 0; s < n_slots; ++s) {
    for (int k = 0; k < 2; ++k) { h[s].g[k].pts = sm.sorted.p; h[s].g[k].start = sm.grid_start.p + h[s].bucket0[k]; }
    sm.h_consts.p[s] = host_pass_consts(h[s].T);
  }
  std::copy(blk_slot[0].begin(), blk_slot[0].end(), sm.h_blk_slot.p);
  std::copy(blk_slot[1].begin(), blk_slot[1].end(), sm.h_blk_slot.p + blocks[0]);
  CK(cudaMemcpyAsync(sm.mslot.p, h, sizeof(MapSlot) * n_slots, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(sm.consts.p, sm.h_consts.p, sizeof(PassConsts) * n_slots, cudaMemcpyHostToDevice, ctx->stream));
  if (blocks[0] + blocks[1])
    CK(cudaMemcpyAsync(sm.blk_slot.p, sm.h_blk_slot.p, sizeof(int) * (blocks[0] + blocks[1]), cudaMemcpyHostToDevice, ctx->stream));
  sm.n_slots = n_slots; sm.buckets = nb_tot; sm.points = pts; sm.blocks[0] = blocks[0]; sm.blocks[1] = blocks[1];
  return LINS_OK;
}

int map_queue_grids(lins_ctx* ctx, ScanToMap& sm) {
  using namespace lins_map;
  const int pts = sm.points, nb = sm.buckets;
  CK(cudaMemsetAsync(sm.count.p, 0, sizeof(int) * ((size_t)nb + 1), ctx->stream));
  if (pts) lins_grid_count_kernel<<<(pts + 255) / 256, 256, 0, ctx->stream>>>(pts, sm.count.p, sm.mslot.p, sm.n_slots);
  size_t bytes = sm.scan_temp.cap;
  CK(cub::DeviceScan::ExclusiveSum(sm.scan_temp.p, bytes, sm.count.p, sm.grid_start.p, nb + 1, ctx->stream));
  CK(cudaMemcpyAsync(sm.cursor.p, sm.grid_start.p, sizeof(int) * nb, cudaMemcpyDeviceToDevice, ctx->stream));
  if (pts) lins_grid_scatter_kernel<<<(pts + 255) / 256, 256, 0, ctx->stream>>>(pts, sm.cursor.p, sm.sorted.p, sm.mslot.p, sm.n_slots);
  CK(cudaGetLastError());
  ctx->launches += pts ? 3 : 1;
  return LINS_OK;
}

int map_queue_loop(lins_ctx* ctx, ScanToMap& sm) {
  using namespace lins_map;
  lins_map_gate_kernel<<<(sm.n_slots + 127) / 128, 128, 0, ctx->stream>>>(sm.loop.p, sm.mslot.p, sm.n_slots);
  CK(cudaGetLastError());
  ctx->launches += 1;
  // per pass one 5-NN and one fit launch per kind over every slot, one LM launch of a warp per slot
  for (int iter = 0; iter < LINS_MAP_MAX_ITER; ++iter) {
    for (int k = 0; k < 2; ++k) {
      if (!sm.blocks[k]) continue;
      queue_knn_grid(ctx, sm, k, sm.loop.p);
      queue_fit(ctx, sm, k, 1, sm.loop.p, nullptr, nullptr, nullptr);
      ctx->launches += 2;
    }
    lins_map_lm_kernel<<<sm.n_slots, 32, 0, ctx->stream>>>(sm.partial.p, sm.blocks[0], iter, sm.loop.p, sm.consts.p, sm.mslot.p);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  CK(cudaMemcpyAsync(sm.h_loop.p, sm.loop.p, sizeof(MapLoopState) * sm.n_slots, cudaMemcpyDeviceToHost, ctx->stream));
  return LINS_OK;
}

// the report of the loop whose state st holds
void map_loop_report(const lins_map::MapLoopState& st, float* T, lins_map_report* rep) {
  lins_map_report r;
  std::memset(&r, 0, sizeof(r));
  for (int i = 0; i < 6; ++i) T[i] = st.T[i];
  // a call whose first pass selects < 50 points takes no LM step (its later passes see the same transform), so nothing
  // was projected: it reports 0, like the reference's LMOptimization, while matP / isDegenerate persist for later calls
  r.iters = st.iters; r.converged = st.converged; r.degenerate = st.n_sel[0] >= 50 ? st.isDegenerate : 0;
  for (int i = 0; i < LINS_MAP_MAX_ITER; ++i) { r.n_sel[i] = st.n_sel[i]; r.delta_r[i] = st.delta_r[i]; r.delta_t[i] = st.delta_t[i]; }
  *rep = r;
}

}  // namespace lins_capi

namespace {

// the queries of the one-slot table in ctx->mp (lins_gpu_map_set has set its maps): checked, uploaded and, with the start
// transform T, in the table, which is filled and uploaded
int map_stage_queries(lins_ctx* ctx, const lins_point* corner, int nc, const lins_point* surf, int ns, const float* T) {
  if (check_cloud(ctx, corner, nc, "bad corner feature cloud") != LINS_OK || check_cloud(ctx, surf, ns, "bad surf feature cloud") != LINS_OK)
    return LINS_E_INVALID;
  lins_ctx::MapState& m = ctx->mp;
  if (m.n_map_c < 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_map_set has not been called");
  const int rc = upload2(ctx, m.q_c, corner, nc, m.q_s, surf, ns);
  if (rc != LINS_OK) return rc;
  lins_map::MapSlot& v = m.stm.h_mslot.p[0];
  v.q[0] = m.q_c.p; v.q[1] = m.q_s.p; v.nq[0] = nc; v.nq[1] = ns;
  for (int i = 0; i < 6; ++i) v.T[i] = T[i];
  return map_fill_table(ctx, m.stm, 1);
}

}  // namespace

extern "C" {

int lins_gpu_map_set(lins_ctx* ctx, const lins_point* corner, int nc, const lins_point* surf, int ns) {
  if (!ctx) return LINS_E_INVALID;
  if (check_cloud(ctx, corner, nc, "bad corner map cloud") != LINS_OK || check_cloud(ctx, surf, ns, "bad surf map cloud") != LINS_OK)
    return LINS_E_INVALID;
  CK(cudaSetDevice(ctx->device));
  lins_ctx::MapState& m = ctx->mp;
  int rc = upload2(ctx, m.map_c, corner, nc, m.map_s, surf, ns);
  if (rc != LINS_OK) return rc;
  const int n[2] = {nc, ns};
  CK(m.n_map.reserve(2));
  CK(cudaMemcpyAsync(m.n_map.p, n, sizeof(n), cudaMemcpyHostToDevice, ctx->stream));  // (pageable: staged before the call returns)
  m.n_map_c = nc; m.n_map_s = ns;
  // a one-slot table whose maps' capacities are their sizes, each grid's origin its cloud's finite minimum
  CK(m.stm.h_mslot.reserve(1));
  lins_map::MapSlot& v = m.stm.h_mslot.p[0];
  std::memset(&v, 0, sizeof(v));
  v.run = 1;
  const lins_point* src[2] = {corner, surf};
  for (int k = 0; k < 2; ++k) {
    v.map[k] = (k ? m.map_s : m.map_c).p; v.cap[k] = n[k]; v.n_map[k] = m.n_map.p + k;
    map_grid_origin(src[k], n[k], v.g[k]);
  }
  if ((rc = map_fill_table(ctx, m.stm, 1)) != LINS_OK || (rc = map_queue_grids(ctx, m.stm)) != LINS_OK) return rc;
  CK(cudaStreamSynchronize(ctx->stream));  // (the next call rewrites the table's pinned staging)
  return LINS_OK;
}

int lins_gpu_scan2map(lins_ctx* ctx, const lins_point* corner, int nc, const lins_point* surf, int ns, float* T, lins_map_report* rep) {
  if (!ctx) return LINS_E_INVALID;
  if (!T) return fail(ctx, LINS_E_INVALID, "null transform");
  CK(cudaSetDevice(ctx->device));
  lins_map_report r;
  std::memset(&r, 0, sizeof(r));
  lins_ctx::MapState& m = ctx->mp;
  if (m.n_map_c < 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_map_set has not been called");
  if (!(m.n_map_c > 10 && m.n_map_s > 100)) {  // :1636
    r.skipped = 1;
    if (rep) *rep = r;
    return LINS_OK;
  }
  int rc = map_stage_queries(ctx, corner, nc, surf, ns, T);
  if (rc != LINS_OK) return rc;
  ScanToMap& sm = m.stm;
  // isDegenerate / matP are members of the reference's mapping node (:226-227, :395-396): they start at 0 and survive the
  // calls — a call whose first pass selects < 50 points keeps using the previous scan's values
  if (!sm.loop.p) {
    CK(sm.loop.reserve(1)); CK(sm.h_loop.reserve(1));
    CK(cudaMemsetAsync(sm.loop.p, 0, sizeof(lins_map::MapLoopState), ctx->stream));
  }
  if ((rc = map_queue_loop(ctx, sm)) != LINS_OK) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  map_loop_report(*sm.h_loop.p, T, &r);
  if (rep) *rep = r;
  return LINS_OK;
}

int lins_gpu_map_associate(lins_ctx* ctx, const lins_point* corner, int nc, const lins_point* surf, int ns, const float* T,
                           int32_t* cknn, int32_t* sknn, float* ccoeff, float* scoeff, uint8_t* cmask, uint8_t* smask) {
  using namespace lins_map;
  if (!ctx) return LINS_E_INVALID;
  if (!T) return fail(ctx, LINS_E_INVALID, "null transform");
  CK(cudaSetDevice(ctx->device));
  int rc = map_stage_queries(ctx, corner, nc, surf, ns, T);
  if (rc != LINS_OK) return rc;
  lins_ctx::MapState& m = ctx->mp;
  ScanToMap& sm = m.stm;
  const MapSlot& v = sm.h_mslot.p[0];
  // the parity hook: brute force by default (exact neighbours for EVERY point, also those the 1 m gate rejects), over
  // enough (query block, map slice) pairs for ~8 CTAs per SM (the scan is latency bound: profiles/r01_map_*); a slice is
  // at least 256 map points.  The grid leaves one list per query.
  const bool grid = map_use_grid();
  int slices[2] = {1, 1}, slice_len[2] = {0, 0};
  size_t part = 0;
  for (int k = 0; k < 2; ++k) {
    if (grid || !sm.blocks[k]) continue;
    const int S = std::max(1, std::min((8 * ctx->sm_count + sm.blocks[k] - 1) / sm.blocks[k], std::min(64, (v.cap[k] + 255) / 256)));
    slices[k] = S;
    slice_len[k] = std::max(1, (v.cap[k] + S - 1) / S);
    part = std::max(part, (size_t)v.nq[k] * S * 5);
  }
  CK(sm.part_d.grow(part + 1)); CK(sm.part_i.grow(part + 1));
  CK(m.knn_c.reserve(5 * (size_t)nc + 1)); CK(m.knn_s.reserve(5 * (size_t)ns + 1)); CK(m.coeff_c.reserve(4 * (size_t)nc + 1));
  CK(m.coeff_s.reserve(4 * (size_t)ns + 1)); CK(m.mask_c.reserve((size_t)nc + 1)); CK(m.mask_s.reserve((size_t)ns + 1));
  int32_t* knn[2] = {m.knn_c.p, m.knn_s.p};
  float* coeff[2] = {m.coeff_c.p, m.coeff_s.p};
  uint8_t* mask[2] = {m.mask_c.p, m.mask_s.p};
  for (int k = 0; k < 2; ++k) {
    if (!sm.blocks[k]) continue;
    if (grid)
      queue_knn_grid(ctx, sm, k, nullptr);
    else
      lins_map_knn_kernel<<<dim3(sm.blocks[k], slices[k]), kKnnThreads, 0, ctx->stream>>>(v.q[k], v.nq[k], v.map[k], v.cap[k], slice_len[k], sm.consts.p,
                                                                                          nullptr, sm.part_d.p, sm.part_i.p);
    queue_fit(ctx, sm, k, slices[k], nullptr, knn[k], coeff[k], mask[k]);
    CK(cudaGetLastError());
    ctx->launches += 2;
  }
  CK(d2h(ctx, cknn, m.knn_c.p, sizeof(int32_t) * 5 * (size_t)nc));
  CK(d2h(ctx, sknn, m.knn_s.p, sizeof(int32_t) * 5 * (size_t)ns));
  CK(d2h(ctx, ccoeff, m.coeff_c.p, sizeof(float) * 4 * (size_t)nc));
  CK(d2h(ctx, scoeff, m.coeff_s.p, sizeof(float) * 4 * (size_t)ns));
  CK(d2h(ctx, cmask, m.mask_c.p, (size_t)nc));
  CK(d2h(ctx, smask, m.mask_s.p, (size_t)ns));
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}

}  // extern "C"
