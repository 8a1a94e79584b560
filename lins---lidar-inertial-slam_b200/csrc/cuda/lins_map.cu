// lins_map.cu — host side of row F2 (SURVEY.md §8(f)): the mapping node's scan-to-map refinement, whose kernels are in
// lins_map.cuh.
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

// which 5-NN search a pass uses: the hashed grid (exact for every point that can be accepted) or the brute-force slices
// (exact for every point).  LINS_MAP_KNN=grid|brute overrides the caller's default.
bool map_use_grid(bool dflt) {
  const char* e = std::getenv("LINS_MAP_KNN");  // (read per call: tests flip it between calls)
  return !e || !*e ? dflt : std::strcmp(e, "grid") == 0;
}

// the kernels' view of a grid (lins_ctx.hpp keeps its parts: that header cannot include lins_map.cuh)
lins_map::GridIndex grid_index(const lins_ctx::MapState::Grid& g) {
  lins_map::GridIndex gi;
  gi.pts = g.sorted.p; gi.start = g.start.p; gi.mask = g.mask; gi.ox = g.origin[0]; gi.oy = g.origin[1]; gi.oz = g.origin[2];
  return gi;
}

}  // namespace

namespace lins_capi {

// the grid origin of a host cloud: its finite minimum (cells are addressed by hash: the extent does not matter)
void map_grid_origin(const lins_point* host_pts, int n, float origin[3]) {
  float mn[3] = {3.0e38f, 3.0e38f, 3.0e38f};
  for (int i = 0; i < n; ++i) {
    const float v[3] = {host_pts[i].x, host_pts[i].y, host_pts[i].z};
    for (int k = 0; k < 3; ++k) if (v[k] == v[k] && std::fabs(v[k]) < 1.0e30f && v[k] < mn[k]) mn[k] = v[k];
  }
  for (int k = 0; k < 3; ++k) origin[k] = mn[k] < 3.0e38f ? mn[k] : 0.f;
}

// bucket-sort one device-resident map cloud into its grid (≙ kdtree*FromMap->setInputCloud, :1637-1638).  Any finite
// origin gives the same 5-NN: the cells are exact (lins_map.cuh: grid_cell) and addressed by hash.
int map_build_grid(lins_ctx* ctx, lins_ctx::MapState::Grid& g, const float4* map, int n, const float origin[3]) {
  using namespace lins_map;
  g.n = n;
  if (n <= 0) return LINS_OK;
  unsigned nb = 4096;
  while (nb < 2u * (unsigned)n && nb < (1u << 24)) nb <<= 1;
  CK(g.start.reserve((size_t)nb + 2)); CK(g.count.reserve((size_t)nb + 2)); CK(g.cursor.reserve((size_t)nb + 2)); CK(g.sorted.reserve((size_t)n + 1));
  g.mask = nb - 1;
  for (int k = 0; k < 3; ++k) g.origin[k] = origin[k];
  const GridIndex gi = grid_index(g);
  CK(cudaMemsetAsync(g.count.p, 0, sizeof(int) * nb, ctx->stream));
  lins_grid_count_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(map, n, gi, g.count.p, nullptr, 0);
  lins_grid_scan_kernel<<<1, 1024, 0, ctx->stream>>>(g.count.p, g.start.p, g.cursor.p, (int)nb);
  lins_grid_scatter_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(map, n, gi, g.cursor.p, g.sorted.p, nullptr, 0);
  CK(cudaGetLastError());
  ctx->launches += 3;
  return LINS_OK;
}

}  // namespace lins_capi

namespace {

// queue one cornerOptimization + surfOptimization pass (5-NN, fits, block partials) that reads its constants from
// m.consts (device); nothing is synchronised.  Returns the number of partial blocks.
int map_queue_pass(lins_ctx* ctx, int nc, int ns, bool dense, bool grid, const lins_map::MapLoopState* st, int* nblocks_out) {
  using namespace lins_map;
  lins_ctx::MapState& m = ctx->mp;
  const int qb[2] = {(nc + kKnnThreads - 1) / kKnnThreads, (ns + kKnnThreads - 1) / kKnnThreads};
  const int nq[2] = {nc, ns}, nm[2] = {std::max(m.n_map_c, 0), std::max(m.n_map_s, 0)};
  const float4* q[2] = {m.q_c.p, m.q_s.p};
  const float4* mp[2] = {m.map_c.p, m.map_s.p};
  const lins_ctx::MapState::Grid* gr[2] = {&m.grid_c, &m.grid_s};
  int slices[2], slice_len[2];
  size_t part = 0;
  for (int k = 0; k < 2; ++k) {
    // brute force: enough (query block, map slice) pairs for ~8 CTAs per SM (the scan is latency bound: profiles/r01_map_*);
    // a slice is at least 256 map points.  grid: one list per query
    int S = qb[k] > 0 ? (8 * ctx->sm_count + qb[k] - 1) / qb[k] : 1;
    S = std::max(1, std::min(S, std::min(64, (nm[k] + 255) / 256)));
    if (grid) S = 1;
    slices[k] = S;
    slice_len[k] = std::max(1, (nm[k] + S - 1) / S);
    part = std::max(part, (size_t)nq[k] * S * 5);
  }
  CK(m.part_d.reserve(part + 1)); CK(m.part_i.reserve(part + 1));
  const int nblocks = qb[0] + qb[1];
  CK(m.partial.reserve((size_t)(nblocks + 1) * (kRowAcc + 1))); CK(m.h_partial.reserve((size_t)(nblocks + 1) * (kRowAcc + 1)));
  if (dense) {
    CK(m.knn_c.reserve(5 * (size_t)nc + 1)); CK(m.knn_s.reserve(5 * (size_t)ns + 1)); CK(m.coeff_c.reserve(4 * (size_t)nc + 1));
    CK(m.coeff_s.reserve(4 * (size_t)ns + 1)); CK(m.mask_c.reserve((size_t)nc + 1)); CK(m.mask_s.reserve((size_t)ns + 1));
  }
  for (int k = 0; k < 2; ++k) {
    if (nq[k] == 0) continue;
    if (grid && nm[k] > 0)
      lins_map_knn_grid_kernel<<<(nq[k] + kGridKnnWarps - 1) / kGridKnnWarps, kGridKnnWarps * 32, 0, ctx->stream>>>(q[k], nq[k], grid_index(*gr[k]), m.consts.p, st, m.part_d.p, m.part_i.p, nullptr, nullptr, k);
    else
      lins_map_knn_kernel<<<dim3(qb[k], slices[k]), kKnnThreads, 0, ctx->stream>>>(q[k], nq[k], mp[k], nm[k], slice_len[k], m.consts.p, st, m.part_d.p, m.part_i.p);
    double* partial = m.partial.p + (size_t)(k == 0 ? 0 : qb[0]) * (kRowAcc + 1);
    if (k == 0)
      lins_map_fit_kernel<true><<<qb[k], kFitThreads, 0, ctx->stream>>>(q[k], nq[k], mp[k], slices[k], m.part_d.p, m.part_i.p, m.consts.p, st, dense ? m.knn_c.p : nullptr,
                                                                       dense ? m.coeff_c.p : nullptr, dense ? m.mask_c.p : nullptr, partial, nullptr, nullptr);
    else
      lins_map_fit_kernel<false><<<qb[k], kFitThreads, 0, ctx->stream>>>(q[k], nq[k], mp[k], slices[k], m.part_d.p, m.part_i.p, m.consts.p, st, dense ? m.knn_s.p : nullptr,
                                                                        dense ? m.coeff_s.p : nullptr, dense ? m.mask_s.p : nullptr, partial, nullptr, nullptr);
    CK(cudaGetLastError());
    ctx->launches += 2;
  }
  *nblocks_out = nblocks;
  return LINS_OK;
}

int map_stage_queries(lins_ctx* ctx, const lins_point* corner, int nc, const lins_point* surf, int ns) {
  if (check_cloud(ctx, corner, nc, "bad corner feature cloud") != LINS_OK || check_cloud(ctx, surf, ns, "bad surf feature cloud") != LINS_OK)
    return LINS_E_INVALID;
  if (ctx->mp.n_map_c < 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_map_set has not been called");
  return upload2(ctx, ctx->mp.q_c, corner, nc, ctx->mp.q_s, surf, ns);
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

// the iteration loop of scan2MapOptimization (:1640-1648) on the queries in ctx->mp.q_c / q_s and the map set up
// in ctx->mp, queued up front with the loop state's D2H into mp.h_loop; nothing is synchronised
int map_queue_loop(lins_ctx* ctx, int nc, int ns, const float* T) {
  using namespace lins_map;
  lins_ctx::MapState& m = ctx->mp;
  // The whole iteration loop (:1640-1648) is queued up front: transformTobeMapped, matP / isDegenerate and the report live
  // on the device (MapLoopState); the first pass uses libm sin / cos of the caller's transform (bit-identical to the
  // reference's first pass), later ones the constants the LM kernel derived on the device.
  if (!m.loop.p) {  // isDegenerate / matP are members of the reference's mapping node (:226-227, :395-396): they survive the
    CK(m.loop.reserve(1));  // calls — a call whose first pass selects < 50 points keeps using the previous scan's values
    CK(cudaMemsetAsync(m.loop.p, 0, sizeof(MapLoopState), ctx->stream));
  }
  CK(m.h_loop.reserve(1)); CK(m.consts.reserve(1));
  const PassConsts pc0 = host_pass_consts(T);
  CK(cudaMemcpyAsync(m.loop.p, T, sizeof(float) * 6, cudaMemcpyHostToDevice, ctx->stream));  // (pageable sources: staged before the call returns)
  CK(cudaMemsetAsync(reinterpret_cast<char*>(m.loop.p) + offsetof(MapLoopState, done), 0, sizeof(MapLoopState) - offsetof(MapLoopState, done), ctx->stream));
  CK(cudaMemcpyAsync(m.consts.p, &pc0, sizeof(pc0), cudaMemcpyHostToDevice, ctx->stream));
  const bool grid = map_use_grid(true);
  for (int iter = 0; iter < LINS_MAP_MAX_ITER; ++iter) {
    int nblocks = 0;
    const int rc = map_queue_pass(ctx, nc, ns, false, grid, m.loop.p, &nblocks);
    if (rc != LINS_OK) return rc;
    lins_map_lm_kernel<<<1, 32, 0, ctx->stream>>>(m.partial.p, nblocks, iter, m.loop.p, m.consts.p, nullptr);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  CK(cudaMemcpyAsync(m.h_loop.p, m.loop.p, sizeof(MapLoopState), cudaMemcpyDeviceToHost, ctx->stream));
  return LINS_OK;
}

int map_queue_slots(lins_ctx* ctx, MappersState& ms, int n_slots) {
  using namespace lins_map;
  MapSlot* h = ms.h_mslot.p;
  // per slot: map_build_grid's bucket rule for each map, fit blocks that start with the slot's queries
  int nb_tot = 0, pts = 0, blocks[2] = {0, 0};
  std::vector<int> blk_slot[2];
  for (int s = 0; s < n_slots; ++s) {
    MapSlot& v = h[s];
    for (int k = 0; k < 2; ++k) {
      unsigned nb = v.run ? 4096 : 1;  // (a slot that does not run searches nothing)
      while (v.run && nb < 2u * (unsigned)v.cap[k] && nb < (1u << 24)) nb <<= 1;
      v.g[k].mask = nb - 1; v.g[k].ox = v.g[k].oy = v.g[k].oz = 0.f;  // (any finite origin gives the same 5-NN)
      v.bucket0[k] = nb_tot; nb_tot += (int)nb;
      v.m0[k] = pts; pts += v.cap[k];
      v.blk[k] = blocks[k];
      v.nblk[k] = v.run ? (v.nq[k] + kFitThreads - 1) / kFitThreads : 0;
      blocks[k] += v.nblk[k];
      blk_slot[k].insert(blk_slot[k].end(), v.nblk[k], s);
    }
  }
  size_t scan_bytes = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, ms.grid_count.p, ms.grid_start.p, nb_tot + 1, ctx->stream));
  CK(ms.scan_temp.grow(scan_bytes + 16));
  CK(ms.grid_start.grow((size_t)nb_tot + 2)); CK(ms.grid_count.grow((size_t)nb_tot + 2)); CK(ms.grid_cursor.grow((size_t)nb_tot + 2));
  CK(ms.grid_sorted.grow((size_t)pts + 1));
  const size_t rows = (size_t)std::max(blocks[0], blocks[1]) * kFitThreads;
  CK(ms.part_d.grow(5 * rows + 1)); CK(ms.part_i.grow(5 * rows + 1));
  CK(ms.partial.grow((size_t)(blocks[0] + blocks[1] + 1) * (kRowAcc + 1)));
  CK(ms.blk_slot.grow((size_t)blocks[0] + blocks[1] + 1)); CK(ms.h_blk_slot.grow((size_t)blocks[0] + blocks[1] + 1));
  CK(ms.consts.grow(n_slots)); CK(ms.h_consts.grow(n_slots)); CK(ms.mslot.grow(n_slots));
  for (int s = 0; s < n_slots; ++s) {
    for (int k = 0; k < 2; ++k) { h[s].g[k].pts = ms.grid_sorted.p; h[s].g[k].start = ms.grid_start.p + h[s].bucket0[k]; }
    ms.h_consts.p[s] = host_pass_consts(h[s].T);
  }
  std::copy(blk_slot[0].begin(), blk_slot[0].end(), ms.h_blk_slot.p);
  std::copy(blk_slot[1].begin(), blk_slot[1].end(), ms.h_blk_slot.p + blocks[0]);
  CK(cudaMemcpyAsync(ms.mslot.p, h, sizeof(MapSlot) * n_slots, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ms.consts.p, ms.h_consts.p, sizeof(PassConsts) * n_slots, cudaMemcpyHostToDevice, ctx->stream));
  if (blocks[0] + blocks[1])
    CK(cudaMemcpyAsync(ms.blk_slot.p, ms.h_blk_slot.p, sizeof(int) * (blocks[0] + blocks[1]), cudaMemcpyHostToDevice, ctx->stream));
  // every slot's two grids: one count, one scan of all buckets, one scatter
  CK(cudaMemsetAsync(ms.grid_count.p, 0, sizeof(int) * ((size_t)nb_tot + 1), ctx->stream));
  const GridIndex g0{};
  if (pts) lins_grid_count_kernel<<<(pts + 255) / 256, 256, 0, ctx->stream>>>(nullptr, pts, g0, ms.grid_count.p, ms.mslot.p, n_slots);
  size_t bytes = ms.scan_temp.cap;
  CK(cub::DeviceScan::ExclusiveSum(ms.scan_temp.p, bytes, ms.grid_count.p, ms.grid_start.p, nb_tot + 1, ctx->stream));
  CK(cudaMemcpyAsync(ms.grid_cursor.p, ms.grid_start.p, sizeof(int) * nb_tot, cudaMemcpyDeviceToDevice, ctx->stream));
  if (pts) lins_grid_scatter_kernel<<<(pts + 255) / 256, 256, 0, ctx->stream>>>(nullptr, pts, g0, ms.grid_cursor.p, ms.grid_sorted.p, ms.mslot.p, n_slots);
  lins_map_gate_kernel<<<(n_slots + 127) / 128, 128, 0, ctx->stream>>>(ms.loop.p, ms.mslot.p, n_slots);
  CK(cudaGetLastError());
  ctx->launches += pts ? 4 : 2;
  // the loop: per pass one 5-NN and one fit launch per kind over every slot, one LM launch of a warp per slot
  double* partial_s = ms.partial.p + (size_t)blocks[0] * (kRowAcc + 1);
  for (int iter = 0; iter < LINS_MAP_MAX_ITER; ++iter) {
    if (blocks[0]) {
      lins_map_knn_grid_kernel<<<blocks[0] * kFitThreads / kGridKnnWarps, kGridKnnWarps * 32, 0, ctx->stream>>>(
          nullptr, blocks[0] * kFitThreads, g0, ms.consts.p, ms.loop.p, ms.part_d.p, ms.part_i.p, ms.mslot.p, ms.blk_slot.p, 0);
      lins_map_fit_kernel<true><<<blocks[0], kFitThreads, 0, ctx->stream>>>(nullptr, 0, nullptr, 1, ms.part_d.p, ms.part_i.p, ms.consts.p, ms.loop.p,
                                                                            nullptr, nullptr, nullptr, ms.partial.p, ms.mslot.p, ms.blk_slot.p);
      ctx->launches += 2;
    }
    if (blocks[1]) {
      lins_map_knn_grid_kernel<<<blocks[1] * kFitThreads / kGridKnnWarps, kGridKnnWarps * 32, 0, ctx->stream>>>(
          nullptr, blocks[1] * kFitThreads, g0, ms.consts.p, ms.loop.p, ms.part_d.p, ms.part_i.p, ms.mslot.p, ms.blk_slot.p + blocks[0], 1);
      lins_map_fit_kernel<false><<<blocks[1], kFitThreads, 0, ctx->stream>>>(nullptr, 0, nullptr, 1, ms.part_d.p, ms.part_i.p, ms.consts.p, ms.loop.p,
                                                                             nullptr, nullptr, nullptr, partial_s, ms.mslot.p, ms.blk_slot.p + blocks[0]);
      ctx->launches += 2;
    }
    lins_map_lm_kernel<<<n_slots, 32, 0, ctx->stream>>>(ms.partial.p, blocks[0], iter, ms.loop.p, ms.consts.p, ms.mslot.p);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  CK(cudaMemcpyAsync(ms.h_loop.p, ms.loop.p, sizeof(MapLoopState) * n_slots, cudaMemcpyDeviceToHost, ctx->stream));
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

extern "C" {

int lins_gpu_map_set(lins_ctx* ctx, const lins_point* corner, int nc, const lins_point* surf, int ns) {
  if (!ctx) return LINS_E_INVALID;
  if (check_cloud(ctx, corner, nc, "bad corner map cloud") != LINS_OK || check_cloud(ctx, surf, ns, "bad surf map cloud") != LINS_OK)
    return LINS_E_INVALID;
  CK(cudaSetDevice(ctx->device));
  int rc = upload2(ctx, ctx->mp.map_c, corner, nc, ctx->mp.map_s, surf, ns);
  if (rc != LINS_OK) return rc;
  ctx->mp.n_map_c = nc; ctx->mp.n_map_s = ns;
  float oc[3], os[3];
  map_grid_origin(corner, nc, oc);
  map_grid_origin(surf, ns, os);
  rc = map_build_grid(ctx, ctx->mp.grid_c, ctx->mp.map_c.p, nc, oc);
  if (rc != LINS_OK) return rc;
  return map_build_grid(ctx, ctx->mp.grid_s, ctx->mp.map_s.p, ns, os);
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
  int rc = map_stage_queries(ctx, corner, nc, surf, ns);
  if (rc != LINS_OK) return rc;
  rc = map_queue_loop(ctx, nc, ns, T);
  if (rc != LINS_OK) return rc;
  CK(cudaStreamSynchronize(ctx->stream));
  map_loop_report(*m.h_loop.p, T, &r);
  if (rep) *rep = r;
  return LINS_OK;
}

int lins_gpu_map_associate(lins_ctx* ctx, const lins_point* corner, int nc, const lins_point* surf, int ns, const float* T,
                           int32_t* cknn, int32_t* sknn, float* ccoeff, float* scoeff, uint8_t* cmask, uint8_t* smask) {
  if (!ctx) return LINS_E_INVALID;
  if (!T) return fail(ctx, LINS_E_INVALID, "null transform");
  CK(cudaSetDevice(ctx->device));
  int rc = map_stage_queries(ctx, corner, nc, surf, ns);
  if (rc != LINS_OK) return rc;
  lins_ctx::MapState& m = ctx->mp;
  CK(m.consts.reserve(1));
  const lins_map::PassConsts pc = host_pass_consts(T);
  CK(cudaMemcpyAsync(m.consts.p, &pc, sizeof(pc), cudaMemcpyHostToDevice, ctx->stream));
  int nblocks = 0;
  // the parity hook: brute force by default (exact neighbours for EVERY point, also those the 1 m gate rejects)
  rc = map_queue_pass(ctx, nc, ns, true, map_use_grid(false), nullptr, &nblocks);
  if (rc != LINS_OK) return rc;
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
