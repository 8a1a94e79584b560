// lins_mappers.cu — the mapping node's cycle for many drives in lockstep (lins_gpu_mappers_*) and for one
// (lins_gpu_mapper_*, a run of one slot of its own): one MapperNode per slot, each stepped by the host logic of
// lins_mapper.cu, with one queue of device work per step for every processed slot.
//
// Per step (one synchronisation): the scans of the processed slots in one H2D (or, from device clouds, in the gather
// launch that follows: sequence mode's publish step, lins_seq.cu); one gather launch of every slot's window
// into its local-map clouds; one segmented VoxelGrid over the five clouds of every slot (map corner 0.2 m, map surf
// 0.4 m, corner 0.2 m, surf 0.4 m, outlier 0.4 m), one gather of each slot's surf DS + outlier DS and one segmented
// VoxelGrid of those (0.4 m); every slot's grids and scan-to-map loop (lins_map.cu, grid origin 0); the read-back of
// the VoxelGrid records and loop states.  After it, the host tail of each slot and one transform launch for every key
// frame saved (and, on a slot with loop closure, for its body-frame clouds into the host store and, after correctPoses,
// for its device store re-transformed from the host store).
//
// The host store (DESIGN.md §4.14) is the run's arena of pinned, mapped memory (lins_kf_arena.hpp).  Device work reads
// and writes it only on the context's stream, and host code touches a chunk only where the stream is idle: a save
// reads it after its synchronisation, a load writes it after a synchronisation at its start, and open and destroy free
// the slabs after one.  A reset hands its chunks back without touching them; the next writer of a chunk is a later
// kernel on the stream or a load.  The VoxelGrids' outputs are sized by their inputs and padded with NaN, and the later launches take those
// capacities.  The segments of a VoxelGrid keep their input ranges and each slot's fit blocks cover its own queries
// only, so every slot's clouds, sums and steps are those of a run of one slot.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include "lins_ctx.hpp"
#include "lins_map_types.cuh"

using namespace lins_capi;

namespace {

int need_open(lins_ctx* ctx) {
  return ctx->mappers.n > 0 ? LINS_OK : fail(ctx, LINS_E_NOMAP, "lins_gpu_mappers_open has not been called");
}

// the odometry fields of a lockstep descriptor, as lins_gpu_mappers_step and _fuse check them
int check_odometry(lins_ctx* ctx, const lins_mappers_desc* d) {
  if (!ctx) return LINS_E_INVALID;
  if (!d) return fail(ctx, LINS_E_INVALID, "null desc");
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  if (d->n_slots != ctx->mappers.n) return fail(ctx, LINS_E_INVALID, "n_slots differs from the open run's");
  if (!d->time || !d->quat || !d->pos) return fail(ctx, LINS_E_INVALID, "null time / quat / pos");
  return LINS_OK;
}

const char* const kBad = "VoxelGrid: the leaf is too small for the cloud's extent (div_x * div_y * div_z > INT32_MAX)";

}  // namespace

namespace lins_capi {

// the host store's slabs: pinned and mapped, at one address for the host and the device (UVA; anything else fails)
lins_arena::Allocator pinned_mapped_allocator() {
  auto alloc = [](size_t bytes, void*) -> void* {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocMapped) != cudaSuccess) return nullptr;
    void* d = nullptr;
    if (cudaHostGetDevicePointer(&d, p, 0) != cudaSuccess || d != p) { cudaFreeHost(p); return nullptr; }
    return p;
  };
  auto release = [](void* p, void*) { cudaFreeHost(p); };
  return lins_arena::Allocator{alloc, release, nullptr};
}

// n_slots fresh mapping nodes in ms, replacing any open run
int mappers_open(lins_ctx* ctx, MappersState& ms, int n_slots) {
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));  // (queued work may still write the host stores' slabs)
  ms.n = 0;
  ms.node = std::vector<MapperNode>(n_slots);  // (constructed in place: a node is not copyable)
  ms.store.release();
  ms.ds = std::vector<std::array<Buf<float4>, 6>>(n_slots);
  CK(ms.stm.loop.reserve(n_slots)); CK(ms.stm.h_loop.reserve(n_slots)); CK(ms.stm.h_mslot.reserve(n_slots));
  CK(cudaMemsetAsync(ms.stm.loop.p, 0, sizeof(lins_map::MapLoopState) * n_slots, ctx->stream));  // matP, isDegenerate
  ms.n = n_slots;
  return LINS_OK;
}

// the slots with mask[s] != 0 back to the fresh state
int mappers_reset(lins_ctx* ctx, MappersState& ms, const uint8_t* mask) {
  CK(cudaSetDevice(ctx->device));
  for (int s = 0; s < ms.n; ++s)
    if (mask[s]) {
      mapper_node_reset(ms.node[s], ms.store);
      CK(cudaMemsetAsync(ms.stm.loop.p + s, 0, sizeof(lins_map::MapLoopState), ctx->stream));
    }
  return LINS_OK;
}

}  // namespace lins_capi

namespace {

// imuHandler for every slot: slot s's rows are [off[s], off[s + 1])
void mappers_imu(MappersState& ms, const int32_t* off, const double* time, const double* roll, const double* pitch) {
  for (int s = 0; s < ms.n; ++s) mapper_node_imu(ms.node[s].s, time + off[s], roll + off[s], pitch + off[s], off[s + 1] - off[s]);
}

}  // namespace

namespace lins_capi {

// one step of every present slot of ms on a checked descriptor (d->n_slots == ms.n, valid offsets and arrays).  dev
// (M x 3: corner, surf, outlier, or null): the slots' clouds are device ranges in XYZ order, copied YZX-permuted into the
// VoxelGrids' input by the local maps' gather launch; d's clouds are then not read.
int mappers_step(lins_ctx* ctx, MappersState& ms, const lins_mappers_desc* d, lins_mapper_report* reps, const MapPiece* dev,
                 const double* period) {
  const int M = ms.n;
  const lins_point* src[3] = {d->corner, d->surf, d->outlier};
  const int32_t* off[3] = {d->corner_off, d->surf_off, d->outlier_off};
  auto count = [&](int k, int s) { return dev ? dev[3 * s + k].len : off[k][s + 1] - off[k][s]; };
  CK(cudaSetDevice(ctx->device));

  // the host head of every present slot's cycle, on copies of its scalars (committed after the read-back)
  std::vector<MapperScalars> sc(M);
  std::vector<lins_mapper_report> rr(M);
  std::vector<int> proc, skipped;  // processed slots; interval-skipped slots
  for (int s = 0; s < M; ++s) {
    if (d->present && !d->present[s]) continue;
    ms.node[s].stepped = true;
    sc[s] = ms.node[s].s;
    (mapper_cycle_begin(ms.node[s], sc[s], d->time[s], d->quat + 4 * s, d->pos + 3 * s, rr[s]) ? proc : skipped).push_back(s);
  }
  const int P = (int)proc.size();
  auto finish = [&]() {
    for (int s : skipped) ms.node[s].s = sc[s];
    for (int s = 0; s < M; ++s)  // timeLaserOdometry, which a skipped cycle's odometry replaces too
      if ((!d->present || d->present[s]) && ms.node[s].loops.enabled) ms.node[s].loops.time = d->time[s];
    if (reps) for (int s = 0; s < M; ++s) if (!d->present || d->present[s]) reps[s] = rr[s];
    return LINS_OK;
  };
  if (P == 0) return finish();

  // round 1: segment 3p + k = scan cloud k of processed slot p (one H2D, or gathered), 3P + 2p + k = its local map k; round 2:
  // segment p = its surf DS + outlier DS.  Every capacity is known here: the outputs are sized by the inputs.
  std::vector<int> h_off1(5 * P + 1), h_off2(P + 1), mapc(2 * P);
  std::vector<float> leaf1(5 * P), leaf2(P, 0.4f);
  std::vector<float4*> out(6 * P);
  int n_scan = 0;
  for (int p = 0; p < P; ++p) {
    const int s = proc[p];
    for (int k = 0; k < 3; ++k) { h_off1[3 * p + k] = n_scan; n_scan += count(k, s); leaf1[3 * p + k] = k == 0 ? 0.2f : 0.4f; }
    int nc = 0, nsf = 0;
    if (!ms.node[s].poses.empty()) mapper_window_sizes(ms.node[s], sc[s], nc, nsf);
    mapc[2 * p] = nc; mapc[2 * p + 1] = nsf;
  }
  int n1 = n_scan;
  for (int p = 0; p < P; ++p)
    for (int k = 0; k < 2; ++k) { h_off1[3 * P + 2 * p + k] = n1; n1 += mapc[2 * p + k]; leaf1[3 * P + 2 * p + k] = k == 0 ? 0.2f : 0.4f; }
  h_off1[5 * P] = n1;
  int n2 = 0;
  for (int p = 0; p < P; ++p) { h_off2[p] = n2; n2 += (h_off1[3 * p + 3] - h_off1[3 * p + 1]); }
  h_off2[P] = n2;

  // every buffer of the step first (a growth frees memory queued work may still read)
  int rc;
  if ((rc = voxel_grid_reserve(ctx, ms.vg, std::max(n1, n2), 5 * P)) != LINS_OK) return rc;
  if ((rc = voxel_grid_reserve(ctx, ms.vg, std::max(n1, n2), P)) != LINS_OK) return rc;
  CK(ms.vin[0].grow((size_t)n1 + 1)); CK(ms.vin[1].grow((size_t)n2 + 1)); if (!dev) CK(ms.h_in.grow((size_t)n_scan + 1));
  CK(ms.vg_info.reserve(6 * (size_t)P)); CK(ms.h_vg_info.reserve(6 * (size_t)P)); CK(ms.h_vg_init.reserve(6 * (size_t)P));
  CK(ms.vg_off.reserve(6 * (size_t)P + 2)); CK(ms.h_vg_off.reserve(6 * (size_t)P + 2));
  CK(ms.vg_out.reserve(6 * (size_t)P)); CK(ms.h_vg_out.reserve(6 * (size_t)P));
  size_t n_copies = (dev ? 5 : 2) * (size_t)P;
  for (int p = 0; p < P; ++p) {
    const int s = proc[p];
    auto& ds = ms.ds[s];
    const int cap[6] = {mapc[2 * p], mapc[2 * p + 1], h_off1[3 * p + 1] - h_off1[3 * p], h_off1[3 * p + 2] - h_off1[3 * p + 1],
                        h_off1[3 * p + 3] - h_off1[3 * p + 2], h_off2[p + 1] - h_off2[p]};
    for (int k = 0; k < 6; ++k) CK(ds[k].grow((size_t)cap[k] + 1));
    out[3 * p + 0] = ds[2].p; out[3 * p + 1] = ds[3].p; out[3 * p + 2] = ds[4].p;
    out[3 * P + 2 * p] = ds[0].p; out[3 * P + 2 * p + 1] = ds[1].p;
    out[5 * P + p] = ds[5].p;
    if (!ms.node[s].poses.empty()) n_copies += 3 * sc[s].window.size();
  }
  if ((rc = ms.copies.reserve(ctx, n_copies)) != LINS_OK) return rc;

  // the scans (one H2D; device clouds join the gather below) and the segment tables (outputs: the slots' own DS clouds,
  // which persist for the download)
  std::vector<DevCopy> copies;
  if (dev) {
    for (int p = 0; p < P; ++p)
      for (int k = 0; k < 3; ++k) {
        const MapPiece& c = dev[3 * proc[p] + k];
        copies.push_back(DevCopy{c.src, ms.vin[0].p + h_off1[3 * p + k], c.len, 1});
      }
  } else {
    size_t o = 0;
    for (int p = 0; p < P; ++p)
      for (int k = 0; k < 3; ++k) {
        const int s = proc[p], n = off[k][s + 1] - off[k][s];
        pack_into(ms.h_in.p + o, src[k] + off[k][s], n);
        o += n;
      }
    if (n_scan) CK(cudaMemcpyAsync(ms.vin[0].p, ms.h_in.p, sizeof(float4) * n_scan, cudaMemcpyHostToDevice, ctx->stream));
  }
  std::copy(h_off1.begin(), h_off1.end(), ms.h_vg_off.p);
  std::copy(h_off2.begin(), h_off2.end(), ms.h_vg_off.p + 5 * P + 1);
  std::copy(out.begin(), out.end(), ms.h_vg_out.p);
  CK(cudaMemcpyAsync(ms.vg_off.p, ms.h_vg_off.p, sizeof(int) * (6 * (size_t)P + 2), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ms.vg_out.p, ms.h_vg_out.p, sizeof(float4*) * 6 * (size_t)P, cudaMemcpyHostToDevice, ctx->stream));

  // every slot's local map: corner_i ..., and surf_i, outlier_i interleaved (:1242-1246), one gather launch
  for (int p = 0; p < P; ++p) {
    const MapperNode& m = ms.node[proc[p]];
    if (m.poses.empty()) continue;
    float4* oc = ms.vin[0].p + h_off1[3 * P + 2 * p];
    float4* os = ms.vin[0].p + h_off1[3 * P + 2 * p + 1];
    for (int id : sc[proc[p]].window) {
      const MapperKeyFrame& kf = m.slots[m.slot_of.at(id)];
      copies.push_back(DevCopy{kf.c[0].p, oc, kf.n[0], 0}); oc += kf.n[0];
      copies.push_back(DevCopy{kf.c[1].p, os, kf.n[1], 0}); os += kf.n[1];
      copies.push_back(DevCopy{kf.c[2].p, os, kf.n[2], 0}); os += kf.n[2];
    }
  }
  if ((rc = queue_copies(ctx, ms.copies, copies, 0)) != LINS_OK) return rc;
  VgInfo* info = ms.vg_info.p;
  if ((rc = voxel_grid_queue(ctx, ms.vg, ms.vin[0].p, 5 * P, h_off1.data(), ms.vg_off.p, leaf1.data(), nullptr, ms.vg_out.p, ms.h_vg_init.p,
                             info)) != LINS_OK)
    return rc;
  // laserCloudSurfTotalLast = surf DS + outlier DS: their NaN tails ride along and are dropped by the filter
  copies.clear();
  for (int p = 0; p < P; ++p) {
    const int s = proc[p], ns = h_off1[3 * p + 2] - h_off1[3 * p + 1], no = h_off1[3 * p + 3] - h_off1[3 * p + 2];
    copies.push_back(DevCopy{ms.ds[s][3].p, ms.vin[1].p + h_off2[p], ns, 0});
    copies.push_back(DevCopy{ms.ds[s][4].p, ms.vin[1].p + h_off2[p] + ns, no, 0});
  }
  if ((rc = queue_copies(ctx, ms.copies, copies, (int)(n_copies - 2 * P))) != LINS_OK) return rc;
  if ((rc = voxel_grid_queue(ctx, ms.vg, ms.vin[1].p, P, h_off2.data(), ms.vg_off.p + 5 * P + 1, leaf2.data(), out[5 * P],
                             ms.vg_out.p + 5 * P, ms.h_vg_init.p + 5 * P, info + 5 * P)) != LINS_OK)
    return rc;

  // scan2MapOptimization of every slot with key frames (a slot without runs no pass, like the single mapper's host gate);
  // every grid's origin is 0 (any finite origin gives the same 5-NN)
  bool any_map = false;
  for (int s = 0; s < M; ++s) std::memset(&ms.stm.h_mslot.p[s], 0, sizeof(lins_map::MapSlot));
  for (int p = 0; p < P; ++p) {
    const int s = proc[p];
    if (ms.node[s].poses.empty()) continue;
    lins_map::MapSlot& v = ms.stm.h_mslot.p[s];
    v.run = 1; any_map = true;
    for (int k = 0; k < 2; ++k) { v.map[k] = ms.ds[s][k].p; v.cap[k] = mapc[2 * p + k]; v.n_map[k] = &info[3 * P + 2 * p + k].count; }
    v.q[0] = ms.ds[s][2].p; v.nq[0] = h_off1[3 * p + 1] - h_off1[3 * p];
    v.q[1] = ms.ds[s][5].p; v.nq[1] = h_off2[p + 1] - h_off2[p];
    for (int i = 0; i < 6; ++i) v.T[i] = sc[s].transformTobeMapped[i];
  }
  if (any_map && ((rc = map_fill_table(ctx, ms.stm, M)) != LINS_OK || (rc = map_queue_grids(ctx, ms.stm)) != LINS_OK ||
                  (rc = map_queue_loop(ctx, ms.stm)) != LINS_OK))
    return rc;
  CK(cudaMemcpyAsync(ms.h_vg_info.p, info, sizeof(VgInfo) * 6 * (size_t)P, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));  // the step's one read-back
  for (int s : proc) ms.node[s].last.valid = false;  // (a failed step has overwritten their previous clouds)
  const VgInfo* hi = ms.h_vg_info.p;
  for (int i = 0; i < 6 * P; ++i)
    if (hi[i].toobig) return fail(ctx, LINS_E_TOOBIG, kBad);

  // the host tail of every processed slot, then one transform launch for the key frames saved
  std::vector<KfSave> saves;
  for (int p = 0; p < P; ++p) {
    const int s = proc[p];
    const bool have_map = !ms.node[s].poses.empty();
    const int cnt[6] = {have_map ? hi[3 * P + 2 * p].count : 0, have_map ? hi[3 * P + 2 * p + 1].count : 0, hi[3 * p].count, hi[3 * p + 1].count,
                        hi[3 * p + 2].count, hi[5 * P + p].count};
    const bool gate = cnt[0] > 10 && cnt[1] > 100;
    KfSave sv{};
    bool saved = false;
    mapper_cycle_end(ms.node[s], sc[s], d->time[s], period ? period[s] : ctx->prm.scan_period, cnt, gate ? &ms.stm.h_loop.p[s] : nullptr, rr[s], &sv, &saved);
    MapperNode& m = ms.node[s];
    if (saved) {
      for (int k = 0; k < 3; ++k) sv.ds[k] = ms.ds[s][2 + k].p;
      sv.kp = m.poses.back();  // (correctPoses may have moved it)
      sv.body = nullptr;
      if (m.loops.enabled) {  // its block of the host store, by id (ids are saved in order)
        HostKeyFrame h;
        std::copy(sv.kf->n, sv.kf->n + 3, h.n);
        void* p = nullptr;
        if (!ms.store.take(m.held, sizeof(float4) * ((size_t)h.n[0] + h.n[1] + h.n[2]), &p)) {
          ms.n = 0;  // (this slot and the ones before it have committed their cycles: the run ends, as after a failed load)
          return fail(ctx, LINS_E_CUDA, "the host key-frame store could not allocate pinned memory (the run has ended)");
        }
        h.p = static_cast<float4*>(p);
        m.host.push_back(h);
        sv.body = h.p;
      }
      saves.push_back(sv);
    }
    if (m.loops.rebuild)  // correctPoses: every other key frame of the device store re-transformed from the host store
      for (const auto& kv : m.slot_of) {
        if (saved && kv.first == (int)m.poses.size() - 1) continue;
        MapperKeyFrame& f = m.slots[kv.second];
        const HostKeyFrame& h = m.host[kv.first];
        saves.push_back(KfSave{&f, m.poses[kv.first], {h.p, h.p + h.n[0], h.p + h.n[0] + h.n[1]}, nullptr});
      }
  }
  if ((rc = keyframes_queue(ctx, saves.data(), (int)saves.size(), ms.tf, ms.h_tf)) != LINS_OK) {
    ms.n = 0;  // (the slots' cycles are committed, their key frames not stored: the run ends)
    return rc;
  }
  return finish();
}

}  // namespace lins_capi

namespace {

// the key poses, window and last cycle's clouds of one slot (dst: NULL skips)
int mappers_download(lins_ctx* ctx, MappersState& ms, int slot, double* key_poses, int32_t* window, float* const dst[6]) {
  CK(cudaSetDevice(ctx->device));
  const float4* src[6];
  for (int k = 0; k < 6; ++k) src[k] = ms.ds[slot][k].p;
  return mapper_node_download(ctx, ms.node[slot], src, key_poses, window, dst);
}

// loop closure on the masked slots, all fresh (checked first: all or nothing).  On a run bound by lins_gpu_seq_map_open
// a slot is fresh as lins_gpu_seq_configure / _tune judge it: no sequence step since open or its last restart.
int mappers_loops(lins_ctx* ctx, MappersState& ms, const uint8_t* mask) {
  const bool bound = &ms == &ctx->mappers && ctx->seq.pub.bound;
  for (int s = 0; s < ms.n; ++s)
    if (mask[s] && !ms.node[s].loops.enabled && (ms.node[s].stepped || (bound && !ctx->seq.slot[s].fresh)))
      return fail(ctx, LINS_E_INVALID, "loop closure: a masked slot is not fresh (present in a step since open / reset)");
  for (int s = 0; s < ms.n; ++s) if (mask[s]) ms.node[s].loops.enabled = true;
  return LINS_OK;
}

// the bytes of the masked slots' key-frame stores (host bookkeeping only)
int store_bytes(lins_ctx* ctx, const MappersState& ms, const uint8_t* mask, uint64_t* device, uint64_t* host, uint64_t* host_reserved) {
  if (!mask || !device || !host) return fail(ctx, LINS_E_INVALID, "null mask / device / host");
  for (int s = 0; s < ms.n; ++s) {
    if (!mask[s]) continue;
    const MapperNode& m = ms.node[s];
    uint64_t d = 0, h = 0;
    for (const auto& kv : m.slot_of)
      for (int a = 0; a < 3; ++a) d += (uint64_t)m.slots[kv.second].n[a];
    for (const HostKeyFrame& k : m.host)
      for (int a = 0; a < 3; ++a) h += (uint64_t)k.n[a];
    device[s] = sizeof(float4) * d;
    host[s] = sizeof(float4) * h;
  }
  if (host_reserved) *host_reserved = ms.store.reserved();
  return LINS_OK;
}

// a node's last global map: its key ids and cloud (NULL skips)
int global_map_download(lins_ctx* ctx, const MapperNode& m, int32_t* key_ids, float* cloud) {
  const MapperGlobalMap& g = m.gm;
  if (!g.valid) return fail(ctx, LINS_E_NOMAP, "no global map since the slot's open / reset");
  CK(cudaSetDevice(ctx->device));
  if (key_ids) std::copy(g.keys.begin(), g.keys.end(), key_ids);
  CK(d2h(ctx, cloud, g.cloud.p, sizeof(float4) * (size_t)g.rep.n_map));
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}

// the single mapper: a run of one slot of its own, opened by the first lins_gpu_mapper_* call on the context
int mapper_open(lins_ctx* ctx) {
  return ctx->mapper.n > 0 ? LINS_OK : mappers_open(ctx, ctx->mapper, 1);
}

}  // namespace

extern "C" {

int lins_gpu_mappers_open(lins_ctx* ctx, int32_t n_slots) {
  if (!ctx) return LINS_E_INVALID;
  if (n_slots < 1) return fail(ctx, LINS_E_INVALID, "n_slots < 1");
  ctx->seq.pub.bound = false;  // (a sequence run's mapping nodes are replaced)
  return mappers_open(ctx, ctx->mappers, n_slots);
}

int lins_gpu_mappers_reset(lins_ctx* ctx, const uint8_t* mask) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  return mappers_reset(ctx, ctx->mappers, mask);
}

int lins_gpu_mappers_imu(lins_ctx* ctx, const int32_t* off, const double* time, const double* roll, const double* pitch) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  MappersState& ms = ctx->mappers;
  if (check_csr(ctx, off, ms.n, time, "bad IMU offsets / arrays") != LINS_OK) return LINS_E_INVALID;
  if (off[ms.n] > 0 && (!roll || !pitch)) return fail(ctx, LINS_E_INVALID, "bad IMU offsets / arrays");
  mappers_imu(ms, off, time, roll, pitch);
  return LINS_OK;
}

int lins_gpu_mappers_step(lins_ctx* ctx, const lins_mappers_desc* d, lins_mapper_report* reps) {
  const int rc = check_odometry(ctx, d);
  if (rc != LINS_OK) return rc;
  const int M = ctx->mappers.n;
  const lins_point* src[3] = {d->corner, d->surf, d->outlier};
  const int32_t* off[3] = {d->corner_off, d->surf_off, d->outlier_off};
  static const char* const what[3] = {"bad corner offsets / cloud", "bad surf offsets / cloud", "bad outlier offsets / cloud"};
  for (int k = 0; k < 3; ++k) if (check_csr(ctx, off[k], M, src[k], what[k]) != LINS_OK) return LINS_E_INVALID;
  return mappers_step(ctx, ctx->mappers, d, reps, nullptr, nullptr);
}

int lins_gpu_mappers_fuse(lins_ctx* ctx, const lins_mappers_desc* d, lins_fused_pose* out) {
  const int rc = check_odometry(ctx, d);
  if (rc != LINS_OK) return rc;
  if (!out) return fail(ctx, LINS_E_INVALID, "null out");
  const MappersState& ms = ctx->mappers;
  for (int s = 0; s < ms.n; ++s) {
    if (d->present && !d->present[s]) { std::memset(&out[s], 0, sizeof(out[s])); continue; }
    mapper_node_fuse(ms.node[s], d->time[s], d->quat + 4 * s, d->pos + 3 * s, out[s]);
  }
  return LINS_OK;
}

int lins_gpu_mappers_download(lins_ctx* ctx, int32_t slot, double* key_poses, int32_t* window, float* map_corner_ds, float* map_surf_ds,
                              float* corner_ds, float* surf_ds, float* outlier_ds, float* surf_total_ds) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  if (slot < 0 || slot >= ctx->mappers.n) return fail(ctx, LINS_E_INVALID, "slot out of range");
  float* const dst[6] = {map_corner_ds, map_surf_ds, corner_ds, surf_ds, outlier_ds, surf_total_ds};
  return mappers_download(ctx, ctx->mappers, slot, key_poses, window, dst);
}

int lins_gpu_mappers_loops(lins_ctx* ctx, const uint8_t* mask) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  return mappers_loops(ctx, ctx->mappers, mask);
}

int lins_gpu_mappers_close_loops(lins_ctx* ctx, const uint8_t* mask, lins_loop_report* reps) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  return mappers_close_loops(ctx, ctx->mappers, mask, reps);
}

int lins_gpu_mappers_global_map(lins_ctx* ctx, const uint8_t* mask, lins_global_map_report* reps) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  return mappers_global_map(ctx, ctx->mappers, mask, reps);
}

int lins_gpu_mappers_global_map_download(lins_ctx* ctx, int32_t slot, int32_t* key_ids, float* cloud) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  if (slot < 0 || slot >= ctx->mappers.n) return fail(ctx, LINS_E_INVALID, "slot out of range");
  return global_map_download(ctx, ctx->mappers.node[slot], key_ids, cloud);
}

int lins_gpu_mappers_store_bytes(lins_ctx* ctx, const uint8_t* mask, uint64_t* device, uint64_t* host, uint64_t* host_reserved) {
  if (!ctx) return LINS_E_INVALID;
  if (need_open(ctx) != LINS_OK) return LINS_E_NOMAP;
  return store_bytes(ctx, ctx->mappers, mask, device, host, host_reserved);
}

int lins_gpu_mapper_store_bytes(lins_ctx* ctx, uint64_t* device, uint64_t* host, uint64_t* host_reserved) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  return store_bytes(ctx, ctx->mapper, &all, device, host, host_reserved);
}

int lins_gpu_mapper_global_map(lins_ctx* ctx, lins_global_map_report* rep) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  return mappers_global_map(ctx, ctx->mapper, &all, rep);
}

int lins_gpu_mapper_global_map_download(lins_ctx* ctx, int32_t* key_ids, float* cloud) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  return global_map_download(ctx, ctx->mapper.node[0], key_ids, cloud);
}

int lins_gpu_mapper_loops(lins_ctx* ctx) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  return mappers_loops(ctx, ctx->mapper, &all);
}

int lins_gpu_mapper_close_loop(lins_ctx* ctx, lins_loop_report* rep) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  return mappers_close_loops(ctx, ctx->mapper, &all, rep);
}

int lins_gpu_mapper_reset(lins_ctx* ctx) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  return mappers_reset(ctx, ctx->mapper, &all);
}

int lins_gpu_mapper_imu(lins_ctx* ctx, const double* time, const double* roll, const double* pitch, int n) {
  if (!ctx) return LINS_E_INVALID;
  if (n < 0 || (n > 0 && (!time || !roll || !pitch))) return fail(ctx, LINS_E_INVALID, "bad IMU arrays");
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const int32_t off[2] = {0, n};
  mappers_imu(ctx->mapper, off, time, roll, pitch);
  return LINS_OK;
}

int lins_gpu_mapper_step(lins_ctx* ctx, const lins_mapper_desc* d, lins_mapper_report* rep) {
  if (!ctx) return LINS_E_INVALID;
  if (!d) return fail(ctx, LINS_E_INVALID, "null desc");
  if (check_cloud(ctx, d->corner, d->n_corner, "bad mapper corner cloud") != LINS_OK || check_cloud(ctx, d->surf, d->n_surf, "bad mapper surf cloud") != LINS_OK ||
      check_cloud(ctx, d->outlier, d->n_outlier, "bad mapper outlier cloud") != LINS_OK)
    return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const int32_t off[3][2] = {{0, d->n_corner}, {0, d->n_surf}, {0, d->n_outlier}};
  lins_mappers_desc one = {};
  one.n_slots = 1;
  one.time = &d->time; one.quat = d->quat; one.pos = d->pos;
  one.corner = d->corner; one.corner_off = off[0];
  one.surf = d->surf; one.surf_off = off[1];
  one.outlier = d->outlier; one.outlier_off = off[2];
  return mappers_step(ctx, ctx->mapper, &one, rep, nullptr, nullptr);
}

int lins_gpu_mapper_fuse(lins_ctx* ctx, const lins_mapper_desc* d, lins_fused_pose* out) {
  if (!ctx) return LINS_E_INVALID;
  if (!d || !out) return fail(ctx, LINS_E_INVALID, "null desc / out");
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  mapper_node_fuse(ctx->mapper.node[0], d->time, d->quat, d->pos, *out);
  return LINS_OK;
}

int lins_gpu_mapper_download(lins_ctx* ctx, double* key_poses, int32_t* window, float* map_corner_ds, float* map_surf_ds,
                             float* corner_ds, float* surf_ds, float* outlier_ds, float* surf_total_ds) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  float* const dst[6] = {map_corner_ds, map_surf_ds, corner_ds, surf_ds, outlier_ds, surf_total_ds};
  return mappers_download(ctx, ctx->mapper, 0, key_poses, window, dst);
}

}  // extern "C"
