// lins_seq_save.cu — sequence-mode slots saved to host bytes and loaded into fresh slots (include/lins_gpu.h:
// lins_gpu_seq_save_size, lins_gpu_seq_save, lins_gpu_seq_load).  A slot's blob (lins_slot_blob.hpp) carries what a
// later step, publish or download of the slot reads: its device rows, maps, stale 1-NN cloud and published outlier
// cloud, its mapping node's scalars, key poses, window, stored key frames and scan-to-map loop state, and its host
// bookkeeping.  No kernel of its own: the device side is the gather list every other data movement here uses.
//   save: one gather launch of every masked slot's device pieces into one staging buffer laid out as the caller's
//         buffer, one D2H into pinned staging, one synchronisation; the host records are written after it.
//   load: every masked blob validated in full first; then one H2D of them, and one gather launch that installs their rows
//         and loop states, fills the key frames' buffers and builds the next map and outlier generations (the restart
//         path's compaction, with the loaded slots' pieces in the staging).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <utility>
#include <vector>

#include "lins_ctx.hpp"
#include "lins_map_types.cuh"
#include "lins_slot_blob.hpp"

using namespace lins_capi;
namespace B = lins_blob;

namespace {

static_assert(sizeof(B::PoseRec) == sizeof(MapperKeyPose), "pose record");
static_assert(sizeof(B::Scalars::consts) == sizeof(SeqState::consts), "consts");
static_assert(sizeof(B::Scalars::init_consts) == sizeof(SeqState::init_consts), "init consts");
static_assert(sizeof(lins_map::MapLoopState) % sizeof(float4) == 0, "loop state in float4 records");

B::BuildSizes build_sizes() {
  return B::BuildSizes{(uint32_t)icp_state_bytes(), (uint32_t)sizeof(lins_map::MapLoopState), (uint32_t)LINS_MAPPER_IMU_QUEUE,
                       (uint32_t)(sizeof(SeqState::consts) / sizeof(double)), (uint32_t)(sizeof(SeqState::init_consts) / sizeof(double))};
}

// the stored key frames of a node as (id, store slot), by id (the blob's order)
std::vector<std::pair<int, int>> stored_keyframes(const MapperNode& m) {
  std::vector<std::pair<int, int>> v(m.slot_of.begin(), m.slot_of.end());
  std::sort(v.begin(), v.end());
  return v;
}

// the counts of slot s's blob
B::Counts slot_counts(const lins_ctx* ctx, int s) {
  const SeqState& q = ctx->seq;
  B::Counts c;
  for (int k = 0; k < 4; ++k) c.n_map[k] = current_piece(q.map, k, s).len;
  c.bound = q.pub.bound;
  if (c.bound) {
    const MapperNode& m = ctx->mappers.node[s];
    c.n_outlier = q.pub.h_outl_off[s + 1] - q.pub.h_outl_off[s];
    c.n_poses = (int64_t)m.poses.size();
    c.n_window = (int64_t)m.s.window.size();
    c.n_keyframes = (int64_t)m.slot_of.size();
    for (const auto& kv : m.slot_of)
      for (int a = 0; a < 3; ++a) c.n_kf_points += m.slots[kv.second].n[a];
  }
  return c;
}

// what save_size, save and load check: a lins_gpu_seq_open run, a mask, no pending publish
int check_run(lins_ctx* ctx, const uint8_t* mask, const char* entry) {
  const int rc = check_open_run(ctx, entry, true);
  if (rc != LINS_OK) return rc;
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  if (ctx->seq.pub.bound && ctx->seq.pub.pending) return fail(ctx, LINS_E_INVALID, "the last step's lins_gpu_seq_map_step has not run");
  if (ctx->seq.pub.bound)  // (a blob carries the window's map-frame clouds, not an enabled slot's whole body-frame store)
    for (int s = 0; s < ctx->seq.n; ++s)
      if (mask[s] && ctx->mappers.node[s].loops.enabled) return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": a masked slot's mapper has loop closure enabled").c_str());
  return LINS_OK;
}

void offsets(const lins_ctx* ctx, const uint8_t* mask, uint64_t* off) {
  const int n = ctx->seq.n;
  off[0] = 0;
  for (int s = 0; s < n; ++s) {
    uint64_t len = 0;
    if (mask[s]) { B::Header h; B::layout(slot_counts(ctx, s), build_sizes(), h); len = h.total; }
    off[s + 1] = off[s] + len;
  }
}

// one section's record(s) into the host image: the bytes, then zeros up to the next 16-byte boundary
void put(uint8_t* dst, const void* src, size_t bytes) {
  if (bytes) std::memcpy(dst, src, bytes);
  std::memset(dst + bytes, 0, B::align16(bytes) - bytes);
}

// the device pieces of slot s's blob, as gather copies into dst (the blob's first byte in the device staging): the rows,
// the maps, the outlier cloud, the key frames' clouds (in kf order) and the loop state
void save_copies(lins_ctx* ctx, int s, const B::Header& h, float4* dst, const std::vector<std::pair<int, int>>& kf, std::vector<DevCopy>& v) {
  SeqState& q = ctx->seq;
  auto f4 = [](const void* p) { return reinterpret_cast<const float4*>(p); };
  auto at = [&](int sec) { return dst + h.sec[sec].off / 16; };
  const double* rows[6] = {q.filt.p + 20 * (size_t)s, q.cov.p + 324 * (size_t)s, q.glob.p + 20 * (size_t)s,
                           q.lin.p + 20 * (size_t)s, q.imu_last.p + 8 * (size_t)s, q.pre.p + 20 * (size_t)s};
  const int row_len[6] = {20, 324, 20, 20, 8, 20};
  for (int i = 0; i < 6; ++i) v.push_back(DevCopy{f4(rows[i]), at(B::kRows) + B::kRowOff[i] / 2, row_len[i] / 2, 0});
  float4* o = at(B::kMaps);
  for (int c = 0; c < 4; ++c) { const MapPiece p = current_piece(q.map, c, s); v.push_back(DevCopy{p.src, o, p.len, 0}); o += p.len; }
  if (!q.pub.bound) return;
  const SeqPubState& pb = q.pub;
  v.push_back(DevCopy{pb.outl.p + pb.h_outl_off[s], at(B::kOutlier), pb.h_outl_off[s + 1] - pb.h_outl_off[s], 0});
  const MapperNode& m = ctx->mappers.node[s];
  o = at(B::kKfClouds);
  for (const auto& k : kf)
    for (int a = 0; a < 3; ++a) { const MapperKeyFrame& f = m.slots[k.second]; v.push_back(DevCopy{f.c[a].p, o, f.n[a], 0}); o += f.n[a]; }
  v.push_back(DevCopy{f4(ctx->mappers.stm.loop.p + s), at(B::kLoop), (int)(sizeof(lins_map::MapLoopState) / 16), 0});
}

// the host records of slot s's blob into img (its first byte in the pinned image)
void save_host(lins_ctx* ctx, int s, const B::Counts& c, B::Header h, uint8_t* img, const std::vector<std::pair<int, int>>& kf) {
  const SeqState& q = ctx->seq;
  const SeqSlot& r = q.slot[s];
  h.magic = B::kMagic;
  h.version = B::kVersion;
  h.flags = (q.pub.bound ? B::kBound : 0u) | (r.cfg ? B::kConfigured : 0u) | (r.tune ? B::kTuned : 0u);
  h.sizes = build_sizes();
  h.n_sections = B::kNumSections;
  put(img, &h, sizeof(h));
  B::Scalars sc;
  std::memset(&sc, 0, sizeof(sc));
  sc.fusion = q.fusion[s];
  sc.stale = q.map.h_stale[s];
  for (int k = 0; k < 4; ++k) sc.n_map[k] = (int32_t)c.n_map[k];
  sc.n_outlier = (int32_t)c.n_outlier; sc.n_poses = (int32_t)c.n_poses; sc.n_window = (int32_t)c.n_window; sc.n_keyframes = (int32_t)c.n_keyframes;
  std::copy(q.consts, q.consts + 10, sc.consts);
  std::copy(q.init_consts, q.init_consts + 24, sc.init_consts);
  if (r.cfg) sc.cfg = *r.cfg;
  if (r.tune) { sc.tune = r.tune->t; std::copy(r.tune->R, r.tune->R + 9, sc.align_R); }
  if (q.pub.bound) { sc.yzx = r.yzx; std::copy(r.pose, r.pose + 7, sc.pose); }
  put(img + h.sec[B::kScalars].off, &sc, sizeof(sc));
  if (!q.pub.bound) return;
  const MapperNode& m = ctx->mappers.node[s];
  put(img + h.sec[B::kMapper].off, static_cast<const B::MapperRec*>(&m.s), sizeof(B::MapperRec));
  put(img + h.sec[B::kPoses].off, m.poses.data(), sizeof(B::PoseRec) * m.poses.size());
  const std::vector<int32_t> win(m.s.window.begin(), m.s.window.end());
  put(img + h.sec[B::kWindow].off, win.data(), sizeof(int32_t) * win.size());
  std::vector<B::KeyframeRec> tab;
  for (const auto& k : kf) {
    const MapperKeyFrame& f = m.slots[k.second];
    tab.push_back(B::KeyframeRec{k.first, {f.n[0], f.n[1], f.n[2]}});
  }
  put(img + h.sec[B::kKeyframes].off, tab.data(), sizeof(B::KeyframeRec) * tab.size());
}

// the device part of lins_gpu_seq_save on checked arguments (a failure ends the run)
int save_run(lins_ctx* ctx, const uint8_t* mask, uint8_t* blob, const uint64_t* off) {
  SeqState& q = ctx->seq;
  const int n = q.n;
  const uint64_t total = off[n];
  CK(cudaSetDevice(ctx->device));
  CK(q.blob.reserve(total / 16 + 1)); CK(q.h_blob.reserve(total / 16 + 1));
  std::vector<B::Counts> counts(n);
  std::vector<B::Header> hdr(n);
  std::vector<std::vector<std::pair<int, int>>> kf(n);
  std::vector<DevCopy> copies;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    counts[s] = slot_counts(ctx, s);
    B::layout(counts[s], build_sizes(), hdr[s]);
    if (q.pub.bound) kf[s] = stored_keyframes(ctx->mappers.node[s]);
    save_copies(ctx, s, hdr[s], q.blob.p + off[s] / 16, kf[s], copies);
  }
  copies.erase(std::remove_if(copies.begin(), copies.end(), [](const DevCopy& c) { return c.n <= 0; }), copies.end());
  int rc = q.copies.reserve(ctx, copies.size());
  if (rc == LINS_OK) rc = q.copies.stage(ctx, copies.data(), (int)copies.size(), 0);
  if (rc == LINS_OK) rc = q.copies.launch(ctx, 0, (int)copies.size());
  if (rc != LINS_OK) return rc;
  uint8_t* img = reinterpret_cast<uint8_t*>(q.h_blob.p);
  CK(cudaMemcpyAsync(img, q.blob.p, total, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < n; ++s)
    if (mask[s]) save_host(ctx, s, counts[s], hdr[s], img + off[s], kf[s]);
  std::memcpy(blob, img, total);
  return LINS_OK;
}

// the device and host part of lins_gpu_seq_load on validated blobs v (masked slots; a failure ends the run)
int load_run(lins_ctx* ctx, const uint8_t* mask, const std::vector<B::View>& v) {
  SeqState& q = ctx->seq;
  SeqPubState& pb = q.pub;
  MappersState& ms = ctx->mappers;
  const int n = q.n;
  CK(cudaSetDevice(ctx->device));
  // the blobs back to back in the staging, each at a 16-byte boundary (its length is a multiple of 16)
  std::vector<uint64_t> base(n, 0);
  uint64_t total = 0;
  for (int s = 0; s < n; ++s) if (mask[s]) { base[s] = total; total += v[s].h.total; }
  CK(q.blob.reserve(total / 16 + 1)); CK(q.h_blob.reserve(total / 16 + 1));
  auto at = [&](int s, int sec) { return q.blob.p + (base[s] + v[s].h.sec[sec].off) / 16; };
  // every buffer first: the next map and outlier generations, the key frames' clouds
  std::vector<MapPiece> next(4 * (size_t)n);
  for (int s = 0; s < n; ++s) {
    const float4* p = mask[s] ? at(s, B::kMaps) : nullptr;
    for (int c = 0; c < 4; ++c) {
      if (!mask[s]) { next[4 * (size_t)s + c] = current_piece(q.map, c, s); continue; }
      next[4 * (size_t)s + c] = MapPiece{p, v[s].sc.n_map[c]};
      p += v[s].sc.n_map[c];
    }
  }
  std::vector<DevCopy> copies;
  int rc = build_next_maps(ctx, q.map, next, copies);
  if (rc != LINS_OK) return rc;
  std::vector<MapPiece> onext;
  if (pb.bound) {
    pb.h_noutl_off.assign((size_t)n + 1, 0);
    for (int s = 0; s < n; ++s) {
      onext.push_back(mask[s] ? MapPiece{at(s, B::kOutlier), v[s].sc.n_outlier} : MapPiece{pb.outl.p + pb.h_outl_off[s], pb.h_outl_off[s + 1] - pb.h_outl_off[s]});
      pb.h_noutl_off[s + 1] = pb.h_noutl_off[s] + onext[s].len;
    }
    CK(pb.noutl.reserve((size_t)pb.h_noutl_off[n] + 1));
    for (int s = 0; s < n; ++s) copies.push_back(DevCopy{onext[s].src, pb.noutl.p + pb.h_noutl_off[s], onext[s].len, 0});
  }
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    const B::View& b = v[s];
    double* rows[6] = {q.filt.p + 20 * (size_t)s, q.cov.p + 324 * (size_t)s, q.glob.p + 20 * (size_t)s,
                       q.lin.p + 20 * (size_t)s, q.imu_last.p + 8 * (size_t)s, q.pre.p + 20 * (size_t)s};
    const int row_len[6] = {20, 324, 20, 20, 8, 20};
    for (int i = 0; i < 6; ++i) copies.push_back(DevCopy{at(s, B::kRows) + B::kRowOff[i] / 2, reinterpret_cast<float4*>(rows[i]), row_len[i] / 2, 0});
    if (!pb.bound) continue;
    copies.push_back(DevCopy{at(s, B::kLoop), reinterpret_cast<float4*>(ms.stm.loop.p + s), (int)(sizeof(lins_map::MapLoopState) / 16), 0});
    // the key-frame store of a fresh node: a store slot for each key frame (a free one first), its clouds from the staging
    MapperNode& m = ms.node[s];
    const float4* src = at(s, B::kKfClouds);
    for (int i = 0; i < b.sc.n_keyframes; ++i) {
      const B::KeyframeRec k = b.keyframe(i);
      int slot;
      if (!m.free_slots.empty()) { slot = m.free_slots.back(); m.free_slots.pop_back(); }
      else { slot = (int)m.slots.size(); m.slots.emplace_back(); }
      m.slot_of[k.id] = slot;
      MapperKeyFrame& f = m.slots[slot];
      for (int a = 0; a < 3; ++a) {
        f.n[a] = k.n[a];
        CK(f.c[a].grow((size_t)k.n[a] + 1));
        copies.push_back(DevCopy{src, f.c[a].p, k.n[a], 0});
        src += k.n[a];
      }
    }
  }
  copies.erase(std::remove_if(copies.begin(), copies.end(), [](const DevCopy& c) { return c.n <= 0; }), copies.end());
  if ((rc = q.copies.reserve(ctx, copies.size())) != LINS_OK) return rc;

  // one H2D of the blobs, one gather launch
  uint8_t* img = reinterpret_cast<uint8_t*>(q.h_blob.p);
  for (int s = 0; s < n; ++s) if (mask[s]) std::memcpy(img + base[s], v[s].p, v[s].h.total);
  if (total) CK(cudaMemcpyAsync(q.blob.p, img, total, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = q.copies.stage(ctx, copies.data(), (int)copies.size(), 0)) != LINS_OK) return rc;
  if ((rc = q.copies.launch(ctx, 0, (int)copies.size())) != LINS_OK) return rc;
  swap_maps(q.map);
  if (pb.bound) { std::swap(pb.outl, pb.noutl); pb.h_outl_off.swap(pb.h_noutl_off); }

  // the host bookkeeping of the loaded slots
  bool any_configured = false;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    const B::View& b = v[s];
    const B::Scalars& sc = b.sc;
    q.map.h_stale[s] = (unsigned char)sc.stale;
    q.fusion[s] = sc.fusion;
    q.status[s] = LINS_SEQ_IDLE;
    // the slot's record is the blob's.  The device constants are uploaded again when the slot is configured now or was
    // before (a fresh slot can have been configured: an unconfigured blob then takes the run's constants back, as
    // lins_gpu_seq_restart does)
    SeqSlot& r = q.slot[s];
    any_configured |= r.cfg.has_value();
    r = SeqSlot();
    r.fresh = false;
    if (b.h.flags & B::kConfigured) r.cfg = sc.cfg;
    if (b.h.flags & B::kTuned) { r.tune = SeqSlot::Tuning{sc.tune, {}}; std::copy(sc.align_R, sc.align_R + 9, r.tune->R); }
    any_configured |= r.cfg.has_value();
    if (!pb.bound) continue;
    pb.fused[s] = lins_fused_pose{};  // (a last-step output: none until the slot's next publish)
    r.yzx = sc.yzx != 0;
    std::copy(sc.pose, sc.pose + 7, r.pose);
    MapperNode& m = ms.node[s];
    static_cast<B::MapperRec&>(m.s) = b.m;
    m.s.window.clear();
    for (int i = 0; i < sc.n_window; ++i) m.s.window.push_back(b.window(i));
    m.poses.resize(sc.n_poses);
    for (int i = 0; i < sc.n_poses; ++i) { const B::PoseRec p = b.pose(i); std::memcpy(&m.poses[i], &p, sizeof(p)); }
    m.last = MapperLast();  // (no DS clouds until the slot's next processed cycle)
    m.stepped = true;       // (a loaded node is not fresh: loop closure cannot be enabled on it)
  }
  CK(queue_map_state(ctx, q.map));
  // (upload_slot_consts ends with a synchronisation; the sources above are pageable)
  if (any_configured) return upload_slot_consts(ctx, n);
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}

}  // namespace

extern "C" {

int lins_gpu_seq_save_size(lins_ctx* ctx, const uint8_t* mask, uint64_t* off) {
  const int rc = check_run(ctx, mask, "lins_gpu_seq_save_size");
  if (rc != LINS_OK) return rc;
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  offsets(ctx, mask, off);
  return LINS_OK;
}

int lins_gpu_seq_save(lins_ctx* ctx, const uint8_t* mask, void* blob, const uint64_t* off) {
  int rc = check_run(ctx, mask, "lins_gpu_seq_save");
  if (rc != LINS_OK) return rc;
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  const int n = ctx->seq.n;
  std::vector<uint64_t> want((size_t)n + 1);
  offsets(ctx, mask, want.data());
  if (!std::equal(want.begin(), want.end(), off)) return fail(ctx, LINS_E_INVALID, "offsets differ from lins_gpu_seq_save_size's");
  if (want[n] == 0) return LINS_OK;
  if (!blob) return fail(ctx, LINS_E_INVALID, "null blob");
  rc = save_run(ctx, mask, static_cast<uint8_t*>(blob), off);
  if (rc != LINS_OK) ctx->seq.n = 0;
  return rc;
}

int lins_gpu_seq_load(lins_ctx* ctx, const uint8_t* mask, const void* blob, const uint64_t* off) {
  const char* entry = "lins_gpu_seq_load";
  int rc = check_run(ctx, mask, entry);
  if (rc != LINS_OK) return rc;
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  SeqState& q = ctx->seq;
  const int n = q.n;
  const uint8_t* p = static_cast<const uint8_t*>(blob);
  std::vector<B::View> v(n);
  bool any = false;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    any = true;
    if (!p) return fail(ctx, LINS_E_INVALID, "null blob");
    if (off[s + 1] < off[s]) return fail(ctx, LINS_E_INVALID, "blob offsets decrease");
    if ((rc = check_fresh(ctx, s, entry)) != LINS_OK) return rc;
    const char* bad = B::parse(p + off[s], off[s + 1] - off[s], build_sizes(), v[s]);
    if (bad) return fail(ctx, LINS_E_INVALID, bad);
    const bool bound = v[s].h.flags & B::kBound;
    if (bound != q.pub.bound) return fail(ctx, LINS_E_INVALID, bound ? "a bound slot blob into an unbound run" : "an unbound slot blob into a bound run");
    if (!(v[s].h.flags & B::kConfigured) &&
        (std::memcmp(v[s].sc.consts, q.consts, sizeof(q.consts)) != 0 || std::memcmp(v[s].sc.init_consts, q.init_consts, sizeof(q.init_consts)) != 0))
      return fail(ctx, LINS_E_INVALID, "an unconfigured slot blob of a run with other open constants");
  }
  if (!any) return LINS_OK;
  rc = load_run(ctx, mask, v);
  if (rc != LINS_OK) q.n = 0;
  return rc;
}

}  // extern "C"
