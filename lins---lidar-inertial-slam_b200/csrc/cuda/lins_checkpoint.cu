// lins_checkpoint.cu — slots saved to host bytes and loaded into fresh slots (include/lins_gpu.h), in the formats of
// lins_slot_blob.hpp and lins_mapper_blob.hpp: sequence-mode slots (lins_gpu_seq_save_size / _save / _load: the device
// rows, maps, stale 1-NN and outlier clouds, host bookkeeping and, in a bound run, the mapping node) and mapping-node
// slots of the lockstep mappers or the single mapper (lins_gpu_mappers_* / lins_gpu_mapper_save_size / _save / _load:
// the node and, with loop closure, the key-pose graph, its estimate and MapperLoops' scalars).  One codec (node_*)
// writes and restores the node of either.
//   save: one gather launch of the masked slots' device pieces into the device staging (a sequence-mode blob whole, a
//         mapper blob's device range only: a plain slot's map-frame key-frame clouds and the loop state), one D2H into
//         pinned staging, one synchronisation, then the host records (a loop slot's body-frame clouds from its host
//         store: the synchronisation orders the copy after the last kernel that wrote them).
//   load: every masked blob validated in full first; then one H2D of the blobs and one gather launch that installs their
//         device pieces and fills the plain key frames' device store.  A sequence-mode load also builds the next map and
//         outlier generations (the restart path's compaction).  A mapper load synchronises first (a queued kernel may
//         still write a chunk a reset handed back), fills a loop slot's host store on the host, stages the rebuild's
//         job table behind the blobs and launches lins_mapper_rebuild_kernel, which writes c = T(b, pose) of each key
//         frame a loop slot's device store keeps (those a later window can take: lins_blob::later_window), as every
//         save and correctPoses leave them (DESIGN.md §4.15); one synchronisation at the end.
// A call's staging is the masked blobs' total (and the job table on a mapper load): a caller bounds it with smaller masks.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "lins_ctx.hpp"
#include "lins_kf_arena.hpp"
#include "lins_map_types.cuh"
#include "lins_mapper_blob.hpp"
#include "lins_mapper_tf.cuh"
#include "lins_slot_blob.hpp"

using namespace lins_capi;
using lins_blob::KeyframeRec;
using lins_blob::MapperRec;
using lins_blob::NodeSecs;
using lins_blob::NodeView;
using lins_blob::PoseRec;
using lins_blob::put;
namespace S = lins_blob;
namespace M = lins_mblob;

namespace {

static_assert(sizeof(PoseRec) == sizeof(MapperKeyPose), "pose record");
static_assert(sizeof(S::Scalars::consts) == sizeof(SeqState::consts), "consts");
static_assert(sizeof(S::Scalars::init_consts) == sizeof(SeqState::init_consts), "init consts");
static_assert(sizeof(M::EstRec) == sizeof(lins_pg::Pose3), "estimate record");
static_assert(sizeof(lins_pg::Vec6) == 6 * sizeof(double), "variance record");
static_assert(sizeof(lins_map::MapLoopState) % sizeof(float4) == 0, "loop state in float4 records");
constexpr int kLoopRecs = sizeof(lins_map::MapLoopState) / sizeof(float4);
// MapperLoops::rebuild is not carried: mapper_cycle_end clears it before anything reads it, and only the step that
// processed the slot reads it, right after (lins_mappers.cu, the correctPoses re-transform)

S::BuildSizes seq_sizes() {
  return S::BuildSizes{(uint32_t)icp_state_bytes(), (uint32_t)sizeof(lins_map::MapLoopState), (uint32_t)LINS_MAPPER_IMU_QUEUE,
                       (uint32_t)(sizeof(SeqState::consts) / sizeof(double)), (uint32_t)(sizeof(SeqState::init_consts) / sizeof(double))};
}
M::BuildSizes mapper_sizes() {
  return M::BuildSizes{(uint32_t)sizeof(lins_map::MapLoopState), (uint32_t)LINS_MAPPER_IMU_QUEUE, (uint32_t)LINS_MAPPER_WINDOW,
                       (uint32_t)sizeof(M::FactorRec)};
}

// one loaded key-frame cloud of a slot with loop closure that its device store keeps: its body-frame points in the
// staging (in) transformed by the key pose (k) into c
struct KfRebuild { const float4* in; float4* c; int n, pad; TfConsts k; };

__global__ void __launch_bounds__(256) lins_mapper_rebuild_kernel(const KfRebuild* __restrict__ jobs) {
  const KfRebuild& jb = jobs[blockIdx.x];
  const TfConsts c = jb.k;
  for (int i = threadIdx.x; i < jb.n; i += blockDim.x) jb.c[i] = tf_point(c, jb.in[i]);
}

double ms_since(std::chrono::steady_clock::time_point& t) {
  const auto now = std::chrono::steady_clock::now();
  const double ms = std::chrono::duration<double, std::milli>(now - t).count();
  t = now;
  return ms;
}

// ---- the mapping-node codec -----------------------------------------------------------------------------------------

// the stored key frames of a node as (id, device store slot), by id (the blob's order): a plain node's device store;
// every key frame of a node with loop closure (its host store; the slot is -1)
using Stored = std::vector<std::pair<int, int>>;
Stored stored_keyframes(const MapperNode& m) {
  Stored v;
  if (m.loops.enabled) {
    for (int id = 0; id < (int)m.host.size(); ++id) v.push_back({id, -1});
    return v;
  }
  v.assign(m.slot_of.begin(), m.slot_of.end());
  std::sort(v.begin(), v.end());
  return v;
}

// the cloud sizes of stored key frame k
const int* kf_sizes(const MapperNode& m, const std::pair<int, int>& k) { return m.loops.enabled ? m.host[k.first].n : m.slots[k.second].n; }

// the node's counts in either format's Counts
template <typename Counts>
void node_counts(const MapperNode& m, Counts& c) {
  c.n_poses = (int64_t)m.poses.size();
  c.n_window = (int64_t)m.s.window.size();
  const Stored kf = stored_keyframes(m);
  c.n_keyframes = (int64_t)kf.size();
  for (const auto& k : kf)
    for (int a = 0; a < 3; ++a) c.n_kf_points += kf_sizes(m, k)[a];
}

// the node's device pieces as gather copies into its blob's sections at `at` (blob: the blob's first byte in the device
// staging): a plain node's key-frame clouds, in kf order, and its loop state
void node_save_copies(const MapperNode& m, const Stored& kf, const lins_map::MapLoopState* loop, float4* blob, const NodeSecs& at, std::vector<DevCopy>& v) {
  float4* o = blob + at.kfclouds / 16;
  for (const auto& k : kf)
    for (int a = 0; a < 3 && !m.loops.enabled; ++a) {
      const MapperKeyFrame& f = m.slots[k.second];
      v.push_back(DevCopy{f.c[a].p, o, f.n[a], 0});
      o += f.n[a];
    }
  v.push_back(DevCopy{reinterpret_cast<const float4*>(loop), blob + at.loop / 16, kLoopRecs, 0});
}

// the node's host records into its blob image img: its scalars, key poses, window and key-frame table and, on a node
// with loop closure, its host store's body-frame clouds in table order (the caller has synchronised the stream)
void node_put(const MapperNode& m, const Stored& kf, uint8_t* img, const NodeSecs& at) {
  put(img + at.mapper, static_cast<const MapperRec*>(&m.s), sizeof(MapperRec));
  put(img + at.poses, m.poses.data(), sizeof(PoseRec) * m.poses.size());
  const std::vector<int32_t> win(m.s.window.begin(), m.s.window.end());
  put(img + at.window, win.data(), sizeof(int32_t) * win.size());
  std::vector<KeyframeRec> tab;
  for (const auto& k : kf) {
    const int* n = kf_sizes(m, k);
    tab.push_back(KeyframeRec{k.first, {n[0], n[1], n[2]}});
  }
  put(img + at.keyframes, tab.data(), sizeof(KeyframeRec) * tab.size());
  if (!m.loops.enabled) return;
  uint8_t* o = img + at.kfclouds;
  for (const auto& k : kf) {
    const HostKeyFrame& f = m.host[k.first];
    const size_t bytes = sizeof(float4) * ((size_t)f.n[0] + f.n[1] + f.n[2]);
    if (bytes) std::memcpy(o, f.p, bytes);
    o += bytes;
  }
}

// a loop slot's key frame for its host store: the block, its clouds in the caller's blob, their bytes
struct HostFill { float4* dst; const uint8_t* src; size_t bytes; };

// Parsed node b into slot s's fresh node, its blob at dev in the device staging: gather copies of the loop state and of a
// plain node's key frames into its device store.  A node with loop closure (loops) takes every key frame into its host
// store (fill: the copies the caller makes) and those a later window can take into its device store, by rebuild jobs.
int node_load(lins_ctx* ctx, MappersState& ms, int s, const NodeView& b, bool loops, const float4* dev, std::vector<DevCopy>& copies,
              std::vector<KfRebuild>& jobs, std::vector<HostFill>& fill) {
  MapperNode& m = ms.node[s];
  copies.push_back(DevCopy{dev + b.node.loop / 16, reinterpret_cast<float4*>(ms.stm.loop.p + s), kLoopRecs, 0});
  const float4* src = dev + b.node.kfclouds / 16;
  const uint8_t* hsrc = b.p + b.node.kfclouds;
  std::vector<unsigned char> keep;  // a loop slot: the key frames its device store keeps
  if (loops) {
    keep.assign(b.n_poses, 0);
    lins_blob::later_window(b, [&](int32_t id, int) { keep[id] = 1; return true; });
    m.host.assign(b.n_poses, HostKeyFrame());
  }
  for (int i = 0; i < b.n_keyframes; ++i) {
    const KeyframeRec k = b.keyframe(i);
    TfConsts tc{};
    if (loops) {
      HostKeyFrame& hk = m.host[k.id];
      std::copy(k.n, k.n + 3, hk.n);
      const size_t bytes = sizeof(float4) * ((size_t)k.n[0] + k.n[1] + k.n[2]);
      void* p = nullptr;
      if (!ms.store.take(m.held, bytes, &p)) return fail(ctx, LINS_E_CUDA, "the host key-frame store could not allocate pinned memory");
      hk.p = static_cast<float4*>(p);
      if (bytes) fill.push_back(HostFill{hk.p, hsrc, bytes});
      hsrc += bytes;
      if (!keep[k.id]) { src += k.n[0] + k.n[1] + k.n[2]; continue; }
      MapperKeyPose kp;
      const PoseRec pr = b.pose(k.id);
      std::memcpy(&kp, &pr, sizeof(kp));
      tc = tf_consts(kp);
    }
    MapperKeyFrame& f = store_keyframe(m, k.id, k.n);
    for (int a = 0; a < 3; ++a) {
      CK(f.c[a].grow((size_t)k.n[a] + 1));
      if (!loops) copies.push_back(DevCopy{src, f.c[a].p, k.n[a], 0});
      else if (k.n[a]) jobs.push_back(KfRebuild{src, f.c[a].p, k.n[a], 0, tc});
      src += k.n[a];
    }
  }
  return LINS_OK;
}

// the node's host state from parsed node b: its scalars, window and key poses; no outputs of a last cycle (no DS clouds
// until its next processed cycle), and not fresh (loop closure cannot be enabled on it)
void node_restore(MapperNode& m, const NodeView& b) {
  static_cast<MapperRec&>(m.s) = b.m;
  m.s.window.clear();
  for (int i = 0; i < b.n_window; ++i) m.s.window.push_back(b.window(i));
  m.poses.resize(b.n_poses);
  for (int i = 0; i < b.n_poses; ++i) { const PoseRec p = b.pose(i); std::memcpy(&m.poses[i], &p, sizeof(p)); }
  m.last = MapperLast();
  m.stepped = true;
}


// ---- the entry preambles --------------------------------------------------------------------------------------------

// off[s + 1] = off[s] + the length of slot s's blob, bytes(s), where the mask is set, else 0
template <typename Bytes>
int save_size(lins_ctx* ctx, int n, const uint8_t* mask, uint64_t* off, Bytes bytes) {
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  off[0] = 0;
  for (int s = 0; s < n; ++s) off[s + 1] = off[s] + (mask[s] ? bytes(s) : 0);
  return LINS_OK;
}

// a save on a run of n slots that passed its checks: offsets equal to the save size's (else the message `differ`),
// nothing to write, a blob; then run() (a failure ends the run)
template <typename Bytes, typename Run>
int save(lins_ctx* ctx, int& n, const uint8_t* mask, const void* blob, const uint64_t* off, Bytes bytes, const std::string& differ, Run run) {
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  std::vector<uint64_t> want((size_t)n + 1);
  save_size(ctx, n, mask, want.data(), bytes);
  if (!std::equal(want.begin(), want.end(), off)) return fail(ctx, LINS_E_INVALID, differ.c_str());
  if (want[n] == 0) return LINS_OK;
  if (!blob) return fail(ctx, LINS_E_INVALID, "null blob");
  const int rc = run();
  if (rc != LINS_OK) n = 0;
  return rc;
}

// a load on a run of n slots that passed its checks: each masked slot's blob present, at offsets that do not decrease
// and passing check(s, bytes, length, view) (the slot fresh, the blob valid), every one before anything changes; then
// run(views) (a failure ends the run)
template <typename View, typename Check, typename Run>
int load(lins_ctx* ctx, int& n, const uint8_t* mask, const void* blob, const uint64_t* off, Check check, Run run) {
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  const uint8_t* p = static_cast<const uint8_t*>(blob);
  std::vector<View> v(n);
  bool any = false;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    any = true;
    if (!p) return fail(ctx, LINS_E_INVALID, "null blob");
    if (off[s + 1] < off[s]) return fail(ctx, LINS_E_INVALID, "blob offsets decrease");
    const int rc = check(s, p + off[s], off[s + 1] - off[s], v[s]);
    if (rc != LINS_OK) return rc;
  }
  if (!any) return LINS_OK;
  const int rc = run(v);
  if (rc != LINS_OK) n = 0;
  return rc;
}

// ---- sequence-mode slots --------------------------------------------------------------------------------------------

// slot s's device row i (S::kRowOff[i]: its place in the blob's rows)
constexpr int kRowLen[6] = {20, 324, 20, 20, 8, 20};
double* seq_row(SeqState& q, int s, int i) {
  double* const rows[6] = {q.filt.p, q.cov.p, q.glob.p, q.lin.p, q.imu_last.p, q.pre.p};
  return rows[i] + kRowLen[i] * (size_t)s;
}

S::Counts seq_counts(lins_ctx* ctx, int s) {
  const SeqState& q = ctx->seq;
  S::Counts c;
  for (int k = 0; k < 4; ++k) c.n_map[k] = current_piece(q.map, k, s).len;
  c.bound = q.pub.bound;
  if (c.bound) {
    c.n_outlier = q.pub.h_outl_off[s + 1] - q.pub.h_outl_off[s];
    node_counts(ctx->mappers.node[s], c);
  }
  return c;
}
uint64_t seq_bytes(lins_ctx* ctx, int s) {
  S::Header h;
  S::layout(seq_counts(ctx, s), seq_sizes(), h);
  return h.total;
}

// what save_size, save and load check: a lins_gpu_seq_open run, a mask, no pending publish
int seq_check(lins_ctx* ctx, const uint8_t* mask, const char* entry) {
  const int rc = check_open_run(ctx, entry, true);
  if (rc != LINS_OK) return rc;
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  if (ctx->seq.pub.bound && ctx->seq.pub.pending) return fail(ctx, LINS_E_INVALID, "the last step's lins_gpu_seq_map_step has not run");
  if (ctx->seq.pub.bound)  // (a blob carries the window's map-frame clouds, not an enabled slot's whole body-frame store)
    for (int s = 0; s < ctx->seq.n; ++s)
      if (mask[s] && ctx->mappers.node[s].loops.enabled) return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": a masked slot's mapper has loop closure enabled").c_str());
  return LINS_OK;
}

// the host records of slot s's blob into img (its first byte in the pinned image)
void seq_put(lins_ctx* ctx, int s, const S::Counts& c, S::Header h, uint8_t* img, const Stored& kf) {
  const SeqState& q = ctx->seq;
  const SeqSlot& r = q.slot[s];
  h.magic = S::kMagic;
  h.version = S::kVersion;
  h.flags = (q.pub.bound ? S::kBound : 0u) | (r.cfg ? S::kConfigured : 0u) | (r.tune ? S::kTuned : 0u);
  h.sizes = seq_sizes();
  h.n_sections = S::kNumSections;
  put(img, &h, sizeof(h));
  S::Scalars sc;
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
  put(img + h.sec[S::kScalars].off, &sc, sizeof(sc));
  if (q.pub.bound) node_put(ctx->mappers.node[s], kf, img, S::node_secs(h));
}

// the device part of lins_gpu_seq_save on checked arguments: each blob whole in the device staging, laid out as blob
int seq_save_run(lins_ctx* ctx, const uint8_t* mask, uint8_t* blob, const uint64_t* off) {
  SeqState& q = ctx->seq;
  const int n = q.n;
  const uint64_t total = off[n];
  CK(cudaSetDevice(ctx->device));
  CK(q.blob.reserve(total / 16 + 1)); CK(q.h_blob.reserve(total / 16 + 1));
  std::vector<S::Counts> counts(n);
  std::vector<S::Header> hdr(n);
  std::vector<Stored> kf(n);
  std::vector<DevCopy> copies;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    counts[s] = seq_counts(ctx, s);
    const S::Header& h = hdr[s];
    S::layout(counts[s], seq_sizes(), hdr[s]);
    float4* dst = q.blob.p + off[s] / 16;
    auto at = [&](int sec) { return dst + h.sec[sec].off / 16; };
    for (int i = 0; i < 6; ++i) copies.push_back(DevCopy{reinterpret_cast<const float4*>(seq_row(q, s, i)), at(S::kRows) + S::kRowOff[i] / 2, kRowLen[i] / 2, 0});
    float4* o = at(S::kMaps);
    for (int c = 0; c < 4; ++c) { const MapPiece p = current_piece(q.map, c, s); copies.push_back(DevCopy{p.src, o, p.len, 0}); o += p.len; }
    if (!q.pub.bound) continue;
    const SeqPubState& pb = q.pub;
    copies.push_back(DevCopy{pb.outl.p + pb.h_outl_off[s], at(S::kOutlier), pb.h_outl_off[s + 1] - pb.h_outl_off[s], 0});
    kf[s] = stored_keyframes(ctx->mappers.node[s]);
    node_save_copies(ctx->mappers.node[s], kf[s], ctx->mappers.stm.loop.p + s, dst, S::node_secs(h), copies);
  }
  int rc = q.copies.reserve(ctx, copies.size());
  if (rc == LINS_OK) rc = queue_copies(ctx, q.copies, copies, 0);
  if (rc != LINS_OK) return rc;
  uint8_t* img = reinterpret_cast<uint8_t*>(q.h_blob.p);
  CK(cudaMemcpyAsync(img, q.blob.p, total, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < n; ++s)
    if (mask[s]) seq_put(ctx, s, counts[s], hdr[s], img + off[s], kf[s]);
  std::memcpy(blob, img, total);
  return LINS_OK;
}

// the device and host part of lins_gpu_seq_load on validated blobs v (masked slots)
int seq_load_run(lins_ctx* ctx, const uint8_t* mask, const std::vector<S::View>& v) {
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
  auto dev = [&](int s) { return q.blob.p + base[s] / 16; };
  auto at = [&](int s, int sec) { return dev(s) + v[s].h.sec[sec].off / 16; };
  // every buffer first: the next map and outlier generations, the key frames' clouds
  std::vector<MapPiece> next(4 * (size_t)n);
  for (int s = 0; s < n; ++s) {
    const float4* p = mask[s] ? at(s, S::kMaps) : nullptr;
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
      onext.push_back(mask[s] ? MapPiece{at(s, S::kOutlier), v[s].sc.n_outlier} : MapPiece{pb.outl.p + pb.h_outl_off[s], pb.h_outl_off[s + 1] - pb.h_outl_off[s]});
      pb.h_noutl_off[s + 1] = pb.h_noutl_off[s] + onext[s].len;
    }
    CK(pb.noutl.reserve((size_t)pb.h_noutl_off[n] + 1));
    for (int s = 0; s < n; ++s) copies.push_back(DevCopy{onext[s].src, pb.noutl.p + pb.h_noutl_off[s], onext[s].len, 0});
  }
  std::vector<KfRebuild> jobs;  // (none, nor host-store copies: a bound run's slots have no loop closure)
  std::vector<HostFill> fill;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    for (int i = 0; i < 6; ++i) copies.push_back(DevCopy{at(s, S::kRows) + S::kRowOff[i] / 2, reinterpret_cast<float4*>(seq_row(q, s, i)), kRowLen[i] / 2, 0});
    if (pb.bound && (rc = node_load(ctx, ms, s, v[s], false, dev(s), copies, jobs, fill)) != LINS_OK) return rc;
  }
  if ((rc = q.copies.reserve(ctx, copies.size())) != LINS_OK) return rc;

  // one H2D of the blobs, one gather launch
  uint8_t* img = reinterpret_cast<uint8_t*>(q.h_blob.p);
  for (int s = 0; s < n; ++s) if (mask[s]) std::memcpy(img + base[s], v[s].p, v[s].h.total);
  if (total) CK(cudaMemcpyAsync(q.blob.p, img, total, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = queue_copies(ctx, q.copies, copies, 0)) != LINS_OK) return rc;
  swap_maps(q.map);
  if (pb.bound) { std::swap(pb.outl, pb.noutl); pb.h_outl_off.swap(pb.h_noutl_off); }

  // the host bookkeeping of the loaded slots
  bool any_configured = false;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    const S::View& b = v[s];
    const S::Scalars& sc = b.sc;
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
    if (b.h.flags & S::kConfigured) r.cfg = sc.cfg;
    if (b.h.flags & S::kTuned) { r.tune = SeqSlot::Tuning{sc.tune, {}}; std::copy(sc.align_R, sc.align_R + 9, r.tune->R); }
    any_configured |= r.cfg.has_value();
    if (!pb.bound) continue;
    pb.fused[s] = lins_fused_pose{};  // (a last-step output: none until the slot's next publish)
    r.yzx = sc.yzx != 0;
    std::copy(sc.pose, sc.pose + 7, r.pose);
    node_restore(ms.node[s], b);
  }
  CK(queue_map_state(ctx, q.map));
  // (upload_slot_consts ends with a synchronisation; the sources above are pageable)
  if (any_configured) return upload_slot_consts(ctx, n);
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}

// ---- mapping-node slots ---------------------------------------------------------------------------------------------

// what every mapper entry checks: an open run that lins_gpu_seq_map_open has not bound, and a mask
int mapper_check(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, const char* entry) {
  if (ms.n == 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_mappers_open has not been called");
  if (&ms == &ctx->mappers && ctx->seq.pub.bound)  // (the slot's estimator half would be lost: lins_gpu_seq_save saves both)
    return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": the run is bound to sequence mode (lins_gpu_seq_save saves its slots)").c_str());
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  return LINS_OK;
}

M::Counts mapper_counts(const MapperNode& m) {
  M::Counts c;
  node_counts(m, c);
  c.n_factors = (int64_t)m.loops.graph.size();
  c.n_est = (int64_t)m.loops.est.size();
  return c;
}
uint64_t mapper_bytes(const MappersState& ms, int s) {
  M::Header h;
  M::layout(mapper_counts(ms.node[s]), mapper_sizes(), h);
  return h.total;
}

// the host records of a node's blob into img (its first byte in the caller's buffer)
void mapper_put(const MapperNode& m, const M::Counts& c, M::Header h, uint8_t* img, const Stored& kf) {
  const MapperLoops& L = m.loops;
  h.magic = M::kMagic;
  h.version = M::kVersion;
  h.flags = L.enabled ? M::kLoops : 0u;
  h.sizes = mapper_sizes();
  h.n_sections = M::kNumSections;
  h.pad = 0;
  put(img, &h, sizeof(h));
  M::Scalars sc;
  std::memset(&sc, 0, sizeof(sc));
  sc.n_poses = (int32_t)c.n_poses; sc.n_window = (int32_t)c.n_window; sc.n_keyframes = (int32_t)c.n_keyframes;
  sc.n_factors = (int32_t)c.n_factors; sc.n_est = (int32_t)c.n_est;
  sc.n_loop = L.n_loop; sc.closed = L.closed ? 1 : 0;
  std::memcpy(sc.cur, L.cur, sizeof(sc.cur));
  sc.time = L.time;
  put(img + h.sec[M::kScalars].off, &sc, sizeof(sc));
  node_put(m, kf, img, M::node_secs(h));
  std::vector<M::FactorRec> fac(L.graph.size());
  for (size_t i = 0; i < L.graph.size(); ++i) {
    const lins_pg::Factor& f = L.graph[i];
    M::FactorRec& r = fac[i];
    r.a = f.a; r.b = f.b;
    std::memcpy(r.R, f.z.R, sizeof(r.R));
    std::memcpy(r.t, f.z.t, sizeof(r.t));
    std::copy(f.var.begin(), f.var.end(), r.var);
  }
  put(img + h.sec[M::kFactors].off, fac.data(), sizeof(M::FactorRec) * fac.size());
  put(img + h.sec[M::kEst].off, L.est.data(), sizeof(M::EstRec) * L.est.size());
}

// the device part of a mapper save on checked arguments: only each blob's device range [lo, hi) in the staging (a plain
// slot's key frames' clouds and the loop state, which follows them; a loop slot's loop state), back to back
int mapper_save_run(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, uint8_t* blob, const uint64_t* off) {
  const int n = ms.n;
  CK(cudaSetDevice(ctx->device));
  std::vector<M::Counts> counts(n);
  std::vector<M::Header> hdr(n);
  std::vector<Stored> kf(n);
  std::vector<uint64_t> lo(n, 0), hi(n, 0), doff(n + 1, 0);  // each slot's device range, and its place in the staging
  for (int s = 0; s < n; ++s) {
    doff[s + 1] = doff[s];
    if (!mask[s]) continue;
    const MapperNode& m = ms.node[s];
    counts[s] = mapper_counts(m);
    M::layout(counts[s], mapper_sizes(), hdr[s]);
    kf[s] = stored_keyframes(m);
    lo[s] = hdr[s].sec[m.loops.enabled ? M::kLoop : M::kKfClouds].off;
    hi[s] = hdr[s].sec[M::kLoop].off + hdr[s].sec[M::kLoop].bytes;
    doff[s + 1] += hi[s] - lo[s];
  }
  const uint64_t total = doff[n];
  CK(ms.blob.reserve(total / 16 + 1)); CK(ms.h_blob.reserve(total / 16 + 1));
  std::vector<DevCopy> copies;
  for (int s = 0; s < n; ++s)
    if (mask[s]) node_save_copies(ms.node[s], kf[s], ms.stm.loop.p + s, ms.blob.p + doff[s] / 16 - lo[s] / 16, M::node_secs(hdr[s]), copies);
  int rc = ms.copies.reserve(ctx, copies.size());
  if (rc == LINS_OK) rc = queue_copies(ctx, ms.copies, copies, 0);
  if (rc != LINS_OK) return rc;
  const uint8_t* img = reinterpret_cast<const uint8_t*>(ms.h_blob.p);
  CK(cudaMemcpyAsync(ms.h_blob.p, ms.blob.p, total, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    std::memcpy(blob + off[s] + lo[s], img + doff[s], hi[s] - lo[s]);
    mapper_put(ms.node[s], counts[s], hdr[s], blob + off[s], kf[s]);
  }
  return LINS_OK;
}

// the device and host part of a mapper load on validated blobs v (masked slots).  ph: the host phases (allocation,
// staging, device, bookkeeping; ph[0], the validation, is the caller's)
int mapper_load_run(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, const std::vector<M::View>& v, double* ph) {
  auto t = std::chrono::steady_clock::now();
  const int n = ms.n;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));  // (before the host writes the host stores' chunks)
  // the blobs back to back in the staging, each at a 16-byte boundary (its length is a multiple of 16), then the
  // rebuild's job table
  std::vector<uint64_t> base(n, 0);
  uint64_t total = 0;
  size_t n_jobs = 0;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    base[s] = total;
    total += v[s].h.total;
    if (v[s].loops())
      for (int i = 0; i < v[s].n_keyframes; ++i) {
        const KeyframeRec k = v[s].keyframe(i);
        for (int a = 0; a < 3; ++a) n_jobs += k.n[a] > 0;  // (a bound: only the device store's key frames get jobs)
      }
  }
  const uint64_t job_off = lins_blob::align16(total), staged = job_off + sizeof(KfRebuild) * n_jobs;
  CK(ms.blob.reserve(staged / 16 + 1)); CK(ms.h_blob.reserve(staged / 16 + 1));
  // every buffer first: each device-store key frame's slot and clouds, and each loop slot's host store blocks
  std::vector<DevCopy> copies;
  std::vector<KfRebuild> jobs;
  std::vector<HostFill> fill;
  int rc;
  for (int s = 0; s < n; ++s)
    if (mask[s] && (rc = node_load(ctx, ms, s, v[s], v[s].loops(), ms.blob.p + base[s] / 16, copies, jobs, fill)) != LINS_OK) return rc;
  if ((rc = ms.copies.reserve(ctx, copies.size())) != LINS_OK) return rc;
  ph[1] = ms_since(t);

  // the loop slots' host stores, the blobs and the job table into the pinned image
  for (const HostFill& f : fill) std::memcpy(f.dst, f.src, f.bytes);
  uint8_t* img = reinterpret_cast<uint8_t*>(ms.h_blob.p);
  for (int s = 0; s < n; ++s) if (mask[s]) std::memcpy(img + base[s], v[s].p, v[s].h.total);
  if (!jobs.empty()) std::memcpy(img + job_off, jobs.data(), sizeof(KfRebuild) * jobs.size());
  ph[2] = ms_since(t);

  // one H2D, one gather launch, one rebuild launch, one synchronisation
  CK(cudaMemcpyAsync(ms.blob.p, img, staged, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = queue_copies(ctx, ms.copies, copies, 0)) != LINS_OK) return rc;
  if (!jobs.empty()) {
    lins_mapper_rebuild_kernel<<<(unsigned)jobs.size(), 256, 0, ctx->stream>>>(reinterpret_cast<const KfRebuild*>(ms.blob.p + job_off / 16));
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  CK(cudaStreamSynchronize(ctx->stream));
  ph[3] = ms_since(t);

  // the host bookkeeping of the loaded slots: the node, and its loop closure; no global map until its next call
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    const M::View& b = v[s];
    const M::Scalars& sc = b.sc;
    MapperNode& m = ms.node[s];
    node_restore(m, b);
    MapperLoops L;
    L.enabled = b.loops();
    L.closed = sc.closed != 0;
    L.n_loop = sc.n_loop;
    std::memcpy(L.cur, sc.cur, sizeof(L.cur));
    L.time = sc.time;
    for (int i = 0; i < sc.n_factors; ++i) {
      const M::FactorRec r = b.factor(i);
      lins_pg::Factor f;
      f.a = r.a; f.b = r.b;
      std::memcpy(f.z.R, r.R, sizeof(r.R));
      std::memcpy(f.z.t, r.t, sizeof(r.t));
      std::copy(r.var, r.var + 6, f.var.begin());
      L.graph.push_back(f);
    }
    L.est.resize(sc.n_est);
    for (int i = 0; i < sc.n_est; ++i) { const M::EstRec e = b.est(i); std::memcpy(&L.est[i], &e, sizeof(e)); }
    m.loops = std::move(L);
    m.gm = MapperGlobalMap();
  }
  ph[4] = ms_since(t);
  return LINS_OK;
}

int mapper_save_size(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, uint64_t* off, const char* entry) {
  const int rc = mapper_check(ctx, ms, mask, entry);
  return rc != LINS_OK ? rc : save_size(ctx, ms.n, mask, off, [&](int s) { return mapper_bytes(ms, s); });
}

int mapper_save(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, void* blob, const uint64_t* off, const char* entry) {
  const int rc = mapper_check(ctx, ms, mask, entry);
  if (rc != LINS_OK) return rc;
  return save(ctx, ms.n, mask, blob, off, [&](int s) { return mapper_bytes(ms, s); }, std::string(entry) + ": offsets differ from the save size's",
              [&] { return mapper_save_run(ctx, ms, mask, static_cast<uint8_t*>(blob), off); });
}

int mapper_load(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, const void* blob, const uint64_t* off, const char* entry) {
  auto t = std::chrono::steady_clock::now();
  const int rc = mapper_check(ctx, ms, mask, entry);
  if (rc != LINS_OK) return rc;
  auto check = [&](int s, const uint8_t* p, uint64_t len, M::View& v) {
    if (ms.node[s].stepped) return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": a masked slot is not fresh (present in a step since open / reset)").c_str());
    const char* bad = M::parse(p, len, mapper_sizes(), v);
    return bad ? fail(ctx, LINS_E_INVALID, bad) : LINS_OK;
  };
  return load<M::View>(ctx, ms.n, mask, blob, off, check, [&](const std::vector<M::View>& v) {
    double ph[5];
    ph[0] = ms_since(t);
    const int rc = mapper_load_run(ctx, ms, mask, v, ph);
    if (rc != LINS_OK) return rc;
    std::copy(ph, ph + 5, ctx->mapper_load_ms);
    ctx->mapper_load_valid = true;
    return LINS_OK;
  });
}

// the single mapper: a run of one slot of its own, opened by the first lins_gpu_mapper_* call on the context
int mapper_open(lins_ctx* ctx) {
  return ctx->mapper.n > 0 ? LINS_OK : mappers_open(ctx, ctx->mapper, 1);
}

}  // namespace

extern "C" {

int lins_gpu_seq_save_size(lins_ctx* ctx, const uint8_t* mask, uint64_t* off) {
  const int rc = seq_check(ctx, mask, "lins_gpu_seq_save_size");
  return rc != LINS_OK ? rc : save_size(ctx, ctx->seq.n, mask, off, [ctx](int s) { return seq_bytes(ctx, s); });
}

int lins_gpu_seq_save(lins_ctx* ctx, const uint8_t* mask, void* blob, const uint64_t* off) {
  const int rc = seq_check(ctx, mask, "lins_gpu_seq_save");
  if (rc != LINS_OK) return rc;
  return save(ctx, ctx->seq.n, mask, blob, off, [ctx](int s) { return seq_bytes(ctx, s); }, "offsets differ from lins_gpu_seq_save_size's",
              [&] { return seq_save_run(ctx, mask, static_cast<uint8_t*>(blob), off); });
}

int lins_gpu_seq_load(lins_ctx* ctx, const uint8_t* mask, const void* blob, const uint64_t* off) {
  const char* entry = "lins_gpu_seq_load";
  const int rc = seq_check(ctx, mask, entry);
  if (rc != LINS_OK) return rc;
  const SeqState& q = ctx->seq;
  auto check = [&](int s, const uint8_t* p, uint64_t len, S::View& v) {
    const int rc = check_fresh(ctx, s, entry);
    if (rc != LINS_OK) return rc;
    if (const char* bad = S::parse(p, len, seq_sizes(), v)) return fail(ctx, LINS_E_INVALID, bad);
    const bool bound = v.h.flags & S::kBound;
    if (bound != q.pub.bound) return fail(ctx, LINS_E_INVALID, bound ? "a bound slot blob into an unbound run" : "an unbound slot blob into a bound run");
    if (!(v.h.flags & S::kConfigured) &&
        (std::memcmp(v.sc.consts, q.consts, sizeof(q.consts)) != 0 || std::memcmp(v.sc.init_consts, q.init_consts, sizeof(q.init_consts)) != 0))
      return fail(ctx, LINS_E_INVALID, "an unconfigured slot blob of a run with other open constants");
    return LINS_OK;
  };
  return load<S::View>(ctx, ctx->seq.n, mask, blob, off, check, [&](const std::vector<S::View>& v) { return seq_load_run(ctx, mask, v); });
}

int lins_gpu_mappers_save_size(lins_ctx* ctx, const uint8_t* mask, uint64_t* off) {
  if (!ctx) return LINS_E_INVALID;
  return mapper_save_size(ctx, ctx->mappers, mask, off, "lins_gpu_mappers_save_size");
}

int lins_gpu_mappers_save(lins_ctx* ctx, const uint8_t* mask, void* blob, const uint64_t* off) {
  if (!ctx) return LINS_E_INVALID;
  return mapper_save(ctx, ctx->mappers, mask, blob, off, "lins_gpu_mappers_save");
}

int lins_gpu_mappers_load(lins_ctx* ctx, const uint8_t* mask, const void* blob, const uint64_t* off) {
  if (!ctx) return LINS_E_INVALID;
  return mapper_load(ctx, ctx->mappers, mask, blob, off, "lins_gpu_mappers_load");
}

int lins_gpu_mapper_save_size(lins_ctx* ctx, uint64_t* bytes) {
  if (!ctx) return LINS_E_INVALID;
  if (!bytes) return fail(ctx, LINS_E_INVALID, "null bytes");
  int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  uint64_t off[2];
  if ((rc = mapper_save_size(ctx, ctx->mapper, &all, off, "lins_gpu_mapper_save_size")) != LINS_OK) return rc;
  *bytes = off[1];
  return LINS_OK;
}

int lins_gpu_mapper_save(lins_ctx* ctx, void* blob, uint64_t bytes) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  const uint64_t off[2] = {0, bytes};
  return mapper_save(ctx, ctx->mapper, &all, blob, off, "lins_gpu_mapper_save");
}

int lins_gpu_mapper_load(lins_ctx* ctx, const void* blob, uint64_t bytes) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  const uint64_t off[2] = {0, bytes};
  return mapper_load(ctx, ctx->mapper, &all, blob, off, "lins_gpu_mapper_load");
}

int lins_gpu_mappers_load_phase_ms(lins_ctx* ctx, double* ms) {
  if (!ctx) return LINS_E_INVALID;
  if (!ms) return fail(ctx, LINS_E_INVALID, "null ms");
  if (!ctx->mapper_load_valid) return fail(ctx, LINS_E_NOMAP, "no mapper load has completed on the context");
  std::copy(ctx->mapper_load_ms, ctx->mapper_load_ms + 5, ms);
  return LINS_OK;
}

}  // extern "C"
