// lins_mapper_save.cu — mapping-node slots of the lockstep mappers and of the single mapper saved to host bytes and
// loaded into fresh slots (include/lins_gpu.h: lins_gpu_mappers_save_size / _save / _load, lins_gpu_mapper_save_size /
// _save / _load).  A slot's blob (lins_mapper_blob.hpp) carries what a later step, fuse, download, close_loops or global
// map of the slot reads: its scalars and IMU queue, window, key poses, stored key frames' clouds and scan-to-map loop
// state, and on a slot with loop closure the key-pose graph, its estimate and MapperLoops' scalars.
//   save: one gather launch of every masked slot's device pieces (a plain slot's map-frame key-frame clouds, the loop
//         state) into one staging buffer of the slots' device ranges back to back, one D2H into pinned staging, one
//         synchronisation; the host records are written after it, and a loop slot's body-frame clouds are copied from
//         its host store (the synchronisation orders the copy after the last kernel that wrote them).
//   load: every masked blob validated in full first; then a synchronisation (a queued kernel may still write a chunk a
//         reset handed back), a loop slot's body-frame clouds copied into its host store on the host, one H2D of the
//         blobs (with the rebuild's job table behind them), one gather launch that installs the loop states and fills
//         the plain slots' key frames, and one launch of lins_mapper_rebuild_kernel that writes the transform by the key
//         pose of each key frame a loop slot's device store keeps into that store, c = T(b, pose), as every save and
//         correctPoses leave them (DESIGN.md §4.15); one synchronisation at the end.
// A loop slot's blob carries every key frame (its host store); the loaded device store is the key frames a later window
// can take (lins_slot_blob.hpp's mapper_state_check): the window, the newest key frame and, while the window is short,
// the last 50.
// A call's device and pinned staging is the masked blobs' total (and the job table on a load): a caller bounds it by
// saving and loading with smaller masks.
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

using namespace lins_capi;
namespace B = lins_mblob;

namespace {

static_assert(sizeof(B::PoseRec) == sizeof(MapperKeyPose), "pose record");
static_assert(sizeof(B::EstRec) == sizeof(lins_pg::Pose3), "estimate record");
static_assert(sizeof(lins_pg::Vec6) == 6 * sizeof(double), "variance record");
static_assert(sizeof(lins_map::MapLoopState) % sizeof(float4) == 0, "loop state in float4 records");
// MapperLoops::rebuild is not carried: mapper_cycle_end clears it before anything reads it, and only the step that
// processed the slot reads it, right after (lins_mappers.cu, the correctPoses re-transform)

B::BuildSizes build_sizes() {
  return B::BuildSizes{(uint32_t)sizeof(lins_map::MapLoopState), (uint32_t)LINS_MAPPER_IMU_QUEUE, (uint32_t)LINS_MAPPER_WINDOW,
                       (uint32_t)sizeof(B::FactorRec)};
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

// the stored key frames of a node as (id, device store slot), by id (the blob's order): a plain slot's device store;
// every key frame of a slot with loop closure (its host store; the slot is -1)
std::vector<std::pair<int, int>> stored_keyframes(const MapperNode& m) {
  std::vector<std::pair<int, int>> v;
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

B::Counts node_counts(const MapperNode& m) {
  B::Counts c;
  c.n_poses = (int64_t)m.poses.size();
  c.n_window = (int64_t)m.s.window.size();
  const std::vector<std::pair<int, int>> kf = stored_keyframes(m);
  c.n_keyframes = (int64_t)kf.size();
  for (const auto& k : kf)
    for (int a = 0; a < 3; ++a) c.n_kf_points += kf_sizes(m, k)[a];
  c.n_factors = (int64_t)m.loops.graph.size();
  c.n_est = (int64_t)m.loops.est.size();
  return c;
}

// what every entry checks: an open run that lins_gpu_seq_map_open has not bound, and a mask
int check_run(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, const char* entry) {
  if (ms.n == 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_mappers_open has not been called");
  if (&ms == &ctx->mappers && ctx->seq.pub.bound)  // (the slot's estimator half would be lost: lins_gpu_seq_save saves both)
    return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": the run is bound to sequence mode (lins_gpu_seq_save saves its slots)").c_str());
  if (!mask) return fail(ctx, LINS_E_INVALID, "null mask");
  return LINS_OK;
}

void offsets(const MappersState& ms, const uint8_t* mask, uint64_t* off) {
  off[0] = 0;
  for (int s = 0; s < ms.n; ++s) {
    uint64_t len = 0;
    if (mask[s]) { B::Header h; B::layout(node_counts(ms.node[s]), build_sizes(), h); len = h.total; }
    off[s + 1] = off[s] + len;
  }
}

// one section's record(s) into the host image: the bytes, then zeros up to the next 16-byte boundary
void put(uint8_t* dst, const void* src, size_t bytes) {
  if (bytes) std::memcpy(dst, src, bytes);
  std::memset(dst + bytes, 0, B::align16(bytes) - bytes);
}

// the bytes [lo, hi) of slot s's blob that come from the device: a plain slot's key frames' clouds and the loop state,
// which follows them; a slot with loop closure's loop state (its key frames' clouds come from its host store)
void device_range(const MapperNode& m, const B::Header& h, uint64_t& lo, uint64_t& hi) {
  lo = m.loops.enabled ? h.sec[B::kLoop].off : h.sec[B::kKfClouds].off;
  hi = h.sec[B::kLoop].off + h.sec[B::kLoop].bytes;
}

// the device pieces of slot s's blob, as gather copies into dst (byte lo of the blob's device range in the device
// staging): a plain slot's key frames' clouds (in kf order) and the loop state
void save_copies(MappersState& ms, int s, const B::Header& h, float4* dst, uint64_t lo, const std::vector<std::pair<int, int>>& kf, std::vector<DevCopy>& v) {
  const MapperNode& m = ms.node[s];
  dst -= lo / 16;
  float4* o = dst + h.sec[B::kKfClouds].off / 16;
  for (const auto& k : kf)
    for (int a = 0; a < 3 && !m.loops.enabled; ++a) {
      const MapperKeyFrame& f = m.slots[k.second];
      v.push_back(DevCopy{f.c[a].p, o, f.n[a], 0});
      o += f.n[a];
    }
  v.push_back(DevCopy{reinterpret_cast<const float4*>(ms.stm.loop.p + s), dst + h.sec[B::kLoop].off / 16, (int)(sizeof(lins_map::MapLoopState) / 16), 0});
}

// the host records of slot s's blob into img (its first byte in the caller's buffer), and a loop slot's key-frame clouds
// from its host store
void save_host(const MapperNode& m, const B::Counts& c, B::Header h, uint8_t* img, const std::vector<std::pair<int, int>>& kf) {
  const MapperLoops& L = m.loops;
  h.magic = B::kMagic;
  h.version = B::kVersion;
  h.flags = L.enabled ? B::kLoops : 0u;
  h.sizes = build_sizes();
  h.n_sections = B::kNumSections;
  h.pad = 0;
  put(img, &h, sizeof(h));
  B::Scalars sc;
  std::memset(&sc, 0, sizeof(sc));
  sc.n_poses = (int32_t)c.n_poses; sc.n_window = (int32_t)c.n_window; sc.n_keyframes = (int32_t)c.n_keyframes;
  sc.n_factors = (int32_t)c.n_factors; sc.n_est = (int32_t)c.n_est;
  sc.n_loop = L.n_loop; sc.closed = L.closed ? 1 : 0;
  std::memcpy(sc.cur, L.cur, sizeof(sc.cur));
  sc.time = L.time;
  put(img + h.sec[B::kScalars].off, &sc, sizeof(sc));
  put(img + h.sec[B::kMapper].off, static_cast<const B::MapperRec*>(&m.s), sizeof(B::MapperRec));
  put(img + h.sec[B::kPoses].off, m.poses.data(), sizeof(B::PoseRec) * m.poses.size());
  const std::vector<int32_t> win(m.s.window.begin(), m.s.window.end());
  put(img + h.sec[B::kWindow].off, win.data(), sizeof(int32_t) * win.size());
  std::vector<B::KeyframeRec> tab;
  for (const auto& k : kf) {
    const int* n = kf_sizes(m, k);
    tab.push_back(B::KeyframeRec{k.first, {n[0], n[1], n[2]}});
  }
  put(img + h.sec[B::kKeyframes].off, tab.data(), sizeof(B::KeyframeRec) * tab.size());
  if (L.enabled) {  // the host store's body-frame clouds, in table order (the caller has synchronised the stream)
    uint8_t* o = img + h.sec[B::kKfClouds].off;
    for (const auto& k : kf) {
      const HostKeyFrame& f = m.host[k.first];
      const size_t bytes = sizeof(float4) * ((size_t)f.n[0] + f.n[1] + f.n[2]);
      if (bytes) std::memcpy(o, f.p, bytes);
      o += bytes;
    }
  }
  std::vector<B::FactorRec> fac(L.graph.size());
  for (size_t i = 0; i < L.graph.size(); ++i) {
    const lins_pg::Factor& f = L.graph[i];
    B::FactorRec& r = fac[i];
    r.a = f.a; r.b = f.b;
    std::memcpy(r.R, f.z.R, sizeof(r.R));
    std::memcpy(r.t, f.z.t, sizeof(r.t));
    std::copy(f.var.begin(), f.var.end(), r.var);
  }
  put(img + h.sec[B::kFactors].off, fac.data(), sizeof(B::FactorRec) * fac.size());
  put(img + h.sec[B::kEst].off, L.est.data(), sizeof(B::EstRec) * L.est.size());
}

// the device part of a save on checked arguments (a failure ends the run)
int save_run(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, uint8_t* blob, const uint64_t* off) {
  const int n = ms.n;
  CK(cudaSetDevice(ctx->device));
  std::vector<B::Counts> counts(n);
  std::vector<B::Header> hdr(n);
  std::vector<std::vector<std::pair<int, int>>> kf(n);
  std::vector<uint64_t> lo(n, 0), hi(n, 0), doff(n + 1, 0);  // each slot's device range, and its place in the staging
  for (int s = 0; s < n; ++s) {
    doff[s + 1] = doff[s];
    if (!mask[s]) continue;
    counts[s] = node_counts(ms.node[s]);
    B::layout(counts[s], build_sizes(), hdr[s]);
    kf[s] = stored_keyframes(ms.node[s]);
    device_range(ms.node[s], hdr[s], lo[s], hi[s]);
    doff[s + 1] += hi[s] - lo[s];
  }
  const uint64_t total = doff[n];
  CK(ms.blob.reserve(total / 16 + 1)); CK(ms.h_blob.reserve(total / 16 + 1));
  std::vector<DevCopy> copies;
  for (int s = 0; s < n; ++s)
    if (mask[s]) save_copies(ms, s, hdr[s], ms.blob.p + doff[s] / 16, lo[s], kf[s], copies);
  copies.erase(std::remove_if(copies.begin(), copies.end(), [](const DevCopy& c) { return c.n <= 0; }), copies.end());
  int rc = ms.copies.reserve(ctx, copies.size());
  if (rc == LINS_OK) rc = ms.copies.stage(ctx, copies.data(), (int)copies.size(), 0);
  if (rc == LINS_OK) rc = ms.copies.launch(ctx, 0, (int)copies.size());
  if (rc != LINS_OK) return rc;
  const uint8_t* img = reinterpret_cast<const uint8_t*>(ms.h_blob.p);
  CK(cudaMemcpyAsync(ms.h_blob.p, ms.blob.p, total, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    std::memcpy(blob + off[s] + lo[s], img + doff[s], hi[s] - lo[s]);
    save_host(ms.node[s], counts[s], hdr[s], blob + off[s], kf[s]);
  }
  return LINS_OK;
}

// the device and host part of a load on validated blobs v (masked slots; a failure ends the run).  ph: the host
// phases (allocation, staging, device, bookkeeping; ph[0], the validation, is the caller's)
int load_run(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, const std::vector<B::View>& v, double* ph) {
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
      for (int i = 0; i < v[s].sc.n_keyframes; ++i) {
        const B::KeyframeRec k = v[s].keyframe(i);
        for (int a = 0; a < 3; ++a) n_jobs += k.n[a] > 0;  // (a bound: only the device store's key frames get jobs)
      }
  }
  const uint64_t job_off = B::align16(total), staged = job_off + sizeof(KfRebuild) * n_jobs;
  CK(ms.blob.reserve(staged / 16 + 1)); CK(ms.h_blob.reserve(staged / 16 + 1));
  auto at = [&](int s, int sec) { return ms.blob.p + (base[s] + v[s].h.sec[sec].off) / 16; };
  // every buffer first: each device-store key frame's slot (a free one first) and its clouds, and each loop slot's host
  // store blocks
  std::vector<DevCopy> copies;
  std::vector<KfRebuild> jobs;
  std::vector<std::pair<float4*, const uint8_t*>> host_fill;  // (host-store block, its clouds in the caller's blob)
  std::vector<size_t> host_bytes;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    const B::View& b = v[s];
    MapperNode& m = ms.node[s];
    copies.push_back(DevCopy{at(s, B::kLoop), reinterpret_cast<float4*>(ms.stm.loop.p + s), (int)(sizeof(lins_map::MapLoopState) / 16), 0});
    const float4* src = at(s, B::kKfClouds);
    const uint8_t* hsrc = b.at(B::kKfClouds);
    std::vector<unsigned char> keep;  // a loop slot: the key frames its device store keeps
    if (b.loops()) {
      const int np = b.sc.n_poses;
      keep.assign(np, 0);
      for (int i = 0; i < b.sc.n_window; ++i) keep[b.window(i)] = 1;
      if (np > 0) keep[np - 1] = 1;
      if (b.sc.n_window < LINS_MAPPER_WINDOW)
        for (int id = std::max(0, np - LINS_MAPPER_WINDOW); id < np; ++id) keep[id] = 1;
      m.host.assign(np, HostKeyFrame());
    }
    for (int i = 0; i < b.sc.n_keyframes; ++i) {
      const B::KeyframeRec k = b.keyframe(i);
      if (b.loops()) {
        HostKeyFrame& hk = m.host[k.id];
        std::copy(k.n, k.n + 3, hk.n);
        const size_t bytes = sizeof(float4) * ((size_t)k.n[0] + k.n[1] + k.n[2]);
        void* p = nullptr;
        if (!ms.store.take(m.held, bytes, &p)) return fail(ctx, LINS_E_CUDA, "the host key-frame store could not allocate pinned memory");
        hk.p = static_cast<float4*>(p);
        if (bytes) { host_fill.push_back({hk.p, hsrc}); host_bytes.push_back(bytes); }
        hsrc += bytes;
        if (!keep[k.id]) { src += k.n[0] + k.n[1] + k.n[2]; continue; }
      }
      int slot;
      if (!m.free_slots.empty()) { slot = m.free_slots.back(); m.free_slots.pop_back(); }
      else { slot = (int)m.slots.size(); m.slots.emplace_back(); }
      m.slot_of[k.id] = slot;
      MapperKeyFrame& f = m.slots[slot];
      MapperKeyPose kp;
      const B::PoseRec pr = b.pose(k.id);
      std::memcpy(&kp, &pr, sizeof(kp));
      const TfConsts tc = tf_consts(kp);
      for (int a = 0; a < 3; ++a) {
        f.n[a] = k.n[a];
        CK(f.c[a].grow((size_t)k.n[a] + 1));
        if (b.loops()) {
          if (k.n[a]) jobs.push_back(KfRebuild{src, f.c[a].p, k.n[a], 0, tc});
        } else {
          copies.push_back(DevCopy{src, f.c[a].p, k.n[a], 0});
        }
        src += k.n[a];
      }
    }
  }
  copies.erase(std::remove_if(copies.begin(), copies.end(), [](const DevCopy& c) { return c.n <= 0; }), copies.end());
  int rc;
  if ((rc = ms.copies.reserve(ctx, copies.size())) != LINS_OK) return rc;
  ph[1] = ms_since(t);

  // the loop slots' host stores, the blobs and the job table into the pinned image
  for (size_t i = 0; i < host_fill.size(); ++i) std::memcpy(host_fill[i].first, host_fill[i].second, host_bytes[i]);
  uint8_t* img = reinterpret_cast<uint8_t*>(ms.h_blob.p);
  for (int s = 0; s < n; ++s) if (mask[s]) std::memcpy(img + base[s], v[s].p, v[s].h.total);
  if (!jobs.empty()) std::memcpy(img + job_off, jobs.data(), sizeof(KfRebuild) * jobs.size());
  ph[2] = ms_since(t);

  // one H2D, one gather launch, one rebuild launch, one synchronisation
  CK(cudaMemcpyAsync(ms.blob.p, img, staged, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = ms.copies.stage(ctx, copies.data(), (int)copies.size(), 0)) != LINS_OK) return rc;
  if ((rc = ms.copies.launch(ctx, 0, (int)copies.size())) != LINS_OK) return rc;
  if (!jobs.empty()) {
    lins_mapper_rebuild_kernel<<<(unsigned)jobs.size(), 256, 0, ctx->stream>>>(reinterpret_cast<const KfRebuild*>(ms.blob.p + job_off / 16));
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  CK(cudaStreamSynchronize(ctx->stream));
  ph[3] = ms_since(t);

  // the host bookkeeping of the loaded slots: the blob's scalars, key poses and loop closure; no outputs of a last cycle
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    const B::View& b = v[s];
    const B::Scalars& sc = b.sc;
    MapperNode& m = ms.node[s];
    static_cast<B::MapperRec&>(m.s) = b.m;
    m.s.window.clear();
    for (int i = 0; i < sc.n_window; ++i) m.s.window.push_back(b.window(i));
    m.poses.resize(sc.n_poses);
    for (int i = 0; i < sc.n_poses; ++i) { const B::PoseRec p = b.pose(i); std::memcpy(&m.poses[i], &p, sizeof(p)); }
    MapperLoops L;
    L.enabled = b.loops();
    L.closed = sc.closed != 0;
    L.n_loop = sc.n_loop;
    std::memcpy(L.cur, sc.cur, sizeof(L.cur));
    L.time = sc.time;
    for (int i = 0; i < sc.n_factors; ++i) {
      const B::FactorRec r = b.factor(i);
      lins_pg::Factor f;
      f.a = r.a; f.b = r.b;
      std::memcpy(f.z.R, r.R, sizeof(r.R));
      std::memcpy(f.z.t, r.t, sizeof(r.t));
      std::copy(r.var, r.var + 6, f.var.begin());
      L.graph.push_back(f);
    }
    L.est.resize(sc.n_est);
    for (int i = 0; i < sc.n_est; ++i) { const B::EstRec e = b.est(i); std::memcpy(&L.est[i], &e, sizeof(e)); }
    m.loops = std::move(L);
    m.last = MapperLast();        // (no DS clouds until the slot's next processed cycle)
    m.gm = MapperGlobalMap();     // (no global map until the slot's next global-map call)
    m.stepped = true;             // (a loaded node is not fresh: loop closure cannot be enabled on it)
  }
  ph[4] = ms_since(t);
  return LINS_OK;
}

int save_size(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, uint64_t* off, const char* entry) {
  const int rc = check_run(ctx, ms, mask, entry);
  if (rc != LINS_OK) return rc;
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  offsets(ms, mask, off);
  return LINS_OK;
}

int save(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, void* blob, const uint64_t* off, const char* entry) {
  int rc = check_run(ctx, ms, mask, entry);
  if (rc != LINS_OK) return rc;
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  const int n = ms.n;
  std::vector<uint64_t> want((size_t)n + 1);
  offsets(ms, mask, want.data());
  if (!std::equal(want.begin(), want.end(), off)) return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": offsets differ from the save size's").c_str());
  if (want[n] == 0) return LINS_OK;
  if (!blob) return fail(ctx, LINS_E_INVALID, "null blob");
  rc = save_run(ctx, ms, mask, static_cast<uint8_t*>(blob), off);
  if (rc != LINS_OK) ms.n = 0;
  return rc;
}

int load(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, const void* blob, const uint64_t* off, const char* entry) {
  auto t = std::chrono::steady_clock::now();
  int rc = check_run(ctx, ms, mask, entry);
  if (rc != LINS_OK) return rc;
  if (!off) return fail(ctx, LINS_E_INVALID, "null offsets");
  const int n = ms.n;
  const uint8_t* p = static_cast<const uint8_t*>(blob);
  std::vector<B::View> v(n);
  bool any = false;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    any = true;
    if (!p) return fail(ctx, LINS_E_INVALID, "null blob");
    if (off[s + 1] < off[s]) return fail(ctx, LINS_E_INVALID, "blob offsets decrease");
    if (ms.node[s].stepped) return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": a masked slot is not fresh (present in a step since open / reset)").c_str());
    const char* bad = B::parse(p + off[s], off[s + 1] - off[s], build_sizes(), v[s]);
    if (bad) return fail(ctx, LINS_E_INVALID, bad);
  }
  if (!any) return LINS_OK;
  double ph[5];
  ph[0] = ms_since(t);
  rc = load_run(ctx, ms, mask, v, ph);
  if (rc != LINS_OK) { ms.n = 0; return rc; }
  std::copy(ph, ph + 5, ctx->mapper_load_ms);
  ctx->mapper_load_valid = true;
  return LINS_OK;
}

// the single mapper: a run of one slot of its own, opened by the first lins_gpu_mapper_* call on the context
int mapper_open(lins_ctx* ctx) {
  return ctx->mapper.n > 0 ? LINS_OK : mappers_open(ctx, ctx->mapper, 1);
}

}  // namespace

extern "C" {

int lins_gpu_mappers_save_size(lins_ctx* ctx, const uint8_t* mask, uint64_t* off) {
  if (!ctx) return LINS_E_INVALID;
  return save_size(ctx, ctx->mappers, mask, off, "lins_gpu_mappers_save_size");
}

int lins_gpu_mappers_save(lins_ctx* ctx, const uint8_t* mask, void* blob, const uint64_t* off) {
  if (!ctx) return LINS_E_INVALID;
  return save(ctx, ctx->mappers, mask, blob, off, "lins_gpu_mappers_save");
}

int lins_gpu_mappers_load(lins_ctx* ctx, const uint8_t* mask, const void* blob, const uint64_t* off) {
  if (!ctx) return LINS_E_INVALID;
  return load(ctx, ctx->mappers, mask, blob, off, "lins_gpu_mappers_load");
}

int lins_gpu_mapper_save_size(lins_ctx* ctx, uint64_t* bytes) {
  if (!ctx) return LINS_E_INVALID;
  if (!bytes) return fail(ctx, LINS_E_INVALID, "null bytes");
  int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  uint64_t off[2];
  if ((rc = save_size(ctx, ctx->mapper, &all, off, "lins_gpu_mapper_save_size")) != LINS_OK) return rc;
  *bytes = off[1];
  return LINS_OK;
}

int lins_gpu_mapper_save(lins_ctx* ctx, void* blob, uint64_t bytes) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  const uint64_t off[2] = {0, bytes};
  return save(ctx, ctx->mapper, &all, blob, off, "lins_gpu_mapper_save");
}

int lins_gpu_mapper_load(lins_ctx* ctx, const void* blob, uint64_t bytes) {
  if (!ctx) return LINS_E_INVALID;
  const int rc = mapper_open(ctx);
  if (rc != LINS_OK) return rc;
  const uint8_t all = 1;
  const uint64_t off[2] = {0, bytes};
  return load(ctx, ctx->mapper, &all, blob, off, "lins_gpu_mapper_load");
}

int lins_gpu_mappers_load_phase_ms(lins_ctx* ctx, double* ms) {
  if (!ctx) return LINS_E_INVALID;
  if (!ms) return fail(ctx, LINS_E_INVALID, "null ms");
  if (!ctx->mapper_load_valid) return fail(ctx, LINS_E_NOMAP, "no mapper load has completed on the context");
  std::copy(ctx->mapper_load_ms, ctx->mapper_load_ms + 5, ms);
  return LINS_OK;
}

}  // extern "C"
