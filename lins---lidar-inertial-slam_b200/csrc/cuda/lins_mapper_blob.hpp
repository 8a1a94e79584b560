// lins_mapper_blob.hpp — the byte format of one saved mapping-node slot of the lockstep mappers or the single mapper
// (lins_gpu_mappers_save / _load, lins_gpu_mapper_save / _load, lins_mapper_save.cu): its records, its layout and its
// validation.  Plain C++ with no CUDA, so the CPU suite compiles it with g++ (tests/test_mapper_checkpoint_cpu.py).
// One format for both APIs: a blob of either loads into the other.
//
// A blob is a header, then sections at 16-byte offsets in a fixed order, each sized by the counts of the scalar section
// (so the section table is fully determined by them, and a loader checks it is exactly that):
//   scalars   Scalars: the counts, then MapperLoops' closed, n_loop, cur and time
//   mapper    lins_blob::MapperRec: the node's scalars and IMU queue
//   poses     lins_blob::PoseRec per key pose
//   window    int32 key-frame ids, oldest first (the deque as it is, its duplicate id included)
//   keyframes lins_blob::KeyframeRec per stored key frame, by id
//   kfclouds  each stored key frame's corner, surf and outlier clouds, in table order, as float4 runs: in the map frame
//             (c) on a plain slot, in the body frame (b) on a slot with loop closure, whose loader rebuilds c = T(b, pose)
//   loop      the scan-to-map loop state (the build's MapLoopState bytes)
//   factors   FactorRec per factor of the key-pose graph, in its order (slots with loop closure)
//   est       EstRec per key pose: isamCurrentEstimate of the last save (slots with loop closure)
// The blob records the build's record sizes, and a build whose sizes differ rejects it.  The factor, estimate and
// body-frame store sections are the graph and store of lins_capi::MapperLoops / MapperKeyFrame as they are, so that a
// later sequence-mode format could carry a slot with loop closure in the same records.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../../include/lins_gpu.h"
#include "lins_slot_blob.hpp"

namespace lins_mblob {

using lins_blob::align16;
using lins_blob::KeyframeRec;
using lins_blob::MapperRec;
using lins_blob::PoseRec;
using lins_blob::SectionRec;

constexpr uint64_t kMagic = 0x5250414d534e494cull;  // "LINSMAPR" in little-endian byte order
constexpr uint32_t kVersion = 1;
enum Flags : uint32_t { kLoops = 1u };  // the slot has loop closure enabled
enum Section { kScalars, kMapper, kPoses, kWindow, kKeyframes, kKfClouds, kLoop, kFactors, kEst, kNumSections };

// a factor of the key-pose graph (lins_pg::Factor): keys a, b (b = -1: the prior on a), the measurement z as R
// (row-major) and t, and the variance of each of its six components
struct FactorRec {
  int32_t a, b;
  double R[9], t[3], var[6];
};
static_assert(sizeof(FactorRec) == 8 + 18 * sizeof(double), "FactorRec without padding");
struct EstRec { double R[9], t[3]; };  // lins_pg::Pose3
static_assert(sizeof(EstRec) == 12 * sizeof(double), "EstRec without padding");

// the record sizes of the build that wrote a blob
struct BuildSizes {
  uint32_t loop_state, imu_queue, window, factor;
};
struct Header {
  uint64_t magic;
  uint32_t version, flags;
  BuildSizes sizes;
  uint32_t n_sections, pad;
  uint64_t total;  // the blob's length in bytes
  SectionRec sec[kNumSections];
};
static_assert(sizeof(Header) % 16 == 0, "header");

struct Scalars {
  int32_t n_poses, n_window, n_keyframes, n_factors, n_est;
  int32_t n_loop, closed;  // MapperLoops: loop factors in the graph, aLoopIsClosed
  float cur[3];            // currentRobotPosPoint of the last processed cycle
  double time;             // timeLaserOdometry of the last odometry message
};
static_assert(sizeof(Scalars) == 10 * 4 + 8, "Scalars without padding");

// what the section sizes depend on
struct Counts {
  int64_t n_poses = 0, n_window = 0, n_keyframes = 0, n_kf_points = 0, n_factors = 0, n_est = 0;
};

// the section table and total length of a blob with counts c (h.sec, h.total; nothing else of h)
inline void layout(const Counts& c, const BuildSizes& sz, Header& h) {
  const uint64_t bytes[kNumSections] = {
      sizeof(Scalars),
      sizeof(MapperRec),
      sizeof(PoseRec) * uint64_t(c.n_poses),
      sizeof(int32_t) * uint64_t(c.n_window),
      sizeof(KeyframeRec) * uint64_t(c.n_keyframes),
      16 * uint64_t(c.n_kf_points),
      sz.loop_state,
      sizeof(FactorRec) * uint64_t(c.n_factors),
      sizeof(EstRec) * uint64_t(c.n_est)};
  uint64_t o = align16(sizeof(Header));
  for (int i = 0; i < kNumSections; ++i) {
    h.sec[i].off = o;
    h.sec[i].bytes = bytes[i];
    o = align16(o + bytes[i]);
  }
  h.total = o;
}

// a parsed blob: the header and scalar records copied out, the rest left in place (p: the blob's first byte; it need
// not be aligned, so records are read with memcpy)
struct View {
  const uint8_t* p = nullptr;
  Header h;
  Scalars sc;
  MapperRec m;
  bool loops() const { return h.flags & kLoops; }
  const uint8_t* at(int section) const { return p + h.sec[section].off; }
  PoseRec pose(int i) const { PoseRec r; std::memcpy(&r, at(kPoses) + sizeof(PoseRec) * i, sizeof(r)); return r; }
  int32_t window(int i) const { int32_t r; std::memcpy(&r, at(kWindow) + sizeof(int32_t) * i, sizeof(r)); return r; }
  KeyframeRec keyframe(int i) const { KeyframeRec r; std::memcpy(&r, at(kKeyframes) + sizeof(KeyframeRec) * i, sizeof(r)); return r; }
  FactorRec factor(int i) const { FactorRec r; std::memcpy(&r, at(kFactors) + sizeof(FactorRec) * i, sizeof(r)); return r; }
  EstRec est(int i) const { EstRec r; std::memcpy(&r, at(kEst) + sizeof(EstRec) * i, sizeof(r)); return r; }
};

inline bool finite_n(const double* v, int n) {
  for (int i = 0; i < n; ++i) if (!std::isfinite(v[i])) return false;
  return true;
}

// Validates the len bytes at p as a mapper blob of a build with record sizes sz and fills v.  Returns nullptr when the
// blob is well formed, else what is wrong.  Every count, offset and id a loader uses is checked here, so that a blob
// that passes cannot make it read or write out of bounds.
inline const char* parse(const uint8_t* p, uint64_t len, const BuildSizes& sz, View& v) {
  v.p = p;
  if (!p || len < sizeof(Header)) return "blob shorter than its header";
  std::memcpy(&v.h, p, sizeof(Header));
  const Header& h = v.h;
  if (h.magic != kMagic) return "not a mapper blob (bad magic)";
  if (h.version != kVersion) return "mapper blob of another format version";
  if (std::memcmp(&h.sizes, &sz, sizeof(sz)) != 0) return "mapper blob of another library build (record sizes differ)";
  if (h.flags & ~uint32_t(kLoops)) return "bad mapper blob flags";
  if (h.n_sections != kNumSections || h.pad != 0) return "bad mapper blob section count";
  if (h.total != len) return "mapper blob length differs from its header's";
  for (int i = 0; i < kNumSections; ++i)
    if (h.sec[i].off % 16 || h.sec[i].off < sizeof(Header) || h.sec[i].off > len || h.sec[i].bytes > len - h.sec[i].off)
      return "mapper blob section outside the blob";
  if (h.sec[kScalars].bytes != sizeof(Scalars)) return "bad mapper blob scalar section";
  std::memcpy(&v.sc, v.at(kScalars), sizeof(Scalars));
  const Scalars& s = v.sc;
  const bool loops = v.loops();
  if (s.n_poses < 0 || s.n_window < 0 || s.n_keyframes < 0 || s.n_factors < 0 || s.n_est < 0 || s.n_loop < 0)
    return "negative count in mapper blob";
  if (s.n_window > LINS_MAPPER_WINDOW) return "mapper blob window longer than the mapper's";
  if (s.n_keyframes > s.n_poses) return "mapper blob stores more key frames than key poses";
  if (!loops && s.n_keyframes > lins_blob::kMaxKeyframes) return "mapper blob stores more than 51 key frames";
  if (s.closed != 0 && s.closed != 1) return "bad closed flag in mapper blob";
  if (!std::isfinite(s.time)) return "non-finite odometry time in mapper blob";
  if (!loops && (s.n_factors || s.n_est || s.n_loop || s.closed)) return "mapper blob without loop closure has a key-pose graph";
  // the tables, once their sections are known to lie in the blob with the sizes the counts give
  if (h.sec[kPoses].bytes != sizeof(PoseRec) * (uint64_t)s.n_poses || h.sec[kKeyframes].bytes != sizeof(KeyframeRec) * (uint64_t)s.n_keyframes ||
      h.sec[kFactors].bytes != sizeof(FactorRec) * (uint64_t)s.n_factors)
    return "bad mapper blob pose, key-frame or factor section";
  Counts c;
  c.n_poses = s.n_poses; c.n_window = s.n_window; c.n_keyframes = s.n_keyframes; c.n_factors = s.n_factors; c.n_est = s.n_est;
  std::vector<int32_t> ids(s.n_keyframes);
  std::vector<unsigned char> seen(s.n_poses, 0);
  for (int i = 0; i < s.n_keyframes; ++i) {
    const KeyframeRec k = v.keyframe(i);
    if (k.id < 0 || k.id >= s.n_poses) return "mapper blob key frame of no key pose";
    if (seen[k.id]) return "mapper blob stores a key frame twice";
    seen[k.id] = 1;
    ids[i] = k.id;
    for (int a = 0; a < 3; ++a) {
      if (k.n[a] < 0) return "negative key-frame cloud count in mapper blob";
      c.n_kf_points += k.n[a];
    }
  }
  if (c.n_kf_points > INT32_MAX) return "mapper blob key-frame clouds too large";
  Header want;
  layout(c, sz, want);
  if (want.total != len || std::memcmp(want.sec, h.sec, sizeof(h.sec)) != 0) return "mapper blob section table differs from its counts";
  std::memcpy(&v.m, v.at(kMapper), sizeof(MapperRec));
  const char* bad = lins_blob::mapper_state_check(v.m, s.n_poses, s.n_window, [&](int i) { return v.window(i); }, ids.data(), s.n_keyframes);
  if (bad) return bad;
  if (!loops) return nullptr;
  // a slot with loop closure keeps every key frame (correctPoses re-transforms them all), and an estimate per key pose
  if (s.n_keyframes != s.n_poses) return "mapper blob with loop closure lacks a key pose's key frame";
  if (s.n_est != s.n_poses) return "mapper blob with loop closure has an estimate count other than its key poses'";
  if (s.closed && s.n_loop < 1) return "mapper blob closed a loop without a loop factor";
  // the graph as mapper_loops_save and close_loops build it: the prior (0, -1) first, then the chain factors (n - 1, n) in
  // increasing n, one per later key pose, and n_loop loop factors (latest, closest) among them, both ends key poses
  int32_t chain = 1, n_loop = 0;
  for (int i = 0; i < s.n_factors; ++i) {
    const FactorRec f = v.factor(i);
    if (!finite_n(f.R, 9) || !finite_n(f.t, 3) || !finite_n(f.var, 6)) return "non-finite factor in mapper blob";
    for (int k = 0; k < 6; ++k) if (!(f.var[k] > 0)) return "mapper blob factor with a variance <= 0";
    if (i == 0) {
      if (f.a != 0 || f.b != -1) return "mapper blob graph does not start with the prior";
    } else if (f.b == f.a + 1) {
      if (f.b != chain) return "mapper blob chain factor out of order";
      ++chain;
    } else {
      if (f.a < 0 || f.a >= s.n_poses || f.b < 0 || f.b >= s.n_poses) return "mapper blob loop factor of no key pose";
      ++n_loop;
    }
  }
  if (s.n_poses > 0 && s.n_factors == 0) return "mapper blob graph does not start with the prior";
  if (s.n_poses > 0 ? chain != s.n_poses : s.n_factors != 0) return "mapper blob chain factors differ from its key poses";
  if (n_loop != s.n_loop) return "mapper blob loop factors differ from its loop count";
  for (int i = 0; i < s.n_est; ++i) {
    const EstRec e = v.est(i);
    if (!finite_n(e.R, 9) || !finite_n(e.t, 3)) return "non-finite estimate in mapper blob";
  }
  return nullptr;
}

}  // namespace lins_mblob
