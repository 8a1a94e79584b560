// lins_mapper_blob.hpp — the byte format of one saved mapping-node slot of the lockstep mappers or the single mapper
// (lins_gpu_mappers_save / _load, lins_gpu_mapper_save / _load, lins_checkpoint.cu): its records, its layout and its
// validation, on the core of lins_blob.hpp.  One format for both APIs: a blob of either loads into the other.  Plain C++
// with no CUDA, so the CPU suite compiles it with g++ (tests/test_mapper_checkpoint_cpu.py).
#pragma once
#include "lins_blob.hpp"

namespace lins_mblob {

// Sections: scalars (Scalars: the counts, then MapperLoops' closed, n_loop, cur and time), the node's sections, factors
// (a FactorRec per factor of the key-pose graph, in its order) and est (an EstRec per key pose: isamCurrentEstimate of
// the last save).  A plain slot's kfclouds are in the map frame (c); a slot with loop closure keeps every key frame, in
// the body frame (b), and its loader rebuilds c = T(b, pose) for those a later window can take.  The graph, estimate and
// body-frame store sections are those of lins_capi::MapperLoops / HostKeyFrame as they are, so that a later
// sequence-mode format could carry a slot with loop closure in the same records.
using lins_blob::KeyframeRec;
using lins_blob::MapperRec;
using lins_blob::NodeSecs;
using lins_blob::NodeView;
using lins_blob::PoseRec;
using lins_blob::SectionRec;
using lins_blob::rec;

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
  h.total = lins_blob::section_table(sizeof(Header), bytes, kNumSections, h.sec);
}
inline NodeSecs node_secs(const Header& h) {
  return {h.sec[kMapper].off, h.sec[kPoses].off, h.sec[kWindow].off, h.sec[kKeyframes].off, h.sec[kKfClouds].off, h.sec[kLoop].off};
}

// a parsed blob: the header and scalar records copied out
struct View : NodeView {
  Header h;
  Scalars sc;
  bool loops() const { return h.flags & kLoops; }
  const uint8_t* at(int section) const { return p + h.sec[section].off; }
  FactorRec factor(int i) const { return rec<FactorRec>(at(kFactors), i); }
  EstRec est(int i) const { return rec<EstRec>(at(kEst), i); }
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
  if (const char* bad = lins_blob::check_envelope(h, len, "mapper", kMagic, kVersion, kLoops, sz, h.n_sections == kNumSections && h.pad == 0, sizeof(Scalars)))
    return bad;
  v.sc = rec<Scalars>(v.at(kScalars), 0);
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
  v.node = node_secs(h);
  v.n_poses = s.n_poses; v.n_window = s.n_window; v.n_keyframes = s.n_keyframes;
  Counts c;
  c.n_poses = s.n_poses; c.n_window = s.n_window; c.n_keyframes = s.n_keyframes; c.n_factors = s.n_factors; c.n_est = s.n_est;
  std::vector<int32_t> ids;
  if (const char* bad = lins_blob::check_keyframes(v, "mapper", ids, c.n_kf_points)) return bad;
  Header want;
  layout(c, sz, want);
  if (want.total != len || std::memcmp(want.sec, h.sec, sizeof(h.sec)) != 0) return "mapper blob section table differs from its counts";
  v.m = rec<MapperRec>(v.at(kMapper), 0);
  if (const char* bad = lins_blob::mapper_state_check(v, ids)) return bad;
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
