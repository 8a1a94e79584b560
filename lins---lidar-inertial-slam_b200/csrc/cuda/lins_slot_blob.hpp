// lins_slot_blob.hpp — the byte format of one saved sequence-mode slot (lins_gpu_seq_save / lins_gpu_seq_load,
// lins_seq_save.cu): its records, its layout and its validation.  Plain C++ with no CUDA, so the CPU suite compiles it
// with g++ (tests/test_seq_checkpoint_cpu.py).
//
// A blob is a header, then sections at 16-byte offsets in a fixed order, each sized by the counts of the scalar
// section (so the section table is fully determined by them, and a loader checks it is exactly that):
//   scalars   Scalars: fusion status, stale flag, YZX flag, counts, the run's open constants, config, tuning, pose
//   rows      the filter, covariance, global, linearisation, imu_last and pre-integration rows (kRowDoubles doubles)
//   maps      map_s, map_c, tree_s, tree_c as float4 runs
//   outlier   the published outlier cloud (bound runs)
//   mapper    MapperRec: the mapping node's scalars (bound runs)
//   poses     PoseRec per key pose
//   window    int32 key-frame ids, oldest first (duplicates kept)
//   keyframes KeyframeRec per stored key frame
//   kfclouds  each stored key frame's corner, surf and outlier clouds, in table order, as float4 runs
//   loop      the scan-to-map loop state (the build's MapLoopState bytes; bound runs)
// The blob records the build's record sizes, and a build whose sizes differ rejects it.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>

#include "../../../include/lins_gpu.h"

namespace lins_blob {

constexpr uint64_t kMagic = 0x544f4c53534e494cull;  // "LINSSLOT" in little-endian byte order
constexpr uint32_t kVersion = 1;
enum Flags : uint32_t { kBound = 1u, kConfigured = 2u, kTuned = 4u };
enum Section { kScalars, kRows, kMaps, kOutlier, kMapper, kPoses, kWindow, kKeyframes, kKfClouds, kLoop, kNumSections };
constexpr int kMaxKeyframes = LINS_MAPPER_WINDOW + 1;  // the store keeps the window and the newest key frame
// filt (20), cov (324), glob (20), lin (20), imu_last (8), pre (20): the device rows of one slot, back to back
constexpr int kRowDoubles = 20 + 324 + 20 + 20 + 8 + 20;
constexpr int kRowOff[6] = {0, 20, 344, 364, 384, 392};
// StateEstimator::FusionStatus values a slot can be in
constexpr int32_t kFusionInit = 0, kFusionFirstScan = 1, kFusionRunning = 3;

// the record sizes of the build that wrote a blob
struct BuildSizes {
  uint32_t icp_state, loop_state, imu_queue, n_consts, n_init_consts;
};
struct SectionRec { uint64_t off, bytes; };
struct Header {
  uint64_t magic;
  uint32_t version, flags;
  BuildSizes sizes;
  uint32_t n_sections;
  uint64_t total;  // the blob's length in bytes
  SectionRec sec[kNumSections];
};
static_assert(sizeof(Header) % 16 == 0, "header");

struct Scalars {
  int32_t fusion, stale, yzx, pad;
  int32_t n_map[4];                    // map_s, map_c, tree_s, tree_c points
  int32_t n_outlier, n_poses, n_window, n_keyframes;
  double consts[10], init_consts[24];  // the source run's open-time constants (lins_seq::Consts, InitConsts)
  lins_slot_config cfg;                // read when kConfigured
  lins_slot_tuning tune;               // read when kTuned
  double align_R[9];                   // the tuning's alignIMUtoVehicle rotation
  double pose[7];                      // globalStateYZX_ (bound runs)
};
// the mapping node's scalar members (the base of lins_ctx.hpp's MapperScalars, which adds the window)
struct MapperRec {
  float transformLast[6], transformSum[6], transformIncre[6], transformTobeMapped[6], transformBefMapped[6], transformAftMapped[6];
  double imuTime[LINS_MAPPER_IMU_QUEUE];
  float imuRoll[LINS_MAPPER_IMU_QUEUE], imuPitch[LINS_MAPPER_IMU_QUEUE];
  int32_t imuPointerFront, imuPointerLast;
  double timeLastProcessing;
  int32_t latestFrameID;
  float previousRobotPos[3];
};
// a saved node's record is copied into the blob as it is: it must have no padding bytes, which would not be zero
static_assert(sizeof(MapperRec) == sizeof(float) * (36 + 2 * LINS_MAPPER_IMU_QUEUE + 3) + sizeof(double) * (LINS_MAPPER_IMU_QUEUE + 1) +
                                       sizeof(int32_t) * 3,
              "MapperRec without padding");
struct PoseRec { float x, y, z, roll, pitch, yaw; double time; };  // PointTypePose
struct KeyframeRec { int32_t id, n[3]; };                           // corner, surf, outlier points

// what the section sizes depend on
struct Counts {
  bool bound = false;
  int64_t n_map[4] = {0, 0, 0, 0};
  int64_t n_outlier = 0, n_poses = 0, n_window = 0, n_keyframes = 0, n_kf_points = 0;
};

inline uint64_t align16(uint64_t x) { return (x + 15) & ~uint64_t(15); }

// the section table and total length of a blob with counts c (h.sec, h.total; nothing else of h)
inline void layout(const Counts& c, const BuildSizes& sz, Header& h) {
  const uint64_t bytes[kNumSections] = {
      sizeof(Scalars),
      sizeof(double) * kRowDoubles,
      16 * uint64_t(c.n_map[0] + c.n_map[1] + c.n_map[2] + c.n_map[3]),
      16 * uint64_t(c.n_outlier),
      c.bound ? sizeof(MapperRec) : 0,
      sizeof(PoseRec) * uint64_t(c.n_poses),
      sizeof(int32_t) * uint64_t(c.n_window),
      sizeof(KeyframeRec) * uint64_t(c.n_keyframes),
      16 * uint64_t(c.n_kf_points),
      c.bound ? sz.loop_state : 0};
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
  const uint8_t* at(int section) const { return p + h.sec[section].off; }
  PoseRec pose(int i) const { PoseRec r; std::memcpy(&r, at(kPoses) + sizeof(PoseRec) * i, sizeof(r)); return r; }
  int32_t window(int i) const { int32_t r; std::memcpy(&r, at(kWindow) + sizeof(int32_t) * i, sizeof(r)); return r; }
  KeyframeRec keyframe(int i) const { KeyframeRec r; std::memcpy(&r, at(kKeyframes) + sizeof(KeyframeRec) * i, sizeof(r)); return r; }
};

// The mapping-node checks a sequence-mode blob and a mapper blob (lins_mapper_blob.hpp) share, once the key-frame table
// ids[0..n_keyframes) is known to hold distinct ids of key poses: the IMU queue pointers are in range, every window id
// names a stored key frame, and so do the newest key pose and every key frame the next window can take.
template <typename Window>
inline const char* mapper_state_check(const MapperRec& m, int32_t n_poses, int32_t n_window, Window window, const int32_t* ids, int32_t n_keyframes) {
  if (m.imuPointerFront < 0 || m.imuPointerFront >= LINS_MAPPER_IMU_QUEUE || m.imuPointerLast < -1 || m.imuPointerLast >= LINS_MAPPER_IMU_QUEUE)
    return "bad IMU queue pointer in slot blob";
  auto stored = [&](int32_t id) {
    for (int i = 0; i < n_keyframes; ++i) if (ids[i] == id) return true;
    return false;
  };
  for (int i = 0; i < n_window; ++i) if (!stored(window(i))) return "slot blob window names no stored key frame";
  // the key frames a later cycle's window can take: the newest, and while the window is short the last 50
  if (n_poses > 0 && !stored(n_poses - 1)) return "slot blob lacks its newest key frame";
  if (n_window < LINS_MAPPER_WINDOW)
    for (int32_t id = n_poses > LINS_MAPPER_WINDOW ? n_poses - LINS_MAPPER_WINDOW : 0; id < n_poses; ++id)
      if (!stored(id)) return "slot blob lacks a key frame of its next window";
  return nullptr;
}

inline bool finite_all(const double* v, int n, bool nonneg) {
  for (int i = 0; i < n; ++i) if (!std::isfinite(v[i]) || (nonneg && v[i] < 0)) return false;
  return true;
}
// the value checks of a config and a tuning, in a blob and in lins_gpu_seq_configure / lins_gpu_seq_tune
inline bool config_ok(const lins_slot_config& c) {
  const lins_seq_params& f = c.filter;
  const lins_seq_init_params& i = c.init;
  return std::isfinite(c.scan_period) && c.scan_period > 0 && std::isfinite(c.features.edge_threshold) && std::isfinite(c.features.surf_threshold) &&
         std::isfinite(c.features.imu_lidar_extrinsic_angle) && finite_all(f.noise, 4, true) && finite_all(f.init_pos_std, 3, true) &&
         finite_all(f.init_att_std, 3, true) && finite_all(i.init_vel_std, 3, true) && finite_all(i.init_acc_std, 3, true) &&
         finite_all(i.init_gyr_std, 3, true) && finite_all(i.init_ba, 3, false) && finite_all(i.init_bw, 3, false);
}
inline bool tuning_ok(const lins_slot_tuning& u) {
  return u.num_iter >= 0 && u.num_iter <= LINS_MAX_ITER && u.icp_freq >= 1 && std::isfinite(u.nearest_feature_search_sq_dist) &&
         std::isfinite(u.lidar_std) && std::isfinite(u.lidar_scale) && std::isfinite(u.imu_misalign_angle);
}

// Validates the len bytes at p as a blob of a build with record sizes sz and fills v.  Returns nullptr when the blob is
// well formed, else what is wrong.  Every count, offset and id a loader uses is checked here, so that a blob that passes
// cannot make it read or write out of bounds.
inline const char* parse(const uint8_t* p, uint64_t len, const BuildSizes& sz, View& v) {
  v.p = p;
  if (!p || len < sizeof(Header)) return "blob shorter than its header";
  std::memcpy(&v.h, p, sizeof(Header));
  const Header& h = v.h;
  if (h.magic != kMagic) return "not a slot blob (bad magic)";
  if (h.version != kVersion) return "slot blob of another format version";
  if (std::memcmp(&h.sizes, &sz, sizeof(sz)) != 0) return "slot blob of another library build (record sizes differ)";
  if (h.flags & ~uint32_t(kBound | kConfigured | kTuned)) return "bad slot blob flags";
  if (h.n_sections != kNumSections) return "bad slot blob section count";
  if (h.total != len) return "slot blob length differs from its header's";
  for (int i = 0; i < kNumSections; ++i)
    if (h.sec[i].off % 16 || h.sec[i].off < sizeof(Header) || h.sec[i].off > len || h.sec[i].bytes > len - h.sec[i].off)
      return "slot blob section outside the blob";
  if (h.sec[kScalars].bytes != sizeof(Scalars)) return "bad slot blob scalar section";
  std::memcpy(&v.sc, v.at(kScalars), sizeof(Scalars));
  const Scalars& s = v.sc;
  const bool bound = h.flags & kBound;
  if (s.fusion != kFusionInit && s.fusion != kFusionFirstScan && s.fusion != kFusionRunning) return "bad fusion status in slot blob";
  if (s.stale != 0 && s.stale != 1) return "bad stale flag in slot blob";
  if (s.yzx != 0 && s.yzx != 1) return "bad YZX flag in slot blob";
  if (s.pad != 0) return "bad slot blob padding";
  for (int c = 0; c < 4; ++c) if (s.n_map[c] < 0) return "negative map count in slot blob";
  if (s.n_outlier < 0 || s.n_poses < 0 || s.n_window < 0 || s.n_keyframes < 0) return "negative count in slot blob";
  if (!s.stale && (s.n_map[2] || s.n_map[3])) return "slot blob has a 1-NN cloud of its own without the stale flag";
  if (!bound && (s.n_outlier || s.n_poses || s.n_window || s.n_keyframes || s.yzx)) return "unbound slot blob with mapper state";
  if (s.n_keyframes > kMaxKeyframes) return "slot blob stores more than 51 key frames";
  if (s.n_keyframes > s.n_poses) return "slot blob stores more key frames than key poses";
  if (s.n_window > LINS_MAPPER_WINDOW) return "slot blob window longer than the mapper's";
  if ((h.flags & kConfigured) && !config_ok(s.cfg)) return "bad slot config in slot blob";
  if ((h.flags & kTuned) && !tuning_ok(s.tune)) return "bad slot tuning in slot blob";
  // the key-frame table, once its section is known to lie in the blob with the size the count gives
  if (h.sec[kKeyframes].bytes != sizeof(KeyframeRec) * (uint64_t)s.n_keyframes) return "bad slot blob key-frame section";
  Counts c;
  c.bound = bound;
  for (int k = 0; k < 4; ++k) c.n_map[k] = s.n_map[k];
  c.n_outlier = s.n_outlier; c.n_poses = s.n_poses; c.n_window = s.n_window; c.n_keyframes = s.n_keyframes;
  int32_t ids[kMaxKeyframes];
  for (int i = 0; i < s.n_keyframes; ++i) {
    const KeyframeRec k = v.keyframe(i);
    if (k.id < 0 || k.id >= s.n_poses) return "slot blob key frame of no key pose";
    for (int j = 0; j < i; ++j) if (ids[j] == k.id) return "slot blob stores a key frame twice";
    ids[i] = k.id;
    for (int a = 0; a < 3; ++a) {
      if (k.n[a] < 0) return "negative key-frame cloud count in slot blob";
      c.n_kf_points += k.n[a];
    }
  }
  if (c.n_kf_points > INT32_MAX) return "slot blob key-frame clouds too large";
  Header want;
  layout(c, sz, want);
  if (want.total != len || std::memcmp(want.sec, h.sec, sizeof(h.sec)) != 0) return "slot blob section table differs from its counts";
  if (!bound) return nullptr;
  std::memcpy(&v.m, v.at(kMapper), sizeof(MapperRec));
  return mapper_state_check(v.m, s.n_poses, s.n_window, [&](int i) { return v.window(i); }, ids, s.n_keyframes);
}

}  // namespace lins_blob
