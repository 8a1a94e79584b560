// lins_slot_blob.hpp — the byte format of one saved sequence-mode slot (lins_gpu_seq_save / lins_gpu_seq_load,
// lins_checkpoint.cu): its records, its layout and its validation, on the core of lins_blob.hpp.  Plain C++ with no CUDA,
// so the CPU suite compiles it with g++ (tests/test_seq_checkpoint_cpu.py).
#pragma once
#include "lins_blob.hpp"

namespace lins_blob {

// Sections: scalars (Scalars: fusion status, stale flag, YZX flag, counts, the run's open constants, config, tuning,
// pose), rows (the filter, covariance, global, linearisation, imu_last and pre-integration rows, kRowDoubles doubles),
// maps (map_s, map_c, tree_s, tree_c as float4 runs), outlier (the published outlier cloud), then the node's sections;
// a run that lins_gpu_seq_map_open has not bound has no outlier cloud and no node.

constexpr uint64_t kMagic = 0x544f4c53534e494cull;  // "LINSSLOT" in little-endian byte order
constexpr uint32_t kVersion = 1;
enum Flags : uint32_t { kBound = 1u, kConfigured = 2u, kTuned = 4u };
enum Section { kScalars, kRows, kMaps, kOutlier, kMapper, kPoses, kWindow, kKeyframes, kKfClouds, kLoop, kNumSections };
// filt (20), cov (324), glob (20), lin (20), imu_last (8), pre (20): the device rows of one slot, back to back
constexpr int kRowDoubles = 20 + 324 + 20 + 20 + 8 + 20;
constexpr int kRowOff[6] = {0, 20, 344, 364, 384, 392};
// StateEstimator::FusionStatus values a slot can be in
constexpr int32_t kFusionInit = 0, kFusionFirstScan = 1, kFusionRunning = 3;

// the record sizes of the build that wrote a blob
struct BuildSizes {
  uint32_t icp_state, loop_state, imu_queue, n_consts, n_init_consts;
};
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

// what the section sizes depend on
struct Counts {
  bool bound = false;
  int64_t n_map[4] = {0, 0, 0, 0};
  int64_t n_outlier = 0, n_poses = 0, n_window = 0, n_keyframes = 0, n_kf_points = 0;
};

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
  h.total = section_table(sizeof(Header), bytes, kNumSections, h.sec);
}
inline NodeSecs node_secs(const Header& h) {
  return {h.sec[kMapper].off, h.sec[kPoses].off, h.sec[kWindow].off, h.sec[kKeyframes].off, h.sec[kKfClouds].off, h.sec[kLoop].off};
}

// a parsed blob: the header and scalar records copied out
struct View : NodeView {
  Header h;
  Scalars sc;
  const uint8_t* at(int section) const { return p + h.sec[section].off; }
};

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
  if (const char* bad = check_envelope(h, len, "slot", kMagic, kVersion, kBound | kConfigured | kTuned, sz, h.n_sections == kNumSections, sizeof(Scalars)))
    return bad;
  v.sc = rec<Scalars>(v.at(kScalars), 0);
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
  v.node = node_secs(h);
  v.n_poses = s.n_poses; v.n_window = s.n_window; v.n_keyframes = s.n_keyframes;
  Counts c;
  c.bound = bound;
  for (int k = 0; k < 4; ++k) c.n_map[k] = s.n_map[k];
  c.n_outlier = s.n_outlier; c.n_poses = s.n_poses; c.n_window = s.n_window; c.n_keyframes = s.n_keyframes;
  std::vector<int32_t> ids;
  if (const char* bad = check_keyframes(v, "slot", ids, c.n_kf_points)) return bad;
  Header want;
  layout(c, sz, want);
  if (want.total != len || std::memcmp(want.sec, h.sec, sizeof(h.sec)) != 0) return "slot blob section table differs from its counts";
  if (!bound) return nullptr;
  v.m = rec<MapperRec>(v.at(kMapper), 0);
  return mapper_state_check(v, ids);
}

}  // namespace lins_blob
