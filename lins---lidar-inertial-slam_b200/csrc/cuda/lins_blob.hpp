// lins_blob.hpp — what the byte formats of saved slots share (lins_checkpoint.cu writes and reads them): the
// sequence-mode slot blob (lins_slot_blob.hpp) and the mapper blob (lins_mapper_blob.hpp).  Their common records, the
// section table, the header and key-frame table checks and the mapping-node rules.  Plain C++ with no CUDA, so the CPU
// suite compiles it with g++ (tests/test_seq_checkpoint_cpu.py, tests/test_mapper_checkpoint_cpu.py).
//
// A blob is a header, then sections at 16-byte offsets in a fixed order, each sized by the counts of the scalar section
// (so the section table is fully determined by them, and a loader checks it is exactly that).  The blob records the
// build's record sizes, and a build whose sizes differ rejects it.  Both formats carry a mapping node in the same
// sections (NodeSecs): its MapperRec, a PoseRec per key pose, the window's int32 key-frame ids (oldest first, the deque as
// it is, its duplicate id included), a KeyframeRec per stored key frame by id, those key frames' corner, surf and outlier
// clouds in table order as float4 runs, and the scan-to-map loop state (the build's MapLoopState bytes).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <unordered_set>
#include <vector>

#include "../../../include/lins_gpu.h"

namespace lins_blob {

constexpr int kMaxKeyframes = LINS_MAPPER_WINDOW + 1;  // a plain node's store keeps the window and the newest key frame

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

struct SectionRec { uint64_t off, bytes; };

inline uint64_t align16(uint64_t x) { return (x + 15) & ~uint64_t(15); }

// one section's record(s) into a blob image: the bytes, then zeros up to the next 16-byte boundary
inline void put(uint8_t* dst, const void* src, size_t bytes) {
  if (bytes) std::memcpy(dst, src, bytes);
  std::memset(dst + bytes, 0, align16(bytes) - bytes);
}

// the section table of n sections of the given byte counts behind a header of header_bytes; returns the blob's length
inline uint64_t section_table(uint64_t header_bytes, const uint64_t* bytes, int n, SectionRec* sec) {
  uint64_t o = align16(header_bytes);
  for (int i = 0; i < n; ++i) {
    sec[i] = SectionRec{o, bytes[i]};
    o = align16(o + bytes[i]);
  }
  return o;
}

// record i of the records at p (a blob need not be aligned, so records are read with memcpy)
template <typename T>
T rec(const uint8_t* p, int i) {
  T r;
  std::memcpy(&r, p + sizeof(T) * i, sizeof(T));
  return r;
}

// a validator message naming the format ("slot", "mapper"); it lasts until the thread's next message
inline const char* msg(const char* fmt, const char* name) {
  thread_local char buf[96];
  std::snprintf(buf, sizeof(buf), fmt, name);
  return buf;
}

// The checks of a blob's header h (read from a blob of len bytes) of format `name`: its magic, version, record sizes,
// flags (within `flags`), section count (sections_ok), length, every section aligned and inside the blob, and the
// scalar section's size.
template <typename Header, typename Sizes>
const char* check_envelope(const Header& h, uint64_t len, const char* name, uint64_t magic, uint32_t version, uint32_t flags, const Sizes& sz,
                           bool sections_ok, uint64_t scalar_bytes) {
  if (h.magic != magic) return msg("not a %s blob (bad magic)", name);
  if (h.version != version) return msg("%s blob of another format version", name);
  if (std::memcmp(&h.sizes, &sz, sizeof(sz)) != 0) return msg("%s blob of another library build (record sizes differ)", name);
  if (h.flags & ~flags) return msg("bad %s blob flags", name);
  if (!sections_ok) return msg("bad %s blob section count", name);
  if (h.total != len) return msg("%s blob length differs from its header's", name);
  for (const SectionRec& s : h.sec)
    if (s.off % 16 || s.off < sizeof(Header) || s.off > len || s.bytes > len - s.off) return msg("%s blob section outside the blob", name);
  if (h.sec[0].bytes != scalar_bytes) return msg("bad %s blob scalar section", name);
  return nullptr;
}

// where a blob keeps a mapping node: the byte offsets of its sections
struct NodeSecs { uint64_t mapper, poses, window, keyframes, kfclouds, loop; };

// a parsed blob's mapping node (none: counts 0), the rest of the blob left in place at p
struct NodeView {
  const uint8_t* p = nullptr;
  NodeSecs node{};
  int32_t n_poses = 0, n_window = 0, n_keyframes = 0;
  MapperRec m;
  PoseRec pose(int i) const { return rec<PoseRec>(p + node.poses, i); }
  int32_t window(int i) const { return rec<int32_t>(p + node.window, i); }
  KeyframeRec keyframe(int i) const { return rec<KeyframeRec>(p + node.keyframes, i); }
};

// The key-frame table of v (its section known to lie in the blob with the size its count gives): every id a key pose's
// and none twice, no negative cloud count, at most INT32_MAX points in all.  Fills ids (table order) and points.
inline const char* check_keyframes(const NodeView& v, const char* name, std::vector<int32_t>& ids, int64_t& points) {
  std::unordered_set<int32_t> seen;
  ids.assign(v.n_keyframes, 0);
  points = 0;
  for (int i = 0; i < v.n_keyframes; ++i) {
    const KeyframeRec k = v.keyframe(i);
    if (k.id < 0 || k.id >= v.n_poses) return msg("%s blob key frame of no key pose", name);
    if (!seen.insert(k.id).second) return msg("%s blob stores a key frame twice", name);
    ids[i] = k.id;
    for (int a = 0; a < 3; ++a) {
      if (k.n[a] < 0) return msg("negative key-frame cloud count in %s blob", name);
      points += k.n[a];
    }
  }
  if (points > INT32_MAX) return msg("%s blob key-frame clouds too large", name);
  return nullptr;
}

// The key frames a later cycle's window can take (mapper_cycle_begin): the window's (kind 0), the newest (kind 1) and,
// while the window is short, the last LINS_MAPPER_WINDOW (kind 2).  Calls take(id, kind) for each in that order (an id
// can come more than once) until it returns false; returns whether none did.
template <typename Take>
bool later_window(const NodeView& v, Take take) {
  for (int i = 0; i < v.n_window; ++i) if (!take(v.window(i), 0)) return false;
  if (v.n_poses > 0 && !take(v.n_poses - 1, 1)) return false;
  if (v.n_window < LINS_MAPPER_WINDOW)
    for (int32_t id = std::max(0, v.n_poses - LINS_MAPPER_WINDOW); id < v.n_poses; ++id) if (!take(id, 2)) return false;
  return true;
}

// The mapping-node checks both formats share, once the key-frame table ids is known to hold distinct ids of key poses:
// the IMU queue pointers are in range, and every key frame a later window can take is stored.
inline const char* mapper_state_check(const NodeView& v, const std::vector<int32_t>& ids) {
  if (v.m.imuPointerFront < 0 || v.m.imuPointerFront >= LINS_MAPPER_IMU_QUEUE || v.m.imuPointerLast < -1 || v.m.imuPointerLast >= LINS_MAPPER_IMU_QUEUE)
    return "bad IMU queue pointer in slot blob";
  static const char* const kMissing[3] = {"slot blob window names no stored key frame", "slot blob lacks its newest key frame",
                                          "slot blob lacks a key frame of its next window"};
  const char* bad = nullptr;
  later_window(v, [&](int32_t id, int kind) {
    if (std::find(ids.begin(), ids.end(), id) != ids.end()) return true;
    bad = kMissing[kind];
    return false;
  });
  return bad;
}

}  // namespace lins_blob
