// tools/synth/lins_bag.cpp — C entry points over csrc/host/rosbag_reader.hpp (SURVEY.md §8 row F4) for tools and tests:
// summary of a ROS1 bag, decoded sensor_msgs/Imu, sensor_msgs/PointCloud2 and cloud_msgs/cloud_info messages, and a
// writer of small bags.  No ROS, no PCL, no GPU.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../lins---lidar-inertial-slam_b200/csrc/cuda/lins_cloud2.cuh"
#include "../../lins---lidar-inertial-slam_b200/csrc/host/rosbag_reader.hpp"

using namespace lins;
using namespace lins::rosbag;

namespace {
struct TopicStat { std::string type, md5; long count = 0; double t0 = 1e300, t1 = -1e300; };
}

extern "C" {

// "topic type md5 count first_time last_time" per line -> out (NUL terminated).  Returns 0 or a LINS_BAG_E_* code.
int lins_bag_summary(const char* path, char* out, int cap) {
  Reader rd;
  int rc = rd.open(path);
  if (rc != LINS_BAG_OK) { std::snprintf(out, cap, "%s", rd.error.c_str()); return rc; }
  std::map<std::string, TopicStat> st;
  rc = rd.for_each([&](const MessageView& m) {
    TopicStat& s = st[m.conn->topic];
    s.type = m.conn->type; s.md5 = m.conn->md5sum; s.count++;
    s.t0 = std::min(s.t0, m.time); s.t1 = std::max(s.t1, m.time);
  });
  if (rc != LINS_BAG_OK) { std::snprintf(out, cap, "%s", rd.error.c_str()); return rc; }
  int pos = 0;  // (no iostreams here: this library may be loaded next to a second libstdc++)
  if (cap > 0) out[0] = 0;
  for (const auto& kv : st) {
    if (pos >= cap - 1) break;
    pos += std::snprintf(out + pos, (size_t)(cap - pos), "%s %s %s %ld %.17g %.17g\n", kv.first.c_str(), kv.second.type.c_str(), kv.second.md5.c_str(), kv.second.count,
                         kv.second.t0, kv.second.t1);
  }
  return LINS_BAG_OK;
}

// every sensor_msgs/Imu of `topic`: rows of 8 doubles (header stamp, acc xyz, gyr xyz, record time).  *n = messages found.
int lins_bag_read_imu(const char* path, const char* topic, double* out, int cap_rows, int* n) {
  Reader rd;
  int rc = rd.open(path);
  if (rc != LINS_BAG_OK) return rc;
  int k = 0;
  bool bad = false;
  rc = rd.for_each([&](const MessageView& m) {
    if (m.conn->topic != topic) return;
    ImuMsg im;
    if (!decode_imu(m.data, m.size, im)) { bad = true; return; }
    if (k < cap_rows) {
      double* r = out + 8 * (size_t)k;
      r[0] = im.header.stamp;
      for (int i = 0; i < 3; ++i) { r[1 + i] = im.linear_acceleration[i]; r[4 + i] = im.angular_velocity[i]; }
      r[7] = m.time;
    }
    ++k;
  });
  *n = k;
  return rc != LINS_BAG_OK ? rc : (bad ? LINS_BAG_E_FORMAT : LINS_BAG_OK);
}

// the index-th sensor_msgs/PointCloud2 of `topic` as PointXYZI records.  *n = its point count (also when cap is too small).
int lins_bag_read_cloud(const char* path, const char* topic, int index, lins_point* out, int cap, int* n, double* stamp) {
  Reader rd;
  int rc = rd.open(path);
  if (rc != LINS_BAG_OK) return rc;
  int k = 0;
  bool found = false, bad = false;
  rc = rd.for_each([&](const MessageView& m) {
    if (m.conn->topic != topic || found) return;
    if (k++ != index) return;
    Header h;
    Cloud c;
    if (!decode_pointcloud2(m.data, m.size, h, c)) { bad = true; return; }
    found = true;
    *n = (int)c.size();
    *stamp = h.stamp;
    std::memcpy(out, c.points.data(), sizeof(lins_point) * std::min<size_t>(c.size(), (size_t)std::max(cap, 0)));
  });
  if (rc != LINS_BAG_OK) return rc;
  return bad ? LINS_BAG_E_FORMAT : (found ? LINS_BAG_OK : LINS_BAG_E_IO);
}

// the index-th cloud_msgs/cloud_info of `topic`.  rings: start/end (cap_rings each), ori3 = start, end, diff;
// per point: ground flag, column index, range (cap_pts each).
int lins_bag_read_cloud_info(const char* path, const char* topic, int index, int32_t* start_ring, int32_t* end_ring, int cap_rings,
                             float* ori3, uint8_t* ground, uint32_t* col, float* range, int cap_pts, int* n_rings, int* n_pts, double* stamp) {
  Reader rd;
  int rc = rd.open(path);
  if (rc != LINS_BAG_OK) return rc;
  int k = 0;
  bool found = false, bad = false;
  rc = rd.for_each([&](const MessageView& m) {
    if (m.conn->topic != topic || found) return;
    if (k++ != index) return;
    Header h;
    CloudInfo ci;
    if (!decode_cloud_info(m.data, m.size, h, ci)) { bad = true; return; }
    found = true;
    *n_rings = (int)ci.startRingIndex.size(); *n_pts = (int)ci.segmentedCloudRange.size(); *stamp = h.stamp;
    for (int i = 0; i < std::min(*n_rings, cap_rings); ++i) { start_ring[i] = ci.startRingIndex[i]; end_ring[i] = ci.endRingIndex[i]; }
    ori3[0] = ci.startOrientation; ori3[1] = ci.endOrientation; ori3[2] = ci.orientationDiff;
    for (int i = 0; i < std::min(*n_pts, cap_pts); ++i) { ground[i] = ci.segmentedCloudGroundFlag[i]; col[i] = ci.segmentedCloudColInd[i]; range[i] = ci.segmentedCloudRange[i]; }
  });
  if (rc != LINS_BAG_OK) return rc;
  return bad ? LINS_BAG_E_FORMAT : (found ? LINS_BAG_OK : LINS_BAG_E_IO);
}

// One sensor_msgs/PointCloud2 message's bytes (b, n) -> what fromROSMsg<PointXYZI> reads of it, without decoding a point:
// the layout lins_gpu_decode_cloud2 takes, the data field's byte range inside the message (*data_start, *data_len) and the
// header stamp.  LINS_BAG_E_FORMAT exactly where decode_pointcloud2 rejects the message (extents without 32-bit wrap).
int lins_bag_index_cloud2_msg(const uint8_t* b, size_t n, lins_cloud2_layout* lay, int64_t* data_start, int64_t* data_len, double* stamp) {
  Cursor c(b, n);
  const Header h = read_header(c);
  const uint32_t height = c.get<uint32_t>(), width = c.get<uint32_t>(), nf = c.get<uint32_t>();
  if (!c.ok || nf > 64) return LINS_BAG_E_FORMAT;
  lins_cloud2_layout l;
  std::memset(&l, 0, sizeof(l));
  bool seen[4] = {false, false, false, false};
  for (uint32_t k = 0; k < nf; ++k) {
    const std::string name = c.str();
    const uint32_t off = c.get<uint32_t>();
    const uint8_t dt = c.get<uint8_t>();
    c.get<uint32_t>();  // count
    const int f = name == "x" ? 0 : name == "y" ? 1 : name == "z" ? 2 : name == "intensity" ? 3 : -1;
    if (f >= 0) { l.offset[f] = off; l.datatype[f] = dt; seen[f] = true; }  // (the last field of a name wins, as there)
  }
  l.is_bigendian = c.get<uint8_t>();
  l.point_step = c.get<uint32_t>(); l.row_step = c.get<uint32_t>();
  const uint32_t dlen = c.get<uint32_t>();
  const uint8_t* d = c.bytes(dlen);
  c.get<uint8_t>();  // is_dense
  if (!c.ok || (dlen && !d)) return LINS_BAG_E_FORMAT;
  l.height = height; l.width = width;
  if (!seen[0] || !seen[1] || !seen[2]) return LINS_BAG_E_FORMAT;
  if (seen[3] && l.datatype[3] == 0) return LINS_BAG_E_FORMAT;  // (a named intensity of datatype 0 is rejected there)
  if (lins_cloud2::check_layout(l, dlen)) return LINS_BAG_E_FORMAT;
  *lay = l;
  *data_start = d ? (int64_t)(d - b) : (int64_t)(c.p - b) - 1;
  *data_len = dlen;
  *stamp = h.stamp;
  return LINS_BAG_OK;
}

// decode_pointcloud2 of one message's bytes: *n = its point count (also when cap is too small); LINS_BAG_E_FORMAT where it
// rejects the message.  The host reference of lins_gpu_decode_cloud2.
int lins_bag_decode_cloud2_msg(const uint8_t* b, size_t n, lins_point* out, int cap, int* npts) {
  Header h;
  Cloud cl;
  if (!decode_pointcloud2(b, n, h, cl)) return LINS_BAG_E_FORMAT;
  *npts = (int)cl.size();
  std::memcpy(out, cl.points.data(), sizeof(lins_point) * std::min<size_t>(cl.size(), (size_t)std::max(cap, 0)));
  return LINS_BAG_OK;
}

// decode_pointcloud2 of n whole messages (message i = buf[msg_off[i] .. msg_off[i + 1])) on `threads` std::threads, message
// i's points as packed (x, y, z, intensity) float records at out + 4 * out_off[i] (LINS_POINTS_PACKED16, what
// lins_gpu_seq_step_raw takes with the least upload): the host arm of tools/cloud2_bench.py.  LINS_BAG_E_FORMAT if a message
// is rejected or its point count differs from out_off's.
int lins_bag_decode_cloud2_many(const uint8_t* buf, const int64_t* msg_off, int n, float* out, const int32_t* out_off, int threads) {
  std::atomic<int> next(0), bad(0);
  auto work = [&]() {
    Header h;
    Cloud c;
    for (int i; (i = next.fetch_add(1)) < n;) {
      if (!decode_pointcloud2(buf + msg_off[i], (size_t)(msg_off[i + 1] - msg_off[i]), h, c) || (int)c.size() != out_off[i + 1] - out_off[i]) { bad = 1; continue; }
      float* o = out + 4 * (size_t)out_off[i];
      for (size_t k = 0; k < c.size(); ++k) {
        const lins_point& p = c.points[k];
        o[4 * k] = p.x; o[4 * k + 1] = p.y; o[4 * k + 2] = p.z; o[4 * k + 3] = p.intensity;
      }
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < std::max(threads, 1); ++t) th.emplace_back(work);
  work();
  for (auto& t : th) t.join();
  return bad ? LINS_BAG_E_FORMAT : LINS_BAG_OK;
}

// Writer test hook: a bag with n_scans clouds of n_pts points on `lidar_topic` (deterministic contents: point i of scan k
// = (k + 0.001 i, -0.002 i, 0.5 k, i % 16 + 0.01 k)), 10 Imu messages per scan on `imu_topic`, one cloud_info per scan.
int lins_bag_write_test(const char* path, const char* lidar_topic, const char* imu_topic, const char* info_topic, int n_scans, int n_pts) {
  Writer w;
  if (w.open(path) != LINS_BAG_OK) return LINS_BAG_E_IO;
  const uint32_t cl = w.add_connection(lidar_topic, "sensor_msgs/PointCloud2", "1158d486dd51d683ce2f1be655c3c181", "see sensor_msgs/PointCloud2");
  const uint32_t ci = w.add_connection(imu_topic, "sensor_msgs/Imu", "6a62c6daae103f4ff57a132d6f95cec2", "see sensor_msgs/Imu");
  const uint32_t cf = w.add_connection(info_topic, "cloud_msgs/cloud_info", "af8fa8b8d2f1b1b6d5e4fd4f3a7e4b0a", "see cloud_msgs/msg/cloud_info.msg");
  for (int k = 0; k < n_scans; ++k) {
    const double t = 100.0 + 0.1 * k;
    for (int j = 0; j < 10; ++j) {
      const double ti = t + 0.01 * j;
      const double acc[3] = {0.1 * j, -0.2 * k, 9.81}, gyr[3] = {0.001 * j, 0.002 * k, -0.003};
      w.write(ci, ti, Writer::encode_imu((uint32_t)(10 * k + j), ti, acc, gyr));
    }
    Cloud c;
    for (int i = 0; i < n_pts; ++i) c.push_back(makePoint(k + 0.001f * i, -0.002f * i, 0.5f * k, (float)(i % 16) + 0.01f * k));
    w.write(cl, t + 0.1, Writer::encode_cloud_xyzi((uint32_t)k, t + 0.1, "velodyne", c));
    CloudInfo info;
    info.resize(16, n_pts);
    for (int r = 0; r < 16; ++r) { info.startRingIndex[r] = r * 7 + k; info.endRingIndex[r] = r * 7 + 5; }
    info.startOrientation = 0.25f * k; info.endOrientation = 6.0f + k; info.orientationDiff = 6.2f;
    for (int i = 0; i < n_pts; ++i) { info.segmentedCloudGroundFlag[i] = i % 3 == 0; info.segmentedCloudColInd[i] = (uint32_t)(i * 5 % 1800); info.segmentedCloudRange[i] = 1.5f + 0.01f * i; }
    w.write(cf, t + 0.1, Writer::encode_cloud_info((uint32_t)k, t + 0.1, info));
  }
  return w.close();
}

}  // extern "C"
