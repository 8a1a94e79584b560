// tools/synth/lins_sequence.cpp — offline sequence driver (SURVEY.md §8 row F3): what LinsFusion does between the
// ROS callbacks and the estimator (lins/src/lib/Estimator.cpp:204-252): for every lidar scan, feed the buffered
// IMU samples through processImu, then the segmented cloud through processPCL.  Inputs are synthetic (a smooth
// trajectory through the seeded world of lins_synth.cpp; IMU at 400 Hz; raw scans pushed through the restated
// image projection).  The estimator is the C++ shim fusion::StateEstimator whose hot seams run on the GPU through
// the C-ABI, so this file links against liblins_gpu.so.  Every performIESKF call's inputs / outputs are recorded
// so that tests can replay them through the CPU oracle.  Never includes anything from oracle/.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "lins_synth.cpp"

#include "../../lins---lidar-inertial-slam_b200/csrc/host/state_estimator.hpp"
#include "../../lins---lidar-inertial-slam_b200/csrc/host/rosbag_reader.hpp"
#include <algorithm>
#include <chrono>

using lins::fusion::StateEstimator;

namespace {

struct SeqRecord {
  // one recorded performIESKF unit per RUNNING scan
  std::vector<lins_point> surfFlat, cornerSharp, surfLessFlat, cornerLessSharp;
  std::vector<int32_t> offSF{0}, offCS{0}, offSL{0}, offCL{0};
  std::vector<double> state_in, cov_in, state_out, cov_out;
  std::vector<int32_t> iters, flags, scan_index;
  std::vector<double> rel_true;  // true relative pose of that scan: t (3) + q (x,y,z,w)
  std::vector<int32_t> status;   // estimator status after each scan
  std::vector<double> global_est, global_true;  // per scan: position (3) + quaternion (x,y,z,w)
  // what LinsFusion::publishTopics hands the mapping node after each scan of an initialised estimator
  // (Estimator.cpp:177-318): the stamp, globalStateYZX_ (rn (3) + qbn (x,y,z,w)) and scan_last_'s YZX less-sharp,
  // less-flat and outlier clouds
  std::vector<double> map_time, map_odom;
  std::vector<lins_point> map_cloud[3];
  std::vector<int32_t> map_off[3] = {{0}, {0}, {0}};
};

void append_cloud(std::vector<lins_point>& dst, std::vector<int32_t>& off, const Cloud& c) {
  dst.insert(dst.end(), c.points.begin(), c.points.end());
  off.push_back((int32_t)dst.size());
}

struct Traj {  // smooth body-frame velocity / yaw-rate profile
  double v0, va, vw, w0, wa, ww;
  V3D vbody(double t) const { return V3D(v0 + va * std::sin(vw * t), 0.1 * std::sin(0.7 * vw * t), 0.0); }
  V3D vdot(double t) const { return V3D(va * vw * std::cos(vw * t), 0.07 * vw * std::cos(0.7 * vw * t), 0.0); }
  V3D wbody(double t) const { return V3D(0.0, 0.0, w0 + wa * std::sin(ww * t)); }
};

// one simulated sweep: the raw cloud (sensor frame, PointXYZI with intensity 0 like a driver that has none), the IMU samples
// taken during it (index 1..nimu; index 0 is the sample at the sweep's start) and the true poses at its two ends
struct Sweep {
  Cloud raw;
  std::vector<V3D> accs, gyrs;
  Pose start, end;
  double t_end = 0;
};

struct SimDrive {
  const lins_synth_cfg* cfg;
  Rng rng;
  LidarModel lm;
  World w;
  Traj tr;
  Pose P;
  double t = 0.0;
  static constexpr int nimu = 40;
  // scan_period > 0: the sweep lasts that long (the IMU rate follows: nimu samples per sweep); else the model's SCAN_PERIOD
  SimDrive(const lins_synth_cfg* c, uint64_t seed, double scan_period = 0.0) : cfg(c), rng(seed) {
    lm = cfg->lidar == 1 ? LidarModel::dense64() : LidarModel::vlp16();
    if (scan_period > 0) lm.scan_period = scan_period;
    w = make_world(rng, cfg->world);
    tr = Traj{rng.uni(1.0, 0.6 * cfg->v_max), rng.uni(0.2, 1.0), rng.uni(0.5, 1.5), rng.uni(-0.5, 0.5) * cfg->w_max, 0.5 * cfg->w_max, rng.uni(0.3, 1.0)};
    P.R = math_utils::rpy2Quat(V3D(0.0, 0.0, rng.uni(-M_PI, M_PI))).toRotationMatrix();
    P.p = V3D(rng.uni(-3, 3), rng.uni(-3, 3), 1.5);
  }
  double dt() const { return lm.scan_period / nimu; }
  void next(Sweep& sw) {
    const double T = lm.scan_period, d = dt();
    const int N = lm.scan_num;
    const V3D g_w(0, 0, -filter::G0);
    const V3D ba(0.0, 0.0, 0.0), bw(0.0, 0.0, 0.0);  // the shim initialises its biases from FilterParams
    std::vector<Pose> poses(nimu + 1);
    sw.accs.assign(nimu + 1, V3D()); sw.gyrs.assign(nimu + 1, V3D());
    poses[0] = P;
    sw.start = P;
    for (int i = 0; i <= nimu; ++i) {
      const double ti = t + i * d;
      const V3D wb = tr.wbody(ti), vb = tr.vbody(ti);
      sw.accs[i] = cross(wb, vb) + tr.vdot(ti) - poses[i].R.transpose() * g_w + ba + V3D(0.02 * rng.gauss(), 0.02 * rng.gauss(), 0.02 * rng.gauss());
      sw.gyrs[i] = wb + bw + V3D(5e-4 * rng.gauss(), 5e-4 * rng.gauss(), 5e-4 * rng.gauss());
      if (i < nimu) {  // midpoint step of the true motion
        const double tm = ti + 0.5 * d;
        poses[i + 1].p = poses[i].p + d * (poses[i].R * math_utils::axis2Quat(0.5 * d * tr.wbody(tm)).toRotationMatrix() * tr.vbody(tm));
        poses[i + 1].R = poses[i].R * math_utils::axis2Quat(d * tr.wbody(tm)).toRotationMatrix();
      }
    }
    sw.raw.clear();
    for (int f = 0; f < N; ++f) {
      const double s = (double)f / N * nimu;
      const int i0 = std::min((int)s, nimu - 1);
      const double a = s - i0;
      Pose Pf;
      Pf.p = poses[i0].p + a * (poses[i0 + 1].p - poses[i0].p);
      Pf.R = poses[i0].R * math_utils::axis2Quat(a * d * tr.wbody(t + (i0 + 0.5 * a) * d)).toRotationMatrix();
      const double ori = -M_PI + (f + 0.25) * (2.0 * M_PI / N);
      for (int r = 0; r < lm.line_num; ++r) {
        const double el = (-(double)(lm.ang_bottom - 0.1f) + r * (double)lm.ang_res_y) * M_PI / 180.0;
        const V3D ds(std::cos(el) * std::cos(ori), -std::cos(el) * std::sin(ori), std::sin(el));
        double rg = raycast(w, Pf.p, Pf.R * ds);
        if (!(rg < 100.0)) continue;
        rg += cfg->range_noise * rng.gauss();
        sw.raw.push_back(makePoint((float)(rg * ds.x()), (float)(rg * ds.y()), (float)(rg * ds.z()), 0.f));
      }
    }
    P = poses[nimu];
    t += T;
    sw.end = P;
    sw.t_end = t;
  }
};

// what LinsFusion::processPointClouds does with one scan (Estimator.cpp:204-252) + the bookkeeping of the recorder:
// `imu_dt / acc / gyr` = the processImu calls between the previous scan and this one, in order
void feed_scan(StateEstimator& est, ImageProjection& ip, SeqRecord* rec, int k, double scan_time, const Cloud& raw, const std::vector<double>& imu_dt,
               const std::vector<V3D>& acc, const std::vector<V3D>& gyr, const Pose* start_true, const Pose* end_true, bool verbose) {
  ip.process(raw);
  for (size_t i = 0; i < imu_dt.size(); ++i) est.processImu(imu_dt[i], acc[i], gyr[i]);
  const bool will_run = est.status_ == StateEstimator::STATUS_RUNNING;
  double s_in[19];
  filter::Cov18 P_in;
  std::vector<lins_point> mapS, mapC;
  if (will_run) {
    est.filter_->state_.toArray(s_in);
    P_in = est.filter_->covariance_;
    mapS = est.scan_last_->surfPointsLessFlat_.points;
    mapC = est.scan_last_->cornerPointsLessSharp_.points;
  }
  est.last_report_.iters = 0;
  const bool publishes = est.isInitialized();  // performStateEstimation publishes after every scan but the first
  const V3D a_last = acc.empty() ? V3D(0, 0, filter::G0) : acc.back(), g_last = gyr.empty() ? V3D() : gyr.back();
  est.processPCL(scan_time, lins::sensor_utils::Imu(scan_time, a_last, g_last), ip.segmentedCloud, ip.segMsg, ip.outlierCloud);
  rec->status.push_back((int)est.status_);
  if (publishes) {
    const auto& g = est.globalStateYZX_;
    const double o[7] = {g.rn_.x(), g.rn_.y(), g.rn_.z(), g.qbn_.x(), g.qbn_.y(), g.qbn_.z(), g.qbn_.w()};
    rec->map_time.push_back(scan_time);
    rec->map_odom.insert(rec->map_odom.end(), o, o + 7);
    append_cloud(rec->map_cloud[0], rec->map_off[0], est.scan_last_->cornerPointsLessSharpYZX_);
    append_cloud(rec->map_cloud[1], rec->map_off[1], est.scan_last_->surfPointsLessFlatYZX_);
    append_cloud(rec->map_cloud[2], rec->map_off[2], est.scan_last_->outlierPointCloudYZX_);
  }
  if (verbose) std::fprintf(stderr, "[lins_seq] scan %d: status %d, IESKF iterations %d, %zu segmented points\n", k, (int)est.status_, (int)est.last_report_.iters, ip.segmentedCloud.size());
  if (will_run && est.last_report_.iters > 0) {
    // processScan swapped the scans: scan_last_ now IS the scan whose features were the queries
    append_cloud(rec->surfFlat, rec->offSF, est.scan_last_->surfPointsFlat_);
    append_cloud(rec->cornerSharp, rec->offCS, est.scan_last_->cornerPointsSharp_);
    Cloud ms, mc; ms.points = mapS; mc.points = mapC;
    append_cloud(rec->surfLessFlat, rec->offSL, ms);
    append_cloud(rec->cornerLessSharp, rec->offCL, mc);
    rec->state_in.insert(rec->state_in.end(), s_in, s_in + 19);
    rec->cov_in.insert(rec->cov_in.end(), P_in.data(), P_in.data() + 324);
    // filter_->state_ after performIESKF but BEFORE reset(1) is linState_ (not diverged) — reset(1) zeroes rn/qbn,
    // so take the relative pose from linState_ and the remaining blocks from the filter
    double s_out[19];
    lins::filter::GlobalState so = est.linState_;
    so.toArray(s_out);
    rec->state_out.insert(rec->state_out.end(), s_out, s_out + 19);
    rec->iters.push_back(est.last_report_.iters);
    rec->flags.push_back((est.last_report_.converged ? 1 : 0) | (est.last_report_.diverged ? 2 : 0) | (est.last_report_.has_nan ? 4 : 0));
    rec->scan_index.push_back(k);
    double tv[7] = {0, 0, 0, 0, 0, 0, 1};
    if (start_true && end_true) {  // true relative pose of this sweep
      M3D Rrel = start_true->R.transpose() * end_true->R;
      V3D trel = start_true->R.transpose() * (end_true->p - start_true->p);
      Q4D qrel = math_utils::R2Quat(Rrel);
      const double v[7] = {trel.x(), trel.y(), trel.z(), qrel.x(), qrel.y(), qrel.z(), qrel.w()};
      std::memcpy(tv, v, sizeof(v));
    }
    rec->rel_true.insert(rec->rel_true.end(), tv, tv + 7);
  }
  const double ge[7] = {est.globalState_.rn_.x(), est.globalState_.rn_.y(), est.globalState_.rn_.z(), est.globalState_.qbn_.x(),
                        est.globalState_.qbn_.y(), est.globalState_.qbn_.z(), est.globalState_.qbn_.w()};
  rec->global_est.insert(rec->global_est.end(), ge, ge + 7);
  double gt[7] = {0, 0, 0, 0, 0, 0, 1};
  if (end_true) {
    Q4D qt = math_utils::R2Quat(end_true->R);
    const double v[7] = {end_true->p.x(), end_true->p.y(), end_true->p.z(), qt.x(), qt.y(), qt.z(), qt.w()};
    std::memcpy(gt, v, sizeof(v));
  }
  rec->global_true.insert(rec->global_true.end(), gt, gt + 7);
}

lins::fusion::EstimatorParams seq_params(const LidarModel& lm) {
  lins::fusion::EstimatorParams ep;
  ep.lidar = lm;
  ep.filter.init_ba = V3D(0, 0, 0);
  ep.filter.init_bw = V3D(0, 0, 0);
  return ep;
}

}  // namespace

extern "C" {

void* lins_seq_run(const lins_synth_cfg* cfg, uint64_t seed, int n_scans, int device) {
  SeqRecord* rec = new SeqRecord();
  SimDrive sim(cfg, seed);
  StateEstimator est(seq_params(sim.lm), device);
  ImageProjection ip(sim.lm);
  const bool verbose = std::getenv("LINS_SEQ_VERBOSE") != nullptr;
  Sweep sw;
  for (int k = 0; k < n_scans; ++k) {
    if (verbose) std::fprintf(stderr, "[lins_seq] simulating scan %d\n", k);
    sim.next(sw);
    std::vector<double> dts(SimDrive::nimu, sim.dt());
    std::vector<V3D> acc(sw.accs.begin() + 1, sw.accs.end()), gyr(sw.gyrs.begin() + 1, sw.gyrs.end());
    feed_scan(est, ip, rec, k, sw.t_end, sw.raw, dts, acc, gyr, &sw.start, &sw.end, verbose);
  }
  return rec;
}

// The same simulated drive written as a ROS1 bag (csrc/host/rosbag_reader.hpp): the raw sweeps on `lidar_topic`
// (sensor_msgs/PointCloud2, stamped at the sweep's end like LinsFusion uses them) and the IMU samples on `imu_topic`.
// scan_period: the sweep's duration (lins_seq_write_bag_period; 0 = the model's SCAN_PERIOD, 0.1 s)
int lins_seq_write_bag_period(const lins_synth_cfg* cfg, uint64_t seed, int n_scans, const char* path, const char* lidar_topic, const char* imu_topic,
                              double scan_period) {
  using namespace lins::rosbag;
  SimDrive sim(cfg, seed, scan_period);
  Writer w;
  if (w.open(path) != LINS_BAG_OK) return LINS_BAG_E_IO;
  const uint32_t cl = w.add_connection(lidar_topic, "sensor_msgs/PointCloud2", "1158d486dd51d683ce2f1be655c3c181", "(sensor_msgs/PointCloud2)");
  const uint32_t ci = w.add_connection(imu_topic, "sensor_msgs/Imu", "6a62c6daae103f4ff57a132d6f95cec2", "(sensor_msgs/Imu)");
  Sweep sw;
  const double t0 = 1000.0;  // (bag times are seconds since the epoch; keep them small enough that 400 Hz stamps stay exact to the ns)
  uint32_t seq = 0;
  for (int k = 0; k < n_scans; ++k) {
    const double ts = t0 + sim.t;
    sim.next(sw);
    for (int i = 1; i <= SimDrive::nimu; ++i) {
      const double ti = ts + i * sim.dt();
      const double a[3] = {sw.accs[i].x(), sw.accs[i].y(), sw.accs[i].z()}, g[3] = {sw.gyrs[i].x(), sw.gyrs[i].y(), sw.gyrs[i].z()};
      w.write(ci, ti, Writer::encode_imu(seq++, ti, a, g));
    }
    w.write(cl, t0 + sw.t_end, Writer::encode_cloud_xyzi((uint32_t)k, t0 + sw.t_end, "velodyne", sw.raw));
  }
  return w.close();
}
int lins_seq_write_bag(const lins_synth_cfg* cfg, uint64_t seed, int n_scans, const char* path, const char* lidar_topic, const char* imu_topic) {
  return lins_seq_write_bag_period(cfg, seed, n_scans, path, lidar_topic, imu_topic, 0.0);
}

// BASELINE.json configs[1] runner: replay a bag the way LinsFusion does (Estimator.cpp:123-284): IMU messages are buffered,
// every lidar message is a scan at its header stamp; between two scans the buffered IMU samples are propagated with
// dt = min(imu stamp, scan stamp) - estimator time (:230-236); the raw cloud goes through the restated image projection.
// Returns a record handle like lins_seq_run (status / pose per scan, one recorded unit per performIESKF call) or null.
// rig (lins_seq_run_bag_rig; null = seq_params' defaults): the exp_port.yaml values of one robot, 29 doubles in the order
// scan_period, edge_threshold, surf_threshold, imu_lidar_extrinsic_angle, acc_n, gyr_n, acc_w, gyr_w, then init_pos_std,
// init_vel_std, init_att_std, init_acc_std, init_gyr_std, init_ba, init_bw (3 each)
// tuning (lins_seq_run_bag_tuned; null = the rig's run): the slot tuning of include/lins_gpu.h as 6 doubles, num_iter,
// icp_freq, nearest_feature_search_sq_dist, lidar_std, lidar_scale, imu_misalign_angle (degrees).  EstimatorParams::gpu
// takes the first five, and every decoded IMU sample goes through alignIMUtoVehicle with the angle, as imuCallback does
// (Estimator.cpp:124-135, :286-292).
void* lins_seq_run_bag_tuned(const char* path, const char* lidar_topic, const char* imu_topic, int max_scans, int lidar_model, int device,
                             const double* rig, const double* tuning, int* error);
void* lins_seq_run_bag_rig(const char* path, const char* lidar_topic, const char* imu_topic, int max_scans, int lidar_model, int device,
                           const double* rig, int* error) {
  return lins_seq_run_bag_tuned(path, lidar_topic, imu_topic, max_scans, lidar_model, device, rig, nullptr, error);
}

// alignIMUtoVehicle (Estimator.cpp:286-292) of one vector: R^T v with R = rpy2R((0, 0, deg2rad(angle))) = Rz Ry Rx
// (math_utils.h:164-182), every product entry and output summed (a0 b0 + a1 b1) + a2 b2, in f64
void lins_host_align_imu(double angle, const double* v, double* out) {
  const double y = angle * M_PI / 180.0, p = 0.0, r = 0.0;
  const double Rz[9] = {std::cos(y), -std::sin(y), 0, std::sin(y), std::cos(y), 0, 0, 0, 1};
  const double Ry[9] = {std::cos(p), 0., std::sin(p), 0., 1., 0., -std::sin(p), 0., std::cos(p)};
  const double Rx[9] = {1., 0., 0., 0., std::cos(r), -std::sin(r), 0., std::sin(r), std::cos(r)};
  auto mul = [](const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) C[3 * i + j] = (A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j];
  };
  double T[9], R[9];
  mul(Rz, Ry, T);
  mul(T, Rx, R);
  const double x = v[0], yy = v[1], z = v[2];
  for (int j = 0; j < 3; ++j) out[j] = (R[j] * x + R[3 + j] * yy) + R[6 + j] * z;
}

void* lins_seq_run_bag_tuned(const char* path, const char* lidar_topic, const char* imu_topic, int max_scans, int lidar_model, int device,
                             const double* rig, const double* tuning, int* error) {
  using namespace lins::rosbag;
  if (error) *error = 0;
  Reader rd;
  int rc = rd.open(path);
  if (rc != LINS_BAG_OK) { if (error) *error = rc; return nullptr; }
  struct ImuS { double t; V3D a, g; };
  std::vector<ImuS> imus;
  std::vector<std::pair<double, Cloud>> scans;
  bool bad = false;
  rc = rd.for_each([&](const MessageView& m) {
    if (m.conn->topic == imu_topic) {
      ImuMsg im;
      if (!decode_imu(m.data, m.size, im)) { bad = true; return; }
      double a[3] = {im.linear_acceleration[0], im.linear_acceleration[1], im.linear_acceleration[2]};
      double g[3] = {im.angular_velocity[0], im.angular_velocity[1], im.angular_velocity[2]};
      if (tuning) { const double a0[3] = {a[0], a[1], a[2]}, g0[3] = {g[0], g[1], g[2]}; lins_host_align_imu(tuning[5], a0, a); lins_host_align_imu(tuning[5], g0, g); }
      imus.push_back(ImuS{im.header.stamp, V3D(a[0], a[1], a[2]), V3D(g[0], g[1], g[2])});
    } else if (m.conn->topic == lidar_topic && (max_scans <= 0 || (int)scans.size() < max_scans)) {
      Header h;
      Cloud c;
      if (!decode_pointcloud2(m.data, m.size, h, c)) { bad = true; return; }
      scans.emplace_back(h.stamp, std::move(c));
    }
  });
  if (rc != LINS_BAG_OK || bad) { if (error) *error = rc != LINS_BAG_OK ? rc : LINS_BAG_E_FORMAT; return nullptr; }
  std::stable_sort(imus.begin(), imus.end(), [](const ImuS& x, const ImuS& y) { return x.t < y.t; });
  std::stable_sort(scans.begin(), scans.end(), [](const std::pair<double, Cloud>& x, const std::pair<double, Cloud>& y) { return x.first < y.first; });
  SeqRecord* rec = new SeqRecord();
  LidarModel lm = lidar_model == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  lins::fusion::EstimatorParams ep = seq_params(lm);
  if (rig) {
    lm.scan_period = rig[0];
    ep = seq_params(lm);
    ep.gpu.scan_period = rig[0];
    ep.feature.edge_threshold = rig[1]; ep.feature.surf_threshold = rig[2]; ep.feature.imu_lidar_extrinsic_angle = rig[3];
    ep.filter.acc_n = rig[4]; ep.filter.gyr_n = rig[5]; ep.filter.acc_w = rig[6]; ep.filter.gyr_w = rig[7];
    V3D* v[7] = {&ep.filter.init_pos_std, &ep.filter.init_vel_std, &ep.filter.init_att_std, &ep.filter.init_acc_std, &ep.filter.init_gyr_std,
                 &ep.filter.init_ba, &ep.filter.init_bw};
    for (int k = 0; k < 7; ++k) *v[k] = V3D(rig[8 + 3 * k], rig[9 + 3 * k], rig[10 + 3 * k]);
  }
  if (tuning) {
    ep.gpu.num_iter = (int)tuning[0]; ep.gpu.icp_freq = (int)tuning[1]; ep.gpu.nearest_feature_search_sq_dist = tuning[2];
    ep.gpu.lidar_std = tuning[3]; ep.gpu.lidar_scale = tuning[4];
  }
  StateEstimator est(ep, device);
  ImageProjection ip(lm);
  const bool verbose = std::getenv("LINS_SEQ_VERBOSE") != nullptr;
  size_t next_imu = 0;
  double est_time = scans.empty() ? 0.0 : scans.front().first - lm.scan_period;  // (the estimator's clock starts one sweep before the first scan)
  for (size_t k = 0; k < scans.size(); ++k) {
    const double ts = scans[k].first;
    std::vector<double> dts;
    std::vector<V3D> acc, gyr;
    while (est_time < ts && next_imu < imus.size()) {  // Estimator.cpp:228-236
      const ImuS& im = imus[next_imu];
      if (im.t <= est_time) { ++next_imu; continue; }   // upper_bound(estimator time)
      const double dt = std::min(im.t, ts) - est_time;
      dts.push_back(dt); acc.push_back(im.a); gyr.push_back(im.g);
      est_time += dt;
      if (im.t <= ts) ++next_imu;
    }
    est_time = ts;
    feed_scan(est, ip, rec, (int)k, ts, scans[k].second, dts, acc, gyr, nullptr, nullptr, verbose);
  }
  return rec;
}

void* lins_seq_run_bag(const char* path, const char* lidar_topic, const char* imu_topic, int max_scans, int lidar_model, int device, int* error) {
  return lins_seq_run_bag_rig(path, lidar_topic, imu_topic, max_scans, lidar_model, device, nullptr, error);
}

// ---- feature logs: what the front end hands the estimator per scan, replayable through the shim or sequence mode ------
// clouds[4] in lins_batch_desc order: surfPointsFlat_, cornerPointsSharp_, surfPointsLessFlat_, cornerPointsLessSharp_
typedef struct lins_feature_log_desc {
  int32_t n_scans;
  const double* time;       /* n: scan stamps */
  const double* imu;        /* k x 7 (dt, acc, gyr): the processImu calls before each scan */
  const int32_t* imu_off;   /* n + 1 */
  const double* imu_last;   /* n x 6: the acc / gyr processPCL receives with the scan */
  const lins_point* clouds[4];
  const int32_t* offs[4];   /* n + 1 each */
} lins_feature_log_desc;

struct FeatureLog {
  std::vector<double> time, imu, imu_last;
  std::vector<int32_t> imu_off{0};
  std::vector<lins_point> c[4];
  std::vector<int32_t> off[4] = {{0}, {0}, {0}, {0}};
  // the same scans as processPCL receives them (a "pcl log"): segmented cloud + cloud_info, CSR like lins_pcl_desc
  int line_num = 0;
  std::vector<lins_point> seg;
  std::vector<int32_t> seg_off{0}, start_ring, end_ring;
  std::vector<uint8_t> ground;
  std::vector<uint32_t> col;
  std::vector<float> range, ori;
  // ... and as the LiDAR driver publishes them (a "raw log"): the raw sweeps, CSR like lins_raw_desc
  std::vector<lins_point> raw;
  std::vector<int32_t> raw_off{0};
};

// a pcl log: per scan the IMU calls and processPCL's segmented cloud + cloud_info (lins_pcl_desc, n_scans == n)
typedef struct lins_pcl_log_desc {
  int32_t n_scans;
  const double* time; const double* imu; const int32_t* imu_off; const double* imu_last;
  lins_pcl_desc pcl;
} lins_pcl_log_desc;

// what the shim did with every scan of a replayed log, and its state right after it became RUNNING (the hand-over)
struct ReplayRecord {
  int handover = -1;  // index of the scan after which the shim was RUNNING for the first time
  std::vector<int32_t> code, iters, flags, replaced, est_status;  // code: LINS_SEQ_* (0 before the hand-over)
  std::vector<double> glob, filt, cov, lin;  // n x 19, n x 19, n x 324, n x 19 after each scan
  std::vector<double> scan_s;                // wall time of each scan's processImu calls + processFeatures
  // sequence initialisation: init_code = the code lins_gpu_seq_step_ex gives an opened slot (LINS_SEQ_INIT_WAIT / FIRST /
  // SECOND while initialising, else `code`); where it is LINS_SEQ_SECOND, the scan's estimateTransform result
  std::vector<int32_t> init_code, icp_iters, icp_converged;
  std::vector<double> icp_pose;              // n x 7: t (3) + q (x,y,z,w)
  double h_filt[19], h_glob[19], h_imu[6], h_cov[324];
  std::vector<lins_point> h_surf, h_corner;
};

void* lins_flog_create(const lins_synth_cfg* cfg, uint64_t seed, int n_scans) {
  FeatureLog* L = new FeatureLog();
  SimDrive sim(cfg, seed);
  ImageProjection ip(sim.lm);
  FeatureExtractor ex(sim.lm, FeatureParams());
  Sweep sw;
  for (int k = 0; k < n_scans; ++k) {
    sim.next(sw);
    for (int i = 1; i <= SimDrive::nimu; ++i) {
      const double row[7] = {sim.dt(), sw.accs[i].x(), sw.accs[i].y(), sw.accs[i].z(), sw.gyrs[i].x(), sw.gyrs[i].y(), sw.gyrs[i].z()};
      L->imu.insert(L->imu.end(), row, row + 7);
    }
    L->imu_off.push_back((int32_t)(L->imu.size() / 7));
    const double last[6] = {sw.accs.back().x(), sw.accs.back().y(), sw.accs.back().z(), sw.gyrs.back().x(), sw.gyrs.back().y(), sw.gyrs.back().z()};
    L->imu_last.insert(L->imu_last.end(), last, last + 6);
    L->time.push_back(sw.t_end);
    append_cloud(L->raw, L->raw_off, sw.raw);
    ip.process(sw.raw);
    ScanFeatures f;
    ex.run(ip.segmentedCloud, ip.segMsg, f);
    const Cloud* cl[4] = {&f.surfPointsFlat, &f.cornerPointsSharp, &f.surfPointsLessFlat, &f.cornerPointsLessSharp};
    for (int j = 0; j < 4; ++j) append_cloud(L->c[j], L->off[j], *cl[j]);
    const CloudInfo& ci = ip.segMsg;
    L->line_num = sim.lm.line_num;
    append_cloud(L->seg, L->seg_off, ip.segmentedCloud);
    const size_t m = ip.segmentedCloud.size();
    L->ground.insert(L->ground.end(), ci.segmentedCloudGroundFlag.begin(), ci.segmentedCloudGroundFlag.begin() + m);
    L->col.insert(L->col.end(), ci.segmentedCloudColInd.begin(), ci.segmentedCloudColInd.begin() + m);
    L->range.insert(L->range.end(), ci.segmentedCloudRange.begin(), ci.segmentedCloudRange.begin() + m);
    L->start_ring.insert(L->start_ring.end(), ci.startRingIndex.begin(), ci.startRingIndex.end());
    L->end_ring.insert(L->end_ring.end(), ci.endRingIndex.begin(), ci.endRingIndex.end());
    const float o3[3] = {ci.startOrientation, ci.endOrientation, ci.orientationDiff};
    L->ori.insert(L->ori.end(), o3, o3 + 3);
  }
  return L;
}
// the pcl-log view of a feature log made by lins_flog_create (valid while the log lives)
void lins_plog_desc(void* h, lins_pcl_log_desc* d) {
  FeatureLog* L = static_cast<FeatureLog*>(h);
  d->n_scans = (int32_t)L->time.size();
  d->time = L->time.data(); d->imu = L->imu.data(); d->imu_off = L->imu_off.data(); d->imu_last = L->imu_last.data();
  lins_pcl_desc& p = d->pcl;
  p.n_scans = d->n_scans; p.line_num = L->line_num;
  p.cloud = L->seg.data(); p.cloud_off = L->seg_off.data();
  p.ground_flag = L->ground.data(); p.col_ind = L->col.data(); p.range = L->range.data();
  p.start_ring_index = L->start_ring.data(); p.end_ring_index = L->end_ring.data(); p.orientation = L->ori.data();
  p.point_format = LINS_POINTS_XYZI32;
}
// the raw sweeps of a feature log made by lins_flog_create (valid while the log lives)
void lins_flog_raw(void* h, lins_raw_desc* d) {
  FeatureLog* L = static_cast<FeatureLog*>(h);
  d->n_scans = (int32_t)L->time.size();
  d->cloud = L->raw.data(); d->cloud_off = L->raw_off.data();
  d->point_format = LINS_POINTS_XYZI32;
}
void lins_flog_destroy(void* h) { delete static_cast<FeatureLog*>(h); }
void lins_flog_desc(void* h, lins_feature_log_desc* d) {
  FeatureLog* L = static_cast<FeatureLog*>(h);
  d->n_scans = (int32_t)L->time.size();
  d->time = L->time.data(); d->imu = L->imu.data(); d->imu_off = L->imu_off.data(); d->imu_last = L->imu_last.data();
  for (int j = 0; j < 4; ++j) { d->clouds[j] = L->c[j].data(); d->offs[j] = L->off[j].data(); }
}

// Replay a (possibly edited) feature log through one shim: processImu for every IMU row, then processFeatures.
// gpu: the C-ABI parameters of the shim's context (NULL = the shipped ones); init_std: INIT_POS_STD (3) + INIT_ATT_STD (3,
// degrees) of its filter (NULL = zero)
// One shim over n scans: processImu for every IMU row of scan k, then feed(est, k, f), which hands the scan to the
// estimator and leaves its four feature clouds in f (for the record's gate and code)
}  // extern "C"
template <typename Feed>
static ReplayRecord* replay_scans(int n_scans, const double* time, const double* imu, const int32_t* imu_off, const double* imu_last,
                                  int lidar_model, int device, const lins_params* gpu, const double* init_std, Feed feed);
extern "C" {

void* lins_flog_replay(const lins_feature_log_desc* d, int lidar_model, int device, const lins_params* gpu, const double* init_std) {
  return replay_scans(d->n_scans, d->time, d->imu, d->imu_off, d->imu_last, lidar_model, device, gpu, init_std,
                      [d](StateEstimator& est, int k, const lins::sensor_utils::Imu& im, ScanFeatures& f) {
                        Cloud* cl[4] = {&f.surfPointsFlat, &f.cornerPointsSharp, &f.surfPointsLessFlat, &f.cornerPointsLessSharp};
                        for (int j = 0; j < 4; ++j) cl[j]->points.assign(d->clouds[j] + d->offs[j][k], d->clouds[j] + d->offs[j][k + 1]);
                        est.processFeatures(d->time[k], im, f);
                      });
}

// Replay a (possibly edited) pcl log through one shim: processImu for every IMU row, then processPCL with the scan's
// segmented cloud and cloud_info (the shim's own FeatureExtractor runs; the outlier cloud is empty: the odometry never
// reads it).  Same record as lins_flog_replay.
void* lins_plog_replay(const lins_pcl_log_desc* d, int lidar_model, int device, const lins_params* gpu, const double* init_std) {
  const LidarModel lm0 = lidar_model == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  return replay_scans(d->n_scans, d->time, d->imu, d->imu_off, d->imu_last, lidar_model, device, gpu, init_std,
                      [d, lm0](StateEstimator& est, int k, const lins::sensor_utils::Imu& im, ScanFeatures& f) {
                        const lins_pcl_desc& p = d->pcl;
                        const int a = p.cloud_off[k], b = p.cloud_off[k + 1], L = p.line_num;
                        Cloud cloud, outlier;
                        cloud.points.assign(p.cloud + a, p.cloud + b);
                        CloudInfo info;
                        info.resize(L, b - a);
                        for (int i = 0; i < L; ++i) { info.startRingIndex[i] = p.start_ring_index[(size_t)k * L + i]; info.endRingIndex[i] = p.end_ring_index[(size_t)k * L + i]; }
                        info.startOrientation = p.orientation[3 * k]; info.endOrientation = p.orientation[3 * k + 1]; info.orientationDiff = p.orientation[3 * k + 2];
                        for (int i = a; i < b; ++i) {
                          info.segmentedCloudGroundFlag[i - a] = p.ground_flag[i]; info.segmentedCloudColInd[i - a] = p.col_ind[i]; info.segmentedCloudRange[i - a] = p.range[i];
                        }
                        LidarModel lm = lm0;
                        lm.line_num = L;
                        FeatureExtractor(lm, FeatureParams()).run(cloud, info, f);  // (what processPCL extracts: the record's sizes)
                        est.processPCL(d->time[k], im, cloud, info, outlier);
                      });
}

}  // extern "C"
template <typename Feed>
static ReplayRecord* replay_scans(int n_scans, const double* time, const double* imu, const int32_t* imu_off, const double* imu_last,
                                  int lidar_model, int device, const lins_params* gpu, const double* init_std, Feed feed) {
  ReplayRecord* R = new ReplayRecord();
  const LidarModel lm = lidar_model == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  lins::fusion::EstimatorParams ep = seq_params(lm);
  if (gpu) ep.gpu = *gpu;
  if (init_std) { ep.filter.init_pos_std = V3D(init_std[0], init_std[1], init_std[2]); ep.filter.init_att_std = V3D(init_std[3], init_std[4], init_std[5]); }
  StateEstimator est(ep, device);
  for (int k = 0; k < n_scans; ++k) {
    const auto t0 = std::chrono::steady_clock::now();
    for (int m = imu_off[k]; m < imu_off[k + 1]; ++m) {
      const double* r = imu + (size_t)m * 7;
      est.processImu(r[0], V3D(r[1], r[2], r[3]), V3D(r[4], r[5], r[6]));
    }
    ScanFeatures f;
    const bool running = est.status_ == StateEstimator::STATUS_RUNNING;
    const StateEstimator::FusionStatus before = est.status_;
    est.last_report_ = lins_report();
    const double* il = imu_last + (size_t)k * 6;
    feed(est, k, lins::sensor_utils::Imu(time[k], V3D(il[0], il[1], il[2]), V3D(il[3], il[4], il[5])), f);
    R->scan_s.push_back(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
    int code = LINS_SEQ_IDLE;
    if (running) {
      const bool gate = f.cornerPointsLessSharp.size() <= 5 || f.surfPointsLessFlat.size() <= 10;  // processScan (:436-440)
      code = gate ? LINS_SEQ_SKIPPED : est.last_report_.diverged ? LINS_SEQ_ICP : LINS_SEQ_RAN;
    }
    R->code.push_back(code);
    int icode = code;
    if (before == StateEstimator::STATUS_INIT) icode = est.status_ == StateEstimator::STATUS_FIRST_SCAN ? LINS_SEQ_FIRST : LINS_SEQ_INIT_WAIT;
    else if (before == StateEstimator::STATUS_FIRST_SCAN) icode = est.status_ == StateEstimator::STATUS_RUNNING ? LINS_SEQ_SECOND : LINS_SEQ_INIT_WAIT;
    R->init_code.push_back(icode);
    double ip[7] = {0, 0, 0, 0, 0, 0, 0};
    if (icode == LINS_SEQ_SECOND) {
      const double v[7] = {est.linState_.rn_.x(), est.linState_.rn_.y(), est.linState_.rn_.z(), est.linState_.qbn_.x(),
                           est.linState_.qbn_.y(), est.linState_.qbn_.z(), est.linState_.qbn_.w()};
      std::memcpy(ip, v, sizeof(v));
    }
    R->icp_pose.insert(R->icp_pose.end(), ip, ip + 7);
    R->icp_iters.push_back(icode == LINS_SEQ_SECOND ? est.last_icp_iters_ : 0);
    R->icp_converged.push_back(icode == LINS_SEQ_SECOND ? est.last_icp_converged_ : 0);
    R->iters.push_back(est.last_report_.iters);
    R->flags.push_back((est.last_report_.converged ? 1 : 0) | (est.last_report_.diverged ? 2 : 0) | (est.last_report_.has_nan ? 4 : 0));
    R->replaced.push_back(code >= LINS_SEQ_RAN && est.last_map_replaced_ ? 1 : 0);
    R->est_status.push_back((int)est.status_);
    double g[19], s[19], l[19];
    est.globalState_.toArray(g); est.filter_->state_.toArray(s); est.linState_.toArray(l);
    R->glob.insert(R->glob.end(), g, g + 19);
    R->filt.insert(R->filt.end(), s, s + 19);
    R->lin.insert(R->lin.end(), l, l + 19);
    R->cov.insert(R->cov.end(), est.filter_->covariance_.data(), est.filter_->covariance_.data() + 324);
    if (R->handover < 0 && est.status_ == StateEstimator::STATUS_RUNNING) {
      R->handover = k;
      std::memcpy(R->h_filt, s, sizeof(s)); std::memcpy(R->h_glob, g, sizeof(g));
      std::memcpy(R->h_cov, est.filter_->covariance_.data(), sizeof(R->h_cov));
      const V3D& a = est.filter_->acc_last; const V3D& w = est.filter_->gyr_last;
      const double im[6] = {a.x(), a.y(), a.z(), w.x(), w.y(), w.z()};
      std::memcpy(R->h_imu, im, sizeof(im));
      R->h_surf = est.scan_last_->surfPointsLessFlat_.points;  // (already moved to the scan end by updatePointCloud)
      R->h_corner = est.scan_last_->cornerPointsLessSharp_.points;
    }
  }
  return R;
}
extern "C" {
// k StatePredictor::predict calls (default FilterParams) from state / covariance / acc_last + gyr_last, in place: the
// host side of the predict stage check
void lins_host_predict(double* state, double* cov, double* imu_last, const double* rows, int k) {
  filter::StatePredictor sp;
  sp.initialization(0.0, V3D(), V3D(), V3D(), V3D(), V3D(imu_last[0], imu_last[1], imu_last[2]), V3D(imu_last[3], imu_last[4], imu_last[5]));
  sp.state_ = filter::GlobalState::fromArray(state);
  std::memcpy(sp.covariance_.data(), cov, sizeof(double) * 324);
  for (int m = 0; m < k; ++m) {
    const double* r = rows + 7 * m;
    sp.predict(r[0], V3D(r[1], r[2], r[3]), V3D(r[4], r[5], r[6]), true);
  }
  sp.state_.toArray(state);
  std::memcpy(cov, sp.covariance_.data(), sizeof(double) * 324);
  const double il[6] = {sp.acc_last.x(), sp.acc_last.y(), sp.acc_last.z(), sp.gyr_last.x(), sp.gyr_last.y(), sp.gyr_last.z()};
  std::memcpy(imu_last, il, sizeof(il));
}

// seconds per call of StatePredictor::predict (the host IMU propagation sequence mode replaces) over `rows` (k x 7)
double lins_bench_host_predict(const double* rows, int k, int reps) {
  filter::StatePredictor sp;
  sp.initialization(0.0, V3D(), V3D(), V3D(), V3D(), V3D(0, 0, 9.81), V3D());
  const auto t0 = std::chrono::steady_clock::now();
  for (int r = 0; r < reps; ++r)
    for (int m = 0; m < k; ++m) sp.predict(rows[7 * m], V3D(rows[7 * m + 1], rows[7 * m + 2], rows[7 * m + 3]), V3D(rows[7 * m + 4], rows[7 * m + 5], rows[7 * m + 6]), true);
  const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  volatile double sink = sp.covariance_.a[0];
  (void)sink;
  return s / ((double)reps * (k > 0 ? k : 1));
}

void lins_replay_destroy(void* h) { delete static_cast<ReplayRecord*>(h); }
int lins_replay_handover(void* h) { return static_cast<ReplayRecord*>(h)->handover; }
const int32_t* lins_replay_ints(void* h, int which) {
  ReplayRecord* R = static_cast<ReplayRecord*>(h);
  const std::vector<int32_t>* v[8] = {&R->code, &R->iters, &R->flags, &R->replaced, &R->est_status, &R->init_code, &R->icp_iters, &R->icp_converged};
  return which >= 0 && which < 8 ? v[which]->data() : nullptr;
}
const double* lins_replay_doubles(void* h, int which) {
  ReplayRecord* R = static_cast<ReplayRecord*>(h);
  switch (which) {
    case 0: return R->glob.data();
    case 1: return R->filt.data();
    case 2: return R->cov.data();
    case 3: return R->lin.data();
    case 4: return R->h_filt;
    case 5: return R->h_glob;
    case 6: return R->h_cov;
    case 7: return R->h_imu;
    case 8: return R->scan_s.data();
    case 9: return R->icp_pose.data();
  }
  return nullptr;
}
// the hand-over's maps: which 0 = surf, 1 = corner; returns the point count
int lins_replay_handover_cloud(void* h, int which, const lins_point** pts) {
  ReplayRecord* R = static_cast<ReplayRecord*>(h);
  const std::vector<lins_point>& c = which == 0 ? R->h_surf : R->h_corner;
  *pts = c.data();
  return (int)c.size();
}

void lins_seq_destroy(void* h) { delete static_cast<SeqRecord*>(h); }
// the mapping node's inputs of a record: n published scans; time (n), odom (n x 7: YZX position, quaternion x y z w), and
// the YZX clouds (which: 0 less-sharp, 1 less-flat, 2 outlier) with their CSR offsets (n + 1)
int lins_seq_map_count(void* h) { return (int)static_cast<SeqRecord*>(h)->map_time.size(); }
const double* lins_seq_map_array(void* h, int which) {
  SeqRecord* r = static_cast<SeqRecord*>(h);
  return which == 0 ? r->map_time.data() : r->map_odom.data();
}
const lins_point* lins_seq_map_cloud(void* h, int which, const int32_t** off) {
  SeqRecord* r = static_cast<SeqRecord*>(h);
  *off = r->map_off[which].data();
  return r->map_cloud[which].data();
}
int lins_seq_num_units(void* h) { return (int)static_cast<SeqRecord*>(h)->iters.size(); }
int lins_seq_num_scans(void* h) { return (int)static_cast<SeqRecord*>(h)->status.size(); }
void lins_seq_desc(void* h, lins_batch_desc* d) {
  SeqRecord* r = static_cast<SeqRecord*>(h);
  d->n_scans = (int32_t)r->iters.size();
  d->surf_flat = r->surfFlat.data(); d->surf_flat_off = r->offSF.data();
  d->corner_sharp = r->cornerSharp.data(); d->corner_sharp_off = r->offCS.data();
  d->surf_less_flat = r->surfLessFlat.data(); d->surf_less_flat_off = r->offSL.data();
  d->corner_less_sharp = r->cornerLessSharp.data(); d->corner_less_sharp_off = r->offCL.data();
  d->state_in = r->state_in.data(); d->cov_in = r->cov_in.data();
  d->point_format = LINS_POINTS_XYZI32;
}
const double* lins_seq_array(void* h, int which) {
  SeqRecord* r = static_cast<SeqRecord*>(h);
  switch (which) {
    case 0: return r->state_out.data();
    case 1: return r->rel_true.data();
    case 2: return r->global_est.data();
    case 3: return r->global_true.data();
  }
  return nullptr;
}
const int32_t* lins_seq_ints(void* h, int which) {
  SeqRecord* r = static_cast<SeqRecord*>(h);
  switch (which) {
    case 0: return r->iters.data();
    case 1: return r->flags.data();
    case 2: return r->scan_index.data();
    case 3: return r->status.data();
  }
  return nullptr;
}

}  // extern "C"
