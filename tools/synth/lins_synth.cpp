// tools/synth/lins_synth.cpp — synthetic input generator (SURVEY.md §8(d) configs 1/3/4/5).
//
// Not part of the hot path and not an oracle: it manufactures the INPUTS (scan pairs + IMU priors) that the
// CUDA path, the oracle and the benchmarks all consume.  The reference ships no dataset (README.md:51 links an
// external bag) so every workload here is synthetic:
//   world  : ground plane + rectangular room (walls) + vertical poles + boxes, seeded
//   sensor : VLP-16 (16 x 1800, parameters.h:82-84) or a 64 x 1024 dense shape; clockwise firing, one column
//            per firing, constant body twist over the scan (the motion model transformToStart assumes,
//            StateEstimator.hpp:1066-1080); range noise N(0, sigma)
//   stages : the product's own host-side CPU restatements — ImageProjection (image_projection_node.cpp:191-415),
//            FeatureExtractor (StateEstimator.hpp:619-827), StatePredictor (KalmanFilter.hpp:125-186, :314-354)
//   unit   : (scan A -> targets in A's end frame, scan B -> queries, prior state + covariance from 40 IMU steps)
// Never includes anything from oracle/.
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../../lins---lidar-inertial-slam_b200/csrc/host/feature_extraction.hpp"
#include "../../lins---lidar-inertial-slam_b200/csrc/host/image_projection.hpp"
#include "../../lins---lidar-inertial-slam_b200/csrc/host/kalman_filter.hpp"

using namespace lins;
using lins::filter::GlobalState;
using lins::filter::StatePredictor;

namespace {

// ---- deterministic RNG (splitmix64 + Box-Muller), identical on every platform -----------------------------
struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ull + 0x1234567ull) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uni() { return (next() >> 11) * (1.0 / 9007199254740992.0); }  // [0,1)
  double uni(double a, double b) { return a + (b - a) * uni(); }
  double gauss() {
    double u1 = uni(), u2 = uni();
    if (u1 < 1e-300) u1 = 1e-300;
    return std::sqrt(-2.0 * std::log(u1)) * std::cos(2.0 * M_PI * u2);
  }
};

struct Pole { double cx, cy, r; };
struct Box { double x0, x1, y0, y1, h; };
struct World {
  double Lx = 20, Ly = 15;  // walls at x = +-Lx, y = +-Ly
  bool walls = true;
  std::vector<Pole> poles;
  std::vector<Box> boxes;
};

World make_world(Rng& rng, int kind) {
  World w;
  if (kind == 0) {
    w.Lx = rng.uni(15, 25); w.Ly = rng.uni(10, 20);
    int np = 12 + (int)(rng.uni() * 6);
    for (int i = 0; i < np; ++i) w.poles.push_back(Pole{rng.uni(-w.Lx + 2, w.Lx - 2), rng.uni(-w.Ly + 2, w.Ly - 2), rng.uni(0.15, 0.3)});
    int nb = 4 + (int)(rng.uni() * 4);
    for (int i = 0; i < nb; ++i) {
      double cx = rng.uni(-w.Lx + 3, w.Lx - 3), cy = rng.uni(-w.Ly + 3, w.Ly - 3), sx = rng.uni(0.5, 2.0), sy = rng.uni(0.5, 2.0);
      w.boxes.push_back(Box{cx - sx, cx + sx, cy - sy, cy + sy, rng.uni(0.8, 3.0)});
    }
  } else {  // open flat ground, sparse poles, a few buildings; no enclosing walls (sky = no return)
    w.walls = false;
    w.Lx = w.Ly = 1e9;
    int np = 16 + (int)(rng.uni() * 10);
    for (int i = 0; i < np; ++i) w.poles.push_back(Pole{rng.uni(-30, 30), rng.uni(-30, 30), rng.uni(0.15, 0.4)});
    int nb = 5 + (int)(rng.uni() * 4);
    for (int i = 0; i < nb; ++i) {
      double cx = rng.uni(-35, 35), cy = rng.uni(-35, 35), sx = rng.uni(1.0, 6.0), sy = rng.uni(1.0, 6.0);
      if (std::fabs(cx) < 12 && std::fabs(cy) < 12) { cx += cx >= 0 ? 14 : -14; }  // keep the sensor's start area free
      w.boxes.push_back(Box{cx - sx, cx + sx, cy - sy, cy + sy, rng.uni(2.0, 8.0)});
    }
  }
  return w;
}

// nearest positive hit distance along o + t d (|d| = 1), or +inf
double raycast(const World& w, const V3D& o, const V3D& d) {
  double best = INFINITY;
  auto upd = [&](double t) { if (t > 0.3 && t < best) best = t; };
  if (d.z() < -1e-12) upd(-o.z() / d.z());  // ground z = 0
  if (w.walls) {
    if (d.x() > 1e-12) upd((w.Lx - o.x()) / d.x()); else if (d.x() < -1e-12) upd((-w.Lx - o.x()) / d.x());
    if (d.y() > 1e-12) upd((w.Ly - o.y()) / d.y()); else if (d.y() < -1e-12) upd((-w.Ly - o.y()) / d.y());
  }
  const double a = d.x() * d.x() + d.y() * d.y();
  if (a > 1e-12) {
    for (const auto& p : w.poles) {
      double ox = o.x() - p.cx, oy = o.y() - p.cy;
      double b = ox * d.x() + oy * d.y(), c = ox * ox + oy * oy - p.r * p.r;
      double disc = b * b - a * c;
      if (disc <= 0) continue;
      double t = (-b - std::sqrt(disc)) / a;
      if (t > 0.3 && t < best && o.z() + t * d.z() >= 0) best = t;
    }
  }
  for (const auto& bx : w.boxes) {
    double tmin = -INFINITY, tmax = INFINITY;
    const double lo[3] = {bx.x0, bx.y0, 0.0}, hi[3] = {bx.x1, bx.y1, bx.h};
    bool miss = false;
    for (int k = 0; k < 3 && !miss; ++k) {
      double ok = o(k), dk = d(k);
      if (std::fabs(dk) < 1e-12) { if (ok < lo[k] || ok > hi[k]) miss = true; continue; }
      double t0 = (lo[k] - ok) / dk, t1 = (hi[k] - ok) / dk;
      if (t0 > t1) std::swap(t0, t1);
      tmin = std::max(tmin, t0); tmax = std::min(tmax, t1);
      if (tmin > tmax) miss = true;
    }
    if (!miss) upd(tmin);
  }
  return best;
}

struct Pose { M3D R; V3D p; };        // sensor -> world
struct Twist { V3D phi, t; };          // end-of-scan pose relative to start-of-scan frame

// One rotation of the sensor. Firing k (k = 0..N-1) happens at motion fraction k/N with
// ori_k = -pi + (k + 0.25) * 2pi/N (ori = -atan2(y, x), increasing = clockwise), all rings at once.
void simulate_scan(const World& w, const LidarModel& lm, const Pose& T0, const Twist& tw, double range_noise, Rng& rng, Cloud& raw) {
  raw.clear();
  const int N = lm.scan_num;
  for (int k = 0; k < N; ++k) {
    double s = (double)k / N;
    Q4D qs = math_utils::axis2Quat(s * tw.phi);
    M3D Rs = T0.R * qs.toRotationMatrix();
    V3D ps = T0.p + T0.R * (s * tw.t);
    double ori = -M_PI + (k + 0.25) * (2.0 * M_PI / N);
    for (int r = 0; r < lm.line_num; ++r) {
      double el = (-(double)(lm.ang_bottom - 0.1f) + r * (double)lm.ang_res_y) * M_PI / 180.0;
      V3D ds(std::cos(el) * std::cos(ori), -std::cos(el) * std::sin(ori), std::sin(el));
      V3D dw = Rs * ds;
      double t = raycast(w, ps, dw);
      if (!(t < 100.0)) continue;
      t += range_noise * rng.gauss();
      raw.push_back(makePoint((float)(t * ds.x()), (float)(t * ds.y()), (float)(t * ds.z()), 0.f));
    }
  }
}

// transformToEnd with the host math (generator only; the product's on-device version is lins_gpu_update_map)
void to_end_frame(Cloud& c, const Twist& tw, double scan_period) {
  Q4D q = math_utils::axis2Quat(tw.phi);
  for (auto& p : c.points) {
    double s = (1.f / scan_period) * (p.intensity - int(p.intensity));
    V3D P(p.x, p.y, p.z);
    V3D P1 = math_utils::axis2Quat(s * tw.phi) * P + s * tw.t;
    V3D P2 = q.inverse() * (P1 - tw.t);
    p.x = (float)P2.x(); p.y = (float)P2.y(); p.z = (float)P2.z();
  }
}

}  // namespace

extern "C" {

typedef struct lins_synth_cfg {
  int32_t lidar;           // 0 = VLP-16 16x1800, 1 = dense 64x1024
  int32_t world;           // 0 = room + poles + boxes, 1 = open flat ground + sparse poles
  int32_t fixed_motion;    // 1 = config-1 motion: v = (2.0, 0.2, 0) m/s, yaw rate 0.15 rad/s
  int32_t stress_queries;  // 1 = use scan B's less-flat / less-sharp clouds as the queries ("1b")
  double v_max;            // |v| ~ U(0, v_max) m/s
  double w_max;            // yaw rate ~ U(-w_max, w_max) rad/s
  double range_noise;      // sigma of the range noise, m
  double prior_vel_sigma;  // sigma of the velocity error in the prior, m/s
} lins_synth_cfg;

struct Unit {
  Cloud surfFlat, cornerSharp, surfLessFlat, cornerLessSharp;
  // scan B's own less-* clouds, still in B's distorted frame (input of lins_gpu_update_map, row F1)
  Cloud newSurfLessFlat, newCornerLessSharp;
  double state[19];
  double cov[324];
  double truth[7];  // true relative pose of scan B: t (3) + q (x,y,z,w)
};

struct SynthBatch {
  std::vector<Unit> units;
  // concatenated views
  std::vector<lins_point> surfFlat, cornerSharp, surfLessFlat, cornerLessSharp, newSurfLessFlat, newCornerLessSharp;
  std::vector<int32_t> surfFlatOff, cornerSharpOff, surfLessFlatOff, cornerLessSharpOff, newSurfLessFlatOff, newCornerLessSharpOff;
  std::vector<double> state, cov, truth;
};

static void gen_unit(uint64_t seed, const lins_synth_cfg& cfg, Unit& u) {
  Rng rng(seed);
  LidarModel lm = cfg.lidar == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  const double T = lm.scan_period;
  World w = make_world(rng, cfg.world);
  // start pose: inside the central region, random yaw, small tilt, sensor height 1.2 .. 1.8 m
  Pose T0;
  double yaw = rng.uni(-M_PI, M_PI), roll = rng.uni(-0.02, 0.02), pitch = rng.uni(-0.02, 0.02);
  T0.R = math_utils::rpy2Quat(V3D(roll, pitch, yaw)).toRotationMatrix();
  double cx = cfg.world == 0 ? w.Lx * 0.4 : 10.0, cy = cfg.world == 0 ? w.Ly * 0.4 : 10.0;
  T0.p = V3D(rng.uni(-cx, cx), rng.uni(-cy, cy), rng.uni(1.2, 1.8));
  // body-frame motion
  V3D vA, wA;
  if (cfg.fixed_motion) {
    vA = V3D(2.0, 0.2, 0.0); wA = V3D(0, 0, 0.15);
  } else {
    double sp = rng.uni(0, cfg.v_max), hd = rng.uni(-0.3, 0.3);
    vA = V3D(sp * std::cos(hd), sp * std::sin(hd), rng.uni(-0.05, 0.05));
    wA = V3D(rng.uni(-0.02, 0.02), rng.uni(-0.02, 0.02), rng.uni(-cfg.w_max, cfg.w_max));
  }
  // scan B continues with a slightly different twist (bounded acceleration)
  V3D vB = vA + V3D(rng.uni(-0.1, 0.1), rng.uni(-0.05, 0.05), rng.uni(-0.01, 0.01));
  V3D wB = wA + V3D(rng.uni(-0.005, 0.005), rng.uni(-0.005, 0.005), rng.uni(-0.02, 0.02));
  Twist twA{T * wA, T * vA}, twB{T * wB, T * vB};
  Pose T1;
  T1.R = T0.R * math_utils::axis2Quat(twA.phi).toRotationMatrix();
  T1.p = T0.p + T0.R * twA.t;

  Cloud rawA, rawB;
  simulate_scan(w, lm, T0, twA, cfg.range_noise, rng, rawA);
  simulate_scan(w, lm, T1, twB, cfg.range_noise, rng, rawB);

  ImageProjection ip(lm);
  FeatureExtractor fe(lm);
  ScanFeatures fa, fb;
  ip.process(rawA);
  fe.run(ip.segmentedCloud, ip.segMsg, fa);
  ip.process(rawB);
  fe.run(ip.segmentedCloud, ip.segMsg, fb);

  // targets: scan A's less-* features re-projected to A's end frame (= B's start frame) with A's pose as the
  // filter would have estimated it: truth + a small estimation error
  Twist twAest = twA;
  twAest.t = twAest.t + V3D(2e-3 * rng.gauss(), 2e-3 * rng.gauss(), 2e-3 * rng.gauss());
  twAest.phi = twAest.phi + V3D(2e-4 * rng.gauss(), 2e-4 * rng.gauss(), 2e-4 * rng.gauss());
  u.surfLessFlat = fa.surfPointsLessFlat;
  u.cornerLessSharp = fa.cornerPointsLessSharp;
  to_end_frame(u.surfLessFlat, twAest, T);
  to_end_frame(u.cornerLessSharp, twAest, T);
  if (cfg.stress_queries) {
    u.surfFlat = fb.surfPointsLessFlat; u.cornerSharp = fb.cornerPointsLessSharp;
  } else {
    u.surfFlat = fb.surfPointsFlat; u.cornerSharp = fb.cornerPointsSharp;
  }
  u.newSurfLessFlat = fb.surfPointsLessFlat;
  u.newCornerLessSharp = fb.cornerPointsLessSharp;

  // prior: reset(1)-like state at B's start + 40 IMU steps (400 Hz) of the constant-twist motion
  filter::FilterParams fp;
  StatePredictor filt(fp);
  V3D g_w(0, 0, -filter::G0);
  M3D R1t = T1.R.transpose();
  V3D gn = R1t * g_w;                      // gravity in B's start frame
  V3D ba_true(rng.uni(-0.02, 0.02), rng.uni(-0.02, 0.02), rng.uni(-0.02, 0.02));
  V3D bw_true(rng.uni(-0.002, 0.002), rng.uni(-0.002, 0.002), rng.uni(-0.002, 0.002));
  V3D v0 = vB + V3D(cfg.prior_vel_sigma * rng.gauss(), cfg.prior_vel_sigma * rng.gauss(), cfg.prior_vel_sigma * rng.gauss());
  V3D ba0 = ba_true + V3D(0.005 * rng.gauss(), 0.005 * rng.gauss(), 0.005 * rng.gauss());
  V3D bw0 = bw_true + V3D(2e-4 * rng.gauss(), 2e-4 * rng.gauss(), 2e-4 * rng.gauss());
  const int nimu = 40;
  const double dt = T / nimu;
  auto imu_at = [&](double s, V3D& acc, V3D& gyr) {
    M3D Rs = math_utils::axis2Quat(s * twB.phi).toRotationMatrix();
    // constant linear velocity in the start frame => zero acceleration: acc = R^T (0 - gn) + ba
    acc = Rs.transpose() * (-gn) + ba_true + V3D(0.02 * rng.gauss(), 0.02 * rng.gauss(), 0.02 * rng.gauss());
    gyr = wB + bw_true + V3D(5e-4 * rng.gauss(), 5e-4 * rng.gauss(), 5e-4 * rng.gauss());
  };
  V3D acc, gyr;
  imu_at(0.0, acc, gyr);
  filt.initialization(0.0, V3D(0, 0, 0), v0, Q4D(), ba0, bw0, acc, gyr);
  filt.state_.gn_ = gn + V3D(0.01 * rng.gauss(), 0.01 * rng.gauss(), 0.01 * rng.gauss());
  filt.state_.gn_ = filt.state_.gn_ * 9.81 / filt.state_.gn_.norm();
  // covariance after reset(1): pos/att = init std (0), vel / ba / bw / g blocks carried over from steady state
  filt.covariance_.setZero();
  double sv = cfg.prior_vel_sigma > 0.02 ? cfg.prior_vel_sigma : 0.02;
  filt.covariance_.setDiag3(GlobalState::vel_, V3D(sv * sv, sv * sv, sv * sv));
  filt.covariance_.setDiag3(GlobalState::acc_, V3D(1e-4, 1e-4, 4e-4));
  filt.covariance_.setDiag3(GlobalState::gyr_, V3D(4e-6, 4e-6, 4e-6));
  filt.covariance_.setDiag3(GlobalState::gra_, V3D(0.01, 0.01, 0.01));
  for (int k = 1; k <= nimu; ++k) {
    imu_at((double)k / nimu, acc, gyr);
    filt.predict(dt, acc, gyr, true);
  }
  filt.state_.toArray(u.state);
  std::memcpy(u.cov, filt.covariance_.data(), sizeof(u.cov));
  Q4D qB = math_utils::axis2Quat(twB.phi);
  u.truth[0] = twB.t.x(); u.truth[1] = twB.t.y(); u.truth[2] = twB.t.z();
  u.truth[3] = qB.x(); u.truth[4] = qB.y(); u.truth[5] = qB.z(); u.truth[6] = qB.w();
}

static void append(std::vector<lins_point>& dst, std::vector<int32_t>& off, const Cloud& c) {
  dst.insert(dst.end(), c.points.begin(), c.points.end());
  off.push_back((int32_t)dst.size());
}

// Generate n units with seeds seed0 .. seed0+n-1 on n_threads threads.
void* lins_synth_batch_create(const lins_synth_cfg* cfg, uint64_t seed0, int n, int n_threads) {
  SynthBatch* b = new SynthBatch();
  b->units.resize(n);
  if (n_threads < 1) n_threads = 1;
  std::atomic<int> next(0);
  auto worker = [&]() {
    for (;;) {
      int i = next.fetch_add(1);
      if (i >= n) break;
      gen_unit(seed0 + (uint64_t)i, *cfg, b->units[i]);
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < n_threads; ++t) th.emplace_back(worker);
  worker();
  for (auto& t : th) t.join();
  b->surfFlatOff.push_back(0); b->cornerSharpOff.push_back(0); b->surfLessFlatOff.push_back(0);
  b->cornerLessSharpOff.push_back(0); b->newSurfLessFlatOff.push_back(0); b->newCornerLessSharpOff.push_back(0);
  for (int i = 0; i < n; ++i) {
    const Unit& u = b->units[i];
    append(b->surfFlat, b->surfFlatOff, u.surfFlat);
    append(b->cornerSharp, b->cornerSharpOff, u.cornerSharp);
    append(b->surfLessFlat, b->surfLessFlatOff, u.surfLessFlat);
    append(b->cornerLessSharp, b->cornerLessSharpOff, u.cornerLessSharp);
    append(b->newSurfLessFlat, b->newSurfLessFlatOff, u.newSurfLessFlat);
    append(b->newCornerLessSharp, b->newCornerLessSharpOff, u.newCornerLessSharp);
    b->state.insert(b->state.end(), u.state, u.state + 19);
    b->cov.insert(b->cov.end(), u.cov, u.cov + 324);
    b->truth.insert(b->truth.end(), u.truth, u.truth + 7);
  }
  b->units.clear();
  b->units.shrink_to_fit();
  return b;
}
void lins_synth_batch_destroy(void* h) { delete static_cast<SynthBatch*>(h); }

// Fills a lins_batch_desc whose pointers alias the batch's storage (valid until destroy).
void lins_synth_batch_desc(void* h, lins_batch_desc* d) {
  SynthBatch* b = static_cast<SynthBatch*>(h);
  d->n_scans = (int32_t)b->surfFlatOff.size() - 1;
  d->surf_flat = b->surfFlat.data(); d->surf_flat_off = b->surfFlatOff.data();
  d->corner_sharp = b->cornerSharp.data(); d->corner_sharp_off = b->cornerSharpOff.data();
  d->surf_less_flat = b->surfLessFlat.data(); d->surf_less_flat_off = b->surfLessFlatOff.data();
  d->corner_less_sharp = b->cornerLessSharp.data(); d->corner_less_sharp_off = b->cornerLessSharpOff.data();
  d->state_in = b->state.data(); d->cov_in = b->cov.data();
  d->point_format = LINS_POINTS_XYZI32;
}
const double* lins_synth_batch_truth(void* h) { return static_cast<SynthBatch*>(h)->truth.data(); }
// scan B's own less-* clouds (distorted frame): which = 0 surf, 1 corner
void lins_synth_batch_new_less(void* h, int which, const lins_point** pts, const int32_t** off) {
  SynthBatch* b = static_cast<SynthBatch*>(h);
  if (which == 0) { *pts = b->newSurfLessFlat.data(); *off = b->newSurfLessFlatOff.data(); }
  else { *pts = b->newCornerLessSharp.data(); *off = b->newCornerLessSharpOff.data(); }
}


// ---- row F2: one scan-to-map unit (what scan2MapOptimization sees, lidar_mapping_node.cpp:1635-1652) --------------------
// K key-frames along a straight-ish drive through the seeded world: every key-frame's less-sharp corners and
// less-flat surfs + outliers, moved to the map frame with its (slightly noisy) key pose, YZX axis order like the
// clouds the estimator publishes (StateEstimator.hpp:1125-1150), voxel down-sampled with the mapping node's leaves
// (0.2 m corners, 0.4 m surfs) -> laserCloudCornerFromMapDS / laserCloudSurfFromMapDS.  The newest scan's features
// (down-sampled the same way, its own frame) are the queries; `truth` is its pose as transformTobeMapped
// (rx, ry, rz, tx, ty, tz of pointAssociateToMap, :594-608), `guess` = truth + the odometry error to be refined.
struct MapUnit {
  std::vector<lins_point> cornerMap, surfMap, cornerLast, surfLast;
  float truth[6], guess[6];
};

static lins_point yzx(const lins_point& p) { return makePoint(p.y, p.z, p.x, p.intensity); }
static void euler_of(const M3D& Rw, const V3D& pw, float out[6]) {
  // camera-convention rotation: Rc = P Rw P^T with P = (x,y,z) -> (y,z,x);  Rc = Ry(ry) Rx(rx) Rz(rz)
  const int perm[3] = {1, 2, 0};
  double Rc[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rc[i][j] = Rw(perm[i], perm[j]);
  out[0] = (float)std::asin(-Rc[1][2]);
  out[1] = (float)std::atan2(Rc[0][2], Rc[2][2]);
  out[2] = (float)std::atan2(Rc[1][0], Rc[1][1]);
  out[3] = (float)pw.y(); out[4] = (float)pw.z(); out[5] = (float)pw.x();
}

void* lins_synth_map_unit_create(const lins_synth_cfg* cfg, uint64_t seed, int n_keyframes, double sigma_t, double sigma_r) {
  MapUnit* u = new MapUnit();
  Rng rng(seed);
  LidarModel lm = cfg->lidar == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  World w = make_world(rng, cfg->world);
  Pose T;
  double yaw = rng.uni(-M_PI, M_PI);
  T.p = V3D(rng.uni(-3, 3), rng.uni(-3, 3), rng.uni(1.3, 1.7));
  ImageProjection ip(lm);
  FeatureExtractor fe(lm);
  Cloud cornerAcc, surfAcc;
  Twist still{V3D(0, 0, 0), V3D(0, 0, 0)};
  for (int k = 0; k <= n_keyframes; ++k) {
    T.R = math_utils::rpy2Quat(V3D(rng.uni(-0.02, 0.02), rng.uni(-0.02, 0.02), yaw)).toRotationMatrix();
    Cloud raw;
    simulate_scan(w, lm, T, still, cfg->range_noise, rng, raw);
    ip.process(raw);
    ScanFeatures f;
    fe.run(ip.segmentedCloud, ip.segMsg, f);
    if (k < n_keyframes) {  // a key-frame of the map: its pose is known up to the back-end's residual error
      Pose Tk = T;
      Tk.p = Tk.p + V3D(5e-3 * rng.gauss(), 5e-3 * rng.gauss(), 5e-3 * rng.gauss());
      Tk.R = Tk.R * math_utils::axis2Quat(V3D(3e-4 * rng.gauss(), 3e-4 * rng.gauss(), 3e-4 * rng.gauss())).toRotationMatrix();
      auto to_map = [&](const Cloud& c, Cloud& acc) {
        for (const auto& p : c.points) {
          V3D q = Tk.R * V3D(p.x, p.y, p.z) + Tk.p;
          acc.push_back(makePoint((float)q.y(), (float)q.z(), (float)q.x(), p.intensity));
        }
      };
      to_map(f.cornerPointsLessSharp, cornerAcc);
      to_map(f.surfPointsLessFlat, surfAcc);
      to_map(ip.outlierCloud, surfAcc);
      // drive on: 0.8 .. 1.6 m forward, gentle heading change
      yaw += rng.uni(-0.5, 0.5) * cfg->w_max;
      const double step = rng.uni(0.8, 1.6);
      T.p = T.p + V3D(step * std::cos(yaw), step * std::sin(yaw), 0.0);
    } else {  // the newest scan: the queries
      Cloud c, s, cds, sds;
      for (const auto& p : f.cornerPointsLessSharp.points) c.push_back(yzx(p));
      for (const auto& p : f.surfPointsLessFlat.points) s.push_back(yzx(p));
      for (const auto& p : ip.outlierCloud.points) s.push_back(yzx(p));
      VoxelGrid vc, vs;
      vc.setLeafSize(0.2f, 0.2f, 0.2f); vs.setLeafSize(0.4f, 0.4f, 0.4f);
      vc.filter(c, cds); vs.filter(s, sds);
      u->cornerLast = cds.points; u->surfLast = sds.points;
      euler_of(T.R, T.p, u->truth);
      for (int i = 0; i < 3; ++i) u->guess[i] = u->truth[i] + (float)(sigma_r * rng.gauss());
      for (int i = 3; i < 6; ++i) u->guess[i] = u->truth[i] + (float)(sigma_t * rng.gauss());
    }
  }
  Cloud cds, sds;
  VoxelGrid vc, vs;
  vc.setLeafSize(0.2f, 0.2f, 0.2f); vs.setLeafSize(0.4f, 0.4f, 0.4f);
  vc.filter(cornerAcc, cds); vs.filter(surfAcc, sds);
  u->cornerMap = cds.points; u->surfMap = sds.points;
  return u;
}
void lins_synth_map_unit_destroy(void* h) { delete static_cast<MapUnit*>(h); }
// which: 0 corner map, 1 surf map, 2 corner last, 3 surf last
int lins_synth_map_unit_cloud(void* h, int which, const lins_point** pts) {
  MapUnit* u = static_cast<MapUnit*>(h);
  const std::vector<lins_point>* v = which == 0 ? &u->cornerMap : which == 1 ? &u->surfMap : which == 2 ? &u->cornerLast : &u->surfLast;
  *pts = v->data();
  return (int)v->size();
}
void lins_synth_map_unit_transforms(void* h, float* truth, float* guess) {
  MapUnit* u = static_cast<MapUnit*>(h);
  std::memcpy(truth, u->truth, sizeof(u->truth));
  std::memcpy(guess, u->guess, sizeof(u->guess));
}

// ---- the mapping node's input along a drive: what the estimator publishes per scan ------------------------------------
// One VLP-16 / 64-ring sweep at each given sensor pose (world x, y, z, yaw; roll = pitch = 0) of a seeded world, run through
// the product's CPU front end: the less-sharp corners, less-flat surfs and outliers in the YZX frame the estimator
// publishes them in (StateEstimator.hpp:1125-1150), and the pose as the mapping node's transform (rx, ry, rz, tx, ty, tz).
struct MapDrive {
  std::vector<std::vector<lins_point>> clouds[3];
  std::vector<float> truth;
};
void* lins_synth_map_drive_create(const lins_synth_cfg* cfg, uint64_t seed, int n, const double* xyzyaw) {
  MapDrive* d = new MapDrive();
  Rng rng(seed);
  LidarModel lm = cfg->lidar == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  World w = make_world(rng, cfg->world);
  ImageProjection ip(lm);
  FeatureExtractor fe(lm);
  Twist still{V3D(0, 0, 0), V3D(0, 0, 0)};
  d->truth.resize(6 * (size_t)n);
  for (int k = 0; k < n; ++k) {
    Pose T;
    T.p = V3D(xyzyaw[4 * k], xyzyaw[4 * k + 1], xyzyaw[4 * k + 2]);
    T.R = math_utils::rpy2Quat(V3D(0, 0, xyzyaw[4 * k + 3])).toRotationMatrix();
    Cloud raw;
    simulate_scan(w, lm, T, still, cfg->range_noise, rng, raw);
    ip.process(raw);
    ScanFeatures f;
    fe.run(ip.segmentedCloud, ip.segMsg, f);
    const Cloud* src[3] = {&f.cornerPointsLessSharp, &f.surfPointsLessFlat, &ip.outlierCloud};
    for (int c = 0; c < 3; ++c) {
      std::vector<lins_point> v;
      for (const auto& p : src[c]->points) v.push_back(yzx(p));
      d->clouds[c].push_back(std::move(v));
    }
    euler_of(T.R, T.p, &d->truth[6 * (size_t)k]);
  }
  return d;
}
void lins_synth_map_drive_destroy(void* h) { delete static_cast<MapDrive*>(h); }
// which: 0 less-sharp corners, 1 less-flat surfs, 2 outliers
int lins_synth_map_drive_cloud(void* h, int scan, int which, const lins_point** pts) {
  const std::vector<lins_point>& v = static_cast<MapDrive*>(h)->clouds[which][scan];
  *pts = v.data();
  return (int)v.size();
}
void lins_synth_map_drive_truth(void* h, float* out) {
  const MapDrive* d = static_cast<MapDrive*>(h);
  std::memcpy(out, d->truth.data(), sizeof(float) * d->truth.size());
}

// The product's CPU front end alone (csrc/host/image_projection.hpp + feature_extraction.hpp) on one raw sweep, for the
// tests that check these restatements against an independent Python one (tests/pyfront.py).  Every output array has room
// for `cap` entries (>= line_num * scan_num); counts: n[0] segmented, n[1] outlier, n[2] sharp, n[3] less sharp, n[4] flat,
// n[5] less flat.
int lins_frontend_run(const lins_point* raw, int n_raw, int lidar_model, int cap, lins_point* seg, lins_point* outlier, int32_t* start_ring,
                      int32_t* end_ring, float* ori3, uint8_t* ground, uint32_t* col, float* range, lins_point* undist, lins_point* sharp,
                      lins_point* less_sharp, lins_point* flat, lins_point* less_flat, int32_t* n) {
  const LidarModel lm = lidar_model == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  Cloud in;
  in.points.assign(raw, raw + n_raw);
  ImageProjection ip(lm);
  ip.process(in);
  FeatureExtractor fe(lm);
  ScanFeatures f;
  fe.run(ip.segmentedCloud, ip.segMsg, f);
  auto put = [&](const Cloud& c, lins_point* dst, int32_t& cnt) {
    cnt = (int32_t)c.size();
    std::memcpy(dst, c.points.data(), sizeof(lins_point) * std::min<size_t>(c.size(), (size_t)cap));
  };
  put(ip.segmentedCloud, seg, n[0]); put(ip.outlierCloud, outlier, n[1]);
  put(f.cornerPointsSharp, sharp, n[2]); put(f.cornerPointsLessSharp, less_sharp, n[3]);
  put(f.surfPointsFlat, flat, n[4]); put(f.surfPointsLessFlat, less_flat, n[5]);
  int32_t nu = 0;
  put(f.undistPointCloud, undist, nu);
  for (int i = 0; i < lm.line_num; ++i) { start_ring[i] = ip.segMsg.startRingIndex[i]; end_ring[i] = ip.segMsg.endRingIndex[i]; }
  ori3[0] = ip.segMsg.startOrientation; ori3[1] = ip.segMsg.endOrientation; ori3[2] = ip.segMsg.orientationDiff;
  for (int i = 0; i < std::min(n[0], cap); ++i) { ground[i] = ip.segMsg.segmentedCloudGroundFlag[i]; col[i] = ip.segMsg.segmentedCloudColInd[i]; range[i] = ip.segMsg.segmentedCloudRange[i]; }
  return 0;
}

// FeatureExtractor::run (csrc/host/feature_extraction.hpp) on a given segmented cloud and cloud_info: the host side of
// lins_gpu_extract_features for hand-built scans.  counts: surfPointsFlat, cornerPointsSharp, surfPointsLessFlat,
// cornerPointsLessSharp (lins_gpu_extract_features' order); every output holds up to n points.
int lins_features_host(const lins_point* seg, int n, int line_num, const int32_t* start_ring, const int32_t* end_ring,
                       const float* ori3, const uint8_t* ground, const uint32_t* col, const float* range, const double* prm4,
                       lins_point* undist, lins_point* surf_flat, lins_point* corner_sharp, lins_point* surf_less_flat,
                       lins_point* corner_less_sharp, int32_t* counts) {
  LidarModel lm;
  lm.line_num = line_num;
  lm.scan_period = prm4[3];
  FeatureParams fp;
  fp.edge_threshold = prm4[0]; fp.surf_threshold = prm4[1]; fp.imu_lidar_extrinsic_angle = prm4[2];
  Cloud in;
  in.points.assign(seg, seg + n);
  CloudInfo info;
  info.resize(line_num, n);
  for (int i = 0; i < line_num; ++i) { info.startRingIndex[i] = start_ring[i]; info.endRingIndex[i] = end_ring[i]; }
  info.startOrientation = ori3[0]; info.endOrientation = ori3[1]; info.orientationDiff = ori3[2];
  for (int i = 0; i < n; ++i) { info.segmentedCloudGroundFlag[i] = ground[i]; info.segmentedCloudColInd[i] = col[i]; info.segmentedCloudRange[i] = range[i]; }
  FeatureExtractor fe(lm, fp);
  ScanFeatures f;
  fe.run(in, info, f);
  const Cloud* outs[4] = {&f.surfPointsFlat, &f.cornerPointsSharp, &f.surfPointsLessFlat, &f.cornerPointsLessSharp};
  lins_point* dst[4] = {surf_flat, corner_sharp, surf_less_flat, corner_less_sharp};
  for (int k = 0; k < 4; ++k) {
    counts[k] = (int32_t)outs[k]->size();
    std::memcpy(dst[k], outs[k]->points.data(), sizeof(lins_point) * std::min<size_t>(outs[k]->size(), (size_t)n));
  }
  std::memcpy(undist, f.undistPointCloud.points.data(), sizeof(lins_point) * (size_t)n);
  return 0;
}

// Wall seconds of `reps` passes of FeatureExtractor::run (shipped parameters, SCAN_PERIOD 0.1) over every scan of d, the
// scans handed out to `threads` std::threads one at a time: the host throughput lins_gpu_extract_features replaces.
// Inputs are converted to Cloud / CloudInfo before the clock starts.
double lins_features_host_bench(const lins_pcl_desc* d, int threads, int reps) {
  const int n = d->n_scans, L = d->line_num;
  std::vector<Cloud> clouds(n);
  std::vector<CloudInfo> infos(n);
  for (int k = 0; k < n; ++k) {
    const int a = d->cloud_off[k], b = d->cloud_off[k + 1];
    clouds[k].points.assign(d->cloud + a, d->cloud + b);
    CloudInfo& info = infos[k];
    info.resize(L, b - a);
    for (int i = 0; i < L; ++i) { info.startRingIndex[i] = d->start_ring_index[(size_t)k * L + i]; info.endRingIndex[i] = d->end_ring_index[(size_t)k * L + i]; }
    info.startOrientation = d->orientation[3 * k]; info.endOrientation = d->orientation[3 * k + 1]; info.orientationDiff = d->orientation[3 * k + 2];
    for (int i = a; i < b; ++i) { info.segmentedCloudGroundFlag[i - a] = d->ground_flag[i]; info.segmentedCloudColInd[i - a] = d->col_ind[i]; info.segmentedCloudRange[i - a] = d->range[i]; }
  }
  LidarModel lm;
  lm.line_num = L;
  std::atomic<long> next(0);
  const long total = (long)n * std::max(reps, 1);
  auto work = [&]() {
    FeatureExtractor fe(lm, FeatureParams());
    ScanFeatures f;
    for (long i; (i = next.fetch_add(1)) < total;) fe.run(clouds[i % n], infos[i % n], f);
  };
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> pool;
  for (int t = 0; t < std::max(threads, 1); ++t) pool.emplace_back(work);
  for (auto& t : pool) t.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

static LidarModel model_of(const lins_lidar_model* m) {
  LidarModel lm;
  lm.line_num = m->line_num; lm.scan_num = m->scan_num; lm.ang_res_x = m->ang_res_x; lm.ang_res_y = m->ang_res_y;
  lm.ang_bottom = m->ang_bottom; lm.ground_scan_ind = m->ground_scan_ind;
  return lm;
}

// ImageProjection::process (csrc/host/image_projection.hpp) of one raw sweep on a fresh object with the given model: the
// host side of lins_gpu_project_scans.  seg / ground / col / range / outlier hold up to max(n, 1) entries; counts:
// segmented, outlier.
int lins_projection_host(const lins_point* raw, int n, const lins_lidar_model* m, lins_point* seg, uint8_t* ground, uint32_t* col,
                         float* range, lins_point* outlier, int32_t* start_ring, int32_t* end_ring, float* ori3, int32_t* counts) {
  const LidarModel lm = model_of(m);
  Cloud in;
  in.points.assign(raw, raw + n);
  ImageProjection ip(lm);
  ip.process(in);
  const size_t ns = ip.segmentedCloud.size(), no = ip.outlierCloud.size();
  counts[0] = (int32_t)ns; counts[1] = (int32_t)no;
  std::memcpy(seg, ip.segmentedCloud.points.data(), sizeof(lins_point) * ns);
  std::memcpy(outlier, ip.outlierCloud.points.data(), sizeof(lins_point) * no);
  for (size_t i = 0; i < ns; ++i) { ground[i] = ip.segMsg.segmentedCloudGroundFlag[i]; col[i] = ip.segMsg.segmentedCloudColInd[i]; range[i] = ip.segMsg.segmentedCloudRange[i]; }
  for (int i = 0; i < lm.line_num; ++i) { start_ring[i] = ip.segMsg.startRingIndex[i]; end_ring[i] = ip.segMsg.endRingIndex[i]; }
  ori3[0] = ip.segMsg.startOrientation; ori3[1] = ip.segMsg.endOrientation; ori3[2] = ip.segMsg.orientationDiff;
  return 0;
}

// Wall seconds of `reps` passes of ImageProjection::process over every sweep of d with model m, the sweeps handed out to
// `threads` std::threads one at a time (one ImageProjection per thread, as a node keeps one): the host throughput
// lins_gpu_project_scans replaces.  Inputs are converted to Clouds before the clock starts.
double lins_projection_host_bench(const lins_raw_desc* d, const lins_lidar_model* m, int threads, int reps) {
  const int n = d->n_scans;
  std::vector<Cloud> clouds(n);
  for (int k = 0; k < n; ++k) {
    clouds[k].points.assign(d->cloud + d->cloud_off[k], d->cloud + d->cloud_off[k + 1]);
  }
  const LidarModel lm = model_of(m);
  std::atomic<long> next(0);
  const long total = (long)n * std::max(reps, 1);
  auto work = [&]() {
    ImageProjection ip(lm);
    for (long i; (i = next.fetch_add(1)) < total;) ip.process(clouds[i % n]);
  };
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> pool;
  for (int t = 0; t < std::max(threads, 1); ++t) pool.emplace_back(work);
  for (auto& t : pool) t.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// one simulated raw sweep of the seeded world (an input for lins_frontend_run): returns the number of points written
int lins_synth_raw_sweep(const lins_synth_cfg* cfg, uint64_t seed, lins_point* out, int cap) {
  Rng rng(seed);
  const LidarModel lm = cfg->lidar == 1 ? LidarModel::dense64() : LidarModel::vlp16();
  World w = make_world(rng, cfg->world);
  Pose T0;
  T0.R = math_utils::rpy2Quat(V3D(rng.uni(-0.02, 0.02), rng.uni(-0.02, 0.02), rng.uni(-M_PI, M_PI))).toRotationMatrix();
  T0.p = V3D(rng.uni(-8, 8), rng.uni(-8, 8), rng.uni(1.2, 1.8));
  const double T = lm.scan_period;
  const double sp = rng.uni(0, cfg->v_max);
  Twist tw{T * V3D(0, 0, rng.uni(-cfg->w_max, cfg->w_max)), T * V3D(sp, 0.1 * sp, 0.0)};
  Cloud raw;
  simulate_scan(w, lm, T0, tw, cfg->range_noise, rng, raw);
  const int n = (int)std::min<size_t>(raw.size(), (size_t)std::max(cap, 0));
  std::memcpy(out, raw.points.data(), sizeof(lins_point) * (size_t)n);
  return n;
}

}  // extern "C"
