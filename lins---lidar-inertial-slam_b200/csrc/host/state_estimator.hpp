// fusion::StateEstimator — host-side mirror of the reference class (lins/include/StateEstimator.hpp:174-1507)
// whose hot seams call the B200 C-ABI (include/lins_gpu.h):
//
//   kdtreeSurf_/kdtreeCorner_->setInputCloud   (:363-364)        -> lins_gpu_set_map
//   performIESKF()                              (:465-600)        -> lins_gpu_ieskf  (all iterations on device)
//   estimateTransform()                         (:1163-1196)      -> lins_gpu_estimate_transform
//   updatePointCloud() XYZ part + index refresh (:1116-1161)      -> lins_gpu_update_map
//
// Everything else stays on the CPU exactly where the reference has it: IMU propagation (StatePredictor), the
// four-stage feature extraction, the status machine, integrateTransformation, the roll/pitch correction and
// the YZX republishing.  Same member names / signatures as the reference so LinsFusion (Estimator.cpp) can use
// it unchanged once PCL / Eigen types are swapped for the layout-compatible ones below (see INTEGRATION.md).
// PRODUCT code: never includes anything from oracle/.
#ifndef LINS_HOST_STATE_ESTIMATOR_HPP_
#define LINS_HOST_STATE_ESTIMATOR_HPP_

#include <cstdio>
#include <memory>
#include <stdexcept>
#include <string>

#include "../../../include/lins_gpu.h"
#include "cloud.hpp"
#include "feature_extraction.hpp"
#include "global_state_yzx.hpp"
#include "kalman_filter.hpp"

namespace lins {

namespace sensor_utils {
struct Imu {  // sensor_utils.hpp:44-54
  Imu() : time(0) {}
  Imu(double t, const V3D& a, const V3D& g) : time(t), acc(a), gyr(g) {}
  double time;
  V3D acc, gyr;
};
}  // namespace sensor_utils

namespace integration {
// Mid-point IMU pre-integration between scan 1 and scan 2 (integrationBase.h:61-85, :141-176); only
// delta_p / delta_q / delta_v / sum_dt are consumed (StateEstimator.hpp:392-396).
class IntegrationBase {
 public:
  IntegrationBase(const V3D& acc0, const V3D& gyr0, const V3D& ba, const V3D& bg)
      : acc_0(acc0), gyr_0(gyr0), linearized_ba(ba), linearized_bg(bg), sum_dt(0.0) {}
  void push_back(double dt, const V3D& acc, const V3D& gyr) { propagate(dt, acc, gyr); }
  void propagate(double dt, const V3D& acc_1, const V3D& gyr_1) {
    V3D un_acc_0 = delta_q * (acc_0 - linearized_ba);
    V3D un_gyr = 0.5 * (gyr_0 + gyr_1) - linearized_bg;
    Q4D rq = delta_q * Q4D(1, un_gyr(0) * dt / 2, un_gyr(1) * dt / 2, un_gyr(2) * dt / 2);
    V3D un_acc_1 = rq * (acc_1 - linearized_ba);
    V3D un_acc = 0.5 * (un_acc_0 + un_acc_1);
    delta_p = delta_p + dt * delta_v + 0.5 * dt * dt * un_acc;
    delta_v = delta_v + dt * un_acc;
    delta_q = rq.normalized();
    sum_dt += dt;
    acc_0 = acc_1; gyr_0 = gyr_1;
  }
  V3D acc_0, gyr_0, linearized_ba, linearized_bg;
  double sum_dt;
  V3D delta_p, delta_v;
  Q4D delta_q;
};
}  // namespace integration

namespace fusion {

using filter::GlobalState;
using filter::StatePredictor;

// the 7 hot-path globals + the feature thresholds (parameters.h:104-153), exp_port.yaml values as defaults
struct EstimatorParams {
  lins_params gpu{30, 1, 25.0, 0.01, 1.0, 0.1, 0, 0};
  FeatureParams feature;
  filter::FilterParams filter;
  LidarModel lidar;
};

// StateEstimator.hpp:74-169
class Scan {
 public:
  Scan() : id_(scan_counter()++), time_(0) {}
  void setPointCloud(double time, const Cloud& dist, const CloudInfo& info, const Cloud& outlier) {
    distPointCloud_ = dist; cloudInfo_ = info; outlierPointCloud_ = outlier; time_ = time;
  }
  static int& scan_counter() { static int c = 0; return c; }
  int id_;
  double time_;
  Cloud distPointCloud_, undistPointCloud_, outlierPointCloud_;
  CloudInfo cloudInfo_;
  Cloud cornerPointsSharp_, cornerPointsLessSharp_, surfPointsFlat_, surfPointsLessFlat_;
  Cloud cornerPointsLessSharpYZX_, surfPointsLessFlatYZX_, outlierPointCloudYZX_;
};
typedef std::shared_ptr<Scan> ScanPtr;

class StateEstimator {
 public:
  enum FusionStatus { STATUS_INIT = 0, STATUS_FIRST_SCAN = 1, STATUS_SECOND_SCAN = 2, STATUS_RUNNING = 3, STATUS_RESET = 4 };

  explicit StateEstimator(const EstimatorParams& p = EstimatorParams(), int device = 0)
      : prm_(p), extractor_(p.lidar, p.feature), preintegration_(nullptr), ctx_(nullptr) {
    filter_ = new StatePredictor(p.filter);
    scan_new_.reset(new Scan());
    scan_last_.reset(new Scan());
    globalState_.setIdentity();
    globalStateYZX_.setIdentity();
    // rotations between the XYZ and YZX conventions (StateEstimator.hpp:217-220)
    M3D R_yzx_to_xyz;
    R_yzx_to_xyz(0, 2) = 1.; R_yzx_to_xyz(1, 0) = 1.; R_yzx_to_xyz(2, 1) = 1.;
    Q_yzx_to_xyz = math_utils::R2Quat(R_yzx_to_xyz);
    Q_xyz_to_yzx = math_utils::R2Quat(R_yzx_to_xyz.transpose());
    status_ = STATUS_INIT;
    int rc = lins_gpu_create(&prm_.gpu, device, nullptr, &ctx_);
    if (rc != LINS_OK) throw std::runtime_error("lins_gpu_create failed (" + std::to_string(rc) + "): no CPU fallback exists");
  }
  ~StateEstimator() {
    delete filter_;
    delete preintegration_;
    if (ctx_) lins_gpu_destroy(ctx_);
  }
  StateEstimator(const StateEstimator&) = delete;
  StateEstimator& operator=(const StateEstimator&) = delete;

  inline double getTime() const { return filter_->time_; }
  inline bool isInitialized() const { return status_ != STATUS_INIT; }

  // StateEstimator.hpp:242-270 (the "for no use here" dead-reckoning block is omitted)
  void processImu(double dt, const V3D& acc, const V3D& gyr) {
    switch (status_) {
      case STATUS_FIRST_SCAN:
        preintegration_->push_back(dt, acc, gyr);
        filter_->time_ += dt;
        break;
      case STATUS_RUNNING:
        filter_->predict(dt, acc, gyr, true);
        break;
      default: break;
    }
  }

  // StateEstimator.hpp:279-328
  void processPCL(double time, const sensor_utils::Imu& imu, const Cloud& distortedPointCloud, const CloudInfo& cloudInfo,
                  const Cloud& outlierPointCloud) {
    scan_new_->setPointCloud(time, distortedPointCloud, cloudInfo, outlierPointCloud);
    ScanFeatures f;
    extractor_.run(scan_new_->distPointCloud_, scan_new_->cloudInfo_, f);  // undistortPcl .. extractFeatures (CPU)
    scan_new_->undistPointCloud_ = f.undistPointCloud;
    scan_new_->cornerPointsSharp_ = f.cornerPointsSharp; scan_new_->cornerPointsLessSharp_ = f.cornerPointsLessSharp;
    scan_new_->surfPointsFlat_ = f.surfPointsFlat; scan_new_->surfPointsLessFlat_ = f.surfPointsLessFlat;
    imu_last_ = imu;
    switch (status_) {
      case STATUS_INIT:
        if (processFirstScan()) status_ = STATUS_FIRST_SCAN;
        break;
      case STATUS_FIRST_SCAN:
        if (processSecondScan()) status_ = STATUS_RUNNING; else status_ = STATUS_INIT;
        break;
      case STATUS_RUNNING:
        if (!processScan()) status_ = STATUS_RUNNING;
        break;
      default: break;
    }
  }

  // processPCL without the extractor: the same status machine on features extracted elsewhere (a replayed feature log)
  void processFeatures(double time, const sensor_utils::Imu& imu, const ScanFeatures& f) {
    scan_new_->time_ = time;
    scan_new_->undistPointCloud_ = f.undistPointCloud;
    scan_new_->cornerPointsSharp_ = f.cornerPointsSharp; scan_new_->cornerPointsLessSharp_ = f.cornerPointsLessSharp;
    scan_new_->surfPointsFlat_ = f.surfPointsFlat; scan_new_->surfPointsLessFlat_ = f.surfPointsLessFlat;
    imu_last_ = imu;
    switch (status_) {
      case STATUS_INIT:
        if (processFirstScan()) status_ = STATUS_FIRST_SCAN;
        break;
      case STATUS_FIRST_SCAN:
        if (processSecondScan()) status_ = STATUS_RUNNING; else status_ = STATUS_INIT;
        break;
      case STATUS_RUNNING:
        if (!processScan()) status_ = STATUS_RUNNING;
        break;
      default: break;
    }
  }

  // StateEstimator.hpp:331-375
  bool processFirstScan() {
    if (scan_new_->cornerPointsLessSharp_.size() < 10 || scan_new_->surfPointsLessFlat_.size() < 100) {
      scan_new_.reset(new Scan());
      return false;
    }
    linState_.setIdentity();
    delete preintegration_;
    preintegration_ = new integration::IntegrationBase(imu_last_.acc, imu_last_.gyr, prm_.filter.init_ba, prm_.filter.init_bw);
    filter_->initialization(scan_new_->time_, V3D(0, 0, 0), V3D(0, 0, 0), V3D(0, 0, 0), V3D(0, 0, 0), imu_last_.acc, imu_last_.gyr);
    setInputCloud(scan_new_);  // kdtreeCorner_/kdtreeSurf_->setInputCloud
    scan_last_.swap(scan_new_);
    scan_new_.reset(new Scan());
    return true;
  }

  // StateEstimator.hpp:379-425
  bool processSecondScan() {
    if (scan_new_->cornerPointsLessSharp_.size() < 10 || scan_new_->surfPointsLessFlat_.size() < 100) {
      scan_new_.reset(new Scan());
      return false;
    }
    V3D ba0, bw0, v0, v1;
    Q4D ql = preintegration_->delta_q;
    V3D pl = preintegration_->delta_p + 0.5 * preintegration_->sum_dt * preintegration_->sum_dt * linState_.gn_;
    estimateTransform(scan_last_, scan_new_, pl, ql);
    estimateInitialState(pl, ql, v0, v1, ba0, bw0);
    filter_->initialization(scan_new_->time_, pl, v1, ba0, bw0, imu_last_.acc, imu_last_.gyr);
    double roll_init, pitch_init;
    calculateRPfromGravity(imu_last_.acc - ba0, roll_init, pitch_init);
    globalState_ = GlobalState(pl, v1, math_utils::rpy2Quat(V3D(roll_init, pitch_init, 0.0)), ba0, bw0);
    updatePointCloud();
    scan_last_.swap(scan_new_);
    scan_new_.reset(new Scan());
    return true;
  }

  // StateEstimator.hpp:435-463
  bool processScan() {
    if (scan_new_->cornerPointsLessSharp_.size() <= 5 || scan_new_->surfPointsLessFlat_.size() <= 10) return false;
    performIESKF();
    integrateTransformation();
    filter_->reset(1);
    double roll, pitch;
    calculateRPfromGravity(filter_->state_.gn_, roll, pitch);
    correctRollPitch(roll, pitch);
    updatePointCloud();
    scan_last_.swap(scan_new_);
    scan_new_.reset(new Scan());
    return true;
  }

  // StateEstimator.hpp:465-600 — the whole iterated update runs on the device
  void performIESKF() {
    double s_in[LINS_STATE_DIM], s_out[LINS_STATE_DIM];
    filter::Cov18 Pk;
    filter_->state_.toArray(s_in);
    last_report_ = lins_report();
    check(lins_gpu_ieskf(ctx_, pts(scan_new_->surfPointsFlat_), (int)scan_new_->surfPointsFlat_.size(),
                         pts(scan_new_->cornerPointsSharp_), (int)scan_new_->cornerPointsSharp_.size(), s_in,
                         filter_->covariance_.data(), s_out, Pk.data(), &last_report_), "lins_gpu_ieskf");
    if (last_report_.diverged) {
      // "======Using ICP Method======" (:585-592): pose from the 6-DoF ICP, covariance untouched
      GlobalState filterState = filter_->state_;
      V3D t = filterState.rn_;
      Q4D q = filterState.qbn_;
      estimateTransform(scan_last_, scan_new_, t, q);
      filterState.rn_ = t; filterState.qbn_ = q;
      filter_->update(filterState, filter_->covariance_);
    } else {
      linState_ = GlobalState::fromArray(s_out);
      filter_->update(linState_, Pk);
    }
  }

  // StateEstimator.hpp:1163-1196
  void estimateTransform(ScanPtr lastScan, ScanPtr newScan, V3D& t, Q4D& q) {
    (void)lastScan;  // the device map already holds lastScan's clouds
    double pose[7] = {t.x(), t.y(), t.z(), q.x(), q.y(), q.z(), q.w()};
    int iters = 0, conv = 0;
    check(lins_gpu_estimate_transform(ctx_, pts(newScan->surfPointsFlat_), (int)newScan->surfPointsFlat_.size(),
                                      pts(newScan->cornerPointsSharp_), (int)newScan->cornerPointsSharp_.size(), pose, &iters, &conv),
          "lins_gpu_estimate_transform");
    t = V3D(pose[0], pose[1], pose[2]);
    q = Q4D(pose[6], pose[3], pose[4], pose[5]);
    linState_.rn_ = t; linState_.qbn_ = q;
    last_icp_iters_ = iters; last_icp_converged_ = conv;
  }

  // StateEstimator.hpp:602-605
  void calculateRPfromGravity(const V3D& fbib, double& roll, double& pitch) {
    pitch = -math_utils::sign(fbib.z()) * std::asin(fbib.x() / filter::G0);
    roll = math_utils::sign(fbib.z()) * std::asin(fbib.y() / filter::G0);
  }
  // StateEstimator.hpp:608-617
  void integrateTransformation() {
    GlobalState filterState = filter_->state_;
    globalState_.rn_ = globalState_.qbn_ * filterState.rn_ + globalState_.rn_;
    globalState_.qbn_ = globalState_.qbn_ * filterState.qbn_;
    globalState_.vn_ = (globalState_.qbn_ * filterState.qbn_.inverse()) * filterState.vn_;
    globalState_.ba_ = filterState.ba_;
    globalState_.bw_ = filterState.bw_;
    globalState_.gn_ = globalState_.qbn_ * filterState.gn_;
  }
  // StateEstimator.hpp:427-431
  void correctRollPitch(const double& roll, const double& pitch) {
    V3D rpy = math_utils::Q2rpy(globalState_.qbn_);
    globalState_.qbn_ = math_utils::rpy2Quat(V3D(roll, pitch, rpy(2)));
  }
  // StateEstimator.hpp:1408-1419
  void estimateInitialState(const V3D& p, const Q4D&, V3D& v0, V3D& v1, V3D& ba, V3D& bw) {
    V3D v = p / preintegration_->sum_dt;
    v0 = v; v1 = v;
    ba = prm_.filter.init_ba; bw = prm_.filter.init_bw;
  }

  // StateEstimator.hpp:1116-1161: transformToEnd of the less-* clouds (device), YZX copies, index refresh
  void updatePointCloud() {
    double lin[LINS_STATE_DIM];
    linState_.toArray(lin);
    int replaced = 0;
    check(lins_gpu_update_map(ctx_, pts(scan_new_->surfPointsLessFlat_), (int)scan_new_->surfPointsLessFlat_.size(),
                              pts(scan_new_->cornerPointsLessSharp_), (int)scan_new_->cornerPointsLessSharp_.size(), lin, &replaced),
          "lins_gpu_update_map");
    last_map_replaced_ = replaced != 0;
    scan_new_->cornerPointsLessSharpYZX_.clear(); scan_new_->surfPointsLessFlatYZX_.clear(); scan_new_->outlierPointCloudYZX_.clear();
    for (const auto& p : scan_new_->cornerPointsLessSharp_.points) scan_new_->cornerPointsLessSharpYZX_.push_back(makePoint(p.y, p.z, p.x, p.intensity));
    for (const auto& p : scan_new_->surfPointsLessFlat_.points) scan_new_->surfPointsLessFlatYZX_.push_back(makePoint(p.y, p.z, p.x, p.intensity));
    for (const auto& p : scan_new_->outlierPointCloud_.points) scan_new_->outlierPointCloudYZX_.push_back(makePoint(p.y, p.z, p.x, p.intensity));
    global_state_yzx(globalState_.rn_.d.data(), globalState_.qbn_.c.data(), globalStateYZX_.rn_.d.data(), globalStateYZX_.qbn_.c.data());
  }

 public:
  EstimatorParams prm_;
  FusionStatus status_;
  StatePredictor* filter_;
  ScanPtr scan_new_, scan_last_;
  GlobalState globalState_, linState_, globalStateYZX_;
  Q4D Q_yzx_to_xyz, Q_xyz_to_yzx;
  sensor_utils::Imu imu_last_;
  lins_report last_report_;
  bool last_map_replaced_ = false;  // the last updatePointCloud rebuilt the 1-NN index (:1156-1157)
  int last_icp_iters_ = 0, last_icp_converged_ = 0;  // the last estimateTransform's iterations and converged flag

 private:
  FeatureExtractor extractor_;
  integration::IntegrationBase* preintegration_;
  lins_ctx* ctx_;

  static lins_point* pts(Cloud& c) { return c.points.empty() ? nullptr : c.points.data(); }
  void setInputCloud(ScanPtr s) {
    check(lins_gpu_set_map(ctx_, pts(s->surfPointsLessFlat_), (int)s->surfPointsLessFlat_.size(), pts(s->cornerPointsLessSharp_),
                           (int)s->cornerPointsLessSharp_.size()), "lins_gpu_set_map");
  }
  void check(int rc, const char* what) {
    if (rc != LINS_OK) throw std::runtime_error(std::string(what) + " failed: " + lins_gpu_last_error(ctx_));
  }
};

}  // namespace fusion
}  // namespace lins
#endif
