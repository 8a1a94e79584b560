"""Sequence initialisation on the CPU: the first / second scan algebra of csrc/cuda/lins_seq_step.cuh (pre-integration,
processFirstScan, processSecondScan, initializeCovariance) against the host shim and filter it replaces, bit for bit; the
ctypes mirror of lins_seq_init_params and the new status codes."""
import ctypes as C
import os
import subprocess

from conftest import ROOT

HOST = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
CUDA = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")

# StateEstimator is compiled with the C-ABI stubbed out: estimateTransform leaves its start pose as it is, so the second
# scan's state depends on the pre-integration and the ICP's start pose only
DRIVER = r'''
#include <cstdio>
#include <cstring>
#include <random>
#include "state_estimator.hpp"
#include "lins_seq_step.cuh"
extern "C" {
int lins_gpu_create(const lins_params*, int, void*, lins_ctx** o) { *o = nullptr; return 0; }
void lins_gpu_destroy(lins_ctx*) {}
const char* lins_gpu_last_error(const lins_ctx*) { return ""; }
int lins_gpu_set_map(lins_ctx*, const lins_point*, int, const lins_point*, int) { return 0; }
int lins_gpu_ieskf(lins_ctx*, const lins_point*, int, const lins_point*, int, const double*, const double*, double*, double*, lins_report*) { return 0; }
int lins_gpu_estimate_transform(lins_ctx*, const lins_point*, int, const lins_point*, int, double*, int*, int*) { return 0; }
int lins_gpu_update_map(lins_ctx*, lins_point*, int, lins_point*, int, const double*, int*) { return 0; }
}
using namespace lins;
static std::mt19937_64 rng(11);
static double U(double a, double b) { return std::uniform_real_distribution<double>(a, b)(rng); }
static bool same(const double* a, const double* b, int n) { return std::memcmp(a, b, sizeof(double) * n) == 0; }
static V3D RV(double a, double b) { return V3D(U(a, b), U(a, b), U(a, b)); }
static void put3(double* d, const V3D& v) { d[0] = v(0); d[1] = v(1); d[2] = v(2); }
// lins_seq.cu set_init_consts
static lins_seq::InitConsts init_consts(const filter::FilterParams& f) {
  lins_seq::InitConsts k;
  for (int i = 0; i < 3; ++i) {
    k.var[lins_seq::kPos + i] = f.init_pos_std(i) * f.init_pos_std(i);
    k.var[lins_seq::kVel + i] = f.init_vel_std(i) * f.init_vel_std(i);
    k.var[lins_seq::kAtt + i] = std::pow(f.init_att_std(i) * M_PI / 180.0, 2);
    k.var[lins_seq::kAcc + i] = f.init_acc_std(i) * f.init_acc_std(i);
    k.var[lins_seq::kGyr + i] = f.init_gyr_std(i) * f.init_gyr_std(i);
    k.var[lins_seq::kGra + i] = 0.01;
    k.ba[i] = f.init_ba(i); k.bw[i] = f.init_bw(i);
  }
  return k;
}
static ScanFeatures features(int corners, int surfs) {
  ScanFeatures f;
  for (int i = 0; i < corners; ++i) f.cornerPointsLessSharp.push_back(makePoint(1.f + i, 2.f, 3.f, 0.f));
  for (int i = 0; i < surfs; ++i) f.surfPointsLessFlat.push_back(makePoint(4.f, 5.f + i, 6.f, 0.f));
  return f;
}
int main() {
  int n_pre = 0, n_zero = 0, bad_pre = 0, bad_fresh = 0, bad_first = 0, bad_start = 0, bad_second = 0, n_second = 0;
  // pre-integration on its own: IntegrationBase over random samples, dt = 0 among them
  for (int trial = 0; trial < 300; ++trial) {
    const V3D a0(U(-1, 1), U(-1, 1), 9.81 + U(-1, 1)), g0 = RV(-.5, .5), ba = RV(-.2, .2), bg = RV(-.01, .01);
    integration::IntegrationBase ib(a0, g0, ba, bg);
    lins_seq::InitConsts k{};
    put3(k.ba, ba); put3(k.bw, bg);
    double imu[6], pre[20];
    put3(imu, a0); put3(imu + 3, g0);
    lins_seq::preint_begin(pre, imu);
    const int n = trial % 50;
    for (int m = 0; m < n; ++m) {
      double dt = m % 9 == 4 ? 0.0 : U(0, 0.005);
      n_zero += dt == 0.0;
      const double acc[3] = {U(-3, 3), U(-3, 3), 9.81 + U(-3, 3)}, gyr[3] = {U(-1, 1), U(-1, 1), U(-1, 1)};
      ib.push_back(dt, V3D(acc[0], acc[1], acc[2]), V3D(gyr[0], gyr[1], gyr[2]));
      lins_seq::preint_propagate(pre, k, dt, acc, gyr);
      ++n_pre;
      double h[20];
      put3(h + lins_seq::pAcc, ib.acc_0); put3(h + lins_seq::pGyr, ib.gyr_0); put3(h + lins_seq::pDp, ib.delta_p); put3(h + lins_seq::pDv, ib.delta_v);
      for (int i = 0; i < 4; ++i) h[lins_seq::pDq + i] = ib.delta_q.c[i];
      h[lins_seq::pSum] = ib.sum_dt;
      if (!same(h, pre, 17)) ++bad_pre;
    }
  }
  // first / second scan through the shim's status machine, with the shipped and with random non-zero init constants
  for (int trial = 0; trial < 200; ++trial) {
    fusion::EstimatorParams ep;
    if (trial % 2) {
      ep.filter.init_pos_std = RV(0, .5); ep.filter.init_vel_std = RV(0, .5); ep.filter.init_att_std = RV(0, 3);
      ep.filter.init_acc_std = RV(0, .1); ep.filter.init_gyr_std = RV(0, .01);
      ep.filter.init_ba = RV(-.2, .2); ep.filter.init_bw = RV(-.01, .01);
    }
    const lins_seq::InitConsts k = init_consts(ep.filter);
    fusion::StateEstimator est(ep);
    double glob[20], filt[20], P[324], lin[20], pre[20], il[8], pose[20];
    lins_seq::fresh_slot(glob, filt, P, k);
    double h[19];
    est.globalState_.toArray(h);
    bool ok = same(h, glob, 19);
    est.filter_->state_.toArray(h);
    ok = ok && same(h, filt, 19) && same(est.filter_->covariance_.data(), P, 324);
    if (!ok) ++bad_fresh;
    // scan 0: the first scan
    double imu[6] = {U(-1, 1), U(-1, 1), 9.81 + U(-1, 1), U(-.2, .2), U(-.2, .2), U(-.2, .2)};
    est.processFeatures(0.1, sensor_utils::Imu(0.1, V3D(imu[0], imu[1], imu[2]), V3D(imu[3], imu[4], imu[5])), features(10, 100));
    lins_seq::first_scan(filt, P, lin, pre, il, imu, k);
    est.filter_->state_.toArray(h);
    ok = est.status_ == fusion::StateEstimator::STATUS_FIRST_SCAN && same(h, filt, 19) && same(est.filter_->covariance_.data(), P, 324);
    est.linState_.toArray(h);
    ok = ok && same(h, lin, 19);
    double hl[6];
    put3(hl, est.filter_->acc_last); put3(hl + 3, est.filter_->gyr_last);
    ok = ok && same(hl, il, 6);
    if (!ok) ++bad_first;
    // the IMU rows between the two scans (none in some trials: p / sum_dt is then not finite, as in the reference)
    const int n = trial % 13 == 0 ? 0 : 1 + trial % 45;
    for (int m = 0; m < n; ++m) {
      const double dt = m % 11 == 7 ? 0.0 : U(0, 0.005);
      const double acc[3] = {U(-3, 3), U(-3, 3), 9.81 + U(-3, 3)}, gyr[3] = {U(-1, 1), U(-1, 1), U(-1, 1)};
      est.processImu(dt, V3D(acc[0], acc[1], acc[2]), V3D(gyr[0], gyr[1], gyr[2]));
      lins_seq::preint_propagate(pre, k, dt, acc, gyr);
    }
    // scan 1: the second scan (the stubbed estimateTransform returns its start pose)
    for (double& v : imu) v = U(-1, 1);
    imu[2] += 9.81;
    est.processFeatures(0.2, sensor_utils::Imu(0.2, V3D(imu[0], imu[1], imu[2]), V3D(imu[3], imu[4], imu[5])), features(10 + trial % 3, 100 + trial % 5));
    lins_seq::second_scan_start(pre, pose);
    double hp[20] = {0};
    put3(hp, est.linState_.rn_);
    for (int i = 0; i < 4; ++i) hp[6 + i] = est.linState_.qbn_.c[i];
    if (!same(hp, pose, 20)) ++bad_start;
    lins_seq::second_scan(glob, filt, P, lin, il, pre, pose, imu, k);
    ok = est.status_ == fusion::StateEstimator::STATUS_RUNNING;
    est.globalState_.toArray(h); ok = ok && same(h, glob, 19);
    est.filter_->state_.toArray(h); ok = ok && same(h, filt, 19);
    est.linState_.toArray(h); ok = ok && same(h, lin, 19);
    ok = ok && same(est.filter_->covariance_.data(), P, 324);
    put3(hl, est.filter_->acc_last); put3(hl + 3, est.filter_->gyr_last);
    ok = ok && same(hl, il, 6);
    if (!ok) ++bad_second;
    ++n_second;
  }
  std::printf("%d %d %d %d %d %d %d %d\n", n_pre, n_zero, n_second, bad_pre, bad_fresh, bad_first, bad_start, bad_second);
  return 0;
}
'''


def test_init_algebra_matches_the_shim_bit_for_bit(tmp_path):
    src = tmp_path / "t.cpp"
    src.write_text(DRIVER)
    exe = str(tmp_path / "t")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", HOST, "-I", CUDA, "-o", exe, str(src)])
    n_pre, n_zero, n_second, *bad = map(int, subprocess.check_output([exe]).split())
    assert n_pre > 5000 and n_zero > 300 and n_second == 200
    assert bad == [0, 0, 0, 0, 0], dict(zip(("pre", "fresh", "first", "start", "second"), bad))


def test_init_struct_mirror_and_codes_match_header(defs, tmp_path):
    cls = defs.LinsSeqInitParams
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "lins_gpu.h"', "int main(){",
             'printf("%zu\\n", sizeof(lins_seq_init_params));']
    lines += [f'printf("%zu\\n", offsetof(lins_seq_init_params, {f}));' for f, _ in cls._fields_]
    lines.append('printf("%d %d %d\\n", LINS_SEQ_INIT_WAIT, LINS_SEQ_FIRST, LINS_SEQ_SECOND); return 0;}')
    (tmp_path / "s.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "s"), str(tmp_path / "s.c")])
    out = [int(x) for x in subprocess.check_output([str(tmp_path / "s")]).split()]
    assert out[:-3] == [C.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    assert out[-3:] == [defs.SEQ_INIT_WAIT, defs.SEQ_FIRST, defs.SEQ_SECOND]


def test_shipped_init_params_are_the_host_filters(defs, tmp_path):
    """LinsSeqInitParams.shipped() holds kalman_filter.hpp's FilterParams defaults bit for bit."""
    (tmp_path / "n.cpp").write_text('''
#include <cstdio>
#include "kalman_filter.hpp"
int main() {
  lins::filter::FilterParams f;
  for (const lins::V3D* v : {&f.init_vel_std, &f.init_acc_std, &f.init_gyr_std, &f.init_ba, &f.init_bw})
    for (int i = 0; i < 3; ++i) std::printf("%a\\n", (*v)(i));
  return 0;
}
''')
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", HOST, "-o", str(tmp_path / "n"), str(tmp_path / "n.cpp")])
    host = [float.fromhex(x) for x in subprocess.check_output([str(tmp_path / "n")]).decode().split()]
    p = defs.LinsSeqInitParams.shipped()
    assert [v for f, _ in p._fields_ for v in getattr(p, f)] == host
