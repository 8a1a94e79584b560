"""Sequence mode on the CPU: the shared filter algebra (csrc/cuda/lins_seq_step.cuh) against the host filter and shim it
replaces, bit for bit; the ctypes mirrors of the new C structs; the edited feature logs the GPU test relies on."""
import ctypes as C
import os
import subprocess

import numpy as np

from conftest import ROOT

HOST = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
CUDA = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")

# StateEstimator is compiled with the C-ABI stubbed out: the test only calls its host-side members
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
static std::mt19937_64 rng(7);
static double U(double a, double b) { return std::uniform_real_distribution<double>(a, b)(rng); }
static bool same(const double* a, const double* b, int n) { return std::memcmp(a, b, sizeof(double) * n) == 0; }
static filter::GlobalState rand_state() {
  filter::GlobalState g;
  g.rn_ = V3D(U(-5, 5), U(-5, 5), U(-1, 1)); g.vn_ = V3D(U(-3, 3), U(-3, 3), U(-.3, .3));
  g.qbn_ = Q4D(U(-1, 1), U(-1, 1), U(-1, 1), U(-1, 1)).normalized();
  g.ba_ = V3D(U(-.1, .1), U(-.1, .1), U(-.1, .1)); g.bw_ = V3D(U(-.01, .01), U(-.01, .01), U(-.01, .01));
  g.gn_ = V3D(U(-.5, .5), U(-.5, .5), -9.81 + U(-.1, .1));
  return g;
}
static void rand_cov(filter::Cov18& P) {
  double A[324];
  for (double& a : A) a = U(-0.1, 0.1);
  for (int i = 0; i < 18; ++i) for (int j = 0; j < 18; ++j) { double s = i == j ? 1e-3 : 0; for (int k = 0; k < 18; ++k) s += A[i * 18 + k] * A[j * 18 + k]; P(i, j) = s; }
}
int main() {
  int bad_predict = 0, bad_reset = 0, bad_post = 0, n_predict = 0, n_zero = 0;
  filter::FilterParams fp;
  fp.init_pos_std = V3D(0.1, 0.2, 0.3); fp.init_att_std = V3D(0.5, 1.0, 2.0);
  for (int trial = 0; trial < 200; ++trial) {
    filter::StatePredictor sp(fp);
    sp.initialization(0.0, V3D(), V3D(), V3D(), V3D(), V3D(U(-1, 1), U(-1, 1), 9.8), V3D(U(-.1, .1), U(-.1, .1), U(-.1, .1)));
    sp.state_ = rand_state();
    rand_cov(sp.covariance_);
    lins_seq::Consts k;
    std::memcpy(k.noise, sp.noise_, sizeof(k.noise));
    for (int i = 0; i < 3; ++i) {
      k.pos_var[i] = fp.init_pos_std(i) * fp.init_pos_std(i);
      k.att_var[i] = std::pow(math_utils::deg2rad(fp.init_att_std(i)), 2);
    }
    double s[19], P[324], al[3], gl[3];
    sp.state_.toArray(s); std::memcpy(P, sp.covariance_.data(), sizeof(P));
    for (int i = 0; i < 3; ++i) { al[i] = sp.acc_last(i); gl[i] = sp.gyr_last(i); }
    // the samples lins_seq_run_bag produces: full 2.5 ms steps, partial first / last ones, and dt = 0
    const int n = 1 + trial % 45;
    for (int m = 0; m < n; ++m) {
      double dt = 0.0025;
      if (m == 0 && trial % 3 == 0) dt = U(0, 0.0025);
      if (m == n - 1 && trial % 4 == 0) dt = U(0, 0.0025);
      if (trial % 5 == 0 && m % 7 == 3) { dt = 0.0; ++n_zero; }
      const double acc[3] = {U(-3, 3), U(-3, 3), 9.81 + U(-3, 3)}, gyr[3] = {U(-1, 1), U(-1, 1), U(-1, 1)};
      sp.predict(dt, V3D(acc[0], acc[1], acc[2]), V3D(gyr[0], gyr[1], gyr[2]), true);
      lins_seq::predict_host(s, P, al, gl, k.noise, dt, acc, gyr);
      double h[19];
      sp.state_.toArray(h);
      ++n_predict;
      if (!same(h, s, 19) || !same(sp.covariance_.data(), P, 324)) ++bad_predict;
    }
    // reset(1)
    sp.reset(1);
    lins_seq::reset1(s, P, k);
    double h[19];
    sp.state_.toArray(h);
    if (!same(h, s, 19) || !same(sp.covariance_.data(), P, 324)) ++bad_reset;
    // integrateTransformation + roll / pitch (the shim's members)
    fusion::StateEstimator est;
    est.globalState_ = rand_state();
    est.filter_->state_ = rand_state();
    double g[19], f[19];
    est.globalState_.toArray(g); est.filter_->state_.toArray(f);
    est.integrateTransformation();
    est.filter_->reset(1);
    double roll, pitch;
    est.calculateRPfromGravity(est.filter_->state_.gn_, roll, pitch);
    est.correctRollPitch(roll, pitch);
    lins_seq::integrate(g, f);
    double fcov[324];
    std::memcpy(fcov, est.filter_->covariance_.data(), sizeof(fcov));
    lins_seq::reset1(f, fcov, k);
    lins_seq::correct_roll_pitch(g, f);
    est.globalState_.toArray(h);
    if (!same(h, g, 19)) ++bad_post;
  }
  std::printf("%d %d %d %d %d\n", n_predict, n_zero, bad_predict, bad_reset, bad_post);
  return 0;
}
'''


def test_step_header_matches_host_filter_and_shim_bit_for_bit(tmp_path):
    src = tmp_path / "t.cpp"
    src.write_text(DRIVER)
    exe = str(tmp_path / "t")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", HOST, "-I", CUDA, "-o", exe, str(src)])
    n_predict, n_zero, bad_predict, bad_reset, bad_post = map(int, subprocess.check_output([exe]).split())
    assert n_predict > 4000 and n_zero > 20
    assert (bad_predict, bad_reset, bad_post) == (0, 0, 0)


def test_seq_struct_mirrors_match_header(defs, tmp_path):
    structs = {"lins_seq_params": defs.LinsSeqParams, "lins_seq_begin_desc": defs.LinsSeqBeginDesc, "lins_seq_step_desc": defs.LinsSeqStepDesc}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "lins_gpu.h"', "int main(){"]
    for name, cls in structs.items():
        lines.append(f'printf("%zu\\n", sizeof({name}));')
        for f, _ in cls._fields_:
            lines.append(f'printf("%zu\\n", offsetof({name}, {f}));')
    lines.append('printf("%d %d %d %d\\n", LINS_SEQ_IDLE, LINS_SEQ_SKIPPED, LINS_SEQ_RAN, LINS_SEQ_ICP); return 0;}')
    (tmp_path / "s.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "s"), str(tmp_path / "s.c")])
    out = subprocess.check_output([str(tmp_path / "s")]).split()
    want = []
    for cls in structs.values():
        want.append(C.sizeof(cls))
        want += [getattr(cls, f).offset for f, _ in cls._fields_]
    assert [int(x) for x in out[:-4]] == want
    assert [int(x) for x in out[-4:]] == [defs.SEQ_IDLE, defs.SEQ_SKIPPED, defs.SEQ_RAN, defs.SEQ_ICP]


def test_case_logs_contain_every_edit(synth):
    import seq_cases as sc

    logs, edits = sc.case_logs(n_seq=12)
    assert sorted({c for c, _ in edits.values()}) == ["gate", "guard", "no_imu"]
    lengths = {len(l["time"]) for l in logs}
    assert len(lengths) > 1 and max(lengths) == sc.N_SCANS  # sequences of different lengths
    assert any(l["lidar"] == 1 for l in logs) and any(l["lidar"] == 0 for l in logs)
    for s, (case, k) in edits.items():
        sc_ = synth.log_scan(logs[s], k)
        n_sl, n_cl = len(sc_["surf_less_flat"]), len(sc_["corner_less_sharp"])
        if case == "gate":
            assert n_sl <= 10
        elif case == "guard":
            assert 10 < n_sl < 20 and n_cl > 5
        else:
            assert case == "no_imu" and len(sc_["imu"]) == 0
    for l in logs:  # unedited scans pass both the gate and the guard
        n = np.diff(l["surf_less_flat_off"])
        assert (n >= 20).sum() >= len(n) - 1


def test_seq_params_noise_is_the_host_predictors(defs, tmp_path):
    """LinsSeqParams.shipped() computes StatePredictor::setNoise's noise_ (kalman_filter.hpp) bit for bit."""
    (tmp_path / "n.cpp").write_text('''
#include <cstdio>
#include "kalman_filter.hpp"
int main() { lins::filter::StatePredictor sp; sp.setNoise(); for (double v : sp.noise_) std::printf("%a\\n", v); return 0; }
''')
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", HOST, "-o", str(tmp_path / "n"), str(tmp_path / "n.cpp")])
    host = [float.fromhex(x) for x in subprocess.check_output([str(tmp_path / "n")]).decode().split()]
    assert list(defs.LinsSeqParams.shipped().noise) == host
