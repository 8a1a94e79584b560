"""Sequence mode's filter algebra against tests/filterref.py, an independent float64 restatement of the reference.

csrc/cuda/lins_seq_step.cuh (what the device kernels run) and csrc/host/kalman_filter.hpp / state_estimator.hpp (the
host mirror) are compiled with g++ into one driver that replays a script of predict / reset(1) / post / initialisation
calls and prints every result in %a.  Every call is checked on its own: filterref gets the driver's inputs of that call.
The scripts walk random chains and the edges where the algebra branches or degenerates.  The restatement itself is pinned
against scipy's Rotation and against mpmath at 50 digits."""
import math
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import filterref as fr
from filterref import check_cov, check_state
from conftest import ROOT

HOST = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
CUDA = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")
M = fr.F64


DRIVER = r'''
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
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
static double rd() { char b[64]; if (std::scanf("%63s", b) != 1) std::exit(2); return std::strtod(b, nullptr); }
static void rdn(double* d, int n) { for (int i = 0; i < n; ++i) d[i] = rd(); }
static V3D rv() { double d[3]; rdn(d, 3); return V3D(d[0], d[1], d[2]); }
static void pr(const char* tag, const double* d, int n) {
  std::printf("%s", tag);
  for (int i = 0; i < n; ++i) std::printf(" %a", d[i]);
  std::printf("\n");
}
int main() {
  filter::FilterParams fp;
  lins_seq::Consts k{};
  lins_seq::InitConsts ik{};
  filter::StatePredictor sp(fp);
  double s[20] = {0}, P[324], al[3], gl[3], pre[20], glob[20], filt[20], lin[20], il[8], pose[20];
  char op[8];
  while (std::scanf("%7s", op) == 1) {
    const std::string o = op;
    if (o == "K") {  // acc_n gyr_n acc_w gyr_w, then pos vel att acc gyr std, init_ba, init_bw
      fp.acc_n = rd(); fp.gyr_n = rd(); fp.acc_w = rd(); fp.gyr_w = rd();
      fp.init_pos_std = rv(); fp.init_vel_std = rv(); fp.init_att_std = rv(); fp.init_acc_std = rv(); fp.init_gyr_std = rv();
      fp.init_ba = rv(); fp.init_bw = rv();
      sp = filter::StatePredictor(fp);
      sp.setNoise();
      std::memcpy(k.noise, sp.noise_, sizeof(k.noise));
      for (int i = 0; i < 3; ++i) {  // lins_seq.cu set_consts / set_init_consts
        k.pos_var[i] = fp.init_pos_std(i) * fp.init_pos_std(i);
        k.att_var[i] = std::pow(fp.init_att_std(i) * M_PI / 180.0, 2);
        ik.var[lins_seq::kPos + i] = k.pos_var[i];
        ik.var[lins_seq::kVel + i] = fp.init_vel_std(i) * fp.init_vel_std(i);
        ik.var[lins_seq::kAtt + i] = k.att_var[i];
        ik.var[lins_seq::kAcc + i] = fp.init_acc_std(i) * fp.init_acc_std(i);
        ik.var[lins_seq::kGyr + i] = fp.init_gyr_std(i) * fp.init_gyr_std(i);
        ik.var[lins_seq::kGra + i] = 0.01;
        ik.ba[i] = fp.init_ba(i); ik.bw[i] = fp.init_bw(i);
      }
    } else if (o == "S") {  // filter state (19), covariance (324, column-major), acc_last, gyr_last
      rdn(s, 19); rdn(P, 324); rdn(al, 3); rdn(gl, 3);
      sp.state_ = filter::GlobalState::fromArray(s);
      std::memcpy(sp.covariance_.data(), P, sizeof(P));
      sp.acc_last = V3D(al[0], al[1], al[2]); sp.gyr_last = V3D(gl[0], gl[1], gl[2]);
      sp.flag_init_state_ = sp.flag_init_imu_ = true;
    } else if (o == "P") {  // one predict call: dt, acc, gyr
      double dt = rd(), a[3], w[3];
      rdn(a, 3); rdn(w, 3);
      sp.predict(dt, V3D(a[0], a[1], a[2]), V3D(w[0], w[1], w[2]), true);
      lins_seq::predict_host(s, P, al, gl, k.noise, dt, a, w);
      double h[19]; sp.state_.toArray(h);
      pr("H", h, 19); pr("H", sp.covariance_.data(), 324); pr("D", s, 19); pr("D", P, 324);
    } else if (o == "R") {  // reset(1)
      sp.reset(1);
      lins_seq::reset1(s, P, k);
      double h[19]; sp.state_.toArray(h);
      pr("H", h, 19); pr("H", sp.covariance_.data(), 324); pr("D", s, 19); pr("D", P, 324);
    } else if (o == "G") {  // processScan's post stage on the current filter state and covariance: global state (19)
      double g[20] = {0}, h[19];
      rdn(g, 19);
      fusion::EstimatorParams ep;
      ep.filter = fp;
      fusion::StateEstimator est(ep);
      est.globalState_ = filter::GlobalState::fromArray(g);
      est.filter_->state_ = sp.state_;
      est.filter_->covariance_ = sp.covariance_;
      est.integrateTransformation();
      est.filter_->reset(1);
      double roll, pitch;
      est.calculateRPfromGravity(est.filter_->state_.gn_, roll, pitch);
      est.correctRollPitch(roll, pitch);
      lins_seq::integrate(g, s);
      lins_seq::reset1(s, P, k);
      lins_seq::correct_roll_pitch(g, s);
      est.globalState_.toArray(h); pr("H", h, 19);
      est.filter_->state_.toArray(h); pr("H", h, 19); pr("H", est.filter_->covariance_.data(), 324);
      pr("D", g, 19); pr("D", s, 19); pr("D", P, 324);
      sp.state_ = est.filter_->state_; sp.covariance_ = est.filter_->covariance_;
    } else if (o == "F") {  // processFirstScan with the scan's IMU sample (acc, gyr)
      double imu[6]; rdn(imu, 6);
      lins_seq::first_scan(filt, P, lin, pre, il, imu, ik);
      pr("D", filt, 19); pr("D", P, 324); pr("D", pre, 17); pr("D", il, 6);
    } else if (o == "Q") {  // one pre-integration row: dt, acc, gyr
      double dt = rd(), a[3], w[3];
      rdn(a, 3); rdn(w, 3);
      lins_seq::preint_propagate(pre, ik, dt, a, w);
      pr("D", pre, 17);
    } else if (o == "T") {  // processSecondScan's ICP start pose
      lins_seq::second_scan_start(pre, pose);
      pr("D", pose, 10);
    } else if (o == "Z") {  // the rest of processSecondScan: the ICP's pose (t, q xyzw), the scan's IMU sample
      double t[7], imu[6]; rdn(t, 7); rdn(imu, 6);
      for (int i = 0; i < 20; ++i) pose[i] = 0.0;
      for (int i = 0; i < 3; ++i) pose[i] = t[i];
      for (int i = 0; i < 4; ++i) pose[6 + i] = t[3 + i];
      lins_seq::second_scan(glob, filt, P, lin, il, pre, pose, imu, ik);
      pr("D", glob, 19); pr("D", filt, 19); pr("D", P, 324); pr("D", il, 6);
    } else {
      return 3;
    }
  }
  return 0;
}
'''


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("filterref")
    (d / "t.cpp").write_text(DRIVER)
    exe = str(d / "t")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", HOST, "-I", CUDA, "-o", exe, str(d / "t.cpp")])

    def run(script):
        out = subprocess.run([exe], input="\n".join(script) + "\n", capture_output=True, text=True, check=True).stdout
        return [(ln.split()[0], np.array([float.fromhex(x) for x in ln.split()[1:]])) for ln in out.splitlines()]
    return run


def hx(*vals):
    return " ".join(float(v).hex() for a in vals for v in np.ravel(a))


# ---- the scripts ----------------------------------------------------------------------------------------------------
def rand_params(rng):
    u = lambda a, b: tuple(rng.uniform(a, b, 3))
    return dict(acc_n=rng.uniform(1e3, 1e5), gyr_n=rng.uniform(0.01, 1), acc_w=rng.uniform(10, 1e3), gyr_w=rng.uniform(0.01, 0.1),
                init_pos_std=u(0, 0.5), init_vel_std=u(0, 0.5), init_att_std=u(0, 3), init_acc_std=u(0, 0.1),
                init_gyr_std=u(0, 0.01), init_ba=u(-0.2, 0.2), init_bw=u(-0.01, 0.01))


def params_line(p):
    return "K " + hx(p["acc_n"], p["gyr_n"], p["acc_w"], p["gyr_w"], *(p[k] for k in (
        "init_pos_std", "init_vel_std", "init_att_std", "init_acc_std", "init_gyr_std", "init_ba", "init_bw")))


def rand_quat(rng, w_negative=False, norm_off=0.0):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    if w_negative and q[3] > 0:
        q = -q
    return q * (1.0 + norm_off)


def rand_state(rng, q=None, gn=None):
    s = np.concatenate([rng.uniform(-5, 5, 3), rng.uniform(-3, 3, 3), rand_quat(rng) if q is None else q,
                        rng.uniform(-0.1, 0.1, 3), rng.uniform(-0.01, 0.01, 3),
                        np.array([*rng.uniform(-0.5, 0.5, 2), -9.81 + rng.uniform(-0.1, 0.1)]) if gn is None else gn])
    return s


def rand_cov(rng):
    A = rng.uniform(-0.1, 0.1, (18, 18))
    return A @ A.T + 1e-3 * np.eye(18)


class Script:
    """The driver's commands plus what the checker needs to rebuild each call's inputs."""

    def __init__(self):
        self.lines, self.ops = [], []

    def add(self, line, op):
        self.lines.append(line)
        self.ops.append(op)


def imu_row(rng, dt=0.0025):
    return dt, np.array([*rng.uniform(-3, 3, 2), 9.81 + rng.uniform(-3, 3)]), rng.uniform(-1, 1, 3)


def chains(seed, n_chains):
    """Random chains of 40 predict calls from edge-case states, each followed by reset(1) or the post stage, and one
    initialisation (first scan, pre-integration, second scan) per chain."""
    rng = np.random.default_rng(seed)
    sc = Script()
    edges = dict(dt0=0, gap=0, spin=0, theta0=0, theta_lo=0, theta_hi=0, w_neg=0, q_off=0, gz_pos=0, gz_zero=0,
                 g_over=0, g_zero=0, sum_dt0=0, gimbal=0)
    for c in range(n_chains):
        p = fr.YAML if c % 4 == 0 else rand_params(rng)
        sc.add(params_line(p), ("K", p))
        kind = c % 6
        q = rand_quat(rng, w_negative=kind == 1, norm_off=(1e-9, -1e-9)[c % 2] if kind == 2 else 0.0)
        edges["w_neg"] += kind == 1
        edges["q_off"] += kind == 2
        gn = None
        if kind == 3:
            up = (c // 6) % 2 == 0
            gn = np.array([*rng.uniform(-0.5, 0.5, 2), (9.81 if up else 0.0)])
            edges["gz_pos" if up else "gz_zero"] += 1
        elif kind == 4:
            gn = np.zeros(3)
            edges["g_zero"] += 1
        s = rand_state(rng, q=q, gn=gn)
        P, al, gl = rand_cov(rng), *imu_row(rng)[1:]
        sc.add("S " + hx(s, P.T, al, gl), ("S", s, P, al, gl))
        bw = s[fr.S_BW:fr.S_BW + 3]
        for n in range(40):
            dt, a, w = imu_row(rng)
            r = n % 10
            if r == 1 and c % 3 == 0:
                dt = 0.0
                edges["dt0"] += 1
            elif r == 2:
                dt = (0.1, 0.5)[c % 2]
                edges["gap"] += 1
                if c % 2:  # theta = |(gyr_last + gyr) / 2 - bw| dt from about 2.5 to 5 rad: up to and past pi
                    w = rng.normal(size=3)
                    w *= rng.uniform(10, 20) / np.linalg.norm(w)
                    theta = np.linalg.norm((0.5 * (sc.ops[-1][3] + w) - bw) * dt)
                    edges["spin"] += theta > math.pi
            elif r == 3:  # gyr == bw: theta = 0 exactly (the previous sample is made equal too)
                w = bw.copy()
            elif r == 4:
                w = bw.copy()
                edges["theta0"] += 1
            elif r in (6, 8):  # theta just below / above 1e-10, from the same sample twice
                d = rng.normal(size=3)
                d *= (0.98e-10 if r == 6 else 1.02e-10) / (np.linalg.norm(d) * dt)
                w = bw + d
            elif r in (7, 9):
                w = sc.ops[-1][3].copy()
                edges["theta_lo" if r == 7 else "theta_hi"] += 1
            sc.add("P " + hx(dt, a, w), ("P", dt, a, w))
        if (c // 2) % 2:
            sc.add("R", ("R",))
        else:
            g = rand_state(rng)
            if c % 8 == 0:  # the integrated attitude's pitch near +-90 degrees: R2rpy divides by cos(pitch)
                s2, P2 = rand_state(rng), rand_cov(rng)
                sc.add("S " + hx(s2, P2.T, al, gl), ("S", s2, P2, al, gl))
                pitch = (1, -1)[c % 16 == 0] * (math.pi / 2 - (1e-2, 1e-4)[(c // 8) % 3 == 0])
                target = fr.rpy2Quat(M, np.array([0.3, pitch, -1.2]))
                g[6:10] = fr.qmul(target, fr.qinverse(M, s2[6:10]))
                edges["gimbal"] += 1
            sc.add("G " + hx(g), ("G", g))
        # an initialisation with non-zero INIT_*: first scan, rows, second scan from the start pose and from a moved one
        imu0 = np.concatenate([imu_row(rng)[1], rng.uniform(-0.5, 0.5, 3)])
        sc.add("F " + hx(imu0), ("F", imu0))
        nrow = 0 if c % 7 == 3 else 1 + c % 45
        edges["sum_dt0"] += nrow == 0
        for n in range(nrow):
            dt, a, w = imu_row(rng, dt=0.0 if n % 11 == 7 else rng.uniform(0, 0.005))
            if n % 13 == 5:
                w = rng.uniform(-20, 20, 3)
            sc.add("Q " + hx(dt, a, w), ("Q", dt, a, w))
        sc.add("T", ("T",))
        imu1 = np.concatenate([imu_row(rng)[1], rng.uniform(-0.5, 0.5, 3)])
        if c % 5 == 1:
            imu1[0] = (1, -1)[c % 2] * rng.uniform(9.9, 12)  # |fx| > G0: a NaN pitch
            edges["g_over"] += 1
        elif c % 5 == 2:
            imu1[2] = p["init_ba"][2]  # fz - ba_z = 0: sign(0) = +1
        pose = np.concatenate([rng.uniform(-0.5, 0.5, 3), rand_quat(rng)])
        sc.add("Z " + hx(pose, imu1), ("Z", pose, imu1))
    return sc, edges


def check(sc, out):
    """Walk the script with the driver's output; every call against filterref from that call's inputs."""
    it = iter(out)

    def nxt(tag):
        t, v = next(it)
        assert t == tag, (t, tag)
        return v
    p = fr.YAML
    noise = fr.noise_diag(p)
    cur = None  # (state, P, acc_last, gyr_last) as the driver holds them
    pre = None
    n_cmp = dict(predict=0, reset=0, post=0, first=0, preint=0, second=0, gimbal_skip=0)
    for op in sc.ops:
        kind = op[0]
        if kind == "K":
            p, noise = op[1], fr.noise_diag(op[1])
        elif kind == "S":
            cur = [op[1], op[2], op[3], op[4]]
        elif kind in ("P", "R"):
            if kind == "P":
                want_s, want_P = fr.predict(M, cur[0], cur[1], cur[2], cur[3], op[1], op[2], op[3], noise)
            else:
                want_s, want_P = fr.reset1(M, cur[0], cur[1], p)
            for side in "HD":
                got_s, got_P = nxt(side), nxt(side)
                check_state(got_s, want_s, (kind, side))
                check_cov(got_P, want_P, (kind, side))
            n_cmp["predict" if kind == "P" else "reset"] += 1
            cur = [got_s, got_P.reshape(18, 18).T, *(op[2:4] if kind == "P" else cur[2:4])]
        elif kind == "G":
            want_g, want_f, want_P = fr.post_step(M, op[1], cur[0], cur[1], p)
            rpy = fr.Q2rpy(M, fr.integrate(M, op[1], cur[0])[6:10])
            skip = range(6, 10) if not math.cos(rpy[1]) > fr.COS_PITCH_MIN else ()
            n_cmp["gimbal_skip"] += len(skip) > 0
            for side in "HD":
                got_g, got_f, got_P = nxt(side), nxt(side), nxt(side)
                check_state(got_g, want_g, ("G global", side), skip=skip)
                check_state(got_f, want_f, ("G filter", side))
                check_cov(got_P, want_P, ("G", side))
            n_cmp["post"] += 1
            cur = [got_f, got_P.reshape(18, 18).T, cur[2], cur[3]]
        elif kind == "F":
            want_f, want_P, pre, al, gl = fr.first_scan(M, op[1], p)
            got_f, got_P, got_pre, got_il = nxt("D"), nxt("D"), nxt("D"), nxt("D")
            check_state(got_f, want_f, "first filter")
            check_cov(got_P, want_P, "first")
            check_state(got_pre, preint_vec(pre), "first preint")
            check_state(got_il, np.concatenate([al, gl]), "first imu_last")
            n_cmp["first"] += 1
        elif kind == "Q":
            # from the driver's own pre-integration state: restate its 17 numbers into a Preint
            pre.push_back(op[1], op[2], op[3])
            got = nxt("D")
            check_state(got, preint_vec(pre), "preint")
            pre = preint_from(got, p)
            n_cmp["preint"] += 1
        elif kind == "T":
            pl, ql = fr.second_scan_start(M, pre)
            got = nxt("D")
            check_state(got[:3], pl, "start t")
            check_state(got[6:10], ql, "start q")
        elif kind == "Z":
            pose, imu1 = op[1], op[2]
            want_g, want_f, want_P, al, gl = fr.second_scan(M, pre, pose[:3], pose[3:], imu1, p)
            got_g, got_f, got_P, got_il = nxt("D"), nxt("D"), nxt("D"), nxt("D")
            check_state(got_g, want_g, "second global")
            check_state(got_f, want_f, "second filter")
            check_cov(got_P, want_P, "second")
            check_state(got_il, np.concatenate([al, gl]), "second imu_last")
            n_cmp["second"] += 1
    assert next(it, None) is None
    return n_cmp


def preint_vec(pre):
    """The device's 17-number pre-integration: acc_0 gyr_0 delta_p delta_v delta_q(x, y, z, w) sum_dt"""
    return np.concatenate([pre.acc_0, pre.gyr_0, pre.delta_p, pre.delta_v, pre.delta_q, [pre.sum_dt]]).astype(float)


def preint_from(v, p):
    pre = fr.Preint(M, v[0:3], v[3:6], p["init_ba"], p["init_bw"])
    pre.delta_p, pre.delta_v, pre.delta_q, pre.sum_dt = v[6:9].copy(), v[9:12].copy(), v[12:16].copy(), float(v[16])
    return pre


# ---- tests ----------------------------------------------------------------------------------------------------------
def test_filter_algebra_matches_the_restated_reference(driver):
    sc, edges = chains(seed=3, n_chains=96)
    n = check(sc, driver(sc.lines))
    assert n["predict"] == 96 * 40 and n["reset"] == 48 and n["post"] == 48 and n["second"] == 96, n
    assert n["preint"] > 1500, n
    assert all(v > 0 for v in edges.values()), edges
    print(n, edges)


def test_edges_produce_the_reference_nan_and_inf(driver):
    """gn = 0 before reset(1) makes the reset's gravity NaN (0 / 0), a second scan with no IMU rows divides by sum_dt = 0
    and |fx| > G0 makes the hand-over pitch NaN: the header must reproduce these, not guard them."""
    sc, _ = chains(seed=5, n_chains=30)
    out = driver(sc.lines)
    check(sc, out)
    flat = np.concatenate([v for _, v in out])
    assert np.isnan(flat).any() and np.isinf(flat).any()


def test_shipped_constants_are_the_yaml_values(defs):
    """LinsSeqParams.shipped().noise and LinsSeqInitParams.shipped() against exp_port.yaml through parameters.h."""
    ulp = lambda a, b: abs(a - b) <= math.ulp(max(abs(a), abs(b)))
    sp = defs.LinsSeqParams.shipped()
    for got, want in zip(sp.noise, fr.noise_diag()):
        assert ulp(got, want), (got, want)
    assert list(sp.init_pos_std) == list(fr.YAML["init_pos_std"]) and list(sp.init_att_std) == list(fr.YAML["init_att_std"])
    ip = defs.LinsSeqInitParams.shipped()
    for f in ("init_vel_std", "init_acc_std", "init_gyr_std", "init_ba", "init_bw"):
        assert all(ulp(a, b) for a, b in zip(getattr(ip, f), fr.YAML[f])), f
    # the filter's noise comes from parameters.h's ACC_N / GYR_N / ..., not integrationBase.h's integration:: constants
    assert fr.noise_diag()[0] > 0.4 and fr.noise_diag()[1] < 1e-10


# ---- the restatement against scipy and mpmath -----------------------------------------------------------------------
def test_rotation_pieces_match_scipy():
    rng = np.random.default_rng(1)
    for _ in range(200):
        q = rand_quat(rng)
        r = Rotation.from_quat(q)
        v = rng.normal(size=3)
        assert np.allclose(fr.qrot(q, v), r.apply(v), rtol=0, atol=1e-14)
        assert np.allclose(fr.qtoR(q), r.as_matrix(), rtol=0, atol=1e-15)
        q2 = rand_quat(rng)
        assert np.allclose(fr.qmul(q, q2), (r * Rotation.from_quat(q2)).as_quat(canonical=False), atol=1e-15) or \
            np.allclose(fr.qmul(q, q2), -(r * Rotation.from_quat(q2)).as_quat(canonical=False), atol=1e-15)
        assert np.allclose(fr.qtoR(fr.qinverse(M, q)), r.inv().as_matrix(), atol=1e-15)
        w = rng.normal(size=3) * rng.uniform(0, 3)
        assert np.allclose(fr.qtoR(fr.axis2Quat(M, w)), Rotation.from_rotvec(w).as_matrix(), atol=1e-14)
        rpy = np.array([rng.uniform(-3, 3), rng.uniform(-1.5, 1.5), rng.uniform(-3, 3)])
        R = Rotation.from_euler("ZYX", rpy[::-1]).as_matrix()  # R = Rz(yaw) Ry(pitch) Rx(roll)
        assert np.allclose(fr.qtoR(fr.rpy2Quat(M, rpy)), R, atol=1e-14)
        assert np.allclose(fr.Q2rpy(M, fr.rpy2Quat(M, rpy)), rpy, atol=1e-12)
    assert np.array_equal(fr.axis2Quat(M, np.array([1e-11, 0, 0])), [0, 0, 0, 1])
    assert fr.sign(0.0) == 1 and fr.sign(-0.0) == 1 and fr.sign(float("nan")) == -1


def test_restatement_matches_mpmath_at_50_digits():
    """predict, reset(1) and the pre-integration in float64 against the same functions at 50 digits."""
    import mpmath

    mpmath.mp.dps = 50
    MP = fr.mp_backend()
    rng = np.random.default_rng(2)
    to_mp = lambda a: np.array([mpmath.mpf(float(x)) for x in np.ravel(a)], dtype=object).reshape(np.shape(a))
    worst = 0.0

    def rel(f, m):
        nonlocal worst
        f = np.asarray(f, float)
        m = np.array([float(x) for x in np.ravel(m)]).reshape(f.shape)
        # states entry-wise against max(|x|, 1), covariances normwise (against max |P|)
        e = np.abs(f - m) / (np.abs(m).max() if m.ndim == 2 else np.maximum(np.abs(m), 1.0))
        worst = max(worst, e.max())
        assert e.max() <= 1e-14, e.max()

    for t in range(50):
        p = fr.YAML if t % 2 else rand_params(rng)
        noise = fr.noise_diag(p)
        s, P = rand_state(rng), rand_cov(rng)
        dt, a, w = imu_row(rng, dt=(0.0025, 0.1, 0.5)[t % 3])
        al, gl = imu_row(rng)[1:]
        fs, fP = fr.predict(M, s, P, al, gl, dt, a, w, noise)
        ms, mP = fr.predict(MP, to_mp(s), to_mp(P), al, gl, dt, a, w, noise)
        rel(fs, ms)
        rel(fP, mP)
        fs, fP = fr.reset1(M, s, P, p)
        ms, mP = fr.reset1(MP, to_mp(s), to_mp(P), p)
        rel(fs, ms)
        rel(fP, mP)
        imu0 = rng.normal(size=6)
        f_pre, m_pre = fr.Preint(M, imu0[:3], imu0[3:], p["init_ba"], p["init_bw"]), fr.Preint(MP, imu0[:3], imu0[3:], p["init_ba"], p["init_bw"])
        for _ in range(20):
            dt, a, w = imu_row(rng, dt=rng.uniform(0, 0.005))
            f_pre.push_back(dt, a, w)
            m_pre.push_back(dt, a, w)
        rel(preint_vec(f_pre), np.array([float(x) for x in np.concatenate([m_pre.acc_0, m_pre.gyr_0, m_pre.delta_p, m_pre.delta_v, m_pre.delta_q, [m_pre.sum_dt]])]))
    print("worst relative float64 - mpmath", worst)
