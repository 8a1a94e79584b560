"""CPU checks of transform fusion (csrc/host/transform_fusion.hpp, the pose transform_fusion_node publishes on
/integrated_to_init): the header, compiled with g++ behind a small C shim, equals the restatement of tests/fusionref.py
byte for byte on random and adversarial inputs; the restatement's setRPY is tf's, pinned against scipy; the restatement
agrees with f64 pose composition T_mapped = T_aft T_bef^-1 T_sum; and lins_fused_pose has one layout in the C header and
in ctypes."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import fusionref as fr
import mapper_drive
from conftest import pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_DIR = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
F = np.float32

SHIM = r"""
#include <cstddef>
#include "transform_fusion.hpp"
#include "lins_gpu.h"
extern "C" void tf_fuse(const double* quat, const double* pos, int published, const float* aft, const float* bef, float* T,
                        double* pos_out, double* quat_out) {
  lins_tf::transform_fusion(quat, pos, published != 0, aft, bef, T, pos_out, quat_out);
}
extern "C" void tf_pair(const float* aft, const float* bef, float* a, float* b) { lins_tf::published_pair(aft, bef, a, b); }
extern "C" void tf_setrpy(double r, double p, double y, double* q) { lins_tf::tf_set_rpy(r, p, y, q); }
extern "C" void fused_layout(long* out) {
  out[0] = sizeof(lins_fused_pose); out[1] = offsetof(lins_fused_pose, pos); out[2] = offsetof(lins_fused_pose, quat);
  out[3] = offsetof(lins_fused_pose, transform_mapped); out[4] = offsetof(lins_fused_pose, valid);
}
"""


@pytest.fixture(scope="module")
def tf_lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ is not available")
    d = tmp_path_factory.mktemp("tf")
    src, so = d / "shim.cpp", d / "libtf.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-Wall", "-Werror", "-shared", "-fPIC", "-I", HOST_DIR, "-I", os.path.join(ROOT, "include"),
                           "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.tf_fuse.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp]
    L.tf_pair.argtypes = [vp] * 4
    L.tf_setrpy.argtypes = [C.c_double, C.c_double, C.c_double, vp]
    L.fused_layout.argtypes = [vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def header_fuse(L, quat, pos, published, aft, bef):
    q, p = np.ascontiguousarray(quat, np.float64), np.ascontiguousarray(pos, np.float64)
    a, b = np.ascontiguousarray(aft, F), np.ascontiguousarray(bef, F)
    T, po, qo = np.zeros(6, F), np.zeros(3), np.zeros(4)
    L.tf_fuse(_p(q), _p(p), int(published), _p(a), _p(b), _p(T), _p(po), _p(qo))
    return T, po, qo


def _cases():
    """(quat, pos, published, aft, bef): random drives and the adversarial corners."""
    rng = np.random.default_rng(1)
    out = []
    ident = (0.0, 0.0, 0.0, 1.0)
    z6 = np.zeros(6, F)
    out += [(ident, (0.0, 0.0, 0.0), p, z6, z6) for p in (False, True)]  # zero state, before and after a publish
    for _ in range(400):  # random, moderate
        T = rng.uniform(-1, 1, 6) * [1.2, math.pi, 1.2, 50, 10, 50]
        aft = (rng.uniform(-1, 1, 6) * [1.2, math.pi, 1.2, 50, 10, 50]).astype(F)
        bef = (rng.uniform(-1, 1, 6) * [1.2, math.pi, 1.2, 50, 10, 50]).astype(F)
        out.append((mapper_drive.odometry_quat(T), T[3:], True, aft, bef))
    specials = [math.pi, -math.pi, float(F(math.pi)), -float(F(math.pi)), 3.5, -4.0, 7.0, math.pi / 2, -math.pi / 2,
                float(F(math.pi / 2)), math.pi / 2 - 1e-4, -math.pi / 2 + 1e-4, 1.5707, 0.0, -0.0]
    for k in range(600):  # angles at and beyond +-pi, |rx| near pi / 2, NaN, off-unit quaternions, positions near 1e4 m
        T = rng.uniform(-1, 1, 6) * [1.5, math.pi, 1.5, 30, 5, 30]
        aft = (rng.uniform(-1, 1, 6) * [1.5, math.pi, 1.5, 30, 5, 30]).astype(F)
        bef = (rng.uniform(-1, 1, 6) * [1.5, math.pi, 1.5, 30, 5, 30]).astype(F)
        for arr in (T, aft, bef):
            for i in range(3):
                if rng.random() < 0.3:
                    arr[i] = specials[rng.integers(len(specials))]
            if rng.random() < 0.3:
                arr[3:] += rng.uniform(-1, 1, 3) * 1e4
        for arr in (aft, bef):
            if rng.random() < 0.15:
                arr[rng.integers(6)] = np.nan
        q = np.array(mapper_drive.odometry_quat(T)) * (rng.uniform(0.5, 2.0) if k % 3 == 0 else 1.0)
        if k % 50 == 7:
            q = np.array([0.0, 0.0, 0.0, 2.0])
        out.append((q, T[3:], k % 11 != 0, aft, bef))
    return out


def test_header_equals_restatement(tf_lib):
    n_nan_in = n_wrap = 0
    for i, (q, p, pub, aft, bef) in enumerate(_cases()):
        got = header_fuse(tf_lib, q, p, pub, aft, bef)
        ref = fr.fuse(q, p, pub, aft, bef)
        for g, r in zip(got, ref):
            assert g.tobytes() == np.asarray(r, g.dtype).tobytes(), (i, q, p, pub, aft, bef, got, ref)
        n_nan_in += bool(np.isnan(aft).any() or np.isnan(bef).any())
        n_wrap += bool(np.abs(aft[:3]).max() > math.pi)
    assert n_nan_in >= 50 and n_wrap >= 50


def test_published_pair(tf_lib):
    """NaN -> 0 in both arrays; aft's angles wrap into getRPY's ranges and keep their rotation; positions and bef pass."""
    aft = np.array([np.nan, 4.0, -3.5, np.nan, 2.5, 1e4], F)
    bef = np.array([0.1, np.nan, 7.0, 1.0, np.nan, -3.0], F)
    a, b = np.zeros(6, F), np.zeros(6, F)
    tf_lib.tf_pair(_p(aft), _p(bef), _p(a), _p(b))
    ra, rb = fr.published_pair(aft, bef)
    assert a.tobytes() == ra.tobytes() and b.tobytes() == rb.tobytes()
    assert b.tolist() == [F(0.1), 0.0, 7.0, 1.0, 0.0, -3.0]
    assert a[3:].tolist() == [0.0, 2.5, 1e4] and np.abs(a[:3]).max() <= math.pi
    assert np.abs(_loam_R(a) - _loam_R(np.array([0.0, 4.0, -3.5]))).max() < 1e-6
    # the zero pair, once published, comes back with a negative zero (-yaw of yaw = +0)
    tf_lib.tf_pair(_p(np.zeros(6, F)), _p(np.zeros(6, F)), _p(a), _p(b))
    assert np.signbit(a).tolist() == [False, True, False, False, False, False]


def test_set_rpy_is_tfs(tf_lib):
    """tf's setRPY(roll, pitch, yaw) = scipy's extrinsic xyz Euler rotation Rz(yaw) Ry(pitch) Rx(roll), to ~1e-15, and the
    header's equals the restatement bit for bit."""
    rng = np.random.default_rng(3)
    for r, p, y in list(rng.uniform(-7, 7, (300, 3))) + [(0, 0, 0), (math.pi, 0, 0), (0, math.pi / 2, 0), (0, 0, -math.pi), (1, -math.pi / 2, 2)]:
        q = np.array(fr.set_rpy(r, p, y))
        h = np.zeros(4)
        tf_lib.tf_setrpy(r, p, y, _p(h))
        assert h.tobytes() == q.tobytes()
        s = Rotation.from_euler("xyz", [r, p, y]).as_quat()
        assert min(np.abs(q - s).max(), np.abs(q + s).max()) < 2e-15, (r, p, y, q, s)


def _rx(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def _ry(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def _rz(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def _loam_R(T):
    """the rotation of a LOAM transform (rx, ry, rz): Ry(ry) Rx(rx) Rz(rz) (transformPointCloud's order)"""
    return _ry(float(T[1])) @ _rx(float(T[0])) @ _rz(float(T[2]))


def test_restatement_is_pose_composition():
    """transformMapped = T_aft T_bef^-1 T_sum in f64 (rotation R = Ry Rx Rz, p_map = R p + t), within f32 rounding: the
    inputs are f32, each of the ~40 f32 operations on the path to an angle or a translation rounds by 6e-8 relative, and
    |rx| <= 1.2 keeps 1 / cos(rx) below 3, so 2e-5 on rotation entries and 2e-5 * (1 + |t|) on translations is a margin
    of a few times the accumulated rounding.  The published orientation is the same rotation in the odometry's frame
    shuffle."""
    rng = np.random.default_rng(5)
    for _ in range(500):
        S, A, B = ((rng.uniform(-1, 1, 6) * [1.2, math.pi, 1.2, 80, 10, 80]).astype(F) for _ in range(3))
        q = mapper_drive.odometry_quat(S)
        T, pos, quat = fr.fuse(q, S[3:], True, A, B)
        Sum = fr.odometry_transform(q, S[3:])
        Ra, Rb, Rs = _loam_R(A), _loam_R(B), _loam_R(Sum)
        Rm = Ra @ Rb.T @ Rs
        tm = A[3:].astype(float) + Ra @ Rb.T @ (Sum[3:].astype(float) - B[3:].astype(float))
        if abs(math.asin(max(-1.0, min(1.0, -Rm[1, 2])))) > 1.2:
            continue  # (near |rx| = pi / 2 the Euler extraction loses precision)
        assert np.abs(_loam_R(T) - Rm).max() < 2e-5
        assert np.abs(pos - tm).max() < 2e-5 * (1 + np.abs(tm).max())
        # the published quaternion, read back as the odometry is, gives the same rotation
        assert np.abs(_loam_R(fr.odometry_transform(quat, pos)) - Rm).max() < 2e-5


def test_fused_pose_layout(tf_lib):
    defs = pkg("ctypes_defs")
    out = (C.c_long * 5)()
    tf_lib.fused_layout(out)
    P = defs.LinsFusedPose
    assert list(out) == [C.sizeof(P), P.pos.offset, P.quat.offset, P.transform_mapped.offset, P.valid.offset] == [96, 8, 32, 64, 88]
