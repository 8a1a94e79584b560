"""CPU suite for the mapping node's cycle: the CPU oracle's pieces (tests/mapperref.py) pinned against independent
restatements — its VoxelGrid against tests/pyfront.voxel_grid, tf's getRPY and gtsam's RzRyRx / xyz() round trip against
scipy's Rotation, the window's deque bookkeeping (duplicate included) against the reference's lines replayed by hand —
the C-ABI structs against the header, and the oracle's cycle on a short synthetic drive."""
import collections
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import mapperref
import pyfront
from conftest import ROOT


def _cloud(rng, n, lo, hi, nan_every=0):
    p = rng.uniform(lo, hi, (n, 4)).astype(np.float32)
    p[:, 3] = rng.uniform(0, 16, n).astype(np.float32)
    if nan_every:
        p[::nan_every, rng.integers(0, 3)] = np.nan
        p[1::nan_every * 3, 1] = np.inf
    return p


@pytest.mark.parametrize("leaf", [0.2, 0.4])
@pytest.mark.parametrize("case", ["spread", "dense", "negative", "nonfinite", "all_nan"])
def test_oracle_voxel_grid_equals_pyfront(leaf, case):
    rng = np.random.default_rng(7)
    p = dict(spread=lambda: _cloud(rng, 4000, -30, 30), dense=lambda: _cloud(rng, 3000, 0.01, 0.9),
             negative=lambda: _cloud(rng, 3000, -12.3, -0.05), nonfinite=lambda: _cloud(rng, 3000, -5, 5, nan_every=11),
             all_nan=lambda: np.full((5, 4), np.nan, np.float32))[case]()
    a, b = mapperref.voxel_grid(p, leaf), pyfront.voxel_grid(p, leaf)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_oracle_voxel_grid_too_big():
    p = np.array([[-1e5, -1e5, -1e5, 0], [1e5, 1e5, 1e5, 0]], np.float32)
    with pytest.raises(mapperref.TooBig):
        mapperref.voxel_grid(p, 0.01)
    assert len(mapperref.voxel_grid(p, 400.0)) == 2


def test_get_rpy_matches_scipy():
    rng = np.random.default_rng(3)
    for _ in range(500):
        rpy = rng.uniform([-3.1, -1.4, -3.1], [3.1, 1.4, 3.1])  # away from gimbal lock
        q = Rotation.from_euler("ZYX", rpy[::-1]).as_quat()  # x, y, z, w; R = Rz(yaw) Ry(pitch) Rx(roll)
        q = q * rng.uniform(0.5, 2.0)  # getRPY normalises through 2 / |q|^2
        assert np.allclose(mapperref.get_rpy(*q), rpy, atol=1e-12)


def test_rot3_round_trip_matches_scipy():
    rng = np.random.default_rng(4)
    for _ in range(500):
        x, y, z = rng.uniform([-3.1, -1.4, -3.1], [3.1, 1.4, 3.1])
        R = np.array(mapperref.rot3_rzryrx(x, y, z))
        assert np.allclose(R, Rotation.from_euler("ZYX", [z, y, x]).as_matrix(), atol=1e-14)
        assert np.allclose(mapperref.rot3_xyz(R.tolist()), (x, y, z), atol=1e-12)
    # f32 in, f32 out: the stored PointTypePose equals the f32 transform to within an ulp
    T = np.float32([0.1, -0.7, 2.5])
    x, y, z = mapperref.rot3_xyz(mapperref.rot3_rzryrx(float(T[2]), float(T[0]), float(T[1])))
    assert np.allclose(np.float32([y, z, x]), T, rtol=0, atol=4e-7)


def _literal_window(saves):
    """extractSurroundingKeyFrames :1204-1240 replayed by hand on a list of per-cycle 'saved a key frame' flags:
    numPoses is the number of key frames saved by earlier cycles."""
    recent, latestFrameID, numPoses, out = [], 0, 0, []
    for saved in saves:
        if numPoses:
            if len(recent) < 50:
                recent = []
                i = numPoses - 1
                while i >= 0:
                    recent.insert(0, i)
                    if len(recent) >= 50:
                        break
                    i -= 1
            else:
                if latestFrameID != numPoses - 1:
                    recent.pop(0)
                    latestFrameID = numPoses - 1
                    recent.append(latestFrameID)
        out.append(list(recent))
        numPoses += int(saved)
    return out


@pytest.mark.parametrize("stall", [None, 50, 51, 60])
def test_window_bookkeeping_with_the_duplicate(stall):
    saves = [k != stall for k in range(70)]
    expect = _literal_window(saves)
    window, latest, n, got = collections.deque(), [0], 0, []
    for saved in saves:
        mapperref.extract_window(window, latest, n)
        got.append(list(window))
        n += int(saved)
    assert got == expect
    assert all(len(w) <= 50 for w in got)
    if stall == 50:  # the cycle that fills the window saves nothing: key frame 0 leaves and 49 enters a second time
        assert got[51] == list(range(1, 50)) + [49] and got[52] == list(range(2, 50)) + [49, 50]
        assert got[69].count(49) == 2 and len(got[69]) == 50  # it shifts through the window with the rest
    else:
        assert all(len(set(w)) == len(w) for w in got)


def test_mapper_structs_match_header(defs):
    assert C.sizeof(defs.LinsMapperDesc) == 8 + 32 + 24 + 3 * 8 + 4 * 4
    assert C.sizeof(defs.LinsMapperReport) == 12 * 4 + 12 * 4 + C.sizeof(defs.LinsMapReport)
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "lins_gpu.h"\nint main(){printf("%zu %zu %zu %zu\\n", sizeof(lins_mapper_desc), '
           'sizeof(lins_mapper_report), offsetof(lins_mapper_report, map), offsetof(lins_mapper_desc, n_corner));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "s"), os.path.join(d, "s.c")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [C.sizeof(defs.LinsMapperDesc), C.sizeof(defs.LinsMapperReport), defs.LinsMapperReport.map.offset,
                     defs.LinsMapperDesc.n_corner.offset]


def test_odometry_quaternion_round_trip():
    import mapper_drive

    rng = np.random.default_rng(5)
    for _ in range(100):
        T = rng.uniform([-0.5, -3.0, -0.5], [0.5, 3.0, 0.5])
        qx, qy, qz, qw = mapper_drive.odometry_quat(T)
        roll, pitch, yaw = mapperref.get_rpy(qz, -qx, -qy, qw)  # laserOdometryHandler :715-719
        assert np.allclose([-pitch, -yaw, roll], T, atol=1e-12)


def test_oracle_cycle_on_a_short_drive(synth, ob, defs):
    """The oracle alone: the first cycle keeps the map empty, later ones refine towards the truth and save key frames;
    interval-skipped messages change nothing but transformSum; memory follows the window."""
    import mapper_drive

    ev = mapper_drive.make_drive(synth, n_out=8, stall_at=-1)
    m = mapperref.MappingOracle(ob.MapOracle(), defs.POINT_DTYPE)
    reps = []
    for e in ev:
        if e[0] == "imu":
            m.imu(*e[1:])
        else:
            reps.append(m.step(*e[1:7]))
    done = [r for r in reps if r["processed"]]
    assert done[0]["map_skipped"] == 1 and done[0]["keyframe_saved"] == 1
    assert all(r["map_skipped"] == 0 for r in done[1:])
    assert sum(r["skipped_interval"] for r in reps) == sum(1 for e in ev if e[0] == "odom" and e[-1] == -1)
    assert len(m.poses) == sum(r["keyframe_saved"] for r in done) >= len(done) - 1  # (the turn moves only 0.3 m)
