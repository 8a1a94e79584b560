"""CPU suite for the global map: the restatement's radius search (tests/globalmapref.py) against scipy's k-d tree and a
plain loop; csrc/host/global_map.hpp compiled with g++ against the restatement on adversarial key poses; the PCD
writer and reader; the replay options refused before any device work."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

import globalmapref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
F = np.float32


def test_radius_selection_matches_kdtree_and_a_loop():
    rng = np.random.default_rng(1)
    poses = (rng.random((4000, 3)) * 1600 - 800).astype(F)
    for cur in (np.zeros(3, F), np.array([120.5, -3.0, 40.25], F), poses[17]):
        sel = globalmapref.select(poses, cur)
        d = np.linalg.norm(poses.astype(np.float64) - cur.astype(np.float64), axis=1)
        away = np.abs(d - 500.0) > 1e-2  # (away from the boundary, where f32 and f64 may disagree)
        tree = set(cKDTree(poses.astype(np.float64)).query_ball_point(cur.astype(np.float64), 500.0))
        assert set(sel[away[sel]]) == {i for i in tree if away[i]}
        loop = [i for i, p in enumerate(poses) if float(F(F(F(p[0] - cur[0]) ** 2 + F(p[1] - cur[1]) ** 2) + F(p[2] - cur[2]) ** 2)) < 250000.0]
        assert list(sel) == loop


DRIVER = r"""
#include <cstdio>
#include <vector>
#include "global_map.hpp"
struct P { float x, y, z; };
int main(int argc, char** argv) {
  FILE* f = std::fopen(argv[1], "rb");
  float cur[3]; int n;
  if (std::fread(cur, 4, 3, f) != 3 || std::fread(&n, 4, 1, f) != 1) return 2;
  std::vector<P> poses(n);
  if (n && std::fread(poses.data(), sizeof(P), n, f) != (size_t)n) return 2;
  const std::vector<int32_t> sel = lins_gm::select_key_poses(poses, cur);
  const std::vector<int32_t> ids = lins_gm::key_poses_ds(poses, sel);
  std::printf("%zu", sel.size());
  for (int32_t i : ids) std::printf(" %d", i);
  std::printf("\n");
  return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("gm")
    (d / "t.cpp").write_text(DRIVER)
    exe = str(d / "t")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", HOST, "-o", exe, str(d / "t.cpp")])
    return exe, d


def _run(driver, poses, cur):
    exe, d = driver
    path = d / "in.bin"
    with open(path, "wb") as f:
        f.write(np.asarray(cur, F).tobytes() + np.int32(len(poses)).tobytes() + np.asarray(poses, F).reshape(-1, 3).tobytes())
    out = [int(v) for v in subprocess.check_output([exe, str(path)]).split()]
    return out[0], out[1:]


def _check(driver, poses, cur):
    poses = np.asarray(poses, F).reshape(-1, 3)
    n, ids = _run(driver, poses, cur)
    sel, ref = globalmapref.key_frames(poses, cur)
    assert (n, ids) == (len(sel), list(ref))
    return sel, ref


def test_boundary_and_non_finite_poses(driver):
    r = np.float32(500.0)
    poses = [(r, 0, 0), (np.nextafter(r, F(0)), 0, 0), (0, 0, -r), (np.nan, 0, 0), (0, np.inf, 0), (-np.inf, 0, 0), (3, 4, 5)]
    sel, _ = _check(driver, poses, np.zeros(3, F))
    assert list(sel) == [1, 6]  # d^2 = 250000f exactly is excluded


def test_no_pose_in_range(driver):
    sel, ids = _check(driver, [(600, 0, 0), (0, -700, 0)], np.zeros(3, F))
    assert len(sel) == 0 and len(ids) == 0
    _check(driver, np.zeros((0, 3)), np.zeros(3, F))


def test_a_voxel_names_a_key_frame_it_does_not_hold_and_two_voxels_the_same(driver):
    poses = np.full((11, 3), np.nan, F)
    poses[0], poses[10] = (0.2, 0.3, 0.4), (0.7, 0.1, 0.9)  # voxel (0, 0, 0): the mean of 0 and 10 names 5
    poses[5] = (3.5, 0.5, 0.5)                             # voxel (3, 0, 0): 5 itself
    sel, ids = _check(driver, poses, np.zeros(3, F))
    assert list(sel) == [0, 5, 10] and list(ids) == [5, 5]


def test_f32_mean_rounds_up_across_an_integer(driver):
    """Many indices in one voxel, index x count far above 2^23: the f32 sum and division round, and the truncated f32
    mean names the key frame above the floor of the exact mean.  The index set is searched (seeded), then checked."""
    rng = np.random.default_rng(0)
    for _ in range(2000):
        c = int(rng.integers(2, 1500))
        idx = np.sort(rng.choice(np.arange(1000, 40000), c, replace=False))
        named = int(F(np.cumsum(idx.astype(F), dtype=F)[-1] / F(c)))  # (cumsum: sequential f32 sums)
        if named > int(idx.sum()) // c:
            break
    else:
        pytest.fail("no index set rounds up")
    poses = np.full((idx[-1] + 1, 3), np.nan, F)
    poses[idx] = (1.5, 2.5, 3.5)
    _, ids = _check(driver, poses, np.zeros(3, F))
    assert ids == [named]


def test_random_pose_sets(driver):
    rng = np.random.default_rng(5)
    for k in range(5):
        n = int(rng.integers(1, 3000))
        poses = (rng.random((n, 3)) * rng.choice([5.0, 60.0, 1200.0]) - 30).astype(F)
        _check(driver, poses, poses[int(rng.integers(0, n))])


def test_pcd_round_trip(tmp_path):
    pcd = importlib.import_module("lins---lidar-inertial-slam_b200.pcd")
    a = np.random.default_rng(2).standard_normal((37, 4)).astype(F)
    a[3, 1] = np.nan
    path = str(tmp_path / "m.pcd")
    pcd.write_pcd(path, a)
    head, b = pcd.read_pcd(path)
    assert head["FIELDS"] == ["x", "y", "z", "intensity"] and head["TYPE"] == ["F"] * 4 and head["SIZE"] == ["4"] * 4
    assert head["POINTS"] == ["37"] and head["WIDTH"] == ["37"] and head["HEIGHT"] == ["1"] and head["DATA"] == ["binary"]
    assert head["VERSION"] == ["0.7"]
    raw = open(path, "rb").read()
    assert raw.endswith(a.astype("<f4").tobytes())
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    pcd.write_pcd(path, np.zeros((0, 4), F))
    assert pcd.read_pcd(path)[1].shape == (0, 4)


def test_pass_budget_matches_header(defs):
    src = open(os.path.join(ROOT, "include", "lins_gpu.h")).read()
    assert "#define LINS_GLOBAL_MAP_PASS_POINTS (1 << 24)" in src and defs.GLOBAL_MAP_PASS_POINTS == 1 << 24


def test_replay_refuses_global_map_without_loops():
    br = importlib.import_module("lins---lidar-inertial-slam_b200.bag_replay")
    for kw in (dict(global_map=True), dict(map=True, global_map=True)):
        with pytest.raises(ValueError):
            br.replay([], 1, **kw)


@pytest.mark.parametrize("tool,args", [("run_bags.py", ["--map", "--global-map"]), ("run_bags.py", ["--global-map"]),
                                       ("run_bag.py", ["--map", "--global-map"]), ("run_bag.py", ["--global-map"])])
def test_tools_refuse_global_map_without_loops(tool, args, tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", tool), str(tmp_path / "none.bag")] + args,
                       capture_output=True, text=True)
    assert r.returncode == 2 and "--global-map" in r.stderr
