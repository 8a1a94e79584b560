"""Image projection on the CPU: the __host__ __device__ per-pixel code of csrc/cuda/lins_projection.cuh, compiled with g++,
against the host ImageProjection (csrc/host/image_projection.hpp) bit for bit on simulated sweeps — orientations, the range
image (row, column, range) and fullCloud's intensity, the ground test and the segmentation edge test — with NaN and
infinite points mixed in; the ctypes mirrors of the new C-ABI structs; and the labelling model the device runs (min-label
propagation) against labelComponents' sequential BFS on random range images and on scenes built to reach each case, and
against the segmented and outlier clouds of tests/pyfront.py's image_projection on range images it projects itself."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import projcases as pc
from conftest import ROOT

HOST = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
CUDA = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")

# the stages of ImageProjection are private: the driver opens them up to run them one by one
DRIVER = r'''
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <stddef.h>
#define private public
#include "image_projection.hpp"
#undef private
#include "lins_projection.cuh"
using namespace lins;
static bool same(float a, float b) { return std::memcmp(&a, &b, 4) == 0; }
int main(int argc, char** argv) {
  if (argc > 1 && std::strcmp(argv[1], "sizes") == 0) {
    std::printf("%zu %zu %zu %zu %zu\n", sizeof(lins_lidar_model), offsetof(lins_lidar_model, ground_scan_ind), sizeof(lins_raw_desc),
                offsetof(lins_raw_desc, cloud_off), offsetof(lins_raw_desc, point_format));
    return 0;
  }
  // the sweeps: n, L, S, ground_scan_ind (int32), ang_res_x, ang_res_y, ang_bottom (f32), n x 3 points
  FILE* f = std::fopen(argv[1], "rb");
  long bad_ori = 0, bad_rng = 0, bad_full = 0, bad_ground = 0, bad_edge = 0, n_pts = 0, n_pix = 0, n_ground = 0, n_edge = 0, n_edge_ok = 0, n_nan_ori = 0;
  int hdr[4];
  while (std::fread(hdr, 4, 4, f) == 4) {
    float res[3];
    if (std::fread(res, 4, 3, f) != 3) return 2;
    const int n = hdr[0];
    std::vector<float> xyz(3 * (size_t)n);
    if (std::fread(xyz.data(), 4, xyz.size(), f) != xyz.size()) return 2;
    LidarModel lm;
    lm.line_num = hdr[1]; lm.scan_num = hdr[2]; lm.ground_scan_ind = hdr[3];
    lm.ang_res_x = res[0]; lm.ang_res_y = res[1]; lm.ang_bottom = res[2];
    const int L = lm.line_num, S = lm.scan_num, P = L * S;
    Cloud in;
    for (int i = 0; i < n; ++i) in.push_back(makePoint(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], 7.f));
    ImageProjection ip(lm);
    ip.resetParameters();
    ip.findStartEndAngle(in);
    ip.projectPointCloud(in);
    ip.groundRemoval();
    if (n >= 2) {
      float o[3];
      lins_proj::start_end_angle(xyz[0], xyz[1], xyz[3 * (n - 1) + 1], xyz[3 * (n - 2)], o);
      const float h[3] = {ip.segMsg.startOrientation, ip.segMsg.endOrientation, ip.segMsg.orientationDiff};
      for (int k = 0; k < 3; ++k) {
        if (std::isnan(h[k])) { n_nan_ori += k == 0; if (!std::isnan(o[k])) ++bad_ori; }
        else if (!same(o[k], h[k])) ++bad_ori;
      }
    }
    // projectPointCloud: the last point of a pixel wins
    std::vector<int> idx(P, -1);
    for (int i = 0; i < n; ++i) {
      int r, c;
      if (lins_proj::project(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], L, S, lm.ang_res_x, lm.ang_res_y, lm.ang_bottom, r, c)) idx[r * S + c] = i;
    }
    std::vector<float> rng(P);
    for (int p = 0; p < P; ++p) {
      const int k = idx[p], r = p / S, c = p % S;
      rng[p] = k < 0 ? FLT_MAX : lins_proj::point_range(xyz[3 * k], xyz[3 * k + 1], xyz[3 * k + 2]);
      if (!same(rng[p], ip.rangeMat[p])) ++bad_rng;
      const PointType& q = ip.fullCloud.points[p];
      if (k < 0) { if (q.intensity != -1) ++bad_full; continue; }
      ++n_pix;
      if (!same(q.x, xyz[3 * k]) || !same(q.y, xyz[3 * k + 1]) || !same(q.z, xyz[3 * k + 2]) || !same(q.intensity, lins_proj::pixel_intensity(r, c))) ++bad_full;
    }
    n_pts += n;
    // groundRemoval: each column's rows in order
    std::vector<int8_t> g(P, 0);
    for (int j = 0; j < S; ++j)
      for (int i = 0; i < lm.ground_scan_ind; ++i) {
        const int lo = idx[i * S + j], up = idx[(i + 1) * S + j];
        if (lo < 0 || up < 0) { g[i * S + j] = -1; continue; }
        if (lins_proj::ground_pair(xyz[3 * lo], xyz[3 * lo + 1], xyz[3 * lo + 2], xyz[3 * up], xyz[3 * up + 1], xyz[3 * up + 2])) { g[i * S + j] = 1; g[(i + 1) * S + j] = 1; }
      }
    for (int p = 0; p < P; ++p) { if (g[p] != ip.groundMat[p]) ++bad_ground; n_ground += g[p] == 1; }
    // labelComponents' edge test, as the host writes it, on every right / jump / down pair of projected pixels
    const float aX = lm.ang_res_x / 180.0 * M_PI, aY = lm.ang_res_y / 180.0 * M_PI;
    const float ax = lins_proj::segment_alpha(lm.ang_res_x), ay = lins_proj::segment_alpha(lm.ang_res_y);
    if (!same(ax, aX) || !same(ay, aY)) ++bad_edge;
    for (int p = 0; p < P; ++p) {
      if (rng[p] == FLT_MAX) continue;
      const int r = p / S, c = p % S;
      const int t[3] = {r * S + (c + 1 < S ? c + 1 : 0), r * S + (c + 255 < S ? c + 255 : 0), r + 1 < L ? p + S : -1};
      for (int k = 0; k < 3; ++k) {
        if (t[k] < 0 || rng[t[k]] == FLT_MAX) continue;
        const float alpha = k < 2 ? aX : aY;
        const float d1 = std::max(rng[p], rng[t[k]]), d2 = std::min(rng[p], rng[t[k]]);
        const bool host = std::atan2(d2 * std::sin(alpha), (d1 - d2 * std::cos(alpha))) > 1.0472f;
        const bool dev = lins_proj::edge(rng[p], rng[t[k]], std::sin(k < 2 ? ax : ay), std::cos(k < 2 ? ax : ay));
        bad_edge += host != dev;
        ++n_edge;
        n_edge_ok += host;
      }
    }
  }
  std::printf("%ld %ld %ld %ld %ld %ld %ld %ld %ld %ld %ld\n", bad_ori, bad_rng, bad_full, bad_ground, bad_edge, n_pts, n_pix, n_ground, n_edge,
              n_edge_ok, n_nan_ori);
  return 0;
}
'''


def _driver(tmp_path):
    src, exe = tmp_path / "proj_check.cpp", tmp_path / "proj_check"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I", HOST, "-I", CUDA, "-o", str(exe), str(src)])
    return str(exe)


def test_struct_mirrors_match_header(tmp_path, defs):
    out = subprocess.check_output([_driver(tmp_path), "sizes"]).split()
    lm, gsi_off, raw, off_off, pf_off = (int(v) for v in out)
    assert C.sizeof(defs.LinsLidarModel) == lm == 24 and defs.LinsLidarModel.ground_scan_ind.offset == gsi_off
    assert C.sizeof(defs.LinsRawDesc) == raw and defs.LinsRawDesc.cloud_off.offset == off_off and defs.LinsRawDesc.point_format.offset == pf_off
    v, d = defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()
    f = np.float32
    assert (v.line_num, v.scan_num, v.ground_scan_ind, d.line_num, d.scan_num, d.ground_scan_ind) == (16, 1800, 5, 64, 1024, 24)
    assert f(v.ang_bottom) == f(15.0) + f(0.1) and f(d.ang_res_y) == f(45.0) / f(63.0) and f(d.ang_bottom) == f(22.5) + f(0.1)


def _with_non_finite(raw, seed, first_last=False):
    """The sweep with NaN no-returns and +-inf coordinates mixed in (and, if asked, NaN first and last points)."""
    xyz = np.stack([raw["x"], raw["y"], raw["z"]], 1).astype(np.float32)
    rng = np.random.default_rng(seed)
    k = rng.choice(len(xyz), len(xyz) // 20, replace=False)
    xyz[k[: len(k) // 2]] = np.nan
    for j, i in enumerate(k[len(k) // 2:]):
        xyz[i, j % 3] = np.inf if j % 2 else -np.inf
    if first_last:
        xyz[0] = np.nan
        xyz[-1] = np.nan
    return xyz


def test_per_pixel_code_matches_host_projection(tmp_path, synth, defs):
    path = tmp_path / "sweeps.bin"
    with open(path, "wb") as f:
        for config, seeds in (("config3", (11, 12, 13)), ("config1", (21, 22)), ("config4", (31, 32))):
            for seed in seeds:
                raw, m = pc.raw_sweep(synth, defs, config, seed)
                xyz = np.stack([raw["x"], raw["y"], raw["z"]], 1).astype(np.float32)
                variants = [xyz] + ([_with_non_finite(raw, seed, first_last=seed % 2 == 1)] if seed in (11, 12, 21, 31) else [])
                for v in variants:
                    f.write(np.array([len(v), m.line_num, m.scan_num, m.ground_scan_ind], np.int32).tobytes())
                    f.write(np.array([m.ang_res_x, m.ang_res_y, m.ang_bottom], np.float32).tobytes())
                    f.write(np.ascontiguousarray(v, np.float32).tobytes())
    out = subprocess.check_output([_driver(tmp_path), str(path)]).split()
    bad_ori, bad_rng, bad_full, bad_ground, bad_edge, n_pts, n_pix, n_ground, n_edge, n_edge_ok, n_nan_ori = (int(v) for v in out)
    assert n_pts > 200000 and n_pix > 100000 and n_ground > 10000 and n_edge > 100000 and 0 < n_edge_ok < n_edge and n_nan_ori >= 2
    assert (bad_ori, bad_rng, bad_full, bad_ground, bad_edge) == (0, 0, 0, 0, 0)


def _same_labelling(blocked, E):
    o1, f1 = pc.bfs_owners(blocked, E)
    o2, f2, rounds = pc.min_label_owners(blocked, E)
    assert np.array_equal(o1, o2)
    assert f1 == f2
    return o1, f1, rounds


@pytest.mark.parametrize("L,S", [(1, 40), (3, 200), (5, 255), (4, 256), (6, 300), (16, 1800), (64, 1024), (128, 300), (2, 2048)])
def test_min_label_model_equals_bfs_on_random_images(L, S):
    rng = np.random.default_rng(L * 10007 + S)
    reps = 3 if L * S <= 40000 else 1
    for k in range(reps):
        blocked, E = pc.random_graph(rng, L, S, p_block=(0.1, 0.3, 0.5)[k % 3], p_edge=(0.7, 0.5, 0.9)[k % 3])
        owner, feasible, rounds = _same_labelling(blocked, E)
        assert len(feasible) > 1


def _pyfront_pixels(out, key):
    """(row, col) pixels of pyfront.image_projection's segmented or outlier cloud (intensity = row + col / 10000)."""
    pts = out[key]
    rows = np.floor(pts[:, 3]).astype(np.int64)
    cols = out["col"].astype(np.int64) if key == "seg" else np.rint((pts[:, 3].astype(np.float64) - rows) * 10000).astype(np.int64)
    return set(zip(rows.tolist(), cols.tolist()))


@pytest.mark.parametrize("L,S,seed", [(5, 100, 1), (8, 300, 2), (6, 300, 3), (16, 1800, 4)])
def test_min_label_model_predicts_pyfront_segmentation(L, S, seed):
    """The model's owners and feasibility, through cloudSegmentation's rules, give the pixels of the segmented and
    outlier clouds that tests/pyfront.py (its own labelComponents BFS on real points) produces.  The range images hold
    two range levels (5 m and 20 m: equal ranges pass the edge test, the two levels never do) and empty pixels, with
    ground_scan_ind 0 (no ground)."""
    import types

    import pyfront
    rng = np.random.default_rng(seed)
    lv = rng.random((L, S))
    img = np.where(lv < 0.45, 5.0, np.where(lv < 0.75, 20.0, np.nan))
    m = types.SimpleNamespace(ang_res_x=np.float32(360.0) / np.float32(S), ang_res_y=np.float32(2.0), ang_bottom=np.float32(15.1))
    out = pyfront.image_projection(pc.image_points(m, img), lm=pyfront.Lidar(line_num=L, scan_num=S, ang_res_x=m.ang_res_x,
                                                                              ang_res_y=2.0, ang_bottom=15.1, ground_scan_ind=0))
    blocked, E = pc.scene_graph(img)
    owner, feasible, _ = _same_labelling(blocked, E)
    seg, outl = set(), set()
    for r, c in zip(*np.nonzero(~blocked)):
        if feasible[int(owner[r, c])]:
            seg.add((int(r), int(c)))
        elif r > 0 and c % 5 == 0:
            outl.add((int(r), int(c)))
    assert len(seg) > 0 and len(outl) > 0
    assert _pyfront_pixels(out, "seg") == seg
    assert _pyfront_pixels(out, "outlier") == outl


def test_scenes_reach_their_condition():
    got = {}
    for name in pc.SCENES:
        img, _ = pc.scene(name)
        blocked, E = pc.scene_graph(img)
        owner, feasible, _ = _same_labelling(blocked, E)
        got[name] = (img.shape[1], owner, feasible)
    S, o, f = got["earlier_seed_blocks"]
    assert o[1, 5] == 0 * S + 5 and o[1, 4] == 1 * S + 3  # (1, 5) belongs to the earlier seed (0, 5)
    E_row = pc.scene_graph(pc.scene("earlier_seed_blocks")[0])[1][0]
    assert E_row[1, 4]  # ... though the later seed (1, 3) has an edge into it
    S, o, f = got["wrap"]
    assert o[1, 0] == o[1, 1] == S - 1  # reached from (0, S - 1) through the wrap
    S, o, f = got["jump_in_row"]
    assert o[1, 265] == o[2, 269] == 1 * S + 10  # (1, 10) -> (1, 265): the +255 jump inside a 300-column row
    assert got["size30"][2][1 * 80 + 10] and not got["size29"][2][1 * 80 + 10]
    assert got["five_three_rows"][2][0] and not got["five_seed_row_only"][2][7]
