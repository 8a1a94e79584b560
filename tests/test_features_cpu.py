"""Feature extraction on the CPU: the __host__ __device__ per-point code of csrc/cuda/lins_features.cuh, compiled with g++,
against the host FeatureExtractor (csrc/host/feature_extraction.hpp) bit for bit on simulated sweeps — stamps, curvatures,
occlusion flags, voxel keys and centroids — and its atan2f against glibc's; the ctypes mirrors of the new C-ABI structs."""
import ctypes as C
import os
import subprocess

import numpy as np

import featcases as fc
from conftest import ROOT

HOST = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
CUDA = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")

# the stages of FeatureExtractor are private: the driver opens them up to call them one by one
DRIVER = r'''
#include <cstdio>
#include <cstring>
#include <random>
#include <stddef.h>
#define private public
#include "feature_extraction.hpp"
#undef private
#include "lins_features.cuh"
using namespace lins;
static bool same(float a, float b) { return std::memcmp(&a, &b, 4) == 0; }
int main(int argc, char** argv) {
  if (argc > 1 && std::strcmp(argv[1], "sizes") == 0) {
    std::printf("%zu %zu %zu %zu %zu %zu\n", sizeof(lins_feature_params), sizeof(lins_pcl_desc), offsetof(lins_pcl_desc, point_format),
                sizeof(lins_seq_pcl_desc), offsetof(lins_seq_pcl_desc, pcl), (size_t)LINS_FEAT_RING_CAP);
    return 0;
  }
  // atan2f: the fdlibm restatement against glibc on random normal inputs of lidar-like and wide magnitudes
  std::mt19937_64 rng(7);
  long bad_atan = 0, n_atan = 0;
  for (int i = 0; i < 3000000; ++i) {
    const double sc = (i % 3 == 0) ? 1e-3 : (i % 3 == 1 ? 100.0 : 1e6);
    const float y = (float)(std::uniform_real_distribution<double>(-1, 1)(rng) * sc);
    const float x = (float)(std::uniform_real_distribution<double>(-1, 1)(rng) * sc);
    ++n_atan;
    if (!same(std::atan2(y, x), lins_feat::atan2f_fdlibm(y, x))) ++bad_atan;
  }
  // the scans: n, line_num, seg (n x 4), range, col, ground, start, end, ori (3)
  FILE* f = std::fopen(argv[1], "rb");
  long bad_stamp = 0, bad_curv = 0, bad_occ = 0, bad_vox = 0, n_pts = 0, n_vox = 0, n_half = 0, n_occ = 0;
  int n, L;
  while (std::fread(&n, 4, 1, f) == 1) {
    if (std::fread(&L, 4, 1, f) != 1) return 2;
    std::vector<float> seg(4 * (size_t)n), rng_(n), ori(3);
    std::vector<uint32_t> col(n);
    std::vector<uint8_t> ground(n);
    std::vector<int32_t> sr(L), er(L);
    bool ok = std::fread(seg.data(), 4, seg.size(), f) == seg.size() && std::fread(rng_.data(), 4, n, f) == (size_t)n &&
              std::fread(col.data(), 4, n, f) == (size_t)n && std::fread(ground.data(), 1, n, f) == (size_t)n &&
              std::fread(sr.data(), 4, L, f) == (size_t)L && std::fread(er.data(), 4, L, f) == (size_t)L && std::fread(ori.data(), 4, 3, f) == 3;
    if (!ok) return 2;
    LidarModel lm; lm.line_num = L;
    Cloud in;
    for (int i = 0; i < n; ++i) in.push_back(makePoint(seg[4 * i], seg[4 * i + 1], seg[4 * i + 2], seg[4 * i + 3]));
    CloudInfo info;
    info.resize(L, n);
    info.startRingIndex = sr; info.endRingIndex = er;
    info.startOrientation = ori[0]; info.endOrientation = ori[1]; info.orientationDiff = ori[2];
    info.segmentedCloudRange = rng_; info.segmentedCloudColInd = col; info.segmentedCloudGroundFlag = ground;
    for (double angle : {0.0, 11.25}) {
      FeatureParams fp; fp.imu_lidar_extrinsic_angle = angle;
      FeatureExtractor fe(lm, fp);
      const size_t cap = std::max<size_t>((size_t)lm.line_num * lm.scan_num, in.size() + 16);
      fe.cloudCurvature_.assign(cap, 0.0); fe.cloudSmoothness_.assign(cap, Smooth());
      fe.cloudNeighborPicked_.assign(cap, 0); fe.cloudLabel_.assign(cap, 0);
      Cloud und;
      fe.undistortPcl(in, info, und);
      fe.calculateSmoothness(und, info);
      fe.markOccludedPoints(und, info);
      const double y = angle * M_PI / 180.0, c = std::cos(y), s = std::sin(y);
      int half = n;
      for (int i = 0; i < n; ++i) {
        float x2, y2; bool flips;
        lins_feat::rotate_xy(c, s, seg[4 * i], seg[4 * i + 1], x2, y2);
        lins_feat::ori_not_passed(x2, y2, ori[0], flips);
        if (flips) { half = i; break; }
      }
      n_half += half < n;
      std::vector<int> occ(n, 0);
      for (int i = 5; i < n - 6; ++i) {
        const int m = lins_feat::occlusion_marks(&rng_[i - 1], &col[i - 1]);
        if (m & 1) for (int k = -5; k <= 0; ++k) occ[i + k] = 1;
        if (m & 2) for (int k = 1; k <= 6; ++k) occ[i + k] = 1;
        if (m & 4) occ[i] = 1;
      }
      for (int i = 0; i < n; ++i) {
        float x2, y2; bool flips;
        lins_feat::rotate_xy(c, s, seg[4 * i], seg[4 * i + 1], x2, y2);
        const double o = i <= half ? lins_feat::ori_not_passed(x2, y2, ori[0], flips) : lins_feat::ori_passed(x2, y2, ori[1]);
        const float st = lins_feat::stamp(seg[4 * i + 3], o, ori[0], ori[2], lm.scan_period);
        if (!same(st, und.points[i].intensity) || !same(x2, und.points[i].x) || !same(y2, und.points[i].y)) ++bad_stamp;
        const double cv = (i >= 5 && i < n - 5) ? lins_feat::curvature(&rng_[i - 5]) : 0.0;
        if (std::memcmp(&cv, &fe.cloudCurvature_[i], 8) != 0) ++bad_curv;
        if (occ[i] != fe.cloudNeighborPicked_[i]) ++bad_occ;
        n_occ += occ[i];
      }
      n_pts += n;
      // VoxelGrid of every ring's de-skewed points: keys + stable sort + f32 centroids against VoxelGrid::filter
      for (int r = 0; r < L; ++r) {
        Cloud ringc, ref;
        for (int k = std::max(0, sr[r]); k < std::min(n, er[r]); ++k) ringc.push_back(und.points[k]);
        fe.downSizeFilter_.filter(ringc, ref);
        if (ringc.size() == 0) continue;
        float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
        for (auto& p : ringc.points) { const float v[3] = {p.x, p.y, p.z}; for (int d = 0; d < 3; ++d) { mn[d] = fminf(mn[d], v[d]); mx[d] = fmaxf(mx[d], v[d]); } }
        int min_b[3], div[3];
        for (int d = 0; d < 3; ++d) { min_b[d] = lins_feat::voxel_bound(mn[d]); div[d] = lins_feat::voxel_bound(mx[d]) - min_b[d] + 1; }
        const int mul[3] = {1, div[0], div[0] * div[1]};
        std::vector<std::pair<uint32_t, int>> kv;
        for (int k = 0; k < (int)ringc.size(); ++k) kv.emplace_back(lins_feat::voxel_key(ringc.points[k].x, ringc.points[k].y, ringc.points[k].z, min_b, mul), k);
        std::stable_sort(kv.begin(), kv.end(), [](const std::pair<uint32_t, int>& a, const std::pair<uint32_t, int>& b) { return a.first < b.first; });
        size_t v = 0;
        for (size_t a = 0; a < kv.size();) {
          size_t b = a;
          float cx = 0, cy = 0, cz = 0, ci = 0;
          for (; b < kv.size() && kv[b].first == kv[a].first; ++b) { const auto& p = ringc.points[kv[b].second]; cx += p.x; cy += p.y; cz += p.z; ci += p.intensity; }
          const float cnt = (float)(b - a);
          if (v >= ref.size() || !same(cx / cnt, ref.points[v].x) || !same(cy / cnt, ref.points[v].y) || !same(cz / cnt, ref.points[v].z) ||
              !same(ci / cnt, ref.points[v].intensity)) ++bad_vox;
          ++v; a = b;
        }
        if (v != ref.size()) ++bad_vox;
        n_vox += v;
      }
    }
  }
  std::printf("%ld %ld %ld %ld %ld %ld %ld %ld %ld %ld\n", bad_atan, n_atan, bad_stamp, bad_curv, bad_occ, bad_vox, n_pts, n_vox, n_half, n_occ);
  return 0;
}
'''


def _driver(tmp_path):
    src, exe = tmp_path / "feat_check.cpp", tmp_path / "feat_check"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I", HOST, "-I", CUDA, "-o", str(exe), str(src)])
    return str(exe)


def test_struct_mirrors_match_header(tmp_path, defs):
    out = subprocess.check_output([_driver(tmp_path), "sizes"]).split()
    fp, pcl, pf_off, seq, seq_pcl_off, cap = (int(v) for v in out)
    assert C.sizeof(defs.LinsFeatureParams) == fp == 24
    assert C.sizeof(defs.LinsPclDesc) == pcl and defs.LinsPclDesc.point_format.offset == pf_off
    assert C.sizeof(defs.LinsSeqPclDesc) == seq and defs.LinsSeqPclDesc.pcl.offset == seq_pcl_off
    assert defs.FEAT_RING_CAP == cap
    p = defs.LinsFeatureParams.shipped()
    assert (p.edge_threshold, p.surf_threshold, p.imu_lidar_extrinsic_angle) == (0.5, 0.5, 0.0)


def test_per_point_code_matches_host_extractor(tmp_path, synth, defs):
    path = tmp_path / "scans.bin"
    with open(path, "wb") as f:
        for config, seeds in (("config3", (11, 12, 13)), ("config1", (21, 22)), ("config4", (31, 32))):
            for seed in seeds:
                s, ln = fc.segmented(synth, defs, config, seed)
                f.write(np.array([len(s["seg"]), ln], np.int32).tobytes())
                for k, t in (("seg", np.float32), ("range", np.float32), ("col", np.uint32), ("ground", np.uint8), ("start_ring", np.int32),
                             ("end_ring", np.int32), ("ori", np.float32)):
                    f.write(np.ascontiguousarray(s[k], t).tobytes())
    out = subprocess.check_output([_driver(tmp_path), str(path)]).split()
    bad_atan, n_atan, bad_stamp, bad_curv, bad_occ, bad_vox, n_pts, n_vox, n_half, n_occ = (int(v) for v in out)
    assert n_atan == 3000000 and bad_atan == 0
    assert n_pts > 100000 and n_vox > 10000 and n_half > 0 and n_occ > 1000
    assert (bad_stamp, bad_curv, bad_occ, bad_vox) == (0, 0, 0, 0)


def test_scenes_reach_their_condition():
    """The hand-built scans of tests/test_gpu_features.py, checked with pyfront on the host."""
    import featmut
    import pyfront
    import test_gpu_features as t

    s, _ = t._scene("many_corners")
    ref = pyfront.extract_features(s["seg"], s, lm=pyfront.Lidar(line_num=1))
    assert len(ref["less_sharp"]) == 120  # 20 picks in each of the 6 sextants (37 candidates each)
    s, _ = t._scene("ring0_default_entry")
    ref = pyfront.extract_features(s["seg"], s, lm=pyfront.Lidar(line_num=2))
    assert s["ground"][0] == 1 and any(fc.same_bits(p[:3], s["seg"][0, :3]) for p in ref["flat"])
    s, _ = t._scene("wrap_half_passed")
    o = -np.arctan2(s["seg"][:, 1].astype(np.float64), s["seg"][:, 0])
    assert (o > 0).any() and (o < 0).any() and (np.abs(np.diff(o)) > np.pi).any()  # the orientations wrap through +-pi
    ref = pyfront.extract_features(s["seg"], s, lm=pyfront.Lidar(line_num=2))
    assert (ref["undist"][:, 3] % 1 > 0.05).any()  # the late half of the sweep is stamped past half a period
    s, _ = t._scene("abutting_rings")
    assert s["start_ring"][1] == s["end_ring"][0] and s["start_ring"][2] == s["end_ring"][1]
    # suppression really crosses the ring boundary: clipping it to the ring changes the clouds
    assert featmut.differs(featmut.select(s["seg"], s, 3), featmut.select(s["seg"], s, 3, clip_to_ring=True))
    s, _ = t._scene("fourth_flat")
    # the 4th flat point's missing suppression decides a later pick
    assert featmut.differs(featmut.select(s["seg"], s, 1), featmut.select(s["seg"], s, 1, suppress_fourth=True))
    for name in ("column_jump", "many_corners"):
        s, _ = t._scene(name)
        ref = pyfront.extract_features(s["seg"], s, lm=pyfront.Lidar(line_num=len(s["start_ring"])))
        assert not featmut.differs(featmut.select(s["seg"], s, len(s["start_ring"])),
                                   {k: ref[k] for k in ("sharp", "less_sharp", "flat", "less_flat")})  # the variants' base is pyfront
    s, _ = t._scene("column_jump")
    assert (np.abs(np.diff(s["col"].astype(np.int64))) > 10).sum() > 50
    # the constant-range ring: ties decide its flat picks (std::sort's order there is unspecified)
    rows = fc.sweep_ring(600, 6.0, -1.2, ground=1)
    scan = fc.ring_scan([rows, fc.sweep_ring(600, 9.0, 0.4, ground=0, bumps=[(k, 0.1) for k in range(7, 600, 10)])])
    ref = pyfront.extract_features(scan["seg"], scan, lm=pyfront.Lidar(line_num=2))
    assert ref["sort_ties"] > 500 and len(ref["flat"]) == 24
