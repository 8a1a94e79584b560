"""CPU suite: sensor_msgs/PointCloud2 decoding for lins_gpu_decode_cloud2 / lins_gpu_seq_step_cloud2 (DESIGN.md §4.8).

- The per-field conversion (csrc/cuda/lins_cloud2.cuh, host branch) compiled with g++ equals (float)read_scalar(p, dt) of
  csrc/host/rosbag_reader.hpp on every datatype: integer extremes, uint32 above 2^24, doubles that round (halfway cases,
  overflow to inf, subnormal results), +-0, NaN, inf and subnormals.
- The C++ index (tools/synth/lins_bag.cpp) and the Python index (tools/bag_tool.py) give the same layouts and data ranges
  on messages bag_tool.encode_pointcloud2 writes in several layouts, and accept exactly the messages decode_pointcloud2
  accepts; every malformed layout is rejected by all three.
- The layout structs match the header.
"""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bag_tool  # noqa: E402
import cloud2cases as cc  # noqa: E402

PKG = os.path.join(ROOT, "lins---lidar-inertial-slam_b200")

DRIVER = r"""
#include <cstdio>
#include <cstring>
#include "lins_cloud2.cuh"
#include "rosbag_reader.hpp"
// stdin: records of (u8 datatype, 8 bytes); stdout: per record the bits of to_float(load_host) and of (float)read_scalar
int main() {
  unsigned char rec[9];
  while (std::fread(rec, 1, 9, stdin) == 9) {
    const float a = lins_cloud2::to_float(lins_cloud2::load_host(rec + 1, lins_cloud2::type_size(rec[0])), rec[0]);
    const float b = (float)lins::rosbag::read_scalar(rec + 1, rec[0]);
    std::fwrite(&a, 4, 1, stdout);
    std::fwrite(&b, 4, 1, stdout);
  }
  return 0;
}
"""


def test_conversion_equals_read_scalar(tmp_path):
    exe = tmp_path / "conv"
    src = tmp_path / "conv.cpp"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(PKG, "csrc", "cuda"), "-I", os.path.join(PKG, "csrc", "host"),
                           "-o", str(exe), str(src)])
    recs = cc.edge_vectors()
    out = subprocess.run([str(exe)], input=b"".join(recs), stdout=subprocess.PIPE, check=True).stdout
    got = np.frombuffer(out, np.uint32).reshape(-1, 2)
    assert len(got) == len(recs)
    fa, fb = got.view(np.float32)[:, 0], got.view(np.float32)[:, 1]
    nan = np.isnan(fa)
    assert np.array_equal(nan, np.isnan(fb))
    bad = [(recs[i][0], recs[i][1:].hex(), hex(got[i, 0]), hex(got[i, 1])) for i in np.flatnonzero(~nan & (got[:, 0] != got[:, 1]))]
    assert not bad, bad[:10]
    # the edges were reached: -0 kept, an overflow to inf, a subnormal result, a rounded uint32
    dts = np.array([r[0] for r in recs])
    assert ((got[:, 0] == 0x80000000) & (dts == 8)).any() and (np.isinf(fa) & (dts == 8)).any()
    assert ((np.abs(fa) < 1.1754942e-38) & (fa != 0) & (dts == 8)).any()
    assert nan[dts == 7].sum() == 3


@pytest.fixture(scope="module")
def baglib():
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tools", "synth"), "liblins_bag.so"])
    return cc.baglib()


def test_layout_struct_matches_header(defs):
    hdr = open(os.path.join(ROOT, "include", "lins_gpu.h")).read()
    assert "lins_cloud2_layout" in hdr and "/* 40 bytes */" in hdr
    assert C.sizeof(defs.LinsCloud2Layout) == 40 and defs.LinsCloud2Layout.datatype.offset == 32
    assert C.sizeof(defs.LinsCloud2Desc) == 32 and defs.LinsSeqCloud2Desc.cloud2.offset == 32


@pytest.mark.parametrize("name", list(cc.LAYOUTS))
def test_indexes_agree_on_every_layout(baglib, name):
    rng = np.random.default_rng(11)
    for n in (0, 1, 37, 240):
        if name == "organised" and n % 4:
            continue
        msg, _ = cc.message(name, cc.sweep(rng, n))
        py = bag_tool.index_pointcloud2(msg)
        cpp = cc.index_cpp(baglib, msg)
        assert py is not None and cpp is not None, (name, n)
        assert py == cpp, (name, n, py, cpp)
        # the host decoder takes it too, with width * height points
        assert len(cc.decode_cpp(baglib, msg)) == py["width"] * py["height"]


def test_indexes_write_a_bag_and_read_it_back(baglib, tmp_path):
    """Messages of every layout in one bag: the index of each message read back from the bag equals its index as written."""
    rng = np.random.default_rng(12)
    msgs = [cc.message(name, cc.sweep(rng, 40))[0] for name in cc.LAYOUTS]
    p = str(tmp_path / "layouts.bag")
    conns = {0: dict(topic="/velodyne_points", type="sensor_msgs/PointCloud2", md5sum="1158d486dd51d683ce2f1be655c3c181", message_definition="")}
    bag_tool.write_bag(p, conns, [(0, 100.0 + 0.1 * k, m) for k, m in enumerate(msgs)])
    _, back = bag_tool.read_bag(p)
    assert [bag_tool.index_pointcloud2(m) for _, _, m in back] == [cc.index_cpp(baglib, m) for m in msgs]


@pytest.mark.parametrize("case", list(cc.MALFORMED))
def test_malformed_rejected_by_all_three(baglib, case):
    msg = cc.malformed(case)
    assert bag_tool.index_pointcloud2(msg) is None, case
    assert cc.index_cpp(baglib, msg) is None, case
    assert cc.decode_cpp(baglib, msg) is None, case
