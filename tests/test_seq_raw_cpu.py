"""Sequence mode from the raw sweep on the CPU: the C-ABI struct of lins_gpu_seq_step_raw and its ctypes mirror, and the
host reference of a raw log (copyPointCloud's NaN removal in numpy, a fresh host ImageProjection per sweep) against the
pcl log the simulator makes of the same drive."""
import ctypes as C
import os
import subprocess

import numpy as np

import featcases as fc
import projcases as pj
import rawcases as rc
from conftest import ROOT, pkg

SIZES = r'''
#include <cstdio>
#include <stddef.h>
#include "lins_gpu.h"
int main() {
  std::printf("%zu %zu %zu %zu\n", sizeof(lins_seq_raw_desc), offsetof(lins_seq_raw_desc, present), offsetof(lins_seq_raw_desc, imu_off),
              offsetof(lins_seq_raw_desc, raw));
  return 0;
}
'''


def test_struct_mirrors_the_header(defs, tmp_path):
    src, exe = tmp_path / "sizes.cpp", tmp_path / "sizes"
    src.write_text(SIZES)
    subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    T = defs.LinsSeqRawDesc
    assert got == [C.sizeof(T), T.present.offset, T.imu_off.offset, T.raw.offset]


def test_symbol_is_declared_and_bound(defs):
    capi = pkg("capi")
    with open(os.path.join(ROOT, "include", "lins_gpu.h")) as f:
        header = f.read()
    assert "int lins_gpu_seq_step_raw(lins_ctx* ctx, const lins_seq_raw_desc* step" in header
    assert "lins_gpu_seq_step_raw" in capi.EXPORTS
    assert [n for n, _ in defs.LinsSeqRawDesc._fields_] == ["n_seq", "present", "imu", "imu_off", "raw"]
    assert defs.LinsSeqRawDesc._fields_[-1][1] is defs.LinsRawDesc
    if os.path.exists(capi.LIB_PATH):  # (build() made it)
        assert C.CDLL(capi.LIB_PATH).lins_gpu_seq_step_raw is not None


def _same_scan(a, b):
    for k in ("seg", "range", "ori"):
        assert fc.same_bits(np.asarray(a[k], np.float32), np.asarray(b[k], np.float32)), k
    for k in ("ground", "col", "start_ring", "end_ring"):
        assert np.array_equal(a[k], b[k]), k


def test_host_projected_raw_log_is_the_pcl_log(defs, synth):
    """The host reference of a raw log equals synth.pcl_log of the same drive and seed, scan for scan, bit for bit."""
    for config, seed, n in (("config3", 7, 4), ("config4", 8, 2)):
        raw, pcl = synth.raw_log(config, seed=seed, n_scans=n), synth.pcl_log(config, seed=seed, n_scans=n)
        assert raw["line_num"] == pcl["line_num"] and len(raw["sweeps"]) == n
        for k in ("time", "imu", "imu_off", "imu_last"):
            assert np.array_equal(raw[k], pcl[k]), k
        mine = rc.pcl_of(defs, raw)
        for a, b in zip(mine["scans"], pcl["scans"]):
            _same_scan(a, b)


def test_numpy_removal_agrees_on_finite_sweeps(defs, synth):
    """Sweeps without non-finite points: the removal keeps every point, and the host projection of what it keeps equals
    lins_projection_host on the sweep itself."""
    for config, seed in (("config3", 11), ("config1", 12), ("config4", 13)):
        raw, model = pj.raw_sweep(synth, defs, config, seed)
        xyzi = np.stack([raw["x"], raw["y"], raw["z"], raw["intensity"]], 1).astype(np.float32)
        assert np.isfinite(xyzi).all()
        kept = rc.finite(xyzi)
        assert kept.tobytes() == xyzi.tobytes()
        _same_scan(rc.host_scan(defs, xyzi, model), pj.host_projection(defs, raw, model))
    # and on a sweep with non-finite points it drops exactly those, keeping the order
    a = xyzi.copy()
    a[[0, 5, len(a) - 1], [0, 2, 1]] = [np.nan, np.inf, -np.inf]
    a[7, 3] = np.nan  # (intensity is not tested)
    kept = rc.finite(a)
    assert len(kept) == len(a) - 3 and np.array_equal(kept[:, :3], np.delete(a, [0, 5, len(a) - 1], 0)[:, :3])
