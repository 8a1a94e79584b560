"""CPU suite: per-slot estimator tuning (lins_slot_tuning, lins_gpu_seq_tune) at the C-ABI boundary and in the host
helpers: the struct's layout against the header, LinsSlotTuning.shipped, rig_config.load_config / slot_tuning,
tools/run_bags.py --tune, and the alignIMUtoVehicle expression against scipy and the shim's host function."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, pkg
from test_slot_config_cpu import _yaml


def test_slot_tuning_layout_matches_header(defs):
    fields = ("num_iter", "icp_freq", "nearest_feature_search_sq_dist", "lidar_std", "lidar_scale", "imu_misalign_angle")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "lins_gpu.h"\nint main(){printf("%zu'
           + " %zu" * len(fields) + '\\n", sizeof(lins_slot_tuning)'
           + "".join(f", offsetof(lins_slot_tuning, {f})" for f in fields) + ");return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "s"), os.path.join(d, "s.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    T = defs.LinsSlotTuning
    assert got == [C.sizeof(T)] + [getattr(T, f).offset for f in fields]
    assert C.sizeof(T) == 2 * 4 + 4 * 8
    assert "lins_gpu_seq_tune" in pkg("capi").EXPORTS


def test_shipped_slot_tuning_is_exp_port(defs):
    t = defs.LinsSlotTuning.shipped()
    p = defs.LinsParams.shipped()
    for k in ("num_iter", "icp_freq", "nearest_feature_search_sq_dist", "lidar_std", "lidar_scale"):
        assert getattr(t, k) == getattr(p, k), k
    assert t.imu_misalign_angle == 3.0
    o = defs.LinsSlotTuning.shipped(num_iter=12, imu_misalign_angle=-2.5)
    assert (o.num_iter, o.icp_freq, o.imu_misalign_angle) == (12, 1, -2.5)
    with pytest.raises(TypeError):
        defs.LinsSlotTuning.shipped(scan_period=0.05)  # (a rig value: lins_slot_config)


def test_load_config_gives_rig_and_tuning(defs, tmp_path, recwarn):
    rc = pkg("rig_config")
    p = _yaml(tmp_path, "a.yaml", misalign=3.0, num_iter=12)
    rig, tuning = rc.load_config(p)
    assert not [w for w in recwarn.list if "imu_misalign_angle" in str(w.message)]  # (applied now: no warning)
    assert rig == rc.load_rig(_yaml(tmp_path, "b.yaml", num_iter=12))[0]
    assert tuning == dict(num_iter=12, icp_freq=1, nearest_feature_search_sq_dist=25, lidar_std=0.01, lidar_scale=1, imu_misalign_angle=3.0)
    t = rc.slot_tuning(tuning)
    assert bytes(t) == bytes(defs.LinsSlotTuning.shipped(num_iter=12))
    with pytest.warns(UserWarning, match="imu_misalign_angle"):  # load_rig is unchanged
        rc.load_rig(p)
    with pytest.raises(ValueError, match="imu_misalign_angle"):
        rc.load_config(_yaml(tmp_path, "c.yaml", drop="imu_misalign_angle"))
    with pytest.raises(ValueError, match="num_iter"):
        rc.load_config(_yaml(tmp_path, "d.yaml", drop="num_iter"))


def _run_bags():
    import importlib.util
    spec = importlib.util.spec_from_file_location("run_bags", os.path.join(ROOT, "tools", "run_bags.py"))
    rb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rb)
    return rb


def test_run_bags_tune_accepts_files_that_disagree(defs, tmp_path, capsys):
    rb = _run_bags()
    a, b = _yaml(tmp_path, "a.yaml", misalign=3.0), _yaml(tmp_path, "b.yaml", period=0.1, extr=0.0, num_iter=10, misalign=-1.0)
    bags = [os.path.join(GOLDEN, "tiny.bag")] * 3
    prm, cfgs, tunes = rb.bag_tunings(f"{a},{b},{a}", 3)  # num_iter and the misalignment differ
    assert [x.scan_period for x in cfgs] == [0.05, 0.1, 0.05]
    assert [t.num_iter for t in tunes] == [30, 10, 30] and [t.imu_misalign_angle for t in tunes] == [3.0, -1.0, 3.0]
    assert prm.num_iter == 30
    prm, cfgs, tunes = rb.bag_tunings(b, 3)
    assert len(tunes) == 3 and all(bytes(t) == bytes(tunes[0]) for t in tunes) and prm.num_iter == 10
    with pytest.raises(SystemExit):
        rb.main(bags + ["--tune"])  # --tune without --config
    assert "--config" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        rb.main(bags + ["--config", f"{a},{b}", "--tune"])
    assert "2 files for 3 bags" in capsys.readouterr().err
    with pytest.raises(SystemExit):  # without --tune the files must still agree
        rb.main(bags + ["--config", f"{a},{b},{a}"])
    assert "num_iter" in capsys.readouterr().err


ANGLES = (0.0, 3.0, -2.5, 0.1, 45.0, -179.0, 1e-7)


def _vectors():
    rng = np.random.default_rng(7)
    v = [rng.normal(size=3) * s for s in (1e-3, 0.1, 9.81, 300.0) for _ in range(50)]
    return v + [np.array([0.0, 0.0, 9.81]), np.array([1.0, -0.0, 0.0])]


def test_alignment_matches_scipy_within_an_ulp():
    from scipy.spatial.transform import Rotation
    rc = pkg("rig_config")
    for a in ANGLES:
        R = rc.misalign_R(a)
        Rs = Rotation.from_euler("ZYX", [a, 0.0, 0.0], degrees=True).as_matrix()  # Rz(yaw) Ry(0) Rx(0)
        assert np.all(np.abs(np.array(R) - Rs) <= np.spacing(np.abs(Rs)) + 1e-300), a
        assert R[2] == (0.0, 0.0, 1.0) and R[0][2] == 0.0 and R[1][2] == 0.0
        for v in _vectors():
            got = np.array(rc.align_imu(R, v))
            want = Rs.T @ v
            tol = 2 * np.spacing(np.max(np.abs(v)))  # (two products and a sum, each within half an ulp of the exact)
            assert np.all(np.abs(got - want) <= tol), (a, v, got, want)
    # a zero angle is the identity on the values (the product is applied all the same)
    v = np.array([0.25, -3.5, 9.81])
    assert rc.align_imu(rc.misalign_R(0.0), v) == tuple(v)
    # the rotation is the yaw the config names: +90 degrees maps the vehicle x axis onto R^T x = (cos, -sin, 0)
    assert np.allclose(rc.align_imu(rc.misalign_R(90.0), (1.0, 0.0, 0.0)), (0.0, -1.0, 0.0), atol=1e-15)
    assert math.isclose(rc.misalign_R(30.0)[1][0], 0.5, rel_tol=1e-15)


def test_alignment_is_bit_equal_to_the_shim():
    rc, synth = pkg("rig_config"), pkg("synth")
    for a in ANGLES:
        R = rc.misalign_R(a)
        for v in _vectors():
            assert np.array(rc.align_imu(R, v)).tobytes() == synth.host_align_imu(a, v).tobytes(), (a, v)
