"""CPU suite: per-slot rig configuration (lins_slot_config, lins_gpu_seq_configure) at the C-ABI boundary and in the host
helpers: the struct's layout against the header, LinsSlotConfig.shipped, and bag_replay.Recording's scan period rule."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

from conftest import GOLDEN, ROOT, pkg


def test_slot_config_layout_matches_header(defs):
    fields = ("scan_period", "features", "filter", "init")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "lins_gpu.h"\nint main(){printf("%zu'
           + " %zu" * len(fields) + '\\n", sizeof(lins_slot_config)'
           + "".join(f", offsetof(lins_slot_config, {f})" for f in fields) + ");return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "s"), os.path.join(d, "s.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    T = defs.LinsSlotConfig
    assert got == [C.sizeof(T)] + [getattr(T, f).offset for f in fields]
    assert C.sizeof(T) == 8 + 3 * 8 + 10 * 8 + 15 * 8


def test_shipped_slot_config_is_the_shipped_params(defs):
    c = defs.LinsSlotConfig.shipped()
    assert c.scan_period == 0.1
    assert bytes(c.features) == bytes(defs.LinsFeatureParams.shipped())
    assert bytes(c.filter) == bytes(defs.LinsSeqParams.shipped())
    assert bytes(c.init) == bytes(defs.LinsSeqInitParams.shipped())
    o = defs.LinsSlotConfig.shipped(scan_period=0.05, edge_threshold=1.5, acc_n=5e4, init_pos_std=(1, 2, 3), init_ba=(0, 0, 0))
    assert o.scan_period == 0.05 and o.features.edge_threshold == 1.5 and o.features.surf_threshold == 0.5
    assert bytes(o.filter) == bytes(defs.LinsSeqParams.shipped(acc_n=5e4, init_pos_std=(1, 2, 3)))
    assert bytes(o.init) == bytes(defs.LinsSeqInitParams.shipped(init_ba=(0, 0, 0)))
    with pytest.raises(TypeError):
        defs.LinsSlotConfig.shipped(num_iter=3)  # (estimator tuning is per context, not per slot)


def test_recording_scan_period_follows_its_config(defs):
    br = pkg("bag_replay")
    bag = os.path.join(GOLDEN, "tiny.bag")
    cfg = defs.LinsSlotConfig.shipped(scan_period=0.05)
    with pytest.raises(ValueError):
        br.Recording(bag, scan_period=0.1, config=cfg)
    a = br.Recording(bag, config=cfg)
    b = br.Recording(bag, scan_period=0.05)
    c = br.Recording(bag, scan_period=0.05, config=cfg)
    assert a.config is cfg and b.config is None
    for r in (b, c):
        assert len(r.imu) == len(a.imu) and all(x.tobytes() == y.tobytes() for x, y in zip(r.imu, a.imu))
    d = br.Recording(bag)  # the default schedule is 10 Hz, as before
    e = br.Recording(bag, scan_period=0.1)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(d.imu, e.imu))


EXP_PORT = """%YAML:1.0

# settings
calibrate_imu: 0  # 0: no imu calibration and use default values. 1: calibrate imu
imu_lidar_extrinsic_angle: {extr}
imu_misalign_angle: {misalign}
line_num: 16
scan_num: 1800
scan_period: {period}
edge_threshold: 0.6
surf_threshold: 0.4
nearest_feature_search_sq_dist: 25
verbose: 0
icp_freq: 1
num_iter: {num_iter}
lidar_scale: 1
lidar_std: 0.01

# topic names
imu_topic: "/imu/data"

# noice parameters
acc_n: 60000
gyr_n: 0.12
acc_w: 450
gyr_w: 0.06

init_pos_std: !!opencv-matrix
   rows: 3
   cols: 1
   dt: d
   data: [0.01, 0.02, 0.03]

init_vel_std: !!opencv-matrix
   rows: 3
   cols: 1
   dt: d
   data: [0.0, 0.0, 0.0]

init_att_std: !!opencv-matrix
   rows: 3
   cols: 1
   dt: d
   data: [0.1, 0.2, 0.3]

init_acc_std: !!opencv-matrix
   rows: 3
   cols: 1
   dt: d
   data: [0.01, 0.01, 0.02]

init_gyr_std: !!opencv-matrix
   rows: 3
   cols: 1
   dt: d
   data: [0.002, 0.002, 0.002]

init_ba: !!opencv-matrix
   rows: 3
   cols: 1
   dt: d
   data: [-0.015774,0.143237,-0.0263845]

init_bw: !!opencv-matrix
   rows: 3
   cols: 1
   dt: d
   data: [-0.00275058,-0.000165954,0.00262913]

init_rbl: !!opencv-matrix
   rows: 3
   cols: 3
   dt: d
   data:  [1, 0, 0,
           0, 1, 0,
           0, 0, 1]
"""


def _yaml(tmp_path, name, period=0.05, extr=2.5, misalign=0.0, num_iter=30, drop=None):
    text = EXP_PORT.format(period=period, extr=extr, misalign=misalign, num_iter=num_iter)
    if drop:
        text = "\n".join(l for l in text.splitlines() if not l.startswith(drop + ":"))
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def test_yaml_reader_builds_the_slot_config(defs, tmp_path):
    rc = pkg("rig_config")
    y = rc.read_opencv_yaml(_yaml(tmp_path, "a.yaml"))
    assert y["init_rbl"] == [1, 0, 0, 0, 1, 0, 0, 0, 1] and y["imu_topic"] == "/imu/data" and y["num_iter"] == 30
    rig, shared = rc.load_rig(_yaml(tmp_path, "a.yaml"))
    assert shared == dict(num_iter=30, icp_freq=1, nearest_feature_search_sq_dist=25, lidar_std=0.01, lidar_scale=1)
    c = rc.slot_config(rig)
    assert c.scan_period == 0.05
    assert (c.features.edge_threshold, c.features.surf_threshold, c.features.imu_lidar_extrinsic_angle) == (0.6, 0.4, 2.5)
    ref = defs.LinsSeqParams.shipped(acc_n=60000.0, gyr_n=0.12, acc_w=450.0, gyr_w=0.06, init_pos_std=(0.01, 0.02, 0.03), init_att_std=(0.1, 0.2, 0.3))
    assert bytes(c.filter) == bytes(ref)  # the noise as setNoise computes it
    assert list(c.init.init_ba) == [-0.015774, 0.143237, -0.0263845] and list(c.init.init_gyr_std) == [0.002, 0.002, 0.002]
    p = rc.lins_params(shared, scan_period=0.05)
    assert (p.num_iter, p.icp_freq, p.nearest_feature_search_sq_dist, p.lidar_std, p.lidar_scale, p.scan_period) == (30, 1, 25.0, 0.01, 1.0, 0.05)


def test_yaml_reader_rejects_missing_keys_and_warns_on_misalignment(tmp_path):
    rc = pkg("rig_config")
    for k in ("scan_period", "acc_w", "init_bw", "lidar_std"):
        with pytest.raises(ValueError, match=k):
            rc.load_rig(_yaml(tmp_path, f"no_{k}.yaml", drop=k))
    bad = tmp_path / "plain.yaml"
    bad.write_text("scan_period: 0.1\n")
    with pytest.raises(ValueError):
        rc.read_opencv_yaml(str(bad))
    with pytest.warns(UserWarning, match="imu_misalign_angle"):
        rc.load_rig(_yaml(tmp_path, "m.yaml", misalign=3.0))


def test_run_bags_config_argument_errors(tmp_path, capsys):
    import importlib.util
    spec = importlib.util.spec_from_file_location("run_bags", os.path.join(ROOT, "tools", "run_bags.py"))
    rb = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rb)
    a, b = _yaml(tmp_path, "a.yaml"), _yaml(tmp_path, "b.yaml", period=0.1, extr=0.0)
    c = _yaml(tmp_path, "c.yaml", num_iter=10)
    bags = [os.path.join(GOLDEN, "tiny.bag")] * 3
    with pytest.raises(SystemExit):
        rb.main(bags + ["--config", f"{a},{b}"])  # two files for three bags
    assert "2 files for 3 bags" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        rb.main(bags + ["--config", f"{a},{b},{c}"])  # num_iter disagrees
    assert "num_iter" in capsys.readouterr().err
    prm, cfgs = rb.bag_configs(f"{a},{b},{a}", 3)  # rigs may differ, shared keys agree
    assert [x.scan_period for x in cfgs] == [0.05, 0.1, 0.05] and prm.num_iter == 30
    prm, cfgs = rb.bag_configs(a, 3)
    assert len(cfgs) == 3 and all(bytes(x) == bytes(cfgs[0]) for x in cfgs)
