"""GPU suite for the mapping node's cycle (lins_gpu_mapper_*, lins_gpu_voxel_grid) against the CPU oracle of
tests/mapperref.py, cycle by cycle.

Bit-exact: the local map's and the scan's DS clouds, the first LM pass's 5-NN, coefficients and masks, the key-frame
decisions, the key-frame count and the window.  Within the scan-to-map tolerance (1e-5 rad / m; only the A^T A
summation order differs): transformAftMapped and the key poses.  After each cycle the oracle adopts the device's
transformAftMapped and newest key pose, so every cycle starts from bit-identical inputs on both sides."""
import numpy as np
import pytest

import mapcases
import mapper_drive
import mapperref
import pyfront

pytestmark = pytest.mark.gpu
T_TOL = 1e-5


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _run(capi, ob, defs, events, check_pass_every=4):
    gpu, aux = capi.LinsGpu(), capi.LinsGpu()
    gpu.mapper_reset()
    orc = mapperref.MappingOracle(ob.MapOracle(), defs.POINT_DTYPE, scan_period=gpu.params.scan_period)
    mo = ob.MapOracle()
    log = []
    for e in events:
        if e[0] == "imu":
            gpu.mapper_imu(e[1], e[2], e[3])
            orc.imu(*e[1:])
            continue
        rep = gpu.mapper_step(*e[1:7])
        ro = orc.step(*e[1:7])
        ctx = f"event {e[-1]} t {e[1]}"
        assert (rep.processed, rep.skipped_interval) == (ro["processed"], ro["skipped_interval"]), ctx
        log.append((e, rep, ro))
        if not rep.processed:
            continue
        assert np.array_equal(_bits(rep.transform_guess), _bits(ro["transform_guess"])), ctx
        poses, window, clouds = gpu.mapper_download(rep)
        for k, v in orc.clouds.items():
            assert clouds[k].shape == v.shape and np.array_equal(_bits(clouds[k]), _bits(v)), f"{ctx} {k}"
        assert rep.map.skipped == ro["map_skipped"], ctx
        assert (rep.keyframe_saved, rep.n_keyframes, rep.loop_candidate) == (ro["keyframe_saved"], ro["n_keyframes"], ro["loop_candidate"]), ctx
        assert list(window) == ro["window"] and rep.window_len == len(ro["window"]), ctx
        if not rep.map.skipped:
            assert rep.map.iters == ro["map"].iters and list(rep.map.n_sel) == list(ro["map"].n_sel), ctx
            if len(log) % check_pass_every == 0:  # the first LM pass on the cycle's own clouds, at the cycle's guess
                cm, sm = (mapperref.to_points(clouds[k], defs.POINT_DTYPE) for k in ("map_corner_ds", "map_surf_ds"))
                cq, sq = (mapperref.to_points(clouds[k], defs.POINT_DTYPE) for k in ("corner_ds", "surf_total_ds"))
                aux.map_set(cm, sm); mo.set_map(cm, sm)
                a, b = aux.map_associate(cq, sq, rep.transform_guess), mo.associate(cq, sq, ro["transform_guess"])
                for k in a:
                    assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), f"{ctx} first pass {k}"
        assert np.abs(np.array(rep.transform_aft_mapped) - ro["transform_aft_mapped"]).max() <= T_TOL, ctx
        assert len(poses) == len(orc.poses)
        assert np.abs(poses[:, :6] - np.array([p for p, _ in orc.poses])).max() <= T_TOL, ctx
        assert np.array_equal(poses[:, 6], [t for _, t in orc.poses]), ctx
        orc.adopt(np.array(rep.transform_aft_mapped, np.float32), poses[-1] if rep.keyframe_saved else None)
    gpu.close(); aux.close()
    return log


def test_mapper_drive_matches_oracle(capi, ob, defs, synth):
    """71 key frames: the window fills, stalls for one cycle (the duplicate), reaches steady state; interval skips; an
    empty IMU queue, then lagging and leading IMU (both transformUpdate branches) and a wrapped ring; a return past the
    start more than 30 s later raises the loop candidate."""
    log = _run(capi, ob, defs, mapper_drive.make_drive(synth))
    reps = [r for _, r, _ in log if r.processed]
    assert reps[0].map.skipped == 1 and reps[-1].n_keyframes > 60
    assert any(r.skipped_interval for _, r, _ in log)
    wins = [ro["window"] for _, r, ro in log if r.processed]
    assert any(len(w) == 50 and len(set(w)) == 49 for w in wins)  # the duplicate
    assert any(r.loop_candidate >= 0 for r in reps) and reps[-1].loop_candidate >= 0
    assert not any(r.loop_candidate >= 0 for r in reps[:40])


def shim_events(synth, n_scans, seed):
    """The mapper's inputs as the C++ StateEstimator shim publishes them on a simulated drive (odometry = its
    globalStateYZX_, clouds = its YZX less-sharp / less-flat / outlier clouds), with one IMU message per scan whose
    roll / pitch are getRPY of the simulated orientation."""
    rec = synth.run_sequence("config3", seed=seed, n_scans=n_scans)
    times = [m["time"] for m in rec["map_inputs"]]
    ev = []
    for k, m in enumerate(rec["map_inputs"]):
        q = rec["global_true"][k + 1][3:]  # (publishing starts with the second scan)
        roll, pitch, _ = mapperref.get_rpy(*q)
        ev.append(("imu", m["time"] + 0.05, roll, pitch))
        ev.append(("odom", m["time"], tuple(m["quat"]), tuple(m["pos"]), m["corner"], m["surf"], m["outlier"], k))
    assert len(times) == n_scans - 1 and np.all(np.diff(times) > 0)
    return ev


def test_mapper_on_shim_odometry_matches_oracle(capi, ob, defs, synth):
    """The estimator's own odometry and clouds: every scan arrives 0.1 s after the last, so the 0.3 s interval skips
    most of them; the cycles that run match the oracle and save key frames as the drive moves on."""
    log = _run(capi, ob, defs, shim_events(synth, 48, seed=3), check_pass_every=2)
    reps = [r for _, r, _ in log if r.processed]
    assert len(reps) >= 10 and sum(r.skipped_interval for _, r, _ in log) >= 20
    assert reps[-1].n_keyframes >= 5 and sum(1 for r in reps if not r.map.skipped) >= 5


def test_mapper_gate_failure_keeps_stale_transform(capi, ob, defs, synth):
    """A first key frame too sparse for the 10 / 100 gate: transformUpdate never runs, transformAftMapped stays at its
    initial zeros, and the 0.3 m test against it saves no further key frame — the reference's behaviour."""
    ev = [e for e in mapper_drive.make_drive(synth, n_out=6, stall_at=-1, sparse_first=1) if e[0] == "odom"]
    log = _run(capi, ob, defs, ev)
    reps = [r for _, r, _ in log if r.processed]
    assert all(r.map.skipped for r in reps) and reps[-1].n_keyframes == 1
    assert all(list(r.transform_aft_mapped) == [0.0] * 6 for r in reps)


def test_mapper_leaves_the_scan2map_state_alone(capi, synth):
    """map_set + scan2map, then mapper cycles that run scan-to-map, a mapper_reset and scan2map again without map_set:
    the transform and report equal those of a context that never ran the mapper (the map, matP and isDegenerate of
    map_set / scan2map are not the mapper's)."""
    c = mapcases.corridor_scene()
    shared, alone = capi.LinsGpu(), capi.LinsGpu()
    for g in (shared, alone):
        g.map_set(c.corner_map, c.surf_map)
        g.scan2map(c.corner_q, c.surf_q, c.T)
    ev = [e for e in mapper_drive.make_drive(synth, n_out=8, seed=9, stall_at=-1) if e[0] == "odom"]
    reps = [shared.mapper_step(*e[1:7]) for e in ev]
    assert sum(1 for r in reps if r.processed and not r.map.skipped) >= 3
    shared.mapper_reset()
    (t1, m1), (t2, m2) = (g.scan2map(c.corner_q, c.surf_q, c.T) for g in (shared, alone))
    assert m2.degenerate == 1 and not m2.skipped
    assert np.array_equal(t1.view(np.uint32), t2.view(np.uint32)) and bytes(m1) == bytes(m2)
    shared.close(); alone.close()


def test_voxel_grid_million_points(gpu):
    rng = np.random.default_rng(11)
    n = 1_000_000
    p = np.zeros((n, 8), np.float32)
    p[:, :3] = rng.uniform(-20.5, -0.5, (n, 3)).astype(np.float32)
    p[: n // 2, :3] = rng.uniform(-3.0, -2.0, (n // 2, 3)).astype(np.float32)  # hundreds of points per voxel
    p[:, 4] = rng.uniform(0, 16, n).astype(np.float32)
    p[::997, 0] = np.nan
    p[5::1999, 2] = np.inf
    xyzi = p[:, [0, 1, 2, 4]]
    for leaf in (0.2, 0.4):
        g = gpu.voxel_grid(p, leaf)
        o = mapperref.voxel_grid(xyzi, leaf)
        assert g.shape == o.shape and np.array_equal(_bits(g), _bits(o)), leaf
    ref = pyfront.voxel_grid(xyzi, 0.4)
    assert np.array_equal(_bits(gpu.voxel_grid(p, 0.4)), _bits(ref))


def test_voxel_grid_key_overflow(capi, gpu):
    p = np.zeros((3, 8), np.float32)
    p[0, :3], p[1, :3] = -1e5, 1e5
    with pytest.raises(capi.LinsError, match="error -4"):
        gpu.voxel_grid(p, 0.01)
    assert len(gpu.voxel_grid(p, 400.0)) == 3  # (-1e5, 0 and 1e5 lie in three 400 m voxels)
    # the mapper refuses such a scan and keeps its state
    m = capi.LinsGpu()
    m.mapper_reset()
    with pytest.raises(capi.LinsError, match="error -4"):
        m.mapper_step(100.0, (0, 0, 0, 1), (0, 0, 0), p, p[:0], p[:0])
    rep = m.mapper_step(100.0, (0, 0, 0, 1), (0, 0, 0), p[2:], p[:0], p[:0])
    assert rep.processed == 1 and rep.n_keyframes == 1
    m.close()


def test_run_bag_map_writes_both_trajectories(synth, tmp_path):
    """tools/run_bag.py --map on a simulated bag: the mapper runs after every odometry output and the mapped trajectory
    is written next to the odometry one."""
    import os
    import subprocess
    import sys

    bag = str(tmp_path / "drive.bag")
    synth.write_sequence_bag(bag, n_scans=30, seed=2)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call([sys.executable, os.path.join(root, "tools", "run_bag.py"), bag, "--map", "--out", str(tmp_path)], stdout=subprocess.DEVNULL)
    odo = np.loadtxt(tmp_path / "odometry.txt", ndmin=2)
    mapped = np.loadtxt(tmp_path / "mapped.txt", ndmin=2)
    assert len(odo) == len(mapped) == 29 and np.array_equal(odo[:, 0], mapped[:, 0])
    assert mapped[:, 1].sum() >= 6 and np.isfinite(mapped).all() and np.isfinite(odo).all()
    assert np.abs(mapped[mapped[:, 1] == 1][:, 2:8]).max() > 0  # the processed cycles moved the mapped pose
