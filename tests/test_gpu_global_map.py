"""GPU suite for the mapping node's global map (lins_gpu_mapper(s)_global_map(_download)) against the restatement of
tests/globalmapref.py.  Exact: the cloud's f32 bits and the key ids, per call, for one drive or many in lockstep.

The restatement takes currentRobotPosPoint from the last processed report's transformAftMapped: that is the point
itself after a cycle without a loop factor, and on the drives with closures every key pose lies far inside 500 m of
either, so the selection is the same."""
import numpy as np
import pytest

import globalmapref
import mapper_drive
from test_gpu_loops import drifted_drive, parked_drive

pytestmark = pytest.mark.gpu
F = np.float32
NAMES = ("corner_ds", "surf_ds", "outlier_ds")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def check_against_ref(keys, cloud, rep, poses, body, cur, ctx=""):
    ref = globalmapref.global_map(poses, body, cur)
    assert (rep.n_key_poses, rep.n_key_frames, rep.n_points, rep.n_map, rep.unfiltered) == (
        ref["n_key_poses"], len(ref["keys"]), len(ref["points"]), len(ref["map"]), ref["unfiltered"]), ctx
    assert np.array_equal(keys, ref["keys"]), ctx
    assert _same(cloud, ref["map"]), ctx
    return ref


def run_single(capi, events, close=True, check=True, every=1):
    """A drive on the single mapper with loop closure (the 1 Hz tick of tests/test_gpu_loops.py), the global map after
    every `every`-th processed cycle and after every closure call, each against the restatement.  Returns (gpu, log of
    (report, loop report or None, global-map report or None), body clouds)."""
    gpu = capi.LinsGpu()
    gpu.mapper_reset()
    gpu.mapper_loops()
    body, last, tick, log, n_proc = [], None, None, [], 0

    def global_map(ctx):
        rep = gpu.mapper_global_map()
        keys, cloud = gpu.mapper_global_map_download(rep)
        if check:
            poses = gpu.mapper_download(last)[0]
            check_against_ref(keys, cloud, rep, poses, body, np.array(last.transform_aft_mapped[3:], F), ctx)
        return rep

    for e in events:
        if e[0] == "imu":
            gpu.mapper_imu(e[1], e[2], e[3])
            continue
        r = gpu.mapper_step(*e[1:7])
        gr = lr = None
        if r.processed:
            last, n_proc = r, n_proc + 1
            if r.keyframe_saved:
                cl = gpu.mapper_download(r)[2]
                body.append(tuple(cl[k] for k in NAMES))
            if n_proc % every == 0:
                gr = global_map(f"event {e[-1]}")
        if close and last is not None and (tick is None or e[1] - tick >= 1.0):
            tick = e[1]
            lr = gpu.mapper_close_loop()
            if lr.accepted:  # between the closure and its correctPoses
                gr = global_map(f"event {e[-1]} after a closure")
        log.append((r, lr, gr))
    return gpu, log, body


def test_global_map_matches_restatement_around_closures(capi, synth):
    events, _ = drifted_drive(synth, stall_at=62)
    gpu, log, body = run_single(capi, events)
    acc = [i for i, (_, lr, _) in enumerate(log) if lr is not None and lr.accepted]
    assert acc, "no closure on the drifted drive"
    assert any(g is not None for _, _, g in log[:acc[0]]), "no global map before the first closure"
    assert any(g is not None for _, _, g in log[acc[0] + 1:]), "no global map after a correctPoses"
    # every key pose within the radius, every key frame named at least once in this 18 m drive's 1 m voxels
    r = next(g for _, _, g in reversed(log) if g is not None)
    assert r.n_key_poses == len(body) and r.n_map > 0 and not r.unfiltered


def test_parked_drive(capi, synth):
    run_single(capi, parked_drive(synth), every=3)


def test_radius_excludes_far_key_poses(capi, synth):
    """Odometry 10 m per scan for 600 m over the first scan's clouds repeated: the key poses follow the odometry (only the
    ground constrains scan-to-map), and the start leaves the 500 m radius."""
    scans, truth = synth.generate_map_drive(np.array([(-9.0, 0.0, 1.5, 0.0)]), seed=5)
    events, t = [], 100.0
    for k in range(62):
        odo = truth[0].astype(np.float64) + k * np.array([0, 0, 0, 0, 0, 10.0])
        events.append(("odom", t, mapper_drive.odometry_quat(odo), (odo[3], odo[4], odo[5])) + tuple(scans[0]) + (k,))
        t += 0.5
    gpu, log, body = run_single(capi, events, close=False, every=5)
    r = next(g for _, _, g in reversed(log) if g is not None)
    poses = gpu.mapper_download(next(x for x, _, _ in reversed(log) if x.processed))[0]
    assert np.abs(poses[-1, :3] - poses[0, :3]).max() > 500.0
    assert 0 < r.n_key_poses < len(poses)


def test_unfiltered_when_the_global_voxel_grid_overflows(capi, synth):
    """A lone outlier point 3.5 km above the first scan: every VoxelGrid of the mapper stays within INT32_MAX voxels, the
    global map's 0.4 m one over the 100 m drive does not, and the map is the concatenation itself."""
    poses = [(-9.0 + 0.5 * k, 0.0, 1.5, 0.0) for k in range(200)]
    scans, truth = synth.generate_map_drive(np.array(poses), seed=8)
    events, t = [], 100.0
    for k, ((corner, surf, outlier), T) in enumerate(zip(scans, truth)):
        if k == 0:
            high = np.zeros(1, outlier.dtype)
            high["x"], high["y"], high["z"], high["intensity"] = 0.0, 3500.0, 0.0, 0.5
            if "pad0" in outlier.dtype.names:
                high["pad0"] = 1.0
            outlier = np.concatenate([outlier, high])
        odo = T.astype(np.float64)
        events.append(("odom", t, mapper_drive.odometry_quat(odo), (odo[3], odo[4], odo[5]), corner, surf, outlier, k))
        t += 0.5
    gpu, log, body = run_single(capi, events, close=False, check=False, every=1000)
    last = next(x for x, _, _ in reversed(log) if x.processed)
    assert last.n_keyframes > 60
    rep = gpu.mapper_global_map()
    keys, cloud = gpu.mapper_global_map_download(rep)
    assert rep.unfiltered == 1 and rep.n_map == rep.n_points
    poses = gpu.mapper_download(last)[0]
    ref = check_against_ref(keys, cloud, rep, poses, body, np.array(last.transform_aft_mapped[3:], F))
    # the premise of reading the store: the stored map-frame clouds are transformPointCloud of the body-frame ones
    assert _same(cloud, ref["points"])


def _lockstep(capi, drives, M):
    """The drives cycled over M lockstep slots with loop closure enabled (no closure is run).  Returns gpu."""
    gpu = capi.LinsGpu()
    gpu.mappers_open(M)
    gpu.mappers_loops([1] * M)
    its = [iter(drives[s % len(drives)]) for s in range(M)]
    pending = [next(it, None) for it in its]
    while any(p is not None for p in pending):
        imu = [(p[1], p[2], p[3]) if p is not None and p[0] == "imu" else None for p in pending]
        if any(r is not None for r in imu):
            gpu.mappers_imu(imu)
            pending = [next(its[s], None) if imu[s] is not None else pending[s] for s in range(M)]
            continue
        gpu.mappers_step([p[1:7] if p is not None else None for p in pending])
        pending = [next(its[s], None) if pending[s] is not None else None for s in range(M)]
    return gpu


def test_lockstep_slots_match_runs_alone_in_several_passes(capi, defs, synth):
    """Three drifted drives of 50-70 m out and back over 132 slots: each global map gathers 0.25-0.35 M points, so the
    full mask and the random masks exceed one pass's budget.  (Closures are covered by the single-drive checks: here
    the host solve of every slot's key-pose graph would dominate the run.)"""
    drives = [drifted_drive(synth, n_out=140)[0], drifted_drive(synth, n_out=120, seed=9)[0], drifted_drive(synth, n_out=100, seed=11)[0]]
    alone = []
    for ev in drives:
        gpu, log, _ = run_single(capi, ev, close=False, check=False, every=10 ** 6)
        rep = gpu.mapper_global_map()
        alone.append((rep, *gpu.mapper_global_map_download(rep)))
    M = 132
    gpu = _lockstep(capi, drives, M)
    rng = np.random.default_rng(3)
    masks = [np.ones(M, np.uint8)] + [(rng.random(M) < 0.85).astype(np.uint8) for _ in range(3)]
    for mask in masks:
        reps = gpu.mappers_global_map(mask)
        assert sum(r.n_points for r in reps if r is not None) > defs.GLOBAL_MAP_PASS_POINTS  # several passes
        for s in range(M):
            if not mask[s]:
                assert reps[s] is None
                continue
            ra, ka, ca = alone[s % len(drives)]
            assert bytes(reps[s]) == bytes(ra), s
            k, c = gpu.mappers_global_map_download(s, reps[s])
            assert np.array_equal(k, ka) and _same(c, ca), s


def test_global_map_has_no_side_effects(capi, synth):
    """Slot 0 takes a global map after every step, slot 1 runs the same drive without: reports, key poses, windows,
    closure reports and downloads stay bit-identical."""
    events, _ = drifted_drive(synth, stall_at=62)
    gpu = capi.LinsGpu()
    gpu.mappers_open(2)
    gpu.mappers_loops([1, 1])
    last, tick = None, None
    for e in events:
        reps = gpu.mappers_step([e[1:7], e[1:7]])
        assert bytes(reps[0]) == bytes(reps[1]), e[-1]
        if reps[0].processed:
            last = reps
        if last is not None:
            gpu.mappers_global_map([1, 0])
            if tick is None or e[1] - tick >= 1.0:
                tick = e[1]
                lr = gpu.mappers_close_loops([1, 1])
                assert bytes(lr[0]) == bytes(lr[1]), e[-1]
            pa, wa, ca = gpu.mappers_download(0, last[0])
            pb, wb, cb = gpu.mappers_download(1, last[1])
            assert np.array_equal(pa, pb) and np.array_equal(wa, wb), e[-1]
            for k in ca:
                assert _same(ca[k], cb[k]), (e[-1], k)


def test_refusals_and_empty_maps(capi, synth):
    gpu = capi.LinsGpu()
    gpu.mappers_open(3)
    gpu.mappers_loops([1, 1, 0])
    with pytest.raises(capi.LinsError):
        gpu.mappers_global_map_download(0, capi.LinsGlobalMapReport())  # none yet
    reps = gpu.mappers_global_map([0, 1, 0])  # enabled, no key frame: an empty map
    assert (reps[1].n_key_poses, reps[1].n_key_frames, reps[1].n_points, reps[1].n_map, reps[1].unfiltered) == (0, 0, 0, 0, 0)
    keys, cloud = gpu.mappers_global_map_download(1, reps[1])
    assert keys.shape == (0,) and cloud.shape == (0, 4)
    ev = [e for e in mapper_drive.make_drive(synth) if e[0] == "odom"][:4]
    for e in ev:
        gpu.mappers_step([e[1:7]] * 3)
    r0 = gpu.mappers_global_map([1, 0, 0])[0]
    k0, c0 = gpu.mappers_global_map_download(0, r0)
    assert r0.n_key_frames > 0 and r0.n_map > 0
    for mask in ([1, 0, 1], [0, 0, 1]):
        with pytest.raises(capi.LinsError):
            gpu.mappers_global_map(mask)  # a plain slot: refused before anything changes
    k, c = gpu.mappers_global_map_download(0, r0)
    assert np.array_equal(k, k0) and _same(c, c0)
    gpu.mappers_reset([1, 0, 0])
    with pytest.raises(capi.LinsError):
        gpu.mappers_global_map_download(0, r0)  # reset frees it


def test_bound_replay_global_map_matches_single_mapper(capi, synth, tmp_path):
    """replay(map=True, loops=True, global_map=True) of three bags through two slots (handed over mid-run) against each
    bag's published stream fed to a single mapper ticked at the same stamps."""
    br = pytest.importorskip("lins---lidar-inertial-slam_b200.bag_replay")
    paths = []
    for seed, n in ((40, 16), (41, 12), (42, 20)):
        p = str(tmp_path / f"b{seed}.bag")
        synth.write_sequence_bag(p, config="config3", seed=seed, n_scans=n)
        paths.append(p)
    outs = br.replay([br.Recording(p) for p in paths], 2, map=True, loops=True, global_map=True)
    for p, o in zip(paths, outs):
        g = capi.LinsGpu()
        g.mapper_reset()
        g.mapper_loops()
        tick = None
        for m in synth.run_bag(p)["map_inputs"]:
            g.mapper_step(m["time"], m["quat"], m["pos"], m["corner"], m["surf"], m["outlier"])
            if tick is None or m["time"] - tick >= 1.0:
                tick = m["time"]
                g.mapper_close_loop()
        rep = g.mapper_global_map()
        keys, cloud = g.mapper_global_map_download(rep)
        assert rep.n_map > 0, p
        assert np.array_equal(o["global_map_keys"], keys), p
        assert o["global_map"].shape == cloud.shape and np.abs(o["global_map"] - cloud).max() <= 1e-4, p
