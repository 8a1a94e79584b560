"""GPU suite for the mapping node's loop closure (lins_gpu_mapper(s)_loops, lins_gpu_mapper(s)_close_loop(s)) against
the restatement of tests/loopref.py.

Exact: an enabled slot that never closes a loop against a plain slot (reports, key poses, windows, clouds); per call the
candidate's rule, the source and history counts and the first iteration's correspondence count; a lockstep slot
against the same drive run alone.  Within 1e-5: ICP's final transform and (relative) its fitness score, and the loop
factor."""
import math

import numpy as np
import pytest

import loopref
import mapper_drive

pytestmark = pytest.mark.gpu
F = np.float32


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def drifted_drive(synth, n_out=36, seed=6, yaw_bias=2e-3, x_bias=0.02, stall_at=None):
    """Out and back along the road with odometry whose yaw and x drift steadily, back at the start > 30 s later;
    stall_at: a scan index where the sensor stands still for one scan (a processed cycle without a key frame)."""
    xs = [-9.0 + 0.5 * k for k in range(n_out)] + [-9.0 + 0.5 * (n_out - 1 - k) - 0.25 for k in range(1, n_out)]
    poses = [(x, 0.3 * math.sin(0.15 * k), 1.5, 0.0 if k < n_out else math.pi) for k, x in enumerate(xs)]
    if stall_at is not None:
        poses.insert(stall_at, poses[stall_at - 1])
    scans, truth = synth.generate_map_drive(np.array(poses), seed=seed)
    ev, t = [], 100.0
    for k, ((corner, surf, outlier), T) in enumerate(zip(scans, truth)):
        odo = T.astype(np.float64) + k * np.array([0, yaw_bias, 0, x_bias, 0, 0])
        ev.append(("odom", t, mapper_drive.odometry_quat(odo), (odo[3], odo[4], odo[5]), corner, surf, outlier, k))
        t += 0.5
    return ev, truth


class Node:
    """One mapping node driven through the single mapper (slot None) or a lockstep slot, with what the checks need: the
    body-frame corner / surf DS clouds of every key frame and the last processed report."""

    def __init__(self, gpu, slot=None):
        self.gpu, self.slot, self.frames, self.rep, self.last_close = gpu, slot, [], None, None

    def download(self):
        return self.gpu.mapper_download(self.rep) if self.slot is None else self.gpu.mappers_download(self.slot, self.rep)

    def after_step(self, rep):
        if rep.processed:
            self.rep = rep
            if rep.keyframe_saved:
                _, _, cl = self.download()
                self.frames.append((cl["corner_ds"], cl["surf_ds"]))

    def due(self, t):
        """the 1 Hz loop thread, ticked by odometry stamps"""
        if self.last_close is None or t - self.last_close >= 1.0:
            self.last_close = t
            return True
        return False


def run_single(capi, events, loops=True, check=None):
    gpu = capi.LinsGpu()
    gpu.mapper_reset()
    if loops:
        gpu.mapper_loops()
    node, log = Node(gpu), []
    for e in events:
        if e[0] == "imu":
            gpu.mapper_imu(e[1], e[2], e[3])
            continue
        rep = gpu.mapper_step(*e[1:7])
        node.after_step(rep)
        lr = None
        if loops and node.rep is not None and node.due(e[1]):
            poses = node.download()[0]
            lr = gpu.mapper_close_loop()
            if check:
                check(node, poses, lr, e[1])
        log.append((rep, lr, node.download()[0] if node.rep is not None else None))
    return gpu, node, log


def check_call(node, poses, lr, t):
    """one close_loop against the restatement on the node's own key poses and key-frame clouds"""
    c = lr.closest_history_frame_id
    if c < 0:
        assert lr.latest_frame_id == -1 and lr.accepted == 0
        return
    assert lr.latest_frame_id == len(poses) - 1 and abs(poses[c, 6] - t) > 30.0
    src, tgt = loopref.loop_clouds(poses, node.frames, c)
    ref = loopref.icp(src, tgt)
    ctx = f"t {t} closest {c}"
    assert (lr.n_source, lr.n_history_ds, lr.n_corr0) == (ref["n_source"], len(tgt), ref["n_corr0"]), ctx
    fin = np.array(lr.final_transform, np.float64).reshape(4, 4)
    assert np.abs(fin - ref["final"]).max() <= 1e-5, (ctx, fin, ref["final"])
    assert abs(lr.fitness - ref["fitness"]) <= 1e-5 * max(ref["fitness"], 1e-12), ctx
    assert (lr.converged, lr.icp_iters) == (ref["converged"], ref["iters"]), ctx
    margin = abs(ref["fitness"] - float(loopref.FITNESS)) > 1e-3
    if margin:
        assert lr.accepted == int(ref["converged"] == 1 and not ref["fitness"] > float(loopref.FITNESS)), ctx
    if lr.accepted:
        z = loopref.loop_factor(fin.astype(F), poses[lr.latest_frame_id], poses[c])
        assert np.abs(np.array(lr.factor[:3]) - z[:3, 3]).max() <= 1e-5, ctx
        # the angles compared as a rotation matrix: an Euler angle near +-pi may wrap on either side
        R = loopref.Rotation.from_euler("xyz", lr.factor[3:]).as_matrix()
        assert np.abs(R - z[:3, :3]).max() <= 1e-5, ctx
        assert lr.noise == float(F(lr.fitness))


def test_enabled_slot_without_closures_is_a_plain_slot(capi, synth):
    """slot 1 enabled, slot 0 plain, the same drive: every report, key pose, window and cloud is bit-identical."""
    gpu = capi.LinsGpu()
    gpu.mappers_open(2)
    gpu.mappers_loops([0, 1])
    for e in mapper_drive.make_drive(synth):
        if e[0] == "imu":
            gpu.mappers_imu([(e[1], e[2], e[3])] * 2)
            continue
        reps = gpu.mappers_step([e[1:7], e[1:7]])
        a, b = bytes(reps[0]), bytes(reps[1])
        assert a == b, e[-1]
        if reps[0].processed:
            pa, wa, ca = gpu.mappers_download(0, reps[0])
            pb, wb, cb = gpu.mappers_download(1, reps[1])
            assert np.array_equal(pa, pb) and np.array_equal(wa, wb)
            for k in ca:
                assert np.array_equal(_bits(ca[k]), _bits(cb[k])), k


def test_close_loop_matches_restatement_on_out_and_back_drive(capi, synth):
    gpu, node, log = run_single(capi, mapper_drive.make_drive(synth), check=check_call)
    lrs = [lr for _, lr, _ in log if lr is not None]
    assert any(lr.closest_history_frame_id < 0 for lr in lrs) and any(lr.closest_history_frame_id >= 0 for lr in lrs)


def test_close_loop_on_drifted_drive_corrects_the_poses(capi, synth):
    events, truth = drifted_drive(synth)
    gpu, node, log = run_single(capi, events, check=check_call)
    acc = [i for i, (_, lr, _) in enumerate(log) if lr is not None and lr.accepted]
    assert acc, "no loop accepted on the drifted drive"
    # correctPoses in the next processed cycle: the key poses move and the window is rebuilt from the newest ids
    i = acc[0]
    before = log[i][2]
    j = next(k for k in range(i + 1, len(log)) if log[k][0].processed)
    after = log[j][2]
    assert np.abs(after[:len(before), :6] - before[:, :6]).max() > 1e-4
    k = next(k for k in range(j + 1, len(log)) if log[k][0].processed)
    assert log[k][0].window_len == min(50, log[j][0].n_keyframes)
    # sanity, not parity: scan-to-map already removes most of this drive's odometry drift, so the closure may not
    # shorten the end pose's distance to the truth; it must not lengthen it by more than a centimetre
    _, _, plain = run_single(capi, events, loops=False)
    end = np.array(truth[-1], np.float64)

    def err(lg):
        last = next(r for r, _, _ in reversed(lg) if r.processed)
        return np.linalg.norm(np.array(last.transform_aft_mapped[3:], np.float64) - end[3:])

    assert err(log) <= err(plain) + 0.01


def test_lockstep_slots_match_runs_alone(capi, synth):
    drives = [mapper_drive.make_drive(synth, seed=4), drifted_drive(synth)[0]]
    alone = [run_single(capi, ev)[2] for ev in drives]
    M = 132
    gpu = capi.LinsGpu()
    gpu.mappers_open(M)
    gpu.mappers_loops([1] * M)
    nodes = [Node(gpu, s) for s in range(M)]
    its = [iter(drives[s % 2]) for s in range(M)]
    logs = [[] for _ in range(M)]
    pending = [next(it, None) for it in its]
    while any(p is not None for p in pending):
        imu = [(p[1], p[2], p[3]) if p is not None and p[0] == "imu" else None for p in pending]
        if any(r is not None for r in imu):
            gpu.mappers_imu(imu)
            pending = [next(its[s], None) if imu[s] is not None else pending[s] for s in range(M)]
            continue
        reps = gpu.mappers_step([p[1:7] if p is not None else None for p in pending])
        due = np.zeros(M, np.uint8)
        for s in range(M):
            if pending[s] is None:
                continue
            nodes[s].after_step(reps[s])
            due[s] = nodes[s].rep is not None and nodes[s].due(pending[s][1])
        lrs = gpu.mappers_close_loops(due) if due.any() else [None] * M
        for s in range(M):
            if pending[s] is not None:
                logs[s].append((reps[s], lrs[s] if due[s] else None, nodes[s].download()[0] if nodes[s].rep is not None else None))
        pending = [next(its[s], None) if pending[s] is not None else None for s in range(M)]
    for s in range(M):
        ref = alone[s % 2]
        assert len(logs[s]) == len(ref)
        for (ra, la, pa), (rb, lb, pb) in zip(logs[s], ref):
            assert bytes(ra) == bytes(rb)
            assert (la is None) == (lb is None) and (la is None or bytes(la) == bytes(lb))
            assert (pa is None and pb is None) or np.array_equal(pa, pb)


def test_enable_rules(capi, synth):
    gpu = capi.LinsGpu()
    gpu.mappers_open(2)
    e = next(e for e in mapper_drive.make_drive(synth) if e[0] == "odom")
    gpu.mappers_step([e[1:7], None])
    with pytest.raises(Exception):
        gpu.mappers_loops([1, 0])  # stepped: not fresh
    with pytest.raises(Exception):
        gpu.mappers_close_loops([0, 1])  # not enabled
    gpu.mappers_loops([0, 1])
    reps = gpu.mappers_close_loops([0, 1])
    assert reps[1].closest_history_frame_id == -1 and reps[0] is None
    gpu.mappers_reset([1, 1])
    with pytest.raises(Exception):
        gpu.mappers_close_loops([0, 1])  # reset: not enabled
    gpu.mappers_loops([1, 0])


def parked_drive(synth, seed=7):
    """Twelve key frames out, 40 s standing still, then back over them: a candidate whose history window is clipped at
    0 and at latest."""
    poses = [(-4.0 + 0.5 * k, 0.0, 1.5, 0.0) for k in range(12)]
    poses += [poses[-1]] * 80 + [(-4.0 + 0.5 * (11 - k) - 0.25, 0.0, 1.5, math.pi) for k in range(1, 12)]
    scans, truth = synth.generate_map_drive(np.array(poses), seed=seed)
    ev, t = [], 100.0
    for k, ((corner, surf, outlier), T) in enumerate(zip(scans, truth)):
        odo = T.astype(np.float64)
        ev.append(("odom", t, mapper_drive.odometry_quat(odo), (odo[3], odo[4], odo[5]), corner, surf, outlier, k))
        t += 0.5
    return ev


def run_against_oracle(capi, ob, defs, events, force_close=(), tol=1e-5):
    """A whole drive on the single mapper with loop closure, cycle by cycle against loopref.LoopMappingOracle: decisions,
    key-frame counts and windows equal, transformAftMapped and every key pose within tol; each close_loop's candidate and
    counts equal and its final transform within 1e-5 (the oracle's loop factor is then built on the device's ICP result,
    as it adopts the device's transformAftMapped after each cycle).  force_close: event tags after which the loop thread
    ticks whatever the 1 s rule says.  Returns the log of (report, oracle report, loop report or None, oracle close)."""
    gpu = capi.LinsGpu()
    gpu.mapper_reset()
    gpu.mapper_loops()
    orc = loopref.LoopMappingOracle(ob.MapOracle(), defs.POINT_DTYPE, scan_period=gpu.params.scan_period)
    node, log = Node(gpu), []
    for e in events:
        if e[0] == "imu":
            gpu.mapper_imu(e[1], e[2], e[3])
            orc.imu(*e[1:])
            continue
        rep = gpu.mapper_step(*e[1:7])
        ro = orc.step(*e[1:7])
        ctx = f"event {e[-1]} t {e[1]}"
        assert (rep.processed, rep.skipped_interval) == (ro["processed"], ro["skipped_interval"]), ctx
        node.after_step(rep)
        if rep.processed:
            assert (rep.keyframe_saved, rep.n_keyframes, rep.loop_candidate) == (ro["keyframe_saved"], ro["n_keyframes"], ro["loop_candidate"]), ctx
            assert rep.window_len == len(ro["window"]), ctx
            poses, window, _ = gpu.mapper_download(rep)
            if orc.window:  # (after correctPoses the window is empty, as the reference leaves it: nothing is written)
                assert list(window) == list(orc.window), ctx
            assert np.abs(np.array(rep.transform_aft_mapped) - ro["transform_aft_mapped"]).max() <= tol, ctx
            assert np.abs(poses[:, :6] - orc.poses7()[:, :6]).max() <= tol, (ctx, np.abs(poses[:, :6] - orc.poses7()[:, :6]).max())
            orc.adopt(np.array(rep.transform_aft_mapped, np.float32), poses[-1] if rep.keyframe_saved else None)
        lr = oc = None
        if node.rep is not None and (node.due(e[1]) or e[-1] in force_close):
            lr = gpu.mapper_close_loop()
            fin = np.array(lr.final_transform, np.float32).reshape(4, 4)
            oc = orc.close(use=(fin, lr.fitness))
            assert (lr.closest_history_frame_id, lr.latest_frame_id) == (oc["closest"], oc["latest"]), ctx
            if oc["closest"] >= 0:
                ref = oc["icp"]
                assert (lr.n_source, lr.n_history_ds, lr.n_corr0, lr.converged) == (ref["n_source"], oc["n_history"], ref["n_corr0"], ref["converged"]), ctx
                assert np.abs(fin - ref["final"]).max() <= 1e-5, ctx
                assert lr.accepted == oc["accepted"], ctx
        log.append((rep, ro, lr, oc))
    return log


def test_whole_drive_with_loops_matches_oracle(capi, ob, defs, synth):
    """The drifted drive with a scan standing still after a forced closure: correctPoses then runs in a cycle that saved
    no key frame (the stale estimate), and again after a later closure in a cycle that did; both against the oracle."""
    events, _ = drifted_drive(synth, stall_at=62)
    log = run_against_oracle(capi, ob, defs, events, force_close={61})
    acc = [i for i, (_, _, lr, _) in enumerate(log) if lr is not None and lr.accepted]
    assert acc
    corr = [(r.keyframe_saved, ro["corrected"]) for r, ro, _, _ in log if r.processed]
    assert (0, True) in corr, "no correctPoses with a stale estimate"
    assert (1, True) in corr, "no correctPoses after a solve"


def test_parked_drive_clips_the_history_window(capi, ob, defs, synth):
    log = run_against_oracle(capi, ob, defs, parked_drive(synth))
    calls = [(lr, oc) for _, _, lr, oc in log if lr is not None and lr.closest_history_frame_id >= 0]
    assert calls
    assert any(lr.closest_history_frame_id - 25 < 0 and lr.closest_history_frame_id + 25 > lr.latest_frame_id for lr, _ in calls)


def test_seq_save_refuses_an_enabled_slot(capi, defs):
    """a bound run: saving or loading a slot whose mapper closes loops is refused and changes nothing"""
    br = pytest.importorskip("lins---lidar-inertial-slam_b200.bag_replay")
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), br.shim_init_params(), 2)
    g.seq_map_open()
    g.mappers_loops([1, 0])
    blob = g.seq_save([0, 1])[1]
    for call in (lambda: g.seq_save([1, 0]), lambda: g.seq_save([1, 1]), lambda: g.seq_load([1, 0], [blob, None])):
        with pytest.raises(Exception):
            call()
    assert g.seq_save([0, 1])[1] == blob
    g.seq_load([0, 1], [None, blob])  # (a fresh slot without loop closure still loads)
    with pytest.raises(Exception):
        g.mappers_loops([0, 1])  # a loaded slot is not fresh


def test_bound_replay_with_loops_matches_host_composition(capi, synth, tmp_path):
    """replay(map=True, loops=True) of bags through fewer slots than bags against each bag's published stream fed to a
    single mapper with loop closure, ticked at the same stamps: decisions and key-frame counts equal, transformAftMapped
    and the final key poses within 1e-5, the same closures."""
    br = pytest.importorskip("lins---lidar-inertial-slam_b200.bag_replay")
    paths = []
    for seed, n in ((40, 16), (41, 12), (42, 20)):
        p = str(tmp_path / f"b{seed}.bag")
        synth.write_sequence_bag(p, config="config3", seed=seed, n_scans=n)
        paths.append(p)
    outs = br.replay([br.Recording(p) for p in paths], 2, map=True, loops=True)
    for p, o in zip(paths, outs):
        g = capi.LinsGpu()
        g.mapper_reset()
        g.mapper_loops()
        tick, last, acc = None, None, 0
        for k, m in enumerate(synth.run_bag(p)["map_inputs"]):
            rep = g.mapper_step(m["time"], m["quat"], m["pos"], m["corner"], m["surf"], m["outlier"])
            assert (o["map_processed"][k], o["map_keyframes"][k]) == (rep.processed, rep.n_keyframes), (p, k)
            assert np.abs(o["map_aft_mapped"][k] - np.array(rep.transform_aft_mapped)).max() <= 1e-5, (p, k)
            if rep.processed:
                last = rep
            if tick is None or m["time"] - tick >= 1.0:
                tick = m["time"]
                acc += g.mapper_close_loop().accepted
        assert acc == o["loops_accepted"], p
        poses = g.mapper_download(last)[0]
        assert poses.shape == o["key_poses"].shape and np.abs(poses[:, :6] - o["key_poses"][:, :6]).max() <= 1e-5, p
