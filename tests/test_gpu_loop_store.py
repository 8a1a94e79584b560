"""GPU suite for the host key-frame store of slots with loop closure (DESIGN.md §4.14): every key frame's body clouds in
the run's pinned, mapped arena, the device store a plain slot's (the window and the newest key frame).

The drives here run past 51 key frames, so the history sub-maps of close_loops and the global maps read key frames that
exist only in the host store.  Checked: a whole drive cycle by cycle against tests/loopref.py's LoopMappingOracle and its
global maps against the restatement; 132 lockstep slots, plain and with loop closure mixed, bit-identical to each drive
run alone; the store bytes (a loop slot's device store equals its plain twin's, its host store holds 16 bytes per DS
point of every key frame, and reset slots refilled with the same drives reserve nothing new); saves at several points
loaded into fresh slots of either API and continued byte-equal; launch counts."""
import numpy as np
import pytest

import test_gpu_global_map as tgm
import test_gpu_loops as tl
import test_gpu_mapper_checkpoint as tc

pytestmark = pytest.mark.gpu

WINDOW = 50
LONG_OUT = 42  # scans out: 2 * 42 - 1 key frames, well past the device store's 51


def long_drive(synth, **kw):
    kw.setdefault("n_out", LONG_OUT)
    return tl.drifted_drive(synth, **kw)[0]


def ds_points(rep):
    return rep.n_corner_ds + rep.n_surf_ds + rep.n_outlier_ds


def test_long_drive_against_oracle_and_global_map_restatement(capi, ob, defs, synth):
    """A forced closure just before a scan standing still (correctPoses on the stale estimate), then the 1 Hz closures
    on the way back: every cycle and closure against the oracle, and the global maps against the restatement."""
    stall = 2 * LONG_OUT - 10
    events = long_drive(synth, stall_at=stall)
    log = tl.run_against_oracle(capi, ob, defs, events, force_close={stall - 1})
    corr = [(r.keyframe_saved, ro["corrected"]) for r, ro, _, _ in log if r.processed]
    assert (0, True) in corr and (1, True) in corr
    calls = [(r, lr) for r, _, lr, _ in log if lr is not None and lr.closest_history_frame_id >= 0]
    assert calls
    # a history sub-map with key frames outside the device store (older than the newest 51)
    assert any(lr.closest_history_frame_id - 25 < lr.latest_frame_id - WINDOW for _, lr in calls)
    assert any(lr.accepted for _, lr in calls)
    _, glog, body = tgm.run_single(capi, events, every=7)  # (each map checked against the restatement inside)
    assert len(body) > WINDOW + 1
    assert any(gr is not None and gr.n_key_poses > WINDOW + 1 for _, _, gr in glog)  # (maps over host-only key frames)


def _alone(capi, ev, loops):
    gpu, _, log = tl.run_single(capi, ev, loops=loops)
    out = [(bytes(rep), bytes(lr) if lr is not None else None) for rep, lr, _ in log]
    gm = None
    if loops:
        rep = gpu.mapper_global_map()
        k, c = gpu.mapper_global_map_download(rep)
        gm = (bytes(rep), k.tobytes(), c.tobytes())
    return out, gm


def _lockstep_run(gpu, drives, M, loop_mask):
    """the drives cycled over M slots, the loop thread ticked on the loop slots as tests/test_gpu_loops.py ticks it (all
    drives share their event times); returns per slot the (report, loop report) log"""
    n_ev = len(drives[0])
    log = [[] for _ in range(M)]
    last_close, started = None, False
    for i in range(n_ev):
        reps = gpu.mappers_step([drives[s % len(drives)][i][1:7] for s in range(M)])
        started = started or any(r.processed for r in reps)
        t = drives[0][i][1]
        lrs = [None] * M
        if started and (last_close is None or t - last_close >= 1.0):
            last_close = t
            lrs = gpu.mappers_close_loops(loop_mask)
        for s in range(M):
            log[s].append((bytes(reps[s]), bytes(lrs[s]) if lrs[s] is not None else None))
    return log


def test_132_mixed_slots_match_runs_alone(capi, synth):
    drives = [long_drive(synth), long_drive(synth, seed=9, yaw_bias=-1.5e-3), long_drive(synth, seed=11, x_bias=0.01)]
    assert len({tuple(e[1] for e in d) for d in drives}) == 1  # (one event layout)
    alone = {(d, lp): _alone(capi, drives[d], lp) for d in range(3) for lp in (False, True)}
    M = 132
    loop_mask = np.array([(s // 3) % 2 for s in range(M)], np.uint8)  # (every drive on plain and loop slots)
    gpu = capi.LinsGpu()
    gpu.mappers_open(M)
    gpu.mappers_loops(loop_mask)
    for rnd in range(2):  # the second round on the slots reset: the host store reuses its chunks
        log = _lockstep_run(gpu, drives, M, loop_mask)
        for s in range(M):
            want, _ = alone[(s % 3, bool(loop_mask[s]))]
            assert log[s] == want, (rnd, s)
        reps = gpu.mappers_global_map(loop_mask)
        for s in np.flatnonzero(loop_mask):
            k, c = gpu.mappers_global_map_download(s, reps[s])
            assert (bytes(reps[s]), k.tobytes(), c.tobytes()) == alone[(s % 3, True)][1], (rnd, s)
        dev, host, reserved = gpu.mappers_store_bytes()
        for s in range(M):
            saved = [r for r in (capi.LinsMapperReport.from_buffer_copy(b) for b, _ in log[s]) if r.processed and r.keyframe_saved]
            assert host[s] == (16 * sum(ds_points(r) for r in saved) if loop_mask[s] else 0), s
            assert len(saved) > WINDOW + 1
        if rnd == 0:
            first = reserved
            gpu.mappers_reset(np.ones(M, np.uint8))
            assert not gpu.mappers_store_bytes()[1].any()
            gpu.mappers_loops(loop_mask)
        else:
            assert reserved == first


def test_store_bytes_against_plain_twin(capi, synth):
    """An enabled slot that never closes a loop next to a plain slot on the same drive: their device stores are equal
    at every step, the enabled slot's host store is 16 bytes per DS point of every key frame, and a reset and refill
    reserves nothing new."""
    ev = long_drive(synth)
    gpu = capi.LinsGpu()
    gpu.mappers_open(2)
    gpu.mappers_loops([0, 1])
    reserved = None
    for rnd in range(2):
        pts, n_kf = 0, 0
        for e in ev:
            reps = gpu.mappers_step([e[1:7]] * 2)
            assert bytes(reps[0]) == bytes(reps[1])
            if reps[1].processed and reps[1].keyframe_saved:
                pts += ds_points(reps[1])
                n_kf += 1
            dev, host, res = gpu.mappers_store_bytes()
            assert dev[0] == dev[1] and host[0] == 0 and host[1] == 16 * pts, e[-1]
            assert dev[1] <= 16 * pts
        assert n_kf > WINDOW + 1 and dev[1] < host[1]
        if reserved is None:
            reserved = res
            assert res >= host[1]
        else:
            assert res == reserved
        gpu.mappers_reset([1, 1])
        gpu.mappers_loops([0, 1])
    s = capi.LinsGpu()
    s.mapper_reset()
    s.mapper_loops()
    for e in ev:
        s.mapper_step(*e[1:7])
    d, h, r = s.mapper_store_bytes()
    assert (d, h) == (int(dev[1]), int(host[1])) and r >= h


def _store(t):
    if t.s is None:
        return t.g.mapper_store_bytes()[:2]
    dev, host, _ = t.g.mappers_store_bytes(t.mask())
    return int(dev[t.s]), int(host[t.s])


def test_saves_of_a_long_drive_load_and_continue(capi, synth):
    """Saves at several points of a long drive with closures (after a forced closure, on the stale estimate, with the
    newest 51 key frames only a part of the store), each loaded into a fresh slot of either API in another context:
    every later output byte-equal, the blob saved again byte-equal, the host store the source's, the device store at
    most the source's and equal to it from the next key-frame save on."""
    stall = 2 * LONG_OUT - 10
    events = long_drive(synth, stall_at=stall)
    force = {stall - 1}
    src = tc.new_target(capi, "single", loops=True)
    save_at = {30, stall - 1, stall, stall + 4, len(events) - 6}
    last_close, log, ticks, stores, points = None, [], set(), [], {}
    for i, e in enumerate(events):
        f = src.fuse(e)
        rep = src.step(e)
        d = src.download()
        lr = gm = None
        if src.rep is not None:
            due = last_close is None or e[1] - last_close >= 1.0
            if due:
                last_close = e[1]
            if due or e[-1] in force:
                ticks.add(i)
                lr = bytes(src.close())
                gm = src.global_map()
        log.append((f, bytes(rep), d, lr, gm))
        stores.append(_store(src))
        if i in save_at:
            points[i] = src.save()
    assert len(points) == len(save_at)
    for j, (i, blob) in enumerate(sorted(points.items())):
        t = tc.new_target(capi, ["single", "lockstep"][j % 2], loops=j % 4 < 2)
        t.load(blob)
        assert t.save() == blob, i
        dev, host = _store(t)
        assert host == stores[i][1] and dev <= stores[i][0], i
        tc.continue_loops(events, log, ticks, i, False, t)
        assert _store(t) == stores[-1], i
    # a lockstep slot's blob into a single mapper and back (the formats are one)
    last = points[max(points)]
    t = tc.new_target(capi, "lockstep")
    t.load(last)
    u = tc.new_target(capi, "single")
    u.load(t.save())
    assert u.save() == last


def test_launch_counts(capi, synth):
    """step, close_loops, global map, save and load launch what they launched with the whole store on the device: a
    step as a plain slot's, a close_loops one gather, one segmented VoxelGrid and the ICP, a global map one gather and
    one VoxelGrid per pass, a save one gather, a load at most two."""
    ev = long_drive(synth)
    g = capi.LinsGpu()
    g.mappers_open(2)
    g.mappers_loops([1, 0])
    p = capi.LinsGpu()
    p.mappers_open(2)
    for e in ev:
        n0, m0 = g.launch_count(), p.launch_count()
        g.mappers_step([e[1:7]] * 2)
        p.mappers_step([e[1:7]] * 2)
        assert g.launch_count() - n0 == p.launch_count() - m0, e[-1]
    n0 = g.launch_count()
    lr = g.mappers_close_loops([1, 0])[0]
    assert lr.closest_history_frame_id >= 0 and lr.n_source > 0
    assert g.launch_count() - n0 == 1 + 7 + 2 * 101
    n0 = g.launch_count()
    rep = g.mappers_global_map([1, 0])[0]
    assert rep.n_points > 0 and g.launch_count() - n0 == 1 + 7
    n0 = g.launch_count()
    blobs = g.mappers_save([1, 1])
    assert g.launch_count() - n0 == 1
    h = capi.LinsGpu()
    h.mappers_open(2)
    n0 = h.launch_count()
    h.mappers_load([1, 1], blobs)
    assert h.launch_count() - n0 == 2
