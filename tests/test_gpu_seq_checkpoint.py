"""GPU suite: saving sequence-mode slots and loading them into fresh slots (lins_gpu_seq_save_size / _save / _load).

Drives of tests/rawcases.py (one edited so that a running scan fails the map refresh guard) run through a context A
(two slots configured, two tuned, one of them both; bound runs also feed their mappers IMU rows), through seq_step_raw
or seq_step_cloud2.  Every slot of A is saved at every step.  At each step where A first holds a state a load must carry
(a slot in INIT, one in FIRST_SCAN part-way through its pre-integration, a SKIPPED scan, a stale 1-NN index; and at
fixed steps), the blobs are loaded into a fresh context B with more slots at a permutation of the slot indices, one of
the destination slots configured and tuned before the load with a config and a tuning its blob does not have.  A and B
then step on the same inputs to the end, and every slot of B equals its slot of A byte for byte: the rows, statuses and
maps, the IESKF results of the slots that ran, the published poses and sizes, the mapper reports, key poses, window and
clouds of processed cycles.  A twin of A that never saves equals A (save is read-only).  A configured and tuned slot's
blob, loaded and then restarted, replays a drive as a slot that was never configured or tuned does.  Long bound drives
(240 scans) reach a mapper window of 50 key frames with the duplicate id and a first key frame whose clouds fail the
10 / 100 gate, and are loaded there.  A saved slot loaded into a spare slot of its own run continues as its source does.  Rejected loads change nothing.  bag_replay.replay stopped with
a checkpoint and resumed in a new context (seq_step_cloud2) returns what an uninterrupted replay returns, with map=True
and map=False."""
import os

import numpy as np
import pytest

import cloud2cases as c2
import pclcases as pc
import rawcases as rc
from conftest import ROOT, pkg
from test_gpu_seq_init import init_params

pytestmark = pytest.mark.gpu
br = pkg("bag_replay")
synth = pkg("synth")
SEQ_SKIPPED, SEQ_RAN, SEQ_ICP = 1, 2, 3
GUARD_LOG = 3


@pytest.fixture(scope="module")
def logs(capi, defs):
    logs, _ = rc.case_logs(defs, 0, gpu=capi.LinsGpu())
    logs = logs[:8]
    # scan 5 of one drive cut to a window of its sweep (in firing order) whose features pass the processScan gate
    # (ncl > 5 && nsl > 10) but fail the map refresh guard (ncl >= 5 && nsl >= 20): the slot then searches a stale index
    sw, m = logs[GUARD_LOG]["sweeps"][5], rc.model_of(defs, logs[GUARD_LOG])
    for w in range(96, 1200, 48):
        cut = next((sw[a:a + w] for a in range(0, len(sw) - w, 512) if _guard_case(*pc.counts(defs, rc.host_scan(defs, sw[a:a + w], m)))), None)
        if cut is not None:
            logs[GUARD_LOG]["sweeps"][5] = cut.copy()
            break
    assert cut is not None
    return logs


def _guard_case(ncl, nsl):
    return ncl > 5 and 10 < nsl < 20


def _open(capi, defs, n, bound):
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n)
    if bound:
        g.seq_map_open()
    return g


def _cfg(defs):
    return defs.LinsSlotConfig.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0), init_vel_std=(0.5, 0.5, 0.5), acc_n=60000.0)


def _tun(defs):
    return defs.LinsSlotTuning.shipped(num_iter=12, nearest_feature_search_sq_dist=16.0, imu_misalign_angle=1.5)


def _rig(defs, g, slots_cfg, slots_tune, n):
    """slots slots_cfg configured (a rig of other init stds and noise), slots slots_tune tuned (fewer iterations, another
    gate, a misalignment)"""
    m = np.zeros(n, np.uint8); m[slots_cfg] = 1
    g.seq_configure(m, [_cfg(defs) if x else None for x in m])
    m = np.zeros(n, np.uint8); m[slots_tune] = 1
    g.seq_tune(m, [_tun(defs) if x else None for x in m])


def _inputs(logs, t, slot_log, n, empty=()):
    """step t's inputs of n slots, slot j driving logs[slot_log[j]] (None: absent); log 2's 4th step is absent, and the
    scans (log, step) in `empty` are present with an empty sweep"""
    sweeps, imus, scan_imu, time, present = [], [], np.zeros((n, 6)), np.zeros(n), np.zeros(n, np.uint8)
    for j in range(n):
        li = slot_log.get(j)
        if li is None or t >= len(logs[li]["time"]) or (t == 3 and li == 2):
            sweeps.append(np.zeros((0, 4), np.float32)); imus.append(np.zeros((0, 7)))
            continue
        o = logs[li]["imu_off"]
        sweeps.append(np.zeros((0, 4), np.float32) if (li, t) in empty else logs[li]["sweeps"][t]); imus.append(logs[li]["imu"][o[t]:o[t + 1]])
        scan_imu[j], time[j], present[j] = logs[li]["imu_last"][t], logs[li]["time"][t], 1
    step = dict(imu=np.concatenate(imus).reshape(-1, 7), imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32),
                present=present, sweeps=sweeps)
    return step, scan_imu, time


def _msgs(defs, sweeps, present):
    """one PointCloud2 message (layout, data field) per slot, of the slot's sweep as the driver encodes it"""
    out = []
    for sw, p in zip(sweeps, present):
        msg, _ = c2.message("velodyne32", np.asarray(sw, np.float64).reshape(-1, 4))
        out.append(c2.as_input(defs, msg) if p else (defs.LinsCloud2Layout(), b""))
    return out


def _step(g, logs, t, slot_log, n, model, bound, entry="raw", defs=None, empty=()):
    step, scan_imu, time = _inputs(logs, t, slot_log, n, empty)
    if bound:  # IMU messages for the mapping nodes (imuHandler), two per present slot
        g.mappers_imu([(time[j] - np.array([0.02, 0.01]), [0.01 * t, 0.02], [0.0, -0.01 * slot_log[j]]) if step["present"][j] else None
                       for j in range(n)])
    if entry == "cloud2":
        g.seq_step_cloud2(dict(step, msgs=_msgs(defs, step["sweeps"], step["present"])), model=model, scan_imu=scan_imu)
    else:
        g.seq_step_raw(step, model=model, scan_imu=scan_imu)
    return g.seq_map_step(time) if bound else (None, None)


def _slot_state(g, s, d, di, mp, reps, pub, published):
    """slot s's observable state after a step, as bytes"""
    out = [d[k][s].tobytes() for k in ("global_state", "filter_state", "filter_cov", "status")]
    if int(d["status"][s]) in (SEQ_RAN, SEQ_ICP):
        r = np.asarray(d["results"])[s]  # (its scan_id is the slot index)
        out += [r["iters"].tobytes(), r["flags"].tobytes(), r["pose"].tobytes()]
        # the report's per-iteration rows past its iterations are not written by the step
        rp = d["reports"][s]
        k = rp.iters
        out += [(rp.iters, rp.converged, rp.diverged, rp.has_nan)] + [bytes(memoryview(getattr(rp, f)))[:k * 8] for f in ("residual_norm", "update_norm")]
        out += [list(rp.m_surf)[:k], list(rp.m_corner)[:k]]
    out.append(di["fusion_status"][s].tobytes())
    out += [mp[k][s].tobytes() for k in ("surf_map", "corner_map", "surf_tree", "corner_tree")] + [mp["stale"][s].tobytes()]
    if published is not None:
        pose, sizes = published
        out += [pose[s].tobytes(), sizes[s].tobytes(), pub[s].tobytes()]
        if pub[s]:
            out.append(bytes(reps[s]))
            if reps[s].processed:
                kp, win, clouds = g.mappers_download(s, reps[s])
                out += [kp.tobytes(), win.tobytes()] + [clouds[k].tobytes() for k in sorted(clouds)]
    return out


def _state(g, slots, reps, pub, bound):
    d, di, mp = g.seq_download(reports=True), g.seq_download_init(), g.seq_download_maps()
    published = g.seq_map_published() if bound else None
    return [_slot_state(g, s, d, di, mp, reps, pub, published) for s in slots]


def _diff(sa, sb):
    return [(j, i) for j in range(len(sa)) for i in range(max(len(sa[j]), len(sb[j]))) if i >= min(len(sa[j]), len(sb[j])) or sa[j][i] != sb[j][i]]


def _load_into_new(capi, defs, blobs, n, bound, rng, configure=None):
    """the blobs of n slots loaded into a fresh run of n + 3 slots at a permutation; `configure` (a source slot): its
    destination is configured and tuned before the load with a config and a tuning its blob does not carry"""
    perm = rng.permutation(n + 3)[:n]
    b = _open(capi, defs, n + 3, bound)
    if configure is not None:
        m = np.zeros(n + 3, np.uint8); m[perm[configure]] = 1
        b.seq_configure(m, [_cfg(defs) if x else None for x in m])
        b.seq_tune(m, [_tun(defs) if x else None for x in m])
    mask = np.zeros(n + 3, np.uint8); mask[perm] = 1
    bl = [None] * (n + 3)
    for j in range(n):
        bl[perm[j]] = blobs[j]
    b.seq_load(mask, bl)
    assert b.seq_download()["status"][perm].tolist() == [0] * n  # LINS_SEQ_IDLE until the next step
    return b, perm, {int(perm[j]): j for j in range(n)}


@pytest.mark.parametrize("entry", ["raw", "cloud2"])
@pytest.mark.parametrize("bound", [False, True])
def test_continuation_bit_identical(capi, defs, logs, bound, entry):
    n = len(logs)
    model = rc.model_of(defs, logs[0])
    T = max(len(l["time"]) for l in logs)
    slot_log = {j: j for j in range(n)}
    a, twin = _open(capi, defs, n, bound), _open(capi, defs, n, bound)
    for g in (a, twin):
        _rig(defs, g, [0, 1], [1, 4], n)
    resumed = []  # (B, perm, its slot -> log map)
    loaded_states = set()
    history = []  # A's state after each step
    rng = np.random.default_rng(7)
    for t in range(T):
        ra, pa = _step(a, logs, t, slot_log, n, model, bound, entry, defs)
        rt, pt = _step(twin, logs, t, slot_log, n, model, bound, entry, defs)
        sa = _state(a, range(n), ra, pa, bound)
        history.append(sa)
        assert sa == _state(twin, range(n), rt, pt, bound), t  # save is read-only
        for b, perm, blog in resumed:
            rb, pbb = _step(b, logs, t, blog, n + 3, model, bound, entry, defs)
            sb = _state(b, perm, rb, pbb, bound)
            assert sb == sa, (t, perm, _diff(sa, sb))
        d, di, mp = a.seq_download(), a.seq_download_init(), a.seq_download_maps()
        here = {("fusion", int(x)) for x in di["fusion_status"]} | {("status", int(x)) for x in d["status"]}
        here |= {("stale", int(x)) for x in mp["stale"]}
        blobs = a.seq_save(np.ones(n, np.uint8))  # at every step: the twin never saves
        if (here - loaded_states) & REQUIRED or t + 1 in (2, 9):
            loaded_states |= here
            resumed.append(_load_into_new(capi, defs, blobs, n, bound, rng, configure=2))
    # every state a load must carry was in a loaded set of blobs: INIT, FIRST_SCAN (each first scan's pre-integration part-
    # way), RUNNING, a SKIPPED scan, a stale index; the configured and tuned slots are in every one
    assert REQUIRED <= loaded_states, REQUIRED - loaded_states
    assert len(resumed) >= 3
    # slot 1's last blob (configured and tuned) loaded into a fresh run and restarted: the slot then replays log 2 with
    # the run's values, as A's slot 2, never configured or tuned, did
    c = _open(capi, defs, n, bound)
    m = np.eye(n, dtype=np.uint8)[1]
    c.seq_load(m, [blobs[1] if x else None for x in m])
    c.seq_restart(m)
    for t in range(T):
        rc_, pc_ = _step(c, logs, t, {1: 2}, n, model, bound, entry, defs)
        sc = _state(c, [1], rc_, pc_, bound)
        assert sc == [history[t][2]], (t, _diff([history[t][2]], sc))


REQUIRED = {("fusion", 0), ("fusion", 1), ("fusion", 3), ("status", SEQ_SKIPPED), ("stale", 1)}


def test_long_mapper_continuation(capi, defs):
    """Bound runs of 240-scan drives: drive 1's second sweep is empty (its first key frame has no clouds, so the next
    processed cycle fails the 10 / 100 gate); once a slot's mapper holds 50 key poses, its next four sweeps are empty
    (no motion: the cycle that fills the window to 50 saves no key frame, and the next one pushes the newest id again).
    The blobs are loaded at each of those states and every loaded run stays equal to the source to the end."""
    model = defs.LinsLidarModel.vlp16()
    logs = [synth.raw_log("config3", seed=21 + i, n_scans=240) for i in range(2)]
    logs[1]["sweeps"][1] = np.zeros((0, 4), np.float32)
    n = len(logs)
    slot_log = {j: j for j in range(n)}
    a = _open(capi, defs, n, True)
    empty, kf, resumed, seen = set(), [0] * n, [], set()
    rng = np.random.default_rng(11)
    for t in range(240):
        ra, pa = _step(a, logs, t, slot_log, n, model, True, empty=empty)
        sa = _state(a, range(n), ra, pa, True)
        for b, perm, blog in resumed:
            rb, pbb = _step(b, logs, t, blog, n + 3, model, True, empty=empty)
            sb = _state(b, perm, rb, pbb, True)
            assert sb == sa, (t, perm, _diff(sa, sb))
        new = set()
        for j in range(n):
            r = ra[j]
            if r is None or not r.processed:
                continue
            if kf[j] >= 1 and r.map.skipped and "gate" not in seen:
                new.add("gate")
            if r.n_keyframes >= 50 and kf[j] < 50:
                empty |= {(slot_log[j], t + i) for i in range(1, 5)}
            _, win, _ = a.mappers_download(j, r)
            if len(win) == 50 and len(set(win.tolist())) < 50 and "window50_dup" not in seen:
                new.add("window50_dup")
            kf[j] = r.n_keyframes
        if new:
            seen |= new
            resumed.append(_load_into_new(capi, defs, a.seq_save(np.ones(n, np.uint8)), n, True, rng))
    assert seen == {"gate", "window50_dup"}, (seen, kf)


def test_migration_within_a_run(capi, defs, logs):
    n = 4
    model = rc.model_of(defs, logs[0])
    g = _open(capi, defs, n + 1, True)
    slot_log = {j: j for j in range(n)}
    for t in range(len(logs[0]["time"])):
        if t == 4:
            blob = g.seq_save(np.eye(n + 1, dtype=np.uint8)[0])[0]
            g.seq_load(np.eye(n + 1, dtype=np.uint8)[n], [None] * n + [blob])
            slot_log[n] = 0
        reps, pub = _step(g, logs, t, slot_log, n + 1, model, True)
        if t >= 4:
            s0, s1 = _state(g, [0, n], reps, pub, True)
            assert s0 == s1, t


def test_rejections_change_nothing(capi, defs, logs):
    n = 4
    model = rc.model_of(defs, logs[0])
    slot_log = {j: j for j in range(n)}
    a, twin = _open(capi, defs, n + 1, True), _open(capi, defs, n + 1, True)
    for t in range(3):
        _step(a, logs, t, slot_log, n + 1, model, True); _step(twin, logs, t, slot_log, n + 1, model, True)
    blobs = a.seq_save(np.array([1] * n + [0], np.uint8))
    spare = np.eye(n + 1, dtype=np.uint8)[n]
    L = a.L
    bad = []
    good = blobs[0]
    flipped = bytearray(good); flipped[0] ^= 1
    bad.append([None] * n + [bytes(flipped)])                 # a corrupt blob
    bad.append([None] * n + [good[:-16]])                      # a truncated blob
    for blob_list in bad:
        with pytest.raises(capi.LinsError):
            a.seq_load(spare, blob_list)
    with pytest.raises(capi.LinsError):                        # a non-fresh destination
        a.seq_load(np.eye(n + 1, dtype=np.uint8)[1], [None, good] + [None] * (n - 1))
    u = _open(capi, defs, 2, False)                            # a binding mismatch (both ways)
    with pytest.raises(capi.LinsError):
        u.seq_load(np.array([1, 0], np.uint8), [good, None])
    with pytest.raises(capi.LinsError):
        a.seq_load(spare, [None] * n + [u.seq_save(np.array([1, 0], np.uint8))[0]])
    o = capi.LinsGpu()                                         # other open constants, for an unconfigured blob
    o.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), 2)
    with pytest.raises(capi.LinsError):
        o.seq_load(np.array([1, 0], np.uint8), [u.seq_save(np.array([1, 0], np.uint8))[0], None])
    m = np.ascontiguousarray(spare)
    off = np.zeros(n + 2, np.uint64)
    assert L.lins_gpu_seq_save_size(a.h, capi.ptr(m), capi.ptr(off)) == 0
    buf = np.zeros(max(int(off[-1]), 16), np.uint8)
    off2 = off.copy(); off2[-1] += 16
    assert L.lins_gpu_seq_save(a.h, capi.ptr(m), capi.ptr(buf), capi.ptr(off2)) == -1  # offsets other than save_size's
    assert L.lins_gpu_seq_save(a.h, None, capi.ptr(buf), capi.ptr(off)) == -1         # no mask
    assert L.lins_gpu_seq_load(a.h, capi.ptr(m), capi.ptr(buf), None) == -1           # no offsets
    # a pending publish: saving and loading both refuse
    step, scan_imu, time = _inputs(logs, 3, slot_log, n + 1)
    a.seq_step_raw(step, model=model, scan_imu=scan_imu); twin.seq_step_raw(step, model=model, scan_imu=scan_imu)
    with pytest.raises(capi.LinsError):
        a.seq_save(np.ones(n + 1, np.uint8))
    with pytest.raises(capi.LinsError):
        a.seq_load(spare, [None] * n + [good])
    ra, pa = a.seq_map_step(time); rt, pt = twin.seq_map_step(time)
    assert _state(a, range(n + 1), ra, pa, True) == _state(twin, range(n + 1), rt, pt, True)
    for t in range(4, 8):
        ra, pa = _step(a, logs, t, slot_log, n + 1, model, True); rt, pt = _step(twin, logs, t, slot_log, n + 1, model, True)
        assert _state(a, range(n + 1), ra, pa, True) == _state(twin, range(n + 1), rt, pt, True), t


@pytest.mark.parametrize("map_", [False, True])
def test_replay_checkpoint_and_resume(capi, tmp_path, map_):
    bag = os.path.join(ROOT, "tests", "golden", "tiny.bag")
    recs = [br.Recording(bag, max_scans=m) for m in (0, 4, 7, 2, 0)]
    full = br.replay(recs, 2, map=map_)
    steps = sum(1 for _ in br.slot_queue([len(r) for r in recs], 2))
    for k in sorted({k for k in (1, steps // 3, steps // 2, steps - 1) if 1 <= k < steps}):
        ck = str(tmp_path / f"ck{k}_{int(map_)}")
        assert br.replay(recs, 2, map=map_, checkpoint=ck, stop_after=k) is None
        got = br.replay(recs, 2, map=map_, resume=ck)
        for a, b in zip(full, got):
            assert a.keys() == b.keys()
            for key in a:
                x, y = np.asarray(a[key]), np.asarray(b[key])
                assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (k, key)
    # checkpoints written along a run that goes on, and a resume from the last of them
    ck = str(tmp_path / f"every_{int(map_)}")
    again = br.replay(recs, 2, map=map_, checkpoint=ck, checkpoint_every=2)
    got = br.replay(recs, 2, map=map_, resume=ck)
    for a, b, c in zip(full, again, got):
        for key in a:
            assert np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes() == np.asarray(c[key]).tobytes(), key
