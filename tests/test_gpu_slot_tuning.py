"""GPU suite: per-slot estimator tuning and IMU misalignment (lins_gpu_seq_tune), so every value of exp_port.yaml the
odometry reads can differ from slot to slot in one lockstep run.

The contract: a tuned slot is bit-identical to the same recording in the same slot of a twin context whose lins_params
equal its tuning and whose IMU rows and scan_imu samples were rotated on the host by alignIMUtoVehicle
(rig_config.misalign_R / align_imu: Python's math.cos / math.sin, the library's expression); an untuned slot reads the
context's lins_params and its IMU values as they come.
- Twin parity: 24 slots, three tunings that differ in every field (NUM_ITER 30 / 12 / 5, ICP_FREQ 1 / 2 / 3, the gate
  25 / 1 / 400, LIDAR_STD 0.01 / 0.05 / 0.002, LIDAR_SCALE 1 / 0.5 / 2, misalignment 0 / 3 / -2.5 degrees) interleaved
  with untuned slots, so one CTA holds units of different tunings; some tuned slots are configured as well, tuned before
  or after the configuration.  Through seq_step_raw_mixed (VLP-16 and 64 x 1024), seq_step_raw and
  seq_step_cloud2_mixed.  The second scans' batched estimateTransform mixes the caps.
- A pass with LIDAR_SCALE 1e9 in one tuning: only its slots take the estimateTransform fallback, beside slots with
  other caps; icp_iters / icp_pose equal the twins'.
- Every slot tuned to the run's values with no misalignment equals the untuned run, before and after restarts, and an
  untuned run launches what it launched before.
- Bags: two bags whose config files differ in tuning and misalignment replayed together, each against the shim's tuned
  run_bag and against itself alone; one bound run.
- Invalid calls change nothing.
- Gates against the oracle: the gate-1 and gate-400 slots' IESKF against the CPU oracle at their gate, NUM_ITER and
  ICP_FREQ, from their own prior: the correspondence IDs exactly, the posterior to 1e-7."""
import ctypes as C

import numpy as np
import pytest

import cloud2cases as cc
from conftest import pkg
from test_gpu_mixed_models import _slot_rows
from test_gpu_seq_pcl import _snapshot
from test_gpu_slot_config import RIGS, _jobs as _config_jobs, _models, _step_inputs, logs  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
synth = pkg("synth")
br = pkg("bag_replay")
rcfg = pkg("rig_config")

TUNINGS = [dict(num_iter=30, icp_freq=1, nearest_feature_search_sq_dist=25.0, lidar_std=0.01, lidar_scale=1.0, imu_misalign_angle=0.0),
           dict(num_iter=12, icp_freq=2, nearest_feature_search_sq_dist=1.0, lidar_std=0.05, lidar_scale=0.5, imu_misalign_angle=3.0),
           dict(num_iter=5, icp_freq=3, nearest_feature_search_sq_dist=400.0, lidar_std=0.002, lidar_scale=2.0, imu_misalign_angle=-2.5)]


def _rotated(log, angle):
    """A copy of a raw log with every IMU value rotated by alignIMUtoVehicle (rows: dt, acc, gyr; imu_last: acc, gyr)."""
    R = rcfg.misalign_R(angle)
    out = dict(log)
    imu = np.array(log["imu"], np.float64, copy=True).reshape(-1, 7)
    for m in range(len(imu)):
        imu[m, 1:4] = rcfg.align_imu(R, imu[m, 1:4])
        imu[m, 4:7] = rcfg.align_imu(R, imu[m, 4:7])
    last = np.array(log["imu_last"], np.float64, copy=True)
    for k in range(len(last)):
        last[k, 0:3] = rcfg.align_imu(R, last[k, 0:3])
        last[k, 3:6] = rcfg.align_imu(R, last[k, 3:6])
    out["imu"], out["imu_last"] = imu, last
    return out


class Ctx:
    """A context whose lins_params are one tuning (None: the run's) with one rig (None: the run's)."""

    def __init__(self, capi, defs, tune, cfg, n_slots):
        c = cfg or defs.LinsSlotConfig.shipped()
        kw = {k: v for k, v in (tune or {}).items() if k != "imu_misalign_angle"}
        self.g = capi.LinsGpu(defs.LinsParams.shipped(scan_period=c.scan_period, **kw))
        self.g.seq_open(c.filter, c.init, n_slots)
        self.fp = c.features


def drive(capi, defs, jobs, tunes, n_slots, models, raw=False, cloud2=False, tune_first=False, tune_defaults=False):
    """jobs: (tuning index or None, config index or None, model index, raw log).  The main context runs them through
    n_slots slots, tuning (and configuring) a slot with its job's values when it takes the job (tune_defaults: the untuned
    jobs too, with the run's values and no misalignment); one twin per (tuning, config) pair steps the same slots with only
    its own jobs present, their IMU values rotated on the host.  Every present slot equals its twin's slot after every
    step.  Returns (rows[job] = [(scan, slot row)], the set of scan_status codes per tuning)."""
    cfgs = [defs.LinsSlotConfig.shipped(**r) for r in RIGS]
    run_tune = {k: getattr(defs.LinsParams.shipped(), k) for k in TUNINGS[0] if k != "imu_misalign_angle"}
    run_tune["imu_misalign_angle"] = 0.0
    keys = sorted({(j[0], j[1]) for j in jobs}, key=lambda k: tuple(-1 if x is None else x for x in k))
    main = Ctx(capi, defs, None, None, n_slots)
    twins = {k: Ctx(capi, defs, None if k[0] is None else tunes[k[0]], None if k[1] is None else cfgs[k[1]], n_slots) for k in keys}
    tjobs = [(j[0], j[1], j[2], j[3] if j[0] is None else _rotated(j[3], tunes[j[0]]["imu_misalign_angle"])) for j in jobs]
    rows, codes, t = [[] for _ in jobs], {k[0]: set() for k in keys}, 0
    for restart, who in br.slot_queue([len(j[3]["time"]) for j in jobs], n_slots):
        if restart.any():
            for c in [main] + list(twins.values()):
                c.g.seq_restart(restart)
        first = [w is not None and w[1] == 0 for w in who]

        def tune():
            m = np.array([f and (jobs[w[0]][0] is not None or tune_defaults) for w, f in zip(who, first)], np.uint8)
            if m.any():
                main.g.seq_tune(m, [defs.LinsSlotTuning.shipped(**(tunes[jobs[w[0]][0]] if jobs[w[0]][0] is not None else run_tune)) if f else None
                                    for w, f in zip(who, m)])

        def configure():
            m = np.array([f and jobs[w[0]][1] is not None for w, f in zip(who, first)], np.uint8)
            if m.any():
                main.g.seq_configure(m, [cfgs[jobs[w[0]][1]] if f else None for w, f in zip(who, m)])
        for call in ((tune, configure) if tune_first or t % 2 else (configure, tune)):
            call()
        present = np.array([w is not None for w in who], np.uint8)
        of = np.array([jobs[w[0]][2] if w else 0 for w in who], np.int32)
        key = [(jobs[w[0]][0], jobs[w[0]][1]) if w else "absent" for w in who]

        def step(c, pres, js):
            sweeps, imu, imu_off, si = _step_inputs([(a, m, l) for a, _, m, l in js], who, n_slots)
            msgs = [cc.as_input(defs, cc.message("velodyne32", sw, seq=t)[0]) for sw in sweeps] if cloud2 else None
            st = dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=pres, msgs=msgs)
            if cloud2:
                c.g.seq_step_cloud2_mixed(st, models, of, fp=c.fp, scan_imu=si)
            elif raw:
                c.g.seq_step_raw(st, model=models[0], fp=c.fp, scan_imu=si)
            else:
                c.g.seq_step_raw_mixed(st, models, of, fp=c.fp, scan_imu=si)

        step(main, present, jobs)
        rg = _slot_rows(main.g, present)
        for k, tw in twins.items():
            mine = np.array([p and key[s] == k for s, p in enumerate(present)], np.uint8)
            if not mine.any():
                continue
            step(tw, mine, tjobs)
            rt = _slot_rows(tw.g, mine)
            for s in np.flatnonzero(mine):
                assert rg[s] == rt[s], f"step {t}: slot {s} (tuning, config {k}) differs from its twin"
                codes[k[0]].add(int(np.frombuffer(rg[s]["status"], np.int32)[0]))
        for j, w in enumerate(who):
            if w is not None:
                rows[w[0]].append((w[1], rg[j]))
        t += 1
    return rows, codes


def _jobs(logs):
    """24 jobs of test_gpu_slot_config's drives: per tuning key (None, 0, 1, 2) in turn, every other tuned job configured
    with RIGS[0] or RIGS[1] as well."""
    out = []
    for i, (k, _, m, l) in enumerate((k, None, m, l) for k, m, l in _config_jobs(logs)):
        c = None if k is None or (i // 4) % 2 == 0 else (i // 4) % 3 % 2
        out.append((k, c, m, l))
    return out


def _want_codes(defs, codes, icp_key=None):
    for k in (0, 1, 2):
        want = {defs.SEQ_SECOND, defs.SEQ_SKIPPED} | ({defs.SEQ_ICP} if k == icp_key else {defs.SEQ_RAN})
        assert want <= codes[k], (k, codes[k])
        if icp_key is not None and k != icp_key:
            assert defs.SEQ_ICP not in codes[k], (k, codes[k])


def test_tuned_slots_equal_their_twins_mixed(capi, defs, logs):
    jobs = _jobs(logs)
    assert len(jobs) >= 24 and {j[1] for j in jobs if j[0] is not None} >= {None, 0, 1}
    _, codes = drive(capi, defs, jobs, TUNINGS, len(jobs), _models(defs))
    _want_codes(defs, codes)


def test_tuned_slots_equal_their_twins_step_raw(capi, defs, logs):
    jobs = [j for j in _jobs(logs) if j[2] == 0]
    _, codes = drive(capi, defs, jobs, TUNINGS, len(jobs), _models(defs)[:1], raw=True, tune_first=True)
    _want_codes(defs, codes)


def test_tuned_slots_equal_their_twins_cloud2_mixed(capi, defs, logs):
    jobs = _jobs(logs)
    _, codes = drive(capi, defs, jobs, TUNINGS, len(jobs), _models(defs), cloud2=True)
    _want_codes(defs, codes)


def test_only_one_tunings_slots_take_the_fallback(capi, defs, logs):
    """LIDAR_SCALE 1e9 in the NUM_ITER-12 tuning: its running scans diverge and run the estimateTransform fallback capped
    at 12, beside the slots of the 30 and 5 caps that do not; the init rows (icp_pose, icp_iters) equal the twins'."""
    tunes = [dict(t) for t in TUNINGS]
    tunes[1]["lidar_scale"] = 1e9
    _, codes = drive(capi, defs, _jobs(logs), tunes, 24, _models(defs))
    _want_codes(defs, codes, icp_key=1)


def test_tuning_the_run_values_changes_nothing(capi, defs, logs):
    """Every slot tuned to the run's own values with no misalignment, through fewer slots (restarts return slots to
    untuned and they are tuned again): bit-identical to the untuned run; an untuned run launches what it did before."""
    jobs = [(None, None, m, l) for _, _, m, l in _jobs(logs)[::2]]
    plain, _ = drive(capi, defs, jobs, TUNINGS, 5, _models(defs))
    same, _ = drive(capi, defs, jobs, TUNINGS, 5, _models(defs), tune_defaults=True)
    assert plain == same


def test_untuned_run_launch_count(capi, defs, logs):
    """A run without a tuned slot launches no alignment kernel; a tuned slot with IMU rows adds exactly one per step."""
    vlp = logs[0]
    S = 3
    counts = []
    for tuned in (False, True):
        g = capi.LinsGpu()
        g.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
        if tuned:
            g.seq_tune(np.array([0, 1, 0], np.uint8), [None, defs.LinsSlotTuning.shipped(imu_misalign_angle=0.0), None])
        per = []
        for t in range(4):
            sweeps = [vlp[i]["sweeps"][t] for i in range(S)]
            imus = [vlp[i]["imu"][vlp[i]["imu_off"][t]:vlp[i]["imu_off"][t + 1]] for i in range(S)]
            st = dict(sweeps=sweeps, imu=np.concatenate(imus).reshape(-1, 7),
                      imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32))
            si = np.ascontiguousarray(np.stack([vlp[i]["imu_last"][t] for i in range(S)]), np.float64)
            n0 = g.launch_count()
            g.seq_step_raw(st, scan_imu=si)
            per.append(g.launch_count() - n0)
        counts.append(per)
    assert [b - a for a, b in zip(*counts)] == [1, 1, 1, 1], counts


# the bags' config files: exp_port.yaml's tuning with no misalignment, and one that differs in every tuning key and is 3
# degrees misaligned
BAG_TUNINGS = [dict(TUNINGS[0]), dict(num_iter=12, icp_freq=2, nearest_feature_search_sq_dist=9.0, lidar_std=0.02, lidar_scale=0.5,
                                      imu_misalign_angle=3.0)]


def _bag_tuning(k):
    return None if k is None else BAG_TUNINGS[k]


def test_bags_with_their_tuning_and_misalignment(capi, defs, tmp_path):
    """Two bags whose config files differ in tuning and misalignment (0 and 3 degrees) and a bag without either, replayed
    together through 2 slots: each equals its replay alone, and that replay agrees with the shim's tuned run_bag to the
    tolerance of the other bag tests.  Then one run bound to the mappers with the tuned slots."""
    plan = [(1, 1), (None, None), (0, 0)]  # (tuning, rig)
    paths = []
    for s, (_, rig) in enumerate(plan):
        p = str(tmp_path / f"bag{s}.bag")
        synth.write_sequence_bag(p, config="config3", seed=90 + s, n_scans=10 - s, scan_period=None if rig is None else RIGS[rig]["scan_period"])
        paths.append(p)
    recs = [br.Recording(p, config=None if r is None else defs.LinsSlotConfig.shipped(**RIGS[r]),
                         tuning=None if k is None else rcfg.slot_tuning(_bag_tuning(k))) for p, (k, r) in zip(paths, plan)]
    together = br.replay(recs, 2)
    for rec, o, (k, r) in zip(recs, together, plan):
        alone = br.replay([rec], 1)[0]
        for key in o:
            assert o[key].tobytes() == alone[key].tobytes(), (rec.path, key)
        ref = synth.run_bag(rec.path, rig=None if r is None else RIGS[r], tuning=_bag_tuning(k))
        assert np.array_equal(o["status"], ref["status"]), (rec.path, o["status"], ref["status"])
        ran = np.flatnonzero(o["iters"] >= 0)
        assert len(ran) >= 3 and np.array_equal(ran, np.asarray(ref["scan_index"])), (ran, ref["scan_index"])
        assert np.array_equal(o["iters"][ran], ref["iters"]) and np.array_equal(o["flags"][ran], ref["flags"])
        diff = np.abs(o["global_est"] - ref["global_est"]).max()
        assert diff <= 1e-7, (rec.path, diff)
    # the misalignment is applied: the 3 degree bag differs from its replay without tuning
    plain = br.replay([br.Recording(paths[0], config=recs[0].config)], 1)[0]
    assert np.abs(plain["global_est"] - together[0]["global_est"]).max() > 1e-6
    bound = br.replay(recs, 2, map=True)
    for o, m in zip(together, bound):
        assert o["global_est"].tobytes() == m["global_est"].tobytes()
        assert len(m["map_time"]) > 0


def test_invalid_tune_changes_nothing(capi, defs, logs):
    vlp = logs[0]
    S = 3
    good = [defs.LinsSlotTuning.shipped(**t) for t in TUNINGS]
    ref = capi.LinsGpu()
    ref.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
    L = g.L

    def call(mask, ts):
        arr = (defs.LinsSlotTuning * S)(*ts)
        return L.lins_gpu_seq_tune(g.h, np.ascontiguousarray(mask, np.uint8).ctypes.data, C.cast(arr, C.c_void_p))

    bad = []
    for field, v in (("num_iter", -1), ("num_iter", defs.LINS_MAX_ITER + 1), ("icp_freq", 0),
                     ("icp_freq", -3), ("nearest_feature_search_sq_dist", float("nan")), ("lidar_std", float("inf")),
                     ("lidar_scale", float("-inf")), ("imu_misalign_angle", float("nan"))):
        b = defs.LinsSlotTuning.shipped()
        setattr(b, field, v)
        bad.append(b)
    for t in range(5):
        if t in (0, 3):
            assert L.lins_gpu_seq_tune(g.h, None, None) == -1
            arr = (defs.LinsSlotTuning * S)(*good)
            assert L.lins_gpu_seq_tune(g.h, None, C.cast(arr, C.c_void_p)) == -1
            assert L.lins_gpu_seq_tune(g.h, np.ones(S, np.uint8).ctypes.data, None) == -1
            for b in bad:
                assert call([1, 1, 0], [good[1], b, good[2]]) == -1
            if t == 3:
                assert call([1, 0, 0], good) == -1  # slot 0 has stepped
        sweeps = [vlp[i]["sweeps"][t] for i in range(S)]
        imus = [vlp[i]["imu"][vlp[i]["imu_off"][t]:vlp[i]["imu_off"][t + 1]] for i in range(S)]
        st = dict(sweeps=sweeps, imu=np.concatenate(imus).reshape(-1, 7),
                  imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32))
        si = np.ascontiguousarray(np.stack([vlp[i]["imu_last"][t] for i in range(S)]), np.float64)
        for c in (ref, g):
            c.seq_step_raw(st, scan_imu=si)
        a, b = _snapshot(ref), _snapshot(g)
        for k in a:
            same = a[k].tobytes() == b[k].tobytes() if isinstance(a[k], np.ndarray) else a[k] == b[k]
            assert same, f"step {t}: {k}"
    h = capi.LinsGpu()
    arr = (defs.LinsSlotTuning * 1)(good[0])
    assert h.L.lins_gpu_seq_tune(h.h, np.ones(1, np.uint8).ctypes.data, C.cast(arr, C.c_void_p)) == -3
    z = np.zeros((0,), defs.POINT_DTYPE)
    h.seq_begin(defs.LinsSeqParams.shipped(), dict(filter_state=np.zeros((1, 19)), filter_cov=np.eye(18).reshape(1, 324),
                                                 global_state=np.zeros((1, 19)), imu_last=np.zeros((1, 6)), surf_map=z,
                                                 surf_map_off=np.zeros(2, np.int32), corner_map=z, corner_map_off=np.zeros(2, np.int32)))
    assert h.L.lins_gpu_seq_tune(h.h, np.ones(1, np.uint8).ctypes.data, C.cast(arr, C.c_void_p)) == -1


def test_gates_1_and_400_match_the_oracle(capi, defs, ob):
    """The twins above run the same kernel at the same gate, so a defect in how the kernel treats a non-default gate (the
    f64 compares, the f32 gate of the windows, walks and certificates, probe-then-window) would be common to both.  Here
    the gate-1 and gate-400 slots (TUNINGS[1], TUNINGS[2]: also ICP_FREQ 2 / 3 and NUM_ITER 12 / 5) run beside untuned
    and gate-25 slots, and every scan such a slot runs through the IESKF is run again by the CPU oracle at that slot's
    gate, NUM_ITER and ICP_FREQ, from the slot's prior (seq_download_ieskf) on the map the slot searched: the last
    iteration's correspondence IDs are equal, the iteration count and flags too, and the posterior agrees to 1e-7."""
    plan = [1, 2, None, 0, 1, 2]  # tuning per slot
    n_scans = 10
    logs = [synth.feature_log("config3", seed=610 + s, n_scans=n_scans) for s in range(len(plan))]
    S = len(plan)
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
    g.seq_tune(np.array([k is not None for k in plan], np.uint8),
               [None if k is None else defs.LinsSlotTuning.shipped(**TUNINGS[k]) for k in plan])
    checked = {1: 0, 2: 0}
    for k in range(n_scans):
        maps = g.seq_download_maps()
        scans = [synth.log_scan(l, k) for l in logs]
        step = dict(imu=np.concatenate([np.asarray(s["imu"]).reshape(-1, 7) for s in scans]),
                    imu_off=np.concatenate([[0], np.cumsum([len(s["imu"]) for s in scans])]))
        for c in defs.Batch.FIELDS:
            step[c] = np.concatenate([s[c] for s in scans])
            step[c + "_off"] = np.concatenate([[0], np.cumsum([len(s[c]) for s in scans])])
        g.seq_step(step, scan_imu=np.stack([s["imu_last"] for s in scans]))
        d, ie = g.seq_download(), g.seq_download_ieskf()
        for s, t in enumerate(plan):
            if t not in checked or int(d["status"][s]) != defs.SEQ_RAN or maps["stale"][s]:
                continue
            prm = defs.LinsParams.shipped(**{f: v for f, v in TUNINGS[t].items() if f != "imu_misalign_angle"})
            o = ob.Oracle(prm)
            try:
                o.set_map(maps["surf_map"][s], maps["corner_map"][s])
                so, _, rep, tr = o.ieskf_trace(scans[s]["surf_flat"], scans[s]["corner_sharp"], ie["prior_state"][s], ie["prior_cov"][s])
            finally:
                o.close()
            res = d["results"][s]
            assert int(res["iters"]) == rep.iters, (k, s, int(res["iters"]), rep.iters)
            assert int(res["flags"]) == (rep.converged and 1) | (rep.diverged and 2) | (rep.has_nan and 4), (k, s)
            assert np.array_equal(ie["surf_ind"][s], tr["surf_ind"][-1]), (k, s, "surf IDs")
            assert np.array_equal(ie["corner_ind"][s], tr["corner_ind"][-1]), (k, s, "corner IDs")
            diff = np.abs(ie["state_out"][s] - so).max()
            assert diff <= 1e-7, (k, s, diff)
            checked[t] += 1
    assert checked[1] >= 6 and checked[2] >= 6, checked
