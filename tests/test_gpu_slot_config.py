"""GPU suite: per-slot rig configuration (lins_gpu_seq_configure), so recordings of different robots run in one context.

The contract: every configured slot is bit-identical to the same recording in the same slot of a run whose shared values
(the context's scan_period, the step's lins_feature_params, the open's lins_seq_params / lins_seq_init_params) equal its
config; an unconfigured slot is bit-identical to the same slot of a run with the run's own values.
- Twin parity: 24 slots, three configs that differ in every field (periods 0.1, 0.05, 0.075, a 2.5 degree extrinsic) and
  unconfigured slots, VLP-16 and 64 x 1024 drives through seq_step_raw_mixed, VLP-16 drives through seq_step_raw; the
  rawcases edits give SKIPPED scans, and a second pass with lidar_scale = 1e9 in every context (a shared value) makes
  every running scan take the estimateTransform fallback, so the per-unit period runs in MODE_IESKF and in both
  MODE_ICP_REDUCE loops.
- Every slot configured to the run's own values equals an unconfigured run, before and after restarts.
- A queue through fewer slots: restarts change a slot's config and sensor; an unconfigured recording after a configured
  one equals its default twin.
- A run bound to the lockstep mappers, with IMU rows fed so that transformUpdate reads the period.
- Bags replayed together with their own configs equal each bag replayed alone with its config.
- Invalid calls return LINS_E_INVALID and change nothing."""
import ctypes as C

import numpy as np
import pytest

import cloud2cases as cc
import rawcases as rc
from conftest import pkg
from test_gpu_mixed_models import _slot_rows
from test_gpu_seq_pcl import _snapshot

pytestmark = pytest.mark.gpu
synth = pkg("synth")
br = pkg("bag_replay")


# three rigs that differ from each other in every field, as exp_port.yaml's values (rig_config.RIG_KEYS)
RIGS = [dict(scan_period=0.1, edge_threshold=0.6, surf_threshold=0.4, imu_lidar_extrinsic_angle=2.5, acc_n=60000.0, gyr_n=0.12,
              acc_w=450.0, gyr_w=0.06, init_pos_std=(0.01, 0.01, 0.02), init_att_std=(0.1, 0.1, 0.2), init_vel_std=(0.05, 0.05, 0.05),
              init_acc_std=(0.02, 0.02, 0.03), init_gyr_std=(0.003, 0.003, 0.003), init_ba=(-0.01, 0.12, -0.02), init_bw=(-0.002, -0.0001, 0.002)),
        dict(scan_period=0.05, edge_threshold=0.35, surf_threshold=0.7, imu_lidar_extrinsic_angle=-1.5, acc_n=90000.0, gyr_n=0.08,
              acc_w=700.0, gyr_w=0.03, init_pos_std=(0.05, 0.04, 0.03), init_att_std=(0.5, 0.4, 0.3), init_vel_std=(0.1, 0.1, 0.2),
              init_acc_std=(0.005, 0.006, 0.01), init_gyr_std=(0.001, 0.001, 0.004), init_ba=(0.02, -0.05, 0.01), init_bw=(0.001, 0.0002, -0.001)),
        dict(scan_period=0.075, edge_threshold=0.8, surf_threshold=0.2, imu_lidar_extrinsic_angle=4.0, acc_n=30000.0, gyr_n=0.2,
              acc_w=250.0, gyr_w=0.1, init_pos_std=(0.002, 0.003, 0.004), init_att_std=(0.02, 0.03, 0.05), init_vel_std=(0.01, 0.02, 0.03),
              init_acc_std=(0.05, 0.04, 0.06), init_gyr_std=(0.01, 0.008, 0.006), init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0))]


def configs(defs):
    return [defs.LinsSlotConfig.shipped(**r) for r in RIGS]


def run_values(defs):
    """The run's own values as a config: what an unconfigured slot of the main context reads."""
    return defs.LinsSlotConfig.shipped()


class Ctx:
    """A context with the shared values of one config (None: the run's own values)."""

    def __init__(self, capi, defs, cfg, n_slots, lidar_scale=1.0, bind=False):
        c = cfg or run_values(defs)
        self.g = capi.LinsGpu(defs.LinsParams.shipped(scan_period=c.scan_period, lidar_scale=lidar_scale))
        self.g.seq_open(c.filter, c.init, n_slots)
        self.fp = c.features
        if bind:
            self.g.seq_map_open()


def _step_inputs(jobs, who, n_slots):
    sweeps, imus, si = [], [], np.zeros((n_slots, 6))
    for j, w in enumerate(who):
        if w is None:
            sweeps.append(np.zeros((0, 4), np.float32)); imus.append(np.zeros((0, 7)))
            continue
        l, k = jobs[w[0]][2], w[1]
        o = l["imu_off"]
        sweeps.append(l["sweeps"][k]); imus.append(l["imu"][o[k]:o[k + 1]]); si[j] = l["imu_last"][k]
    imu = np.concatenate(imus).reshape(-1, 7)
    imu_off = np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32)
    return sweeps, imu, imu_off, si


def _mapper_imu(jobs, who):
    """Per slot the imuHandler rows of its scan: three stamps around the scan's time, roll / pitch from the scan index."""
    rows = []
    for w in who:
        if w is None:
            rows.append(None)
            continue
        t = float(jobs[w[0]][2]["time"][w[1]])
        rows.append((np.array([t - 0.06, t - 0.01, t + 0.08]), np.array([0.01, 0.012, 0.015]) * (1 + w[1] % 3),
                     np.array([-0.02, -0.018, -0.01]) * (1 + w[1] % 2)))
    return rows


def drive(capi, defs, jobs, cfgs, n_slots, models, lidar_scale=1.0, raw=False, bind=False, configure_defaults=False, cloud2=False):
    """jobs: (config index or None, model index, raw log).  The main context runs them through n_slots slots, configuring a
    slot with its job's config when it takes the job (configure_defaults: also the unconfigured jobs, with the run's own
    values); one twin per config (and one for the unconfigured jobs) steps the same slots with only its own jobs present.
    Every present slot equals its twin's slot after every step.  raw: seq_step_raw with models[0] (every job's model must
    be 0), else seq_step_raw_mixed, or with cloud2 seq_step_cloud2_mixed on the sweeps as Velodyne PointCloud2 messages.  bind: both sides bound to the lockstep mappers, fed IMU rows, their reports and
    downloads compared.  Returns (rows[job] = [(scan, slot row)], the set of scan_status codes per config)."""
    keys = sorted({j[0] for j in jobs}, key=lambda k: -1 if k is None else k)
    main = Ctx(capi, defs, None, n_slots, lidar_scale, bind)
    twins = {k: Ctx(capi, defs, None if k is None else cfgs[k], n_slots, lidar_scale, bind) for k in keys}
    rows, codes, t = [[] for _ in jobs], {k: set() for k in keys}, 0
    n_processed = [0]
    for restart, who in br.slot_queue([len(j[2]["time"]) for j in jobs], n_slots):
        if restart.any():
            for c in [main] + list(twins.values()):
                c.g.seq_restart(restart)
        fresh = np.array([w is not None and w[1] == 0 and (jobs[w[0]][0] is not None or configure_defaults) for w in who], np.uint8)
        if fresh.any():
            main.g.seq_configure(fresh, [(cfgs[jobs[w[0]][0]] if jobs[w[0]][0] is not None else run_values(defs)) if f else None
                                         for w, f in zip(who, fresh)])
        sweeps, imu, imu_off, si = _step_inputs(jobs, who, n_slots)
        present = np.array([w is not None for w in who], np.uint8)
        of = np.array([jobs[w[0]][1] if w else 0 for w in who], np.int32)
        key = [jobs[w[0]][0] if w else "absent" for w in who]
        time = np.array([float(jobs[w[0]][2]["time"][w[1]]) if w else 0.0 for w in who])
        msgs = [cc.as_input(defs, cc.message("velodyne32", sw, seq=t)[0]) for sw in sweeps] if cloud2 else None

        def step(c, pres):
            st = dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=pres, msgs=msgs)
            if cloud2:
                c.g.seq_step_cloud2_mixed(st, models, of, fp=c.fp, scan_imu=si)
            elif raw:
                c.g.seq_step_raw(st, model=models[0], fp=c.fp, scan_imu=si)
            else:
                c.g.seq_step_raw_mixed(st, models, of, fp=c.fp, scan_imu=si)
            if bind:
                c.g.mappers_imu([r if p else None for r, p in zip(_mapper_imu(jobs, who), pres)])
                return c.g.seq_map_step(time)[0]
            return None

        mreps = step(main, present)
        rg = _slot_rows(main.g, present)
        for k, tw in twins.items():
            mine = np.array([p and key[s] == k for s, p in enumerate(present)], np.uint8)
            if not mine.any():
                continue
            treps = step(tw, mine)
            rt = _slot_rows(tw.g, mine)
            for s in np.flatnonzero(mine):
                assert rg[s] == rt[s], f"step {t}: slot {s} (config {k}) differs from its twin"
                codes[k].add(int(np.frombuffer(rg[s]["status"], np.int32)[0]))
                if bind:
                    assert (mreps[s] is None) == (treps[s] is None), (t, s)
                    if mreps[s] is not None:
                        assert bytes(mreps[s]) == bytes(treps[s]), f"step {t}: slot {s} mapper report"
                    if mreps[s] is not None and mreps[s].processed:  # (a download is sized by a processed cycle's report)
                        n_processed[0] += 1
                        (pa, wa, ca), (pb, wb, cb) = main.g.mappers_download(s, mreps[s]), tw.g.mappers_download(s, treps[s])
                        assert pa.tobytes() == pb.tobytes() and wa.tobytes() == wb.tobytes(), (t, s)
                        assert all(ca[k].tobytes() == cb[k].tobytes() for k in ca), (t, s)
        for j, w in enumerate(who):
            if w is not None:
                rows[w[0]].append((w[1], rg[j]))
        t += 1
    assert not bind or n_processed[0] > 0
    return rows, codes


@pytest.fixture(scope="module")
def logs(defs):
    vlp, _ = rc.case_logs(defs, 0, n_seq=8, n_scans=12)   # logs[0] scan 6: the processScan gate (SKIPPED)
    dense, _ = rc.case_logs(defs, 1, n_seq=8, n_scans=12)
    return vlp, dense


def _models(defs):
    return [defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()]


def _jobs(logs):
    """24 jobs: per config key (None, 0, 1, 2) the gated VLP-16 drive, three more VLP-16 drives and both 64 x 1024 drives."""
    vlp, dense = logs
    jobs = []
    for i in range(6):
        for k in (None, 0, 1, 2):
            jobs.append((k, 0, vlp[(0, 1, 2, 4)[i]]) if i < 4 else (k, 1, dense[i - 4]))
    return jobs


def _want_codes(defs, codes, with_icp):
    want = {defs.SEQ_SECOND, defs.SEQ_SKIPPED} | ({defs.SEQ_ICP} if with_icp else {defs.SEQ_RAN})
    for k in (0, 1, 2):
        assert want <= codes[k], (k, codes[k])


@pytest.mark.parametrize("lidar_scale", [1.0, 1e9])
def test_configured_slots_equal_their_twins_mixed(capi, defs, logs, lidar_scale):
    jobs = _jobs(logs)
    assert len(jobs) >= 24
    _, codes = drive(capi, defs, jobs, configs(defs), len(jobs), _models(defs), lidar_scale=lidar_scale)
    _want_codes(defs, codes, lidar_scale > 1)


def test_configured_slots_equal_their_twins_step_raw(capi, defs, logs):
    jobs = [j for j in _jobs(logs) if j[1] == 0]
    _, codes = drive(capi, defs, jobs, configs(defs), len(jobs), _models(defs)[:1], raw=True)
    _want_codes(defs, codes, False)


def test_configured_slots_equal_their_twins_cloud2_mixed(capi, defs, logs):
    jobs = _jobs(logs)
    _, codes = drive(capi, defs, jobs, configs(defs), len(jobs), _models(defs), cloud2=True)
    _want_codes(defs, codes, False)


def test_configuring_the_run_values_changes_nothing(capi, defs, logs):
    """Every slot configured to the run's own values, through fewer slots (so restarts return slots to unconfigured and
    configure them again): bit-identical to the unconfigured run."""
    jobs = [(None, m, l) for _, m, l in _jobs(logs)[::2]]
    plain, _ = drive(capi, defs, jobs, configs(defs), 5, _models(defs))
    same, _ = drive(capi, defs, jobs, configs(defs), 5, _models(defs), configure_defaults=True)
    assert plain == same


def test_queue_changes_config_and_sensor(capi, defs, logs):
    """Recordings through 3 slots: restarts change a slot's config and its sensor, unconfigured recordings follow
    configured ones; each equals its twin, and its rows equal those of the same recording alone in its own slot."""
    jobs = _jobs(logs)[:12]
    rows, _ = drive(capi, defs, jobs, configs(defs), 3, _models(defs))
    full, _ = drive(capi, defs, jobs, configs(defs), len(jobs), _models(defs))
    assert rows == full


def test_bound_mappers_use_the_slot_period(capi, defs, logs):
    jobs = [j for j in _jobs(logs) if j[1] == 0][:8]
    drive(capi, defs, jobs, configs(defs), 4, _models(defs)[:1], raw=True, bind=True)


def test_bags_at_10_and_20_hz_replay_with_their_rigs(capi, defs, tmp_path):
    """Bags recorded at 10 Hz and at 20 Hz, each with its robot's rig (RIGS[0]: 0.1 s, RIGS[1]: 0.05 s) or none, replayed
    together through 2 slots: each equals its own single-config replay, and that replay agrees with the C++
    StateEstimator shim's run_bag under the same rig, to the tolerance of the other bag tests."""
    plan = [(1, 0.05), (None, None), (0, 0.1), (1, 0.05)]  # (rig, sweep duration of the recording)
    paths = []
    for s, (_, period) in enumerate(plan):
        p = str(tmp_path / f"bag{s}.bag")
        synth.write_sequence_bag(p, config="config3", seed=80 + s, n_scans=10 - s, scan_period=period)
        paths.append(p)
    _, msgs = cc.bag_tool.read_bag(paths[0])
    stamps = sorted(cc.bag_tool.index_pointcloud2(b)["stamp"] for _, _, b in msgs if cc.bag_tool.index_pointcloud2(b))
    assert np.allclose(np.diff(stamps), 0.05)  # (a 20 Hz recording)
    recs = [br.Recording(p, config=None if k is None else defs.LinsSlotConfig.shipped(**RIGS[k])) for p, (k, _) in zip(paths, plan)]
    together = br.replay(recs, 2)
    for r, o, (k, _) in zip(recs, together, plan):
        alone = br.replay([r], 1)[0]
        for key in o:
            assert o[key].tobytes() == alone[key].tobytes(), (r.path, key)
        ref = synth.run_bag(r.path, rig=None if k is None else RIGS[k])
        assert np.array_equal(o["status"], ref["status"]), (r.path, o["status"], ref["status"])
        ran = np.flatnonzero(o["iters"] >= 0)
        assert len(ran) >= 3 and np.array_equal(ran, np.asarray(ref["scan_index"])), (ran, ref["scan_index"])
        assert np.array_equal(o["iters"][ran], ref["iters"]) and np.array_equal(o["flags"][ran], ref["flags"])
        diff = np.abs(o["global_est"] - ref["global_est"]).max()
        assert diff <= 1e-7, (r.path, diff)


def test_invalid_configure_changes_nothing(capi, defs, logs):
    vlp = logs[0]
    S = 3
    jobs = [(None, 0, vlp[i]) for i in range(S)]
    cfg = configs(defs)
    ref = capi.LinsGpu()
    ref.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
    L = g.L

    def call(mask, cs):
        arr = (defs.LinsSlotConfig * S)(*cs)
        return L.lins_gpu_seq_configure(g.h, np.ascontiguousarray(mask, np.uint8).ctypes.data, C.cast(arr, C.c_void_p))

    def bad_configs():
        out = []
        for field, v in (("scan_period", 0.0), ("scan_period", -0.1), ("scan_period", float("nan")), ("scan_period", float("inf"))):
            c = defs.LinsSlotConfig.shipped(); setattr(c, field, v); out.append(c)
        for sub, name, i, v in (("features", "edge_threshold", None, float("nan")), ("features", "imu_lidar_extrinsic_angle", None, float("inf")),
                                ("filter", "noise", 2, -1e-9), ("filter", "init_pos_std", 1, -0.1), ("filter", "init_att_std", 0, float("nan")),
                                ("init", "init_vel_std", 2, -1.0), ("init", "init_acc_std", 0, -0.01), ("init", "init_gyr_std", 1, float("inf")),
                                ("init", "init_ba", 0, float("nan")), ("init", "init_bw", 2, float("-inf"))):
            c = defs.LinsSlotConfig.shipped()
            if i is None:
                setattr(getattr(c, sub), name, v)
            else:
                getattr(getattr(c, sub), name)[i] = v
            out.append(c)
        return out

    for t in range(5):
        if t in (0, 3):
            # every rejection: nulls, a bad entry among good ones, a slot that has stepped (t = 3), a begin run elsewhere
            assert L.lins_gpu_seq_configure(g.h, None, None) == -1
            arr = (defs.LinsSlotConfig * S)(*cfg)
            assert L.lins_gpu_seq_configure(g.h, None, C.cast(arr, C.c_void_p)) == -1
            assert L.lins_gpu_seq_configure(g.h, np.ones(S, np.uint8).ctypes.data, None) == -1
            for b in bad_configs():
                assert call([1, 1, 0], [cfg[0], b, cfg[1]]) == -1
            if t == 3:
                assert call([1, 0, 0], [cfg[0], cfg[1], cfg[2]]) == -1  # slot 0 has stepped
        sweeps = [l["sweeps"][t] for _, _, l in jobs]
        imus = [l["imu"][l["imu_off"][t]:l["imu_off"][t + 1]] for _, _, l in jobs]
        st = dict(sweeps=sweeps, imu=np.concatenate(imus).reshape(-1, 7),
                  imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32))
        si = np.ascontiguousarray(np.stack([l["imu_last"][t] for _, _, l in jobs]), np.float64)
        for c in (ref, g):
            c.seq_step_raw(st, scan_imu=si)
        a, b = _snapshot(ref), _snapshot(g)
        for k in a:
            same = a[k].tobytes() == b[k].tobytes() if isinstance(a[k], np.ndarray) else a[k] == b[k]
            assert same, f"step {t}: {k}"
    # no run: LINS_E_NOMAP; a seq_begin run cannot be configured
    h = capi.LinsGpu()
    arr = (defs.LinsSlotConfig * 1)(cfg[0])
    assert h.L.lins_gpu_seq_configure(h.h, np.ones(1, np.uint8).ctypes.data, C.cast(arr, C.c_void_p)) == -3
    z = np.zeros((0,), defs.POINT_DTYPE)
    h.seq_begin(defs.LinsSeqParams.shipped(), dict(filter_state=np.zeros((1, 19)), filter_cov=np.eye(18).reshape(1, 324),
                                                 global_state=np.zeros((1, 19)), imu_last=np.zeros((1, 6)), surf_map=z,
                                                 surf_map_off=np.zeros(2, np.int32), corner_map=z, corner_map_off=np.zeros(2, np.int32)))
    assert h.L.lins_gpu_seq_configure(h.h, np.ones(1, np.uint8).ctypes.data, C.cast(arr, C.c_void_p)) == -1
