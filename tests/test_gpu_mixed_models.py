"""GPU suite: one lidar model per scan (lins_gpu_project_scans_mixed, lins_gpu_seq_step_raw_mixed,
lins_gpu_seq_step_cloud2_mixed), so sweeps of different sensors run in one call and one context.

- Projection: VLP-16 sweeps, 64 x 1024 sweeps and VLP-16 sweeps under a third model whose every field differs, interleaved
  and permuted in one call, in both point formats: every output bit-identical to lins_gpu_project_scans with the sweep's
  own model, the ring entries past its line_num 0; a table listing an unused model changes only the ring stride.
- Sequence mode: recordings of the three models through one context with step_raw_mixed, against one twin context per
  model stepping the same slots with lins_gpu_seq_step_raw; every present slot bit-identical to its twin's slot after
  every step (states, covariances, results, init read-back, IESKF prior / output, correspondence IDs, maps).  Also: a
  queue through fewer slots whose restarts change a slot's sensor, alternating with step_raw, S = 1, a permutation,
  PACKED16 sweeps, and n_models = 1.
- Bags: VLP-16 and 64 x 1024 bags replayed together (bag_replay.replay with one model per bag) equal, per bag, the
  single-model replay of each sensor's bags alone, and synth.run_bag.
- Invalid tables return LINS_E_INVALID and change nothing."""
import ctypes as C

import numpy as np
import pytest

import cloud2cases as cc
import projcases as pj
import rawcases as rc
from conftest import pkg
from test_gpu_projection import _same_ori
from test_gpu_seq_init import init_params
from test_gpu_seq_pcl import _snapshot
from test_gpu_seq_raw import _bad_models

pytestmark = pytest.mark.gpu
synth = pkg("synth")
F = np.float32
PROJ_KEYS = ("seg", "outlier", "range", "ground", "col")


def third_model(defs):
    """A model for VLP-16 sweeps with every field unlike VLP-16's and 64 x 1024's."""
    return defs.LinsLidarModel(20, 1500, F(0.24), F(1.6), F(16.3), 7)


def _models(defs):
    return [defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64(), third_model(defs)]


# ---- projection ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu(capi):
    return capi.LinsGpu()


@pytest.fixture(scope="module")
def mixed_sweeps(synth, defs):
    """(sweeps, model index per sweep): 40 VLP-16, 24 64 x 1024 and 40 VLP-16 sweeps for the third model, interleaved."""
    groups = [[pj.raw_sweep(synth, defs, "config3", s)[0] for s in range(100, 140)],
              [pj.raw_sweep(synth, defs, "config4", s)[0] for s in range(300, 324)],
              [pj.raw_sweep(synth, defs, "config3", s)[0] for s in range(500, 540)]]
    sweeps, of = [], []
    for i in range(max(len(g) for g in groups)):
        for m, g in enumerate(groups):
            if i < len(g):
                sweeps.append(g[i]); of.append(m)
    return sweeps, np.array(of, np.int32)


def _check_against_single(gpu, defs, sweeps, of, models, dev, point_format):
    L_max = max(m.line_num for m in models)
    for m, model in enumerate(models):
        idx = np.flatnonzero(of == m)
        if not len(idx):
            continue
        ref = gpu.project_scans([sweeps[i] for i in idx], model=model, point_format=point_format)
        L = model.line_num
        for i, r in zip(idx, ref):
            d = dev[i]
            for k in PROJ_KEYS:
                assert d[k].tobytes() == r[k].tobytes(), (i, m, k)
            assert _same_ori(d["ori"], r["ori"]), (i, m)
            for k in ("start_ring", "end_ring"):
                assert len(d[k]) == L_max and d[k][:L].tobytes() == r[k].tobytes(), (i, m, k)
                assert not d[k][L:].any(), (i, m, k)


@pytest.mark.parametrize("point_format", [0, 1])
def test_project_scans_mixed_equals_per_model(gpu, defs, mixed_sweeps, point_format):
    sweeps, of = mixed_sweeps
    models = _models(defs)
    assert len(sweeps) >= 100 and set(of) == {0, 1, 2}
    dev = gpu.project_scans_mixed(sweeps, models, of, point_format=point_format)
    _check_against_single(gpu, defs, sweeps, of, models, dev, point_format)
    assert gpu.project_ms() > 0
    assert all(len(dev[i]["seg"]) > 500 for i in range(len(sweeps)))
    # permuted: the same outputs per sweep
    perm = np.random.default_rng(11).permutation(len(sweeps))
    pdev = gpu.project_scans_mixed([sweeps[i] for i in perm], models, of[perm], point_format=point_format)
    for j, i in enumerate(perm):
        for k in PROJ_KEYS + ("start_ring", "end_ring"):
            assert pdev[j][k].tobytes() == dev[i][k].tobytes(), (i, k)
        assert _same_ori(pdev[j]["ori"], dev[i]["ori"])


def test_unused_model_changes_only_the_ring_stride(gpu, defs, mixed_sweeps):
    sweeps, of = mixed_sweeps
    sweeps, of = sweeps[:30], of[:30]
    models = _models(defs)
    dev = gpu.project_scans_mixed(sweeps, models, of)
    big = defs.LinsLidarModel(100, 2000, F(0.18), F(0.5), F(25.0), 50)  # listed, used by no sweep
    wide = gpu.project_scans_mixed(sweeps, [models[0], big, models[1], models[2]], np.array([(0, 2, 3)[m] for m in of], np.int32))
    for a, b in zip(dev, wide):
        for k in PROJ_KEYS:
            assert a[k].tobytes() == b[k].tobytes(), k
        assert _same_ori(a["ori"], b["ori"])
        for k in ("start_ring", "end_ring"):
            assert len(b[k]) == 100 and b[k][:64].tobytes() == a[k].tobytes() and not b[k][64:].any()
    # one model without model_of: project_scans itself
    one = gpu.project_scans_mixed(sweeps, [models[1]], None)
    ref = gpu.project_scans(sweeps, model=models[1])
    for a, b in zip(one, ref):
        for k in PROJ_KEYS + ("start_ring", "end_ring"):
            assert a[k].tobytes() == b[k].tobytes(), k


# ---- sequence mode ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def seq_logs(defs):
    """Raw logs (rawcases.case_logs, with their edits) per model: VLP-16, 64 x 1024, and VLP-16 drives for the third
    model."""
    vlp, _ = rc.case_logs(defs, 0, n_seq=8, n_scans=12)
    dense, _ = rc.case_logs(defs, 1, n_seq=8, n_scans=12)
    third = [synth.raw_log("config3", seed=700 + s, n_scans=12 - 2 * (s % 3)) for s in range(4)]
    return [vlp, dense, third]


def _interleaved(seq_logs):
    """Jobs (model index, log) of every log, the models taking turns."""
    jobs = []
    for i in range(max(len(l) for l in seq_logs)):
        for m, logs in enumerate(seq_logs):
            if i < len(logs):
                jobs.append((m, logs[i]))
    return jobs


def _slot_rows(g, present):
    """Per present slot what a step leaves (None for an absent slot): everything of _snapshot for that slot, with the
    result record (iters, flags, pose), the IESKF's prior and output and its correspondence IDs where the slot ran the
    IESKF (the record's scan_id is the slot's place in its step's batch, which a twin with fewer slots numbers otherwise)."""
    d, di, ie, mp = g.seq_download(), g.seq_download_init(), g.seq_download_ieskf(), g.seq_download_maps()
    out = []
    for s, p in enumerate(present):
        if not p:
            out.append(None)
            continue
        r = {k: np.asarray(d[k][s]).tobytes() for k in ("global_state", "filter_state", "filter_cov", "status")}
        r.update({"init_" + k: np.asarray(v[s]).tobytes() for k, v in di.items()})
        r["maps"] = [mp[k][s].tobytes() for k in ("surf_map", "corner_map", "surf_tree", "corner_tree")] + [int(mp["stale"][s])]
        if int(d["status"][s]) in (2, 3):
            r["results"] = [np.asarray(d["results"][s][f]).tobytes() for f in ("iters", "flags", "pose")]
            r["ieskf"] = [ie[k][s].tobytes() for k in ("prior_state", "prior_cov", "state_out", "cov_out")]
            r["ind"] = [ie["surf_ind"][s].tobytes(), ie["corner_ind"][s].tobytes()]
        out.append(r)
    return out


def drive(capi, defs, jobs, n_slots, models, alt=False, point_format=0, one_model=False):
    """Run jobs ((model index, raw log), each from scan 0) through n_slots slots of one context with seq_step_raw_mixed,
    and through one twin context per model that steps the same slots with seq_step_raw, only the slots holding that
    model's jobs present.  Every present slot must be bit-identical to its twin's slot after every step.  alt: on every
    other step whose present slots share one model, the mixed context calls seq_step_raw instead.  one_model: the table
    has one model and no model_of.  Returns (rows[job] = [(scan, slot row)], the calls made: {"mixed", "raw"})."""
    ctxs = []
    for _ in range(1 + len(models)):
        c = capi.LinsGpu()
        c.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
        ctxs.append(c)
    g, twins = ctxs[0], ctxs[1:]
    rows, calls, t = [[] for _ in jobs], set(), 0
    for restart, who in pkg("bag_replay").slot_queue([len(l["time"]) for _, l in jobs], n_slots):
        if restart.any():
            for c in ctxs:
                c.seq_restart(restart)
        sweeps, imus, si = [], [], np.zeros((n_slots, 6))
        present = np.array([w is not None for w in who], np.uint8)
        of = np.array([jobs[w[0]][0] if w else 0 for w in who], np.int32)
        for j, w in enumerate(who):
            if w is None:
                sweeps.append(np.zeros((0, 4), np.float32)); imus.append(np.zeros((0, 7)))
                continue
            l, k = jobs[w[0]][1], w[1]
            o = l["imu_off"]
            sweeps.append(l["sweeps"][k]); imus.append(l["imu"][o[k]:o[k + 1]]); si[j] = l["imu_last"][k]
        imu = np.concatenate(imus).reshape(-1, 7)
        imu_off = np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32)
        step = dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=present)
        used = set(of[present == 1].tolist())
        if alt and t % 2 and len(used) == 1:
            g.seq_step_raw(step, model=models[used.pop()], scan_imu=si, point_format=point_format)
            calls.add("raw")
        else:
            g.seq_step_raw_mixed(step, models, None if one_model else of, scan_imu=si, point_format=point_format)
            calls.add("mixed" if len(used) > 1 else "mixed_uniform")
        rg = _slot_rows(g, present)
        for m, tw in enumerate(twins):
            mine = present & (of == m)
            if not mine.any():
                continue
            tw.seq_step_raw(dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=mine.astype(np.uint8)), model=models[m], scan_imu=si)
            rt = _slot_rows(tw, mine)
            for s in np.flatnonzero(mine):
                assert rg[s] == rt[s], f"step {t}: slot {s} (model {m}) differs from its twin"
        for j, w in enumerate(who):
            if w is not None:
                rows[w[0]].append((w[1], rg[j]))
        t += 1
    return rows, calls


@pytest.fixture(scope="module")
def full(capi, defs, seq_logs):
    jobs = _interleaved(seq_logs)
    rows, calls = drive(capi, defs, jobs, len(jobs), _models(defs))
    return jobs, rows, calls


def test_every_slot_equals_its_single_model_twin(defs, full):
    jobs, rows, calls = full
    assert "mixed" in calls and len(jobs) >= 20
    codes = {m: set() for m in range(3)}
    for (m, l), r in zip(jobs, rows):
        assert [k for k, _ in r] == list(range(len(l["time"])))
        codes[m] |= {int(np.frombuffer(x["status"], np.int32)[0]) for _, x in r}
    for m in (0, 1):  # the shipped sensors' drives initialise and run
        assert {defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN} <= codes[m], (m, codes[m])


def test_queue_through_fewer_slots_with_sensor_changes_and_step_raw(capi, defs, seq_logs, full):
    """Recordings in model blocks through 4 slots: restarts hand slots recordings of another sensor, and on every other
    step whose slots hold one sensor the run calls seq_step_raw."""
    jobs = [(m, l) for m, logs in enumerate(seq_logs) for l in logs]
    rows, calls = drive(capi, defs, jobs, 4, _models(defs), alt=True)
    assert {"mixed", "raw"} <= calls, calls
    fjobs, frows, _ = full
    for (m, l), r in zip(jobs, rows):
        i = next(i for i, (fm, fl) in enumerate(fjobs) if fm == m and fl is l)
        assert r == frows[i]


def test_single_slot_permutation_and_packed16(capi, defs, full):
    jobs, frows, _ = full
    pick = [0, 1, 2, 4]  # VLP-16, 64 x 1024, third, 64 x 1024 through one slot: the sensor changes at each restart
    rows, _ = drive(capi, defs, [jobs[i] for i in pick], 1, _models(defs))
    for j, i in enumerate(pick):
        assert rows[j] == frows[i]
    perm = list(np.random.default_rng(5).permutation(len(jobs)))
    rows, _ = drive(capi, defs, [jobs[i] for i in perm], len(jobs), _models(defs), point_format=1)
    for j, i in enumerate(perm):
        assert rows[j] == frows[i]


def test_one_model_table_equals_step_raw(capi, defs, seq_logs):
    jobs = [(0, l) for l in seq_logs[1][:4]]
    drive(capi, defs, jobs, len(jobs), [defs.LinsLidarModel.dense64()], one_model=True)


# ---- bags ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed_bags(tmp_path_factory):
    """Two VLP-16 bags and two 64 x 1024 bags, alternating: (paths, lidar per bag)."""
    d = tmp_path_factory.mktemp("mixed_bags")
    lib = cc.baglib()
    paths, lidar = [], []
    for s in range(4):
        p = str(d / f"drive{s}.bag")
        synth.write_sequence_bag(p, config=("config3", "config4")[s % 2], seed=60 + s, n_scans=8 - s)
        paths.append(p); lidar.append(s % 2)
    for p in paths:  # run_bag projects without the NaN removal: the sweeps' ends must be finite for the two to agree
        _, msgs = cc.bag_tool.read_bag(p)
        for _, _, b in msgs:
            pts = cc.decode_cpp(lib, b) if cc.bag_tool.index_pointcloud2(b) else None
            if pts is not None and len(pts):
                assert np.isfinite(pts[[0, -1], :3]).all()
    return paths, lidar


def test_mixed_bag_replay_equals_per_sensor_replay_and_run_bag(capi, defs, mixed_bags):
    br = pkg("bag_replay")
    paths, lidar = mixed_bags
    presets = [defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()]
    recs = [br.Recording(p) for p in paths]
    mixed = br.replay(recs, 3, model=[presets[l] for l in lidar])
    for l in (0, 1):
        idx = [i for i in range(len(paths)) if lidar[i] == l]
        alone = br.replay([recs[i] for i in idx], 1, model=presets[l])
        for i, o in zip(idx, alone):
            for k in o:
                assert mixed[i][k].tobytes() == o[k].tobytes(), (paths[i], k)
    for p, l, o in zip(paths, lidar, mixed):
        ref = synth.run_bag(p, lidar_model=l)
        assert np.array_equal(o["status"], ref["status"])
        ran = np.flatnonzero(o["iters"] >= 0)
        assert np.array_equal(ran, np.asarray(ref["scan_index"])), (ran, ref["scan_index"])
        assert np.array_equal(o["iters"][ran], ref["iters"]) and np.array_equal(o["flags"][ran], ref["flags"])
        diff = np.abs(o["global_est"] - ref["global_est"]).max()
        assert diff <= 1e-7, (p, diff)
        assert len(ran) > 0


# ---- invalid tables -----------------------------------------------------------------------------------------------------
def _bad_tables(defs, S):
    """(what, models list or None, n_models, model_of or None, null models pointer): tables every mixed entry rejects."""
    vlp, dense = defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()
    ok_of = np.array([0, 1, 0][:S], np.int32)
    out = [("n_models 0", [vlp, dense], 0, ok_of, False), ("n_models -1", [vlp, dense], -1, ok_of, False),
           ("null models", [vlp, dense], 2, ok_of, True), ("null model_of", [vlp, dense], 2, None, False),
           ("model_of -1", [vlp, dense], 2, np.array([0, -1, 0][:S], np.int32), False),
           ("model_of == n_models", [vlp, dense], 2, np.array([0, 1, 2][:S], np.int32), False),
           ("one model, model_of 1", [vlp], 1, np.array([0, 1, 0][:S], np.int32), False)]
    for field, v, m in _bad_models(defs):
        out.append((f"model 1 {field}={v}", [vlp, m], 2, ok_of, False))
    return out


def _table(defs, models, n_models, model_of, null_models, keep):
    keep["models"] = (defs.LinsLidarModel * len(models))(*models)
    t = defs.LinsLidarModels()
    t.n_models = n_models
    t.models = None if null_models else C.cast(keep["models"], C.c_void_p)
    if model_of is not None:
        keep["model_of"] = np.ascontiguousarray(model_of, np.int32)
        t.model_of = keep["model_of"].ctypes.data
    return t


def test_invalid_tables_change_nothing(capi, defs, seq_logs):
    logs = [seq_logs[0][0], seq_logs[1][0], seq_logs[0][1]]
    S, n_steps = 3, 4
    models, of = [defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()], np.array([0, 1, 0], np.int32)
    fp = defs.LinsFeatureParams.shipped()

    def step(t):
        imus = [l["imu"][l["imu_off"][t]:l["imu_off"][t + 1]] for l in logs]
        return dict(sweeps=[l["sweeps"][t] for l in logs], imu=np.concatenate(imus).reshape(-1, 7),
                    imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32))

    def scan_imu(t):
        return np.ascontiguousarray(np.stack([l["imu_last"][t] for l in logs]), np.float64)

    ref, g = capi.LinsGpu(), capi.LinsGpu()
    for c in (ref, g):
        c.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), S)
    bad = _bad_tables(defs, S)
    for t in range(n_steps):
        ref.seq_step_raw_mixed(step(t), models, of, scan_imu=scan_imu(t))
        if t in (1, 2):  # (at t = 1 the slots are initialising, at t = 2 they run)
            st, si = step(t + 1), scan_imu(t + 1)
            keep = {"imu": np.ascontiguousarray(st["imu"], np.float64), "imu_off": st["imu_off"]}
            d = defs.LinsSeqRawDesc()
            d.n_seq, d.imu, d.imu_off = S, keep["imu"].ctypes.data, keep["imu_off"].ctypes.data
            d.raw = g._raw_desc(st["sweeps"], 0, keep)
            d2 = defs.LinsSeqCloud2Desc()
            d2.n_seq, d2.imu, d2.imu_off = S, d.imu, d.imu_off
            d2.cloud2 = g.cloud2_desc([cc.as_input(defs, cc.message("velodyne32", s, seq=t)[0]) for s in st["sweeps"]], keep)
            assert g.L.lins_gpu_seq_step_raw_mixed(g.h, C.byref(d), None, C.byref(fp), si.ctypes.data) == -1
            assert g.L.lins_gpu_seq_step_cloud2_mixed(g.h, C.byref(d2), None, C.byref(fp), si.ctypes.data) == -1
            for what, ms, n_models, mo, null in bad:
                tk = {}
                tab = _table(defs, ms, n_models, mo, null, tk)
                assert g.L.lins_gpu_seq_step_raw_mixed(g.h, C.byref(d), C.byref(tab), C.byref(fp), si.ctypes.data) == -1, what
                assert g.L.lins_gpu_seq_step_cloud2_mixed(g.h, C.byref(d2), C.byref(tab), C.byref(fp), si.ctypes.data) == -1, what
        g.seq_step_raw_mixed(step(t), models, of, scan_imu=scan_imu(t))
        a, b = _snapshot(ref), _snapshot(g)
        for k in a:
            same = a[k].tobytes() == b[k].tobytes() if isinstance(a[k], np.ndarray) else a[k] == b[k]
            assert same, f"step {t}: {k}"
    assert {int(v) for v in a["status"]} & {defs.SEQ_RAN, defs.SEQ_ICP}, a["status"]


def test_project_scans_mixed_rejects_bad_tables_and_writes_nothing(gpu, capi, defs, mixed_sweeps):
    sweeps = mixed_sweeps[0][:3]
    keep = {}
    d = gpu._raw_desc(sweeps, 0, keep)
    total = int(keep["cloud_off"][-1])
    outs = [np.full(max(total, 1) * 32, 0x5A, np.uint8) for _ in range(9)]  # (room for every output's records)
    before = [o.copy() for o in outs]
    assert gpu.L.lins_gpu_project_scans_mixed(gpu.h, None, C.byref(d), *[o.ctypes.data for o in outs]) == -1
    for what, ms, n_models, mo, null in _bad_tables(defs, 3):
        tk = {}
        tab = _table(defs, ms, n_models, mo, null, tk)
        assert gpu.L.lins_gpu_project_scans_mixed(gpu.h, C.byref(tab), C.byref(d), *[o.ctypes.data for o in outs]) == -1, what
    for a, b in zip(outs, before):
        assert a.tobytes() == b.tobytes()
    # the context still projects
    dev = gpu.project_scans_mixed(sweeps, _models(defs), np.array([0, 0, 0], np.int32))
    ref = gpu.project_scans(sweeps)
    for a, b in zip(dev, ref):
        assert a["seg"].tobytes() == b["seg"].tobytes()
