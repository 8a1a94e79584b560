"""GPU suite: lins_gpu_seq_step_raw (sequence mode from the raw sweep: image projection with copyPointCloud's NaN removal,
feature extraction and the filter step in one device call) on simulated drives of VLP-16 and of 64 x 1024 sweeps.

At every step a run of step_raw is bit-identical (test_gpu_seq_pcl._snapshot: states, covariances, results, init
read-back, IESKF prior and output, correspondence IDs, maps) to two twins fed with the same sweeps after the removal on
the host: host ImageProjection -> step_pcl, and device project_scans -> step_pcl.  Every recording also matches its own
shim replaying the host-projected pcl log, at test_gpu_seq_init.py's tolerances.  Then: edited sweeps (truncated, empty,
non-finite points, an entirely non-finite sweep), a scan without IMU rows and an absent slot; step_raw / step_pcl /
step_ex alternating; S = 1, a permutation, PACKED16 sweeps, a queue through fewer slots and a run started by seq_begin;
invalid calls that change nothing; the timing hooks."""
import ctypes as C

import numpy as np
import pytest

import featcases as fc
import projcases as pj
import rawcases as rc
from conftest import pkg
from test_gpu_seq_init import check_job, init_params
from test_gpu_seq_pcl import _rows_equal, _snapshot

pytestmark = pytest.mark.gpu
synth = pkg("synth")
ABSENT_JOB = 7  # this job's slot is absent for one step in the middle of its drive


def _build(capi, defs, lidar):
    logs, edits = rc.case_logs(defs, lidar, gpu=capi.LinsGpu())
    print("lidar", lidar, "drives replaced because a tie decides a pick:", edits.pop("tie_skipped"))
    pcls = [rc.pcl_of(defs, l) for l in logs]
    recs = [synth.replay_pcl_log(p) for p in pcls]
    return logs, edits, pcls, recs


@pytest.fixture(scope="module")
def vlp(capi, defs):
    return _build(capi, defs, 0)


@pytest.fixture(scope="module")
def dense(capi, defs):
    return _build(capi, defs, 1)


def _empty_scan(L):
    return dict(seg=np.zeros((0, 4), np.float32), ground=np.zeros(0, np.uint8), col=np.zeros(0, np.uint32), range=np.zeros(0, np.float32),
                start_ring=np.zeros(L, np.int32), end_ring=np.zeros(L, np.int32), ori=np.zeros(3, np.float32))


def _jobs(logs):
    """Every log from scan 0; job ABSENT_JOB skips one step after its third scan."""
    jobs = []
    for i, l in enumerate(logs):
        ev = list(range(len(l["time"])))
        if i == ABSENT_JOB:
            ev = ev[:3] + [None] + ev[3:]
        jobs.append((i, ev))
    return jobs


def _via_ex(g, capi, step, L, scan_imu):
    feats = g.extract_features(step["scans"], line_num=L)
    d = dict(imu=step["imu"], imu_off=step["imu_off"], present=step["present"])
    for k in fc.NAMES:
        clouds = [capi._points_from_xyzi(f[k] if step["present"][s] else np.zeros((0, 4))) for s, f in enumerate(feats)]
        d[k] = np.concatenate(clouds)
        d[k + "_off"] = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    g.seq_step(d, scan_imu=scan_imu)


def _same(a, b, t, who):
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), f"{who} step {t}: {k}"
        else:
            assert a[k] == b[k], f"{who} step {t}: {k}"


def drive(capi, defs, cases, n_slots, jobs, twins=(), point_format=0, hooks=False):
    """Run `jobs` ((log index, events): a scan index, or None for a step the slot is absent) through n_slots opened slots
    with lins_gpu_seq_step_raw, restarting a slot whose job has ended.  Each twin is a second context stepped with the
    same input another way, whose snapshot must be bit-identical after every step: "pcl_host" (step_pcl with the host
    pcl scans), "pcl_dev" (device project_scans of the host-filtered sweeps -> step_pcl), "alt" (step_raw, step_pcl,
    step_ex in turn).  Returns rows[i] = [(scan, row)] of job i."""
    logs, _, pcls, _ = cases
    model = rc.model_of(defs, logs[0])
    L = model.line_num
    ctxs = []
    for _ in range(1 + len(twins)):
        g = capi.LinsGpu()
        g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
        ctxs.append(g)
    g = ctxs[0]
    rows = [[] for _ in jobs]
    t = 0
    for restart, slots in pkg("bag_replay").slot_queue([len(ev) for _, ev in jobs], n_slots):
        if restart.any():
            for c in ctxs:
                c.seq_restart(restart)
        sweeps, scans, present, who, imus, scan_imu = [], [], [], [], [], np.zeros((n_slots, 6))
        for j, w in enumerate(slots):
            k = jobs[w[0]][1][w[1]] if w is not None else None
            if k is None:
                sweeps.append(np.zeros((0, 4), np.float32)); scans.append(_empty_scan(L)); present.append(0); who.append(None)
                imus.append(np.zeros((0, 7)))
                continue
            li = jobs[w[0]][0]
            o = logs[li]["imu_off"]
            sweeps.append(logs[li]["sweeps"][k]); scans.append(pcls[li]["scans"][k]); present.append(1); who.append((w[0], k))
            imus.append(logs[li]["imu"][o[k]:o[k + 1]])
            scan_imu[j] = logs[li]["imu_last"][k]
        imu = np.concatenate(imus).reshape(-1, 7)
        imu_off = np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32)
        pres = np.array(present, np.uint8)
        g.seq_step_raw(dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=pres), model=model, scan_imu=scan_imu, point_format=point_format)
        if hooks:
            assert g.project_ms() > 0 and g.extract_ms() > 0
        for tw, c in zip(twins, ctxs[1:]):
            mode = tw if tw != "alt" else ("raw", "pcl_host", "ex")[t % 3]
            if mode == "raw":
                c.seq_step_raw(dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=pres), model=model, scan_imu=scan_imu)
            elif mode == "ex":
                _via_ex(c, capi, dict(imu=imu, imu_off=imu_off, scans=scans, present=pres), L, scan_imu)
            else:
                sc = scans if mode == "pcl_host" else [
                    {k: p[k] for k in scans[0]} for p in c.project_scans([rc.finite(s) for s in sweeps], model=model)]
                c.seq_step_pcl(dict(imu=imu, imu_off=imu_off, scans=sc, present=pres), scan_imu=scan_imu, line_num=L)
            _same(_snapshot(g), _snapshot(c), t, tw)
        d, di = g.seq_download(), g.seq_download_init()
        for j, w in enumerate(who):
            if w is None:
                continue
            row = {k: np.array(v[j], copy=True) for k, v in d.items()}
            row.update({k: np.array(v[j], copy=True) for k, v in di.items()})
            rows[w[0]].append((w[1], row))
        t += 1
    return rows


def _check_edits(defs, cases, rows):
    logs, edits, _, recs = cases
    for s, (case, k) in edits.items():
        r = recs[s]
        if case == "gate":
            assert r["code"][k] == defs.SEQ_SKIPPED, (case, r["code"][k])
        elif case == "first_gate":
            assert r["init_code"][k] == defs.SEQ_INIT_WAIT, (case, r["init_code"][k])
        elif case == "no_imu":
            assert logs[s]["imu_off"][k + 1] == logs[s]["imu_off"][k] and r["code"][k] in (defs.SEQ_RAN, defs.SEQ_ICP, defs.SEQ_SKIPPED)
        elif case in ("empty", "all_nonfinite"):
            assert len(rc.finite(logs[s]["sweeps"][k])) == 0 and r["code"][k] == defs.SEQ_SKIPPED, (case, r["code"][k])
        elif case == "nonfinite":
            a = logs[s]["sweeps"][k]
            bad = ~np.isfinite(a[:, :3]).all(1)
            assert bad[0] and bad[-2] and bad[-1] and bad[1:-2].sum() > 10
            # without the removal the sweep's orientation would not be finite (the extraction would reject the scan)
            unfiltered = pj.host_projection(defs, defs.make_points(a[:, :3], a[:, 3]), rc.model_of(defs, logs[s]))
            assert not np.isfinite(unfiltered["ori"]).all()
            assert r["code"][k] in (defs.SEQ_RAN, defs.SEQ_ICP), (case, r["code"][k])
    # the absent step of ABSENT_JOB: its rows still cover every scan of its log
    assert [k for k, _ in rows[ABSENT_JOB]] == list(range(len(logs[ABSENT_JOB]["time"])))


@pytest.fixture(scope="module")
def from_zero(capi, defs, vlp):
    return drive(capi, defs, vlp, len(vlp[0]), _jobs(vlp[0]), twins=("pcl_host", "pcl_dev"), hooks=True)


@pytest.mark.parametrize("lidar", ["vlp", "dense"])
def test_twins_at_every_step_and_the_shim(capi, defs, request, lidar):
    """From scan 0, >= 12 raw logs of spread lengths: every step bit-identical to both twins (inside drive), every recording
    against its own shim, every edit reaching its case."""
    cases = request.getfixturevalue(lidar)
    logs, _, _, recs = cases
    rows = request.getfixturevalue("from_zero") if lidar == "vlp" else drive(capi, defs, cases, len(logs), _jobs(logs),
                                                                              twins=("pcl_host", "pcl_dev"))
    assert len(logs) >= 12 and len({len(l["time"]) for l in logs}) > 1
    worst, codes = [0.0], set()
    for i in range(len(logs)):
        assert [k for k, _ in rows[i]] == list(range(len(logs[i]["time"])))
        codes |= set(check_job(defs, rows[i], recs[i], worst))
    assert {defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN, defs.SEQ_SKIPPED, defs.SEQ_INIT_WAIT} <= codes, codes
    _check_edits(defs, cases, rows)
    print(lidar, "worst |device - shim|", worst[0])


def test_alternating_entry_points(capi, defs, vlp, from_zero):
    """step_raw / step_pcl / step_ex in turn: bit-identical to the all-step_raw run at every step."""
    logs = vlp[0]
    rows = drive(capi, defs, vlp, len(logs), _jobs(logs), twins=("alt",))
    for i in range(len(logs)):
        _rows_equal(rows[i], from_zero[i])


def test_single_slot_permutation_and_packed16(capi, defs, vlp, from_zero):
    logs = vlp[0]
    jobs = _jobs(logs)
    for i in (0, 5):
        _rows_equal(drive(capi, defs, vlp, 1, [jobs[i]])[0], from_zero[i])
    perm = list(np.random.default_rng(3).permutation(len(logs)))
    rows = drive(capi, defs, vlp, len(logs), [jobs[i] for i in perm])
    for j, i in enumerate(perm):
        _rows_equal(rows[j], from_zero[i])
    rows = drive(capi, defs, vlp, len(logs), jobs, point_format=1)
    for i in range(len(logs)):
        _rows_equal(rows[i], from_zero[i])


def test_queue_through_fewer_slots(capi, defs, vlp):
    """Twice the recordings through a third of the slots, recycled with lins_gpu_seq_restart."""
    logs, _, _, recs = vlp
    n = len(logs)
    jobs = [(i % n, list(range(len(logs[i % n]["time"])))) for i in range(2 * n)]
    rows = drive(capi, defs, vlp, n // 3, jobs)
    worst = [0.0]
    for j, (i, _) in enumerate(jobs):
        assert [k for k, _ in rows[j]] == list(range(len(logs[i]["time"])))
        check_job(defs, rows[j], recs[i], worst)


def test_run_started_by_seq_begin(capi, defs, vlp):
    """The shim's hand-over (right after processSecondScan) through lins_gpu_seq_begin, then step_raw for every later scan."""
    logs, _, _, recs = vlp
    idx = [i for i in range(len(logs)) if recs[i]["handover_index"] >= 0]
    ho = [recs[i]["handover"] for i in idx]
    h = dict(filter_state=np.stack([x["filter_state"] for x in ho]), filter_cov=np.stack([x["filter_cov"] for x in ho]),
             global_state=np.stack([x["global_state"] for x in ho]), imu_last=np.stack([x["imu_last"] for x in ho]))
    for k in ("surf_map", "corner_map"):
        h[k] = np.concatenate([x[k] for x in ho])
        h[k + "_off"] = np.concatenate([[0], np.cumsum([len(x[k]) for x in ho])]).astype(np.int32)
    g = capi.LinsGpu()
    g.seq_begin(defs.LinsSeqParams.shipped(), h)
    S = len(idx)
    worst, codes = [0.0], set()
    first = [recs[i]["handover_index"] + 1 for i in idx]
    for t in range(max(len(logs[i]["time"]) - f for i, f in zip(idx, first))):
        sweeps, present, rows_imu, who = [], np.zeros(S, np.uint8), [], []
        for j, (i, f) in enumerate(zip(idx, first)):
            k = f + t
            o = logs[i]["imu_off"]
            if k < len(logs[i]["time"]):
                sweeps.append(logs[i]["sweeps"][k]); present[j] = 1; rows_imu.append(logs[i]["imu"][o[k]:o[k + 1]]); who.append((j, i, k))
            else:
                sweeps.append(np.zeros((0, 4), np.float32)); rows_imu.append(np.zeros((0, 7)))
        imu = np.concatenate(rows_imu).reshape(-1, 7)
        imu_off = np.concatenate([[0], np.cumsum([len(r) for r in rows_imu])]).astype(np.int32)
        g.seq_step_raw(dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=present))
        d, di = g.seq_download(), g.seq_download_init()
        for j, i, k in who:
            row = {key: np.array(v[j], copy=True) for key, v in d.items()}
            row.update({key: np.array(v[j], copy=True) for key, v in di.items()})
            codes |= set(check_job(defs, [(k, row)], recs[i], worst))
    assert S >= len(logs) - 3 and defs.SEQ_RAN in codes, (S, codes)


# ---- invalid input ------------------------------------------------------------------------------------------------------
def _raw_call(g, capi, defs, step, model, fp, scan_imu, edit=None):
    """lins_gpu_seq_step_raw through ctypes with the descriptor edited by edit(d, keep); returns the code."""
    keep = {"imu": np.ascontiguousarray(step["imu"], np.float64), "imu_off": np.ascontiguousarray(step["imu_off"], np.int32)}
    d = defs.LinsSeqRawDesc()
    d.raw = g._raw_desc(step["sweeps"], 0, keep)
    d.n_seq = len(keep["imu_off"]) - 1
    d.imu, d.imu_off = keep["imu"].ctypes.data, keep["imu_off"].ctypes.data
    if edit is not None:
        edit(d, keep)
    si = None if scan_imu is None else np.ascontiguousarray(scan_imu, np.float64)
    return g.L.lins_gpu_seq_step_raw(g.h, C.byref(d) if d is not None else None, C.byref(model) if model is not None else None,
                                     C.byref(fp) if fp is not None else None, None if si is None else si.ctypes.data)


def _bad_models(defs):
    out = []
    for field, v in (("line_num", 0), ("line_num", 129), ("scan_num", 1), ("scan_num", defs.FEAT_RING_CAP + 1), ("ang_res_x", 0.0),
                     ("ang_res_x", -0.2), ("ang_res_x", float("nan")), ("ang_res_y", float("inf")), ("ang_res_y", 0.0),
                     ("ang_bottom", float("nan")), ("ang_bottom", float("-inf")), ("ground_scan_ind", -1), ("ground_scan_ind", 16)):
        m = defs.LinsLidarModel.vlp16()
        setattr(m, field, v)
        out.append((field, v, m))
    return out


def _set_off(d, keep, f):
    off = keep["cloud_off"].copy()
    f(off)
    keep["bad_off"] = off
    d.raw.cloud_off = off.ctypes.data


def test_invalid_calls_change_nothing(capi, defs, vlp):
    logs = vlp[0][:3]
    S, n_steps = 3, 4
    model, fp = defs.LinsLidarModel.vlp16(), defs.LinsFeatureParams.shipped()

    def step(t):
        o = [l["imu_off"] for l in logs]
        imus = [l["imu"][oo[t]:oo[t + 1]] for l, oo in zip(logs, o)]
        return dict(sweeps=[l["sweeps"][t] for l in logs], imu=np.concatenate(imus).reshape(-1, 7),
                    imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32))

    def scan_imu(t):
        return np.stack([l["imu_last"][t] for l in logs])

    ref, g = capi.LinsGpu(), capi.LinsGpu()
    for c in (ref, g):
        c.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), S)
    edits = [
        ("offsets start at 1", lambda d, k: _set_off(d, k, lambda o: o.__setitem__(0, 1))),
        ("offsets decrease", lambda d, k: _set_off(d, k, lambda o: o.__setitem__(1, o[2] + 1))),
        ("null cloud", lambda d, k: setattr(d.raw, "cloud", None)),
        ("null offsets", lambda d, k: setattr(d.raw, "cloud_off", None)),
        ("imu without imu_off", lambda d, k: setattr(d, "imu_off", None)),
        ("null imu rows", lambda d, k: setattr(d, "imu", None)),
        ("bad point format", lambda d, k: setattr(d.raw, "point_format", 7)),
        ("n_seq", lambda d, k: setattr(d, "n_seq", S + 1)),
        ("raw.n_scans", lambda d, k: setattr(d.raw, "n_scans", S - 1)),
    ]
    for t in range(n_steps):
        ref.seq_step_raw(step(t), scan_imu=scan_imu(t))
        if t in (1, 2):  # (at t = 1 the slots are initialising, at t = 2 they run)
            st = step(t + 1)
            for field, v, m in _bad_models(defs):
                assert _raw_call(g, capi, defs, st, m, fp, scan_imu(t + 1)) == -1, (field, v)
            for what, e in edits:
                assert _raw_call(g, capi, defs, st, model, fp, scan_imu(t + 1), e) == -1, what
            assert _raw_call(g, capi, defs, st, None, fp, scan_imu(t + 1)) == -1
            assert _raw_call(g, capi, defs, st, model, None, scan_imu(t + 1)) == -1
            assert g.L.lins_gpu_seq_step_raw(g.h, None, C.byref(model), C.byref(fp), None) == -1
            if t == 1:
                assert _raw_call(g, capi, defs, st, model, fp, None) == -1  # initialising slots need scan_imu
        g.seq_step_raw(step(t), scan_imu=scan_imu(t))
        a, b = _snapshot(ref), _snapshot(g)
        _same(a, b, t, "invalid")
    assert {int(v) for v in a["status"]} & {defs.SEQ_RAN, defs.SEQ_ICP}, a["status"]


def test_step_raw_before_seq_open(capi, defs, vlp):
    g = capi.LinsGpu()
    with pytest.raises(capi.LinsError, match="error -3"):
        g.seq_step_raw(dict(imu=np.zeros((0, 7)), imu_off=np.zeros(2, np.int32), sweeps=[vlp[0][0]["sweeps"][0]]))
