"""GPU suite: lins_gpu_seq_step_pcl (sequence mode from segmented clouds) against lins_gpu_extract_features followed by
lins_gpu_seq_step_ex with the extracted clouds — bit-identical poses, filter state, init read-back, IESKF records with their
correspondence IDs, and maps at every step; the two entry points alternating in one run; invalid scans change nothing."""
import numpy as np
import pytest

import featcases as fc
from conftest import pkg

pytestmark = pytest.mark.gpu

S, STEPS = 5, 6


@pytest.fixture(scope="module")
def recordings(synth, defs):
    """S x STEPS segmented VLP-16 sweeps (config3 worlds) with the IMU sample processPCL gets with each scan; slot 3 is
    absent at step 2 and slot 4's scan at step 1 is cut below the first-scan gate."""
    scans = [[fc.segmented(synth, defs, "config3", 1000 + 37 * s + t)[0] for t in range(STEPS)] for s in range(S)]
    sc = scans[4][1]
    keep = np.arange(len(sc["seg"])) < 400  # the first 400 points only: few features
    for k in ("seg", "ground", "col", "range"):
        sc[k] = sc[k][keep]
    sc["start_ring"] = np.zeros(16, np.int32)
    sc["end_ring"] = np.zeros(16, np.int32)
    sc["start_ring"][0], sc["end_ring"][0] = 4, 390
    return scans


def _empty_scan():
    return dict(seg=np.zeros((0, 4), np.float32), ground=np.zeros(0, np.uint8), col=np.zeros(0, np.uint32), range=np.zeros(0, np.float32),
                start_ring=np.zeros(16, np.int32), end_ring=np.zeros(16, np.int32), ori=np.array([0, 6.283, 6.283], np.float32))


def _present(t):
    p = np.ones(S, np.uint8)
    if t == 2:
        p[3] = 0
    return p


def _scan_imu():
    si = np.zeros((S, 6))
    si[:, 2] = 9.81
    return si


def _step(recordings, t):
    p = _present(t)
    scans = [recordings[s][t] if p[s] else _empty_scan() for s in range(S)]
    return dict(imu=np.zeros((0, 7)), imu_off=np.zeros(S + 1, np.int32), scans=scans, present=p)


def _open(capi, defs):
    g = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
    g.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
    return g


def _via_ex(g, capi, step):
    feats = g.extract_features(step["scans"])
    d = dict(imu=step["imu"], imu_off=step["imu_off"], present=step["present"])
    for k in fc.NAMES:
        clouds = [capi._points_from_xyzi(f[k]) if step["present"][s] else capi._points_from_xyzi(np.zeros((0, 4))) for s, f in enumerate(feats)]
        d[k] = np.concatenate(clouds)
        d[k + "_off"] = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    g.seq_step(d, scan_imu=_scan_imu())


def _snapshot(g):
    out = {}
    d = g.seq_download(reports=True)
    for k in ("global_state", "filter_state", "filter_cov", "status"):
        out[k] = np.asarray(d[k]).copy()
    out["results"] = np.asarray(d["results"]).tobytes()
    out.update({"init_" + k: v for k, v in g.seq_download_init().items()})
    ie = g.seq_download_ieskf()
    for k in ("prior_state", "prior_cov", "state_out", "cov_out"):
        out["ieskf_" + k] = ie[k]
    out["ind"] = [None if a is None else a.tobytes() for a in ie["surf_ind"] + ie["corner_ind"]]
    mp = g.seq_download_maps()
    out["maps"] = [c.tobytes() for name in ("surf_map", "corner_map", "surf_tree", "corner_tree") for c in mp[name]] + [mp["stale"].tobytes()]
    return out


def _same(a, b, t):
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), f"step {t}: {k}"
        else:
            assert a[k] == b[k], f"step {t}: {k}"


def test_step_pcl_equals_extract_then_step_ex(capi, defs, recordings):
    g1, g2 = _open(capi, defs), _open(capi, defs)
    seen = set()
    for t in range(STEPS):
        step = _step(recordings, t)
        g1.seq_step_pcl(step, scan_imu=_scan_imu())
        _via_ex(g2, capi, step)
        a, b = _snapshot(g1), _snapshot(g2)
        _same(a, b, t)
        seen.update(int(v) for v in a["status"])
        assert g1.extract_ms() > 0
    # the run went through the first-scan gate, both initialisations, an idle slot and running steps (the recordings'
    # scans come from unrelated sweeps, so a running step's IESKF may diverge into the estimateTransform fallback)
    assert {0, 4, 5, 6} <= seen and seen & {2, 3}, seen


def test_alternating_entry_points(capi, defs, recordings):
    ref, g = _open(capi, defs), _open(capi, defs)
    for t in range(STEPS):
        step = _step(recordings, t)
        ref.seq_step_pcl(step, scan_imu=_scan_imu())
        if t % 2:
            _via_ex(g, capi, step)
        else:
            g.seq_step_pcl(step, scan_imu=_scan_imu())
        _same(_snapshot(ref), _snapshot(g), t)


def test_invalid_scan_changes_nothing(capi, defs, recordings):
    ref, g = _open(capi, defs), _open(capi, defs)
    for t in range(3):
        ref.seq_step_pcl(_step(recordings, t), scan_imu=_scan_imu())
        g.seq_step_pcl(_step(recordings, t), scan_imu=_scan_imu())
        if t == 1:
            bad = _step(recordings, 2)
            bad["scans"] = list(bad["scans"])
            s0 = dict(bad["scans"][0])
            s0["range"] = s0["range"].copy()
            s0["range"][100] = np.nan
            bad["scans"][0] = s0
            with pytest.raises(capi.LinsError, match="error -1"):
                g.seq_step_pcl(bad, scan_imu=_scan_imu())
            with pytest.raises(capi.LinsError, match="error -1"):
                g.seq_step_pcl(_step(recordings, 2))  # initialising slots need scan_imu
    _same(_snapshot(ref), _snapshot(g), 2)


# ---- pcl logs of simulated drives: against the shim through processPCL and against step_ex with host features ---------
import pclcases as pc  # noqa: E402
from test_gpu_seq_init import check_job, init_params  # noqa: E402


@pytest.fixture(scope="module")
def pcases(capi, defs):
    synth = pc.synth
    logs, edits = pc.case_logs(defs, gpu=capi.LinsGpu())
    print("drives replaced because a tie decides a pick:", edits.pop("tie_skipped"))
    recs = [synth.replay_pcl_log(l) for l in logs]
    flogs = [pc.feature_log(defs, l) for l in logs]
    return logs, edits, recs, flogs


def _whole(logs, i):
    return (i, list(range(len(logs[i]["time"]))))


def drive_pcl(capi, defs, logs, flogs, n_slots, jobs, twin=True):
    """Run `jobs` ((log index, scan indices)) through n_slots opened slots with lins_gpu_seq_step_pcl, restarting a slot
    whose job has ended.  With twin, a second context runs the same steps through lins_gpu_seq_step_ex with the host-extracted
    features and every read-back must be bit-identical after every step.  Returns rows[i] = [(scan, row)] of job i."""
    synth = pc.synth
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
    g2 = None
    if twin:
        g2 = capi.LinsGpu()
        g2.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
    rows = [[] for _ in jobs]
    empty = {c: flogs[0][c][:0] for c in defs.Batch.FIELDS}
    for restart, slots in pkg("bag_replay").slot_queue([len(ev) for _, ev in jobs], n_slots):
        if restart.any():
            g.seq_restart(restart)
            if g2:
                g2.seq_restart(restart)
        scans, fscans, present, who, scan_imu = [], [], [], [], np.zeros((n_slots, 6))
        for j, w in enumerate(slots):
            if w is None:
                scans.append(_empty_scan64()); fscans.append(dict(imu=np.zeros((0, 7)), **empty)); present.append(0); who.append(None)
                continue
            i, e = w
            k = jobs[i][1][e]
            li = jobs[i][0]
            scans.append(logs[li]["scans"][k]); fscans.append(synth.log_scan(flogs[li], k)); present.append(1); who.append((i, k))
            scan_imu[j] = logs[li]["imu_last"][k]
        imu = np.concatenate([np.asarray(s["imu"]).reshape(-1, 7) for s in fscans])
        imu_off = np.concatenate([[0], np.cumsum([len(s["imu"]) for s in fscans])]).astype(np.int32)
        pres = np.array(present, np.uint8)
        g.seq_step_pcl(dict(imu=imu, imu_off=imu_off, scans=scans, present=pres), scan_imu=scan_imu, line_num=pc.LINES)
        if g2:
            step = dict(present=pres, imu=imu, imu_off=imu_off)
            for c in defs.Batch.FIELDS:
                step[c] = np.concatenate([s[c] for s in fscans])
                step[c + "_off"] = np.concatenate([[0], np.cumsum([len(s[c]) for s in fscans])])
            g2.seq_step(step, scan_imu=scan_imu)
            _same(_snapshot(g), _snapshot(g2), len(rows))
        d, di = g.seq_download(), g.seq_download_init()
        for j, w in enumerate(who):
            if w is None:
                continue
            row = {k: np.array(v[j], copy=True) for k, v in d.items()}
            row.update({k: np.array(v[j], copy=True) for k, v in di.items()})
            rows[w[0]].append((w[1], row))
    return rows


def _empty_scan64():
    s = _empty_scan()
    s["start_ring"], s["end_ring"] = np.zeros(pc.LINES, np.int32), np.zeros(pc.LINES, np.int32)
    return s


@pytest.fixture(scope="module")
def from_zero(capi, defs, pcases):
    logs, _, _, flogs = pcases
    return drive_pcl(capi, defs, logs, flogs, len(logs), [_whole(logs, i) for i in range(len(logs))])


def test_pcl_logs_match_the_shim_and_step_ex(defs, pcases, from_zero):
    """From scan 0: every step bit-identical to step_ex with the host-extracted features (inside drive_pcl), and every
    recording against its own shim replaying the pcl log through processPCL, to the bar of test_gpu_seq_init.py."""
    logs, edits, recs, _ = pcases
    worst, codes = [0.0], set()
    for i in range(len(logs)):
        assert [k for k, _ in from_zero[i]] == list(range(len(logs[i]["time"])))
        codes |= set(check_job(defs, from_zero[i], recs[i], worst))
    assert {defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN, defs.SEQ_SKIPPED, defs.SEQ_INIT_WAIT} <= codes, codes
    assert any(l["lidar"] == 1 for l in logs) and len({len(l["time"]) for l in logs}) > 1
    # each edit of a segmented cloud reaches its case in the shim's own record
    for s, (case, k) in edits.items():
        r = recs[s]
        if case == "gate":
            assert r["code"][k] == defs.SEQ_SKIPPED, (case, r["code"][k])
        elif case == "guard":
            assert r["code"][k] in (defs.SEQ_RAN, defs.SEQ_ICP) and r["map_replaced"][k] == 0, (case, r["code"][k])
        elif case == "no_imu":
            assert logs[s]["imu_off"][k + 1] == logs[s]["imu_off"][k] and r["code"][k] in (defs.SEQ_RAN, defs.SEQ_ICP, defs.SEQ_SKIPPED)
        elif case == "first_gate":
            assert r["init_code"][k] == defs.SEQ_INIT_WAIT
    print("worst |device - shim|", worst[0])


def _rows_equal(a, b):
    """Bit-identical rows.  The result record is compared where the step ran the IESKF (lins_gpu_seq_download leaves it
    unspecified elsewhere), without its scan_id, the unit's place in that step's batch."""
    assert [k for k, _ in a] == [k for k, _ in b]
    for (_, x), (_, y) in zip(a, b):
        for key in x:
            if key != "results":
                assert np.asarray(x[key]).tobytes() == np.asarray(y[key]).tobytes(), key
        if int(x["status"]) in (2, 3):
            for f in ("iters", "flags", "pose"):
                assert np.asarray(x["results"][f]).tobytes() == np.asarray(y["results"][f]).tobytes(), f


def test_queue_through_fewer_slots(capi, defs, pcases, from_zero):
    """Twice the recordings through a third of the slots, recycled with lins_gpu_seq_restart."""
    logs, _, recs, flogs = pcases
    n = len(logs)
    jobs = [_whole(logs, i % n) for i in range(2 * n)]
    rows = drive_pcl(capi, defs, logs, flogs, n // 3, jobs)
    worst = [0.0]
    for j, (i, _) in enumerate(jobs):
        assert [k for k, _ in rows[j]] == list(range(len(logs[i]["time"])))
        check_job(defs, rows[j], recs[i], worst)


def test_single_slot_and_permutation(capi, defs, pcases, from_zero):
    logs, _, _, flogs = pcases
    for i in (0, 5):
        _rows_equal(drive_pcl(capi, defs, logs, flogs, 1, [_whole(logs, i)], twin=False)[0], from_zero[i])
    perm = list(np.random.default_rng(3).permutation(len(logs)))
    rows = drive_pcl(capi, defs, logs, flogs, len(logs), [_whole(logs, i) for i in perm], twin=False)
    for j, i in enumerate(perm):
        _rows_equal(rows[j], from_zero[i])


def test_run_started_by_seq_begin(capi, defs, pcases):
    """The shim's hand-over (right after processSecondScan) through lins_gpu_seq_begin, then step_pcl for every later scan."""
    logs, _, recs, _ = pcases
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
        scans, present, rows_imu, who = [], np.zeros(S, np.uint8), [], []
        for j, (i, f) in enumerate(zip(idx, first)):
            k = f + t
            o = logs[i]["imu_off"]
            if k < len(logs[i]["time"]):
                scans.append(logs[i]["scans"][k]); present[j] = 1; rows_imu.append(logs[i]["imu"][o[k]:o[k + 1]]); who.append((j, i, k))
            else:
                scans.append(_empty_scan64()); rows_imu.append(np.zeros((0, 7)))
        imu = np.concatenate(rows_imu)
        imu_off = np.concatenate([[0], np.cumsum([len(r) for r in rows_imu])]).astype(np.int32)
        g.seq_step_pcl(dict(imu=imu, imu_off=imu_off, scans=scans, present=present), line_num=pc.LINES)
        d, di = g.seq_download(), g.seq_download_init()
        for j, i, k in who:
            row = {key: np.array(v[j], copy=True) for key, v in d.items()}
            row.update({key: np.array(v[j], copy=True) for key, v in di.items()})
            codes |= set(check_job(defs, [(k, row)], recs[i], worst))
    assert S >= len(logs) - 2 and defs.SEQ_RAN in codes, (S, codes)
