"""Sequence mode from the first scan on the GPU: slots opened by lins_gpu_seq_open run processPCL's whole status machine
(processFirstScan, the IMU pre-integration, processSecondScan with its estimateTransform) and take new recordings through
lins_gpu_seq_restart.  Every recording is compared at every scan with one C++ StateEstimator shim replaying the same
feature log (tools/synth/lins_sequence.cpp)."""
import numpy as np
import pytest

import seq_cases as sc
from conftest import pkg

STATE_TOL = 1e-7
pytestmark = pytest.mark.gpu
N_SEQ = 48


def init_params(defs):
    """The shim's filter constants (lins_sequence.cpp seq_params: zero INIT_BA / INIT_BW, the shipped stds)."""
    return defs.LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0))


@pytest.fixture(scope="module")
def cases():
    synth = pkg("synth")
    logs, edits = sc.case_logs(N_SEQ)
    recs = [synth.replay_feature_log(l) for l in logs]
    return logs, edits, recs


def drive(capi, defs, logs, n_slots, jobs, params=None):
    """Run `jobs` through n_slots opened slots.  A job is (log index, events): one event per step, a scan index of the log
    (present) or None (idle).  Jobs are taken in order by the first free slot; a slot whose job has ended is restarted
    (lins_gpu_seq_restart) and starts the next job on the following step.  Returns (rows, steps): rows[i] = [(scan, row)]
    of job i, steps = per step the list of (slot, job, code) of the present slots."""
    synth = pkg("synth")
    g = capi.LinsGpu(params)
    g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
    rows, steps = [[] for _ in jobs], []
    empty = {c: logs[0][c][:0] for c in defs.Batch.FIELDS}
    for restart, slots in pkg("bag_replay").slot_queue([len(ev) for _, ev in jobs], n_slots):
        if restart.any():
            g.seq_restart(restart)
        scans, present, who, scan_imu = [], [], [], np.zeros((n_slots, 6))
        for j, w in enumerate(slots):
            k = jobs[w[0]][1][w[1]] if w is not None else None
            if k is None:
                scans.append(dict(imu=np.zeros((0, 7)), **empty)); present.append(0); who.append(None)
            else:
                s = synth.log_scan(logs[jobs[w[0]][0]], k)
                scans.append(s); present.append(1); who.append((w[0], k)); scan_imu[j] = s["imu_last"]
        step = dict(present=np.array(present, np.uint8), imu=np.concatenate([np.asarray(s["imu"]).reshape(-1, 7) for s in scans]),
                    imu_off=np.concatenate([[0], np.cumsum([len(s["imu"]) for s in scans])]))
        for c in defs.Batch.FIELDS:
            step[c] = np.concatenate([s[c] for s in scans])
            step[c + "_off"] = np.concatenate([[0], np.cumsum([len(s[c]) for s in scans])])
        g.seq_step(step, scan_imu=scan_imu)
        d, di = g.seq_download(), g.seq_download_init()
        st = []
        for j, w in enumerate(who):
            if w is None:
                continue
            row = {k: np.array(v[j], copy=True) for k, v in d.items()}
            row.update({k: np.array(v[j], copy=True) for k, v in di.items()})
            rows[w[0]].append((w[1], row))
            st.append((j, w[0], int(d["status"][j])))
        steps.append(st)
    g.close()
    return rows, steps


def check_job(defs, rows, rec, worst):
    """One job's rows against its shim replay: codes, status, iterations, flags, the second scan's ICP bit for bit, state
    and covariance within STATE_TOL.  Returns the codes seen."""
    seen = []
    for k, d in rows:
        code = rec["init_code"][k]
        assert d["status"] == code, (k, d["status"], code)
        assert d["fusion_status"] == rec["est_status"][k], (k, d["fusion_status"], rec["est_status"][k])
        if code in (defs.SEQ_RAN, defs.SEQ_ICP):
            assert d["results"]["iters"] == rec["iters"][k] and d["results"]["flags"] == rec["flags"][k], k
        if code == defs.SEQ_SECOND:
            assert np.array_equal(d["icp_pose"], rec["icp_pose"][k]), (k, d["icp_pose"] - rec["icp_pose"][k])
            assert (d["icp_iters"], d["icp_converged"]) == (rec["icp_iters"][k], rec["icp_converged"][k]), k
            assert d["icp_iters"] >= 1
        for key in ("global_state", "filter_state", "filter_cov"):
            diff = np.abs(d[key] - rec[key][k]).max()
            worst[0] = max(worst[0], diff)
            assert diff <= STATE_TOL, (k, key, diff)
        seen.append(int(code))
    return seen


def whole(logs, i):
    return (i, list(range(len(logs[i]["time"]))))


@pytest.fixture(scope="module")
def open48(capi, defs, cases):
    logs, _, _ = cases
    return drive(capi, defs, logs, N_SEQ, [whole(logs, i) for i in range(N_SEQ)])


def test_from_scan_zero_matches_one_shim_per_sequence(defs, cases, open48):
    logs, edits, recs = cases
    rows, _ = open48
    worst, codes = [0.0], set()
    for i in range(N_SEQ):
        assert [k for k, _ in rows[i]] == list(range(len(logs[i]["time"])))
        codes |= set(check_job(defs, rows[i], recs[i], worst))
    assert {defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN, defs.SEQ_SKIPPED} <= codes, codes
    print("worst |device - shim|", worst[0])


def edited(log, edits):
    synth = pkg("synth")
    scans = [synth.log_scan(log, i) for i in range(len(log["time"]))]
    for k, field, n in edits:
        scans[k][field] = scans[k][field][:n].copy()
    return synth.make_log(scans, log["lidar"])


def test_init_edges_match_the_shim(capi, defs, cases):
    """The first scan's gate at exactly 9 / 10 corners and 99 / 100 surfs, a second scan below the gate (back to INIT:
    scan 2 is the new first scan), and a slot idle between its first and second scan."""
    logs, _, _ = cases
    synth = pkg("synth")
    base = [l for l in logs[:12] if l["lidar"] == 0]
    for l in base[:6]:
        s0 = synth.log_scan(l, 0)
        assert len(s0["corner_less_sharp"]) >= 10 and len(s0["surf_less_flat"]) >= 100
    cl, sl = "corner_less_sharp", "surf_less_flat"
    variants = [edited(base[0], [(0, cl, 9)]), edited(base[1], [(0, cl, 10)]), edited(base[2], [(0, sl, 99)]),
                edited(base[3], [(0, sl, 100)]), edited(base[4], [(1, sl, 60)]), base[5]]
    recs = [synth.replay_feature_log(l) for l in variants]
    jobs = [whole(variants, i) for i in range(5)]
    n5 = len(variants[5]["time"])
    jobs.append((5, [0, None, None] + list(range(1, n5))))  # idle for two steps between the first and the second scan
    rows, steps = drive(capi, defs, variants, len(jobs), jobs)
    worst = [0.0]
    seen = [check_job(defs, rows[i], recs[i], worst) for i in range(len(jobs))]
    assert seen[0][:2] == [defs.SEQ_INIT_WAIT, defs.SEQ_FIRST] and seen[2][:2] == [defs.SEQ_INIT_WAIT, defs.SEQ_FIRST]
    assert seen[1][:2] == [defs.SEQ_FIRST, defs.SEQ_SECOND] and seen[3][:2] == [defs.SEQ_FIRST, defs.SEQ_SECOND]
    assert seen[4][:4] == [defs.SEQ_FIRST, defs.SEQ_INIT_WAIT, defs.SEQ_FIRST, defs.SEQ_SECOND]
    assert seen[5][:3] == [defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN]
    assert [w for w in steps[1] if w[1] == 5] == [] and [w for w in steps[2] if w[1] == 5] == []  # (the idle steps)
    print("worst |device - shim|", worst[0])


def test_slots_recycle_through_a_queue_of_recordings(capi, defs, cases):
    """110 recordings of spread lengths (prefixes of the case logs) through 32 slots: a slot that finishes restarts with
    the next recording on the following step, so first, second and running scans mix within steps.  Every recording
    matches its own fresh shim replay at every scan."""
    logs, _, recs = cases
    jobs = []
    for i in range(110):
        li = (7 * i) % N_SEQ
        n = min(len(logs[li]["time"]), 3 + (5 * i) % 19)
        jobs.append((li, list(range(n))))
    jobs[40] = (jobs[40][0], list(range(len(logs[jobs[40][0]]["time"]))))
    rows, steps = drive(capi, defs, logs, 32, jobs)
    worst = [0.0]
    for i, (li, ev) in enumerate(jobs):
        assert [k for k, _ in rows[i]] == ev, i
        check_job(defs, rows[i], recs[li], worst)
    mixed = sum({defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN} <= {c for _, _, c in st} for st in steps)
    assert mixed >= 3, mixed
    # a freed slot takes the next job on the very next step
    first_step = {}
    for t, st in enumerate(steps):
        for j, i, _ in st:
            first_step.setdefault(i, (t, j))
    last_step = {}
    for t, st in enumerate(steps):
        for j, i, _ in st:
            last_step[i] = (t, j)
    handoffs = 0
    for i in range(110):
        t, j = last_step[i]
        nxt = [i2 for i2, (t2, j2) in first_step.items() if j2 == j and t2 > t]
        if nxt:
            assert first_step[min(nxt)][0] == t + 1, (i, t, first_step[min(nxt)])
            handoffs += 1
    assert handoffs >= 70, handoffs
    print("worst |device - shim|", worst[0], "steps", len(steps), "mixed steps", mixed)


def _same(a, b):
    for key in ("global_state", "filter_state", "filter_cov", "status", "fusion_status", "icp_pose", "icp_iters", "icp_converged"):
        if not np.array_equal(a[key], b[key]):
            return key
    if a["status"] in (2, 3) and not (np.array_equal(a["results"]["pose"], b["results"]["pose"]) and a["results"]["iters"] == b["results"]["iters"]):
        return "results"
    return None


def test_outputs_do_not_depend_on_the_other_slots(capi, defs, cases, open48):
    """S = 1, a permutation of the 48 and the VLP-16 logs tiled to S = 300 (several units per CTA in the batched
    estimateTransform and the IESKF): every output, the second scans' ICP included, is bit-identical."""
    logs, _, _ = cases
    full, _ = open48
    rng = np.random.default_rng(5)
    vlp = [i for i in range(N_SEQ) if logs[i]["lidar"] == 0]
    for order in ([3], [int(i) for i in rng.permutation(N_SEQ)], [vlp[j % len(vlp)] for j in range(300)]):
        part, _ = drive(capi, defs, logs, len(order), [whole(logs, i) for i in order])
        for j, i in enumerate(order):
            assert [k for k, _ in part[j]] == [k for k, _ in full[i]]
            for (k, d), (_, e) in zip(part[j], full[i]):
                assert _same(d, e) is None, (len(order), j, i, k, _same(d, e))


def test_bad_calls_are_rejected_and_change_nothing(capi, defs, cases):
    logs, _, _ = cases
    synth = pkg("synth")
    g = capi.LinsGpu()
    L = g.L
    sp, ip = defs.LinsSeqParams.shipped(), init_params(defs)
    assert L.lins_gpu_seq_open(g.h, sp, ip, 0) == -1 and L.lins_gpu_seq_open(g.h, sp, ip, -3) == -1
    assert L.lins_gpu_seq_restart(g.h, np.ones(1, np.uint8).ctypes.data) == -3  # no run yet
    g.seq_open(sp, ip, 2)
    s = [synth.log_scan(logs[i], 0) for i in range(2)]
    step = dict(imu=np.zeros((0, 7)), imu_off=[0, 0, 0])
    for c in defs.Batch.FIELDS:
        step[c] = np.concatenate([x[c] for x in s])
        step[c + "_off"] = [0, len(s[0][c]), len(s[0][c]) + len(s[1][c])]
    before = (g.seq_download(), g.seq_download_init(), g.seq_download_maps())

    def unchanged():
        after = (g.seq_download(), g.seq_download_init(), g.seq_download_maps())
        for a, b in zip(before[:2], after[:2]):
            for k in a:
                assert np.array_equal(a[k], b[k]), k
        for k in ("surf_map", "corner_map"):
            assert all(len(x) == len(y) for x, y in zip(before[2][k], after[2][k]))

    with pytest.raises(capi.LinsError):  # a present slot initialises: scan_imu is required
        g.seq_step(step)
    unchanged()
    assert L.lins_gpu_seq_restart(g.h, None) == -1
    unchanged()
    # with slot 0 absent and slot 1 present, still required; with both absent, not
    with pytest.raises(capi.LinsError):
        g.seq_step(dict(step, present=np.array([0, 1], np.uint8)))
    unchanged()
    g.seq_step(dict(step, present=np.array([0, 0], np.uint8)))
    assert list(g.seq_download()["status"]) == [defs.SEQ_IDLE] * 2
    g.seq_step(step, scan_imu=np.stack([x["imu_last"] for x in s]))
    assert list(g.seq_download()["status"]) == [defs.SEQ_FIRST] * 2
    # restart on a run started by lins_gpu_seq_begin
    recs = synth.replay_feature_log(logs[10])
    h = recs["handover"]
    ho = dict(h, surf_map_off=[0, len(h["surf_map"])], corner_map_off=[0, len(h["corner_map"])])
    for k in ("filter_state", "filter_cov", "global_state", "imu_last"):
        ho[k] = h[k][None]
    g.seq_begin(sp, ho)
    before = (g.seq_download(), g.seq_download_init(), g.seq_download_maps())
    assert L.lins_gpu_seq_restart(g.h, np.ones(1, np.uint8).ctypes.data) == -1
    unchanged()
    assert list(g.seq_download_init()["fusion_status"]) == [defs.FUSION_RUNNING]
    g.close()
