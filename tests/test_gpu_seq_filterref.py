"""Sequence mode on the GPU, stage by stage, against tests/filterref.py (the reference's filter algebra restated in
float64) and the oracle's estimateTransform.  Each step starts from what the device held before it (seq_download) and
every stage's output is checked against filterref from that step's inputs:
  * prior_state / prior_cov = predict over the step's IMU rows (the test tracks acc_last / gyr_last itself);
  * RAN: the post stage (integrateTransformation, reset(1), roll / pitch) of the IESKF's posterior;
  * ICP: the post stage of the prior with estimateTransform's pose (the oracle's, from the prior) and the prior
    covariance, except on a stale 1-NN index;
  * SKIPPED: the prior; IDLE: bit-identical; INIT_WAIT: unchanged;
  * fresh slots: GlobalState() and initializeCovariance; FIRST: processFirstScan; SECOND: processSecondScan with the
    test's own pre-integration of the rows and the device's ICP pose, and that ICP itself (iterations, convergence, pose)
    against the oracle from filterref's start pose.
Three runs: (a) the case logs from scan 0 with the shipped non-zero INIT_BA / INIT_BW, (b) hand-overs, IMU rows and scan
IMU samples edited to hit the edges of the algebra (the IESKF may diverge there; the stage checks still apply), (c) every
running scan forced onto the ICP branch.  The feature logs and the shim's hand-overs only supply inputs; no expected
value comes from this project's own code."""
from collections import Counter

import numpy as np
import pytest

import filterref as fr
import seq_cases as sc
from conftest import pkg
from filterref import check_cov, check_state

pytestmark = pytest.mark.gpu
M = fr.F64
ICP_POSE_TOL = 1.2e-14  # the second scans' estimateTransform against the oracle: 10x the worst of run (a) on an H100 SXM 80 GB (1.2e-15)
POS_STD, VEL_STD, ATT_STD = (0.05, 0.1, 0.02), (0.2, 0.1, 0.05), (0.5, 0.7, 1.5)


def params(defs):
    """The shipped constants (non-zero INIT_BA / INIT_BW) with non-zero INIT_POS / VEL / ATT_STD, for the device and for
    filterref alike."""
    sp = defs.LinsSeqParams.shipped(init_pos_std=POS_STD, init_att_std=ATT_STD)
    ip = defs.LinsSeqInitParams.shipped(init_vel_std=VEL_STD)
    p = dict(fr.YAML, init_pos_std=POS_STD, init_att_std=ATT_STD, init_vel_std=VEL_STD)
    assert any(ip.init_ba) and any(ip.init_bw)
    return sp, ip, p


def cov(c):
    return np.asarray(c, float).reshape(18, 18).T  # the C-ABI's column-major 18x18


def same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def drive(capi, defs, ob, logs, events, lidar_params=None, begin=None):
    """Run slot j through events[j] (scan indices of logs[j], None = absent) from a seq_open run (or, with `begin`, from
    those seq_begin hand-overs) and check every step.  Returns a dict: seen (status codes), worst (ICP pose difference),
    icp_compared / icp_stale (ICP steps whose post stage was / was not compared), second_iters (per step, the icp_iters of
    its second scans) and edges (what the running steps' inputs hit)."""
    synth = pkg("synth")
    sp, ip, p = params(defs)
    noise = fr.noise_diag(p)
    n = len(logs)
    g = capi.LinsGpu(lidar_params)
    if begin is None:
        g.seq_open(sp, ip, n)
        fus = [fr.STATUS_INIT] * n
        imu_last = [None] * n
        st0 = g.seq_download()  # a new StateEstimator: GlobalState() twice and initializeCovariance
        for j in range(n):
            check_state(st0["global_state"][j], fr.global_state(M), ("fresh global", j))
            check_state(st0["filter_state"][j], fr.global_state(M), ("fresh filter", j))
            check_cov(st0["filter_cov"][j], fr.initialize_covariance(M, p), ("fresh", j))
    else:
        g.seq_begin(sp, begin)
        fus = [fr.STATUS_RUNNING] * n
        imu_last = [(np.array(h[:3]), np.array(h[3:])) for h in np.asarray(begin["imu_last"], float)]
    orc = ob.Oracle(lidar_params)
    pre = [None] * n
    seen, worst, n_stale, n_icp = [], [0.0], [0], [0]
    second_iters, edges = [], Counter()
    empty = {c: logs[0][c][:0] for c in defs.Batch.FIELDS}
    for t in range(max(len(e) for e in events)):
        before, maps = g.seq_download(), g.seq_download_maps()
        scans, present, scan_imu = [], np.zeros(n, np.uint8), np.zeros((n, 6))
        for j in range(n):
            k = events[j][t] if t < len(events[j]) else None
            if k is None:
                scans.append(dict(imu=np.zeros((0, 7)), **empty))
            else:
                s = synth.log_scan(logs[j], k)
                scans.append(s)
                present[j] = 1
                scan_imu[j] = s["imu_last"]
        step = dict(present=present, imu=np.concatenate([np.asarray(s["imu"]).reshape(-1, 7) for s in scans]),
                    imu_off=np.concatenate([[0], np.cumsum([len(s["imu"]) for s in scans])]))
        for c in defs.Batch.FIELDS:
            step[c] = np.concatenate([s[c] for s in scans])
            step[c + "_off"] = np.concatenate([[0], np.cumsum([len(s[c]) for s in scans])])
        g.seq_step(step, scan_imu=scan_imu)
        second_iters.append([])
        d, ie, di = g.seq_download(), g.seq_download_ieskf(), g.seq_download_init()
        for j in range(n):
            code = int(d["status"][j])
            seen.append(code)
            gb, fb, pb = before["global_state"][j], before["filter_state"][j], before["filter_cov"][j]
            ga, fa, pa = d["global_state"][j], d["filter_state"][j], d["filter_cov"][j]
            where = (t, j, code)
            if not present[j]:
                assert code == defs.SEQ_IDLE, where
                assert same(ga, gb) and same(fa, fb) and same(pa, pb), where
                continue
            rows = np.asarray(scans[j]["imu"]).reshape(-1, 7)
            s = scans[j]
            if fus[j] == fr.STATUS_RUNNING:
                st = dict(state=fb, P=cov(pb), acc_last=imu_last[j][0], gyr_last=imu_last[j][1])
                q = fb[6:10]
                edges["w_neg"] += q[3] < 0
                edges["q_off"] += 5e-10 < abs(np.linalg.norm(q) - 1) < 2e-9
                edges["gz_pos"] += fb[18] > 0
                edges["gz_zero"] += fb[18] == 0 and fb[16:19].any()
                edges["g_zero"] += not fb[16:19].any()
                for r in rows:
                    th = np.linalg.norm((0.5 * (np.asarray(st["gyr_last"], float) + r[4:7]) - st["state"][13:16]) * r[0])
                    edges["theta0"] += th == 0
                    edges["theta_lo"] += 0 < th < 1e-10
                    edges["theta_hi"] += 1e-10 <= th < 2e-10
                    edges["theta_pi"] += th > np.pi
                    edges["dt0"] += r[0] == 0
                    edges["gap"] += r[0] >= 0.1
                    fr.process_imu(M, fus[j], r[0], r[1:4], r[4:7], filt=st, noise=noise)
                imu_last[j] = (st["acc_last"], st["gyr_last"])
                check_state(ie["prior_state"][j], st["state"], ("prior", where))
                check_cov(ie["prior_cov"][j], st["P"], ("prior", where))
                if code == defs.SEQ_SKIPPED:
                    check_state(fa, st["state"], ("skipped", where))
                    check_cov(pa, st["P"], ("skipped", where))
                    assert same(ga, gb), where
                    continue
                if code == defs.SEQ_RAN:
                    upd, upd_P = ie["state_out"][j], cov(ie["cov_out"][j])
                else:
                    assert code == defs.SEQ_ICP and d["results"]["flags"][j] & 2, where  # (bit 1: the IESKF diverged)
                    # estimateTransform from the prior on the oracle.  After a guard-cut scan the index is stale: its IDs
                    # address the newer map cloud, which the oracle's set_map cannot express, so only the prior is checked
                    if maps["stale"][j]:
                        n_stale[0] += 1
                        continue
                    n_icp[0] += 1
                    orc.set_map(maps["surf_map"][j], maps["corner_map"][j])
                    prior = ie["prior_state"][j]
                    ot, oq, _, _ = orc.estimate_transform(s["surf_flat"], s["corner_sharp"], prior[0:3], prior[6:10])
                    upd, upd_P = fr.icp_prior(prior, ot, oq), cov(ie["prior_cov"][j])
                want_g, want_f, want_P = fr.post_step(M, gb, upd, upd_P, p)
                rpy = fr.Q2rpy(M, fr.integrate(M, gb, upd)[6:10])
                skip = range(6, 10) if not np.cos(rpy[1]) > fr.COS_PITCH_MIN else ()
                check_state(ga, want_g, ("post global", where), skip=skip)
                check_state(fa, want_f, ("post filter", where))
                check_cov(pa, want_P, ("post", where))
                continue
            if fus[j] == fr.STATUS_FIRST_SCAN:
                for r in rows:
                    fr.process_imu(M, fus[j], r[0], r[1:4], r[4:7], pre=pre[j])
            if code == defs.SEQ_INIT_WAIT:
                assert same(ga, gb) and same(fa, fb) and same(pa, pb), where
                fus[j] = fr.STATUS_INIT
            elif code == defs.SEQ_FIRST:
                assert fus[j] == fr.STATUS_INIT, where
                want_f, want_P, pre[j], al, gl = fr.first_scan(M, scan_imu[j], p)
                imu_last[j] = (al, gl)
                check_state(fa, want_f, ("first", where))
                check_cov(pa, want_P, ("first", where))
                assert same(ga, gb), where
                fus[j] = fr.STATUS_FIRST_SCAN
            else:
                assert code == defs.SEQ_SECOND and fus[j] == fr.STATUS_FIRST_SCAN, where
                pl, ql = fr.second_scan_start(M, pre[j])
                orc.set_map(maps["surf_map"][j], maps["corner_map"][j])
                ot, oq, oit, ocv = orc.estimate_transform(s["surf_flat"], s["corner_sharp"], pl, ql)
                assert (int(di["icp_iters"][j]), bool(di["icp_converged"][j])) == (oit, ocv), (where, di["icp_iters"][j], oit)
                second_iters[-1].append(oit)
                edges["sum_dt0"] += pre[j].sum_dt == 0
                edges["fz_zero"] += scan_imu[j][2] - p["init_ba"][2] == 0
                edges["g_over"] += abs(scan_imu[j][0] - p["init_ba"][0]) > fr.G0
                diff = np.abs(di["icp_pose"][j] - np.concatenate([ot, oq])).max()
                worst[0] = max(worst[0], diff)
                assert diff <= ICP_POSE_TOL, (where, diff)
                want_g, want_f, want_P, al, gl = fr.second_scan(M, pre[j], di["icp_pose"][j][:3], di["icp_pose"][j][3:], scan_imu[j], p)
                imu_last[j] = (al, gl)
                check_state(ga, want_g, ("second global", where))
                check_state(fa, want_f, ("second filter", where))
                check_cov(pa, want_P, ("second", where))
                fus[j] = fr.STATUS_RUNNING
        for j in range(n):
            assert int(di["fusion_status"][j]) == fus[j], (t, j)
    g.close()
    orc.close()
    return dict(seen=seen, worst=worst[0], icp_compared=n_icp[0], icp_stale=n_stale[0], second_iters=second_iters, edges=edges)


def edited(log, k, field, n):
    synth = pkg("synth")
    scans = [synth.log_scan(log, i) for i in range(len(log["time"]))]
    scans[k][field] = scans[k][field][:n].copy()
    return synth.make_log(scans, log["lidar"])


@pytest.fixture(scope="module")
def logs():
    lg, _ = sc.case_logs(48)
    lg[6] = edited(lg[6], 0, "corner_less_sharp", 9)  # a first scan below the gate: INIT_WAIT, then scan 1 is the first
    return lg


def test_from_scan_zero_with_the_shipped_biases(capi, defs, ob, logs):
    """Run (a): the 48 case logs from scan 0 with the shipped INIT_BA / INIT_BW and non-zero INIT_*_STD; every fourth
    slot is absent for two steps (once before and once after its second scan).  The second scans of one step run as one
    batched estimateTransform loop in which units end at different iterations."""
    events = []
    for j, l in enumerate(logs):
        ev = list(range(len(l["time"])))
        if j % 4 == 1:
            ev = ev[:1] + [None] + ev[1:5] + [None] + ev[5:]
        events.append(ev)
    r = drive(capi, defs, ob, logs, events)
    seen = r["seen"]
    counts = {c: seen.count(c) for c in set(seen)}
    for c in (defs.SEQ_IDLE, defs.SEQ_INIT_WAIT, defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN, defs.SEQ_SKIPPED):
        assert counts.get(c, 0) > 0, (c, counts)
    assert counts[defs.SEQ_SECOND] >= 48 and counts[defs.SEQ_RAN] >= 500, counts
    assert any(len(set(it)) > 1 for it in r["second_iters"]), r["second_iters"]
    print("codes", counts, "second-scan iterations per step", [sorted(set(it)) for it in r["second_iters"] if it],
          "worst |icp_pose - oracle|", r["worst"])


def _edit_scan(log, k, fn):
    synth = pkg("synth")
    scans = [synth.log_scan(log, i) for i in range(len(log["time"]))]
    scans[k] = dict(scans[k], imu=np.array(scans[k]["imu"], float), imu_last=np.array(scans[k]["imu_last"], float))
    fn(scans[k])
    return synth.make_log(scans, log["lidar"])


def test_edges_from_edited_handovers_and_scans(capi, defs, ob, synth, logs):
    """Run (b): the edges of test_filterref_cpu.py on the device.  Running sequences start (seq_begin) from shim
    hand-overs whose filter state or first IMU rows are edited: q with w < 0, |q| = 1 +- 1e-9, gn with z > 0, z = 0 and
    gn = 0, gyr == bw (theta = 0), theta just below and above 1e-10, |w dt| past pi, dt = 0 and 0.1 / 0.5 s gaps.  Slots
    opened from scan 0 hit the hand-over edges: a second scan without IMU rows (sum_dt = 0), |fx - ba_x| > G0 (a NaN
    pitch) and fz - ba_z = 0 (sign(0)).  A slot whose state turned non-finite is absent afterwards."""
    synth = pkg("synth")
    base = [i for i in range(len(logs)) if logs[i]["lidar"] == 0 and i not in (0, 1, 2, 3, 6)][:6]
    kinds = ["w_neg", "q_plus", "q_minus", "gz_pos", "gz_zero", "g_zero", "theta0", "theta_lo", "theta_hi", "spin", "gaps"]
    n_steps = 4
    ho = dict(filter_state=[], filter_cov=[], global_state=[], imu_last=[], surf_map=[], corner_map=[])
    slot_logs, events = [], []
    for j, kind in enumerate(kinds):
        log = logs[base[j % len(base)]]
        rec = synth.replay_feature_log(log)
        h, k0 = rec["handover"], rec["handover_index"]
        f, il = np.array(h["filter_state"], float), np.array(h["imu_last"], float)
        bw = f[13:16]
        scans = [synth.log_scan(log, k) for k in range(len(log["time"]))]
        rows = np.array(scans[k0 + 1]["imu"], float)
        if kind == "w_neg":
            f[6:10] = -f[6:10]
        elif kind in ("q_plus", "q_minus"):
            f[6:10] *= 1 + (1e-9 if kind == "q_plus" else -1e-9)
        elif kind == "gz_pos":
            f[16:19] = (0.3, -0.2, 9.8)
        elif kind == "gz_zero":
            f[16:19] = (9.81 * 0.6, -9.81 * 0.8, 0.0)
        elif kind == "g_zero":
            f[16:19] = 0.0
        elif kind == "theta0":
            il[3:6] = bw
            rows[:, 4:7] = bw
        elif kind in ("theta_lo", "theta_hi"):
            dvec = np.array([0.6, -0.48, 0.64]) * (0.98e-10 if kind == "theta_lo" else 1.02e-10) / 0.0025
            rows[:, 0] = 0.0025
            il[3:6] = bw + dvec
            rows[:, 4:7] = bw + dvec
        elif kind == "spin":
            w = bw + np.array([6.0, -8.0, 0.0])  # |w| dt = 5 rad over a 0.5 s row
            il[3:6] = w
            rows[0, 0], rows[0, 4:7] = 0.5, w
        else:
            rows[1, 0], rows[2, 0], rows[3, 0] = 0.0, 0.1, 0.5
        scans[k0 + 1] = dict(scans[k0 + 1], imu=rows)
        slot_logs.append(synth.make_log(scans, log["lidar"]))
        ev = list(range(k0 + 1, min(k0 + 1 + n_steps, len(log["time"]))))
        if kind in ("gz_pos", "gz_zero", "g_zero"):
            ev = ev[:1]  # (the post stage leaves these non-finite or far off; one checked step each)
        events.append(ev)
        for key, v in (("filter_state", f), ("filter_cov", h["filter_cov"]), ("global_state", h["global_state"]), ("imu_last", il)):
            ho[key].append(np.asarray(v, float))
        ho["surf_map"].append(h["surf_map"])
        ho["corner_map"].append(h["corner_map"])
    begin = {k: np.stack(ho[k]) for k in ("filter_state", "filter_cov", "global_state", "imu_last")}
    for k in ("surf_map", "corner_map"):
        begin[k] = np.concatenate(ho[k])
        begin[k + "_off"] = np.concatenate([[0], np.cumsum([len(c) for c in ho[k]])])
    r = drive(capi, defs, ob, slot_logs, events, begin=begin)
    e = r["edges"]
    for k in ("w_neg", "q_off", "gz_pos", "gz_zero", "g_zero", "theta0", "theta_lo", "theta_hi", "theta_pi", "dt0", "gap"):
        assert e[k] > 0, (k, e)

    # the hand-over edges, from scan 0 (each slot runs its first and second scan only)
    ba = fr.YAML["init_ba"]
    init_logs = [_edit_scan(logs[base[0]], 1, lambda s: s.update(imu=np.zeros((0, 7)))),
                 _edit_scan(logs[base[1]], 1, lambda s: s["imu_last"].__setitem__(0, ba[0] + 10.5)),
                 _edit_scan(logs[base[2]], 1, lambda s: s["imu_last"].__setitem__(2, ba[2]))]
    r2 = drive(capi, defs, ob, init_logs, [[0, 1]] * 3)
    for k in ("sum_dt0", "g_over", "fz_zero"):
        assert r2["edges"][k] > 0, (k, r2["edges"])
    print("edges", dict(e), dict(r2["edges"]), "codes", Counter(r["seen"]), Counter(r2["seen"]))


def test_icp_branch_with_the_shipped_biases(capi, defs, ob, logs):
    """Run (c): lidar_scale = 1e9 makes every running scan's IESKF diverge, so each one takes the estimateTransform
    fallback and the post stage starts from the prior with its pose."""
    pick = [0, 1, 2, 4, 5, 11]
    r = drive(capi, defs, ob, [logs[i] for i in pick], [list(range(len(logs[i]["time"]))) for i in pick],
              lidar_params=defs.LinsParams.shipped(lidar_scale=1e9))
    seen = r["seen"]
    assert seen.count(defs.SEQ_ICP) >= 80 and defs.SEQ_RAN not in seen, {c: seen.count(c) for c in set(seen)}
    assert r["icp_compared"] >= 80 and r["icp_compared"] + r["icp_stale"] == seen.count(defs.SEQ_ICP), r
    print("ICP steps", seen.count(defs.SEQ_ICP), "compared", r["icp_compared"], "stale", r["icp_stale"],
          "worst |icp_pose - oracle|", r["worst"])
