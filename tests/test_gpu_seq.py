"""Sequence mode on the GPU: many sequences in lockstep through lins_gpu_seq_step against one C++ StateEstimator shim per
sequence replaying the same feature log (tools/synth/lins_sequence.cpp), and each stage of a step against the host
StatePredictor / the single-scan seam at equal inputs."""
import re

import numpy as np
import pytest

import seq_cases as sc
from conftest import pkg

STATE_TOL = 1e-7
PREDICT_RTOL = 1e-12  # the device's f64 sin / cos may differ from glibc's by an ulp
pytestmark = pytest.mark.gpu
N_SEQ = 48


@pytest.fixture(scope="module")
def cases():
    synth = pkg("synth")
    logs, edits = sc.case_logs(N_SEQ)
    recs = [synth.replay_feature_log(l) for l in logs]
    assert all(r["handover_index"] == 1 for r in recs)
    return logs, edits, recs


def run_lockstep(capi, defs, logs, recs, order, params=None, seq_params=None, stages=False):
    """Run the sequences `order` (indices into logs, repeats allowed) in lockstep from their shim hand-overs.  Returns
    (rows, steps): rows[j] = [(scan, download row)] of position j; with stages, steps[t] holds what step t started from
    (filter state, maps) and what its IESKF saw and produced (lins_gpu_seq_download_ieskf)."""
    synth = pkg("synth")
    g = capi.LinsGpu(params)
    hs = [recs[i]["handover"] for i in order]
    ho = {k: np.stack([h[k] for h in hs]) for k in ("filter_state", "filter_cov", "global_state", "imu_last")}
    for k in ("surf_map", "corner_map"):
        ho[k] = np.concatenate([h[k] for h in hs])
        ho[k + "_off"] = np.concatenate([[0], np.cumsum([len(h[k]) for h in hs])])
    g.seq_begin(seq_params or defs.LinsSeqParams.shipped(), ho)
    first = [recs[i]["handover_index"] + 1 for i in order]
    n_steps = max(len(logs[i]["time"]) - f for i, f in zip(order, first))
    rows, steps = [[] for _ in order], []
    for t in range(n_steps):
        scans, present = [], []
        for i, f in zip(order, first):
            k = f + t
            if k < len(logs[i]["time"]):
                scans.append(synth.log_scan(logs[i], k)); present.append(1)
            else:
                scans.append(dict(imu=np.zeros((0, 7)), **{c: logs[i][c][:0] for c in defs.Batch.FIELDS})); present.append(0)
        step = dict(present=np.array(present, np.uint8), imu=np.concatenate([np.asarray(s["imu"]).reshape(-1, 7) for s in scans]),
                    imu_off=np.concatenate([[0], np.cumsum([len(s["imu"]) for s in scans])]))
        for c in defs.Batch.FIELDS:
            step[c] = np.concatenate([s[c] for s in scans])
            step[c + "_off"] = np.concatenate([[0], np.cumsum([len(s[c]) for s in scans])])
        pre = dict(state=g.seq_download(), maps=g.seq_download_maps(), scans=scans) if stages else None
        g.seq_step(step)
        d = g.seq_download(reports=True)
        if stages:
            steps.append(dict(pre, ieskf=g.seq_download_ieskf(), after=d))
        for j, f in enumerate(first):
            if present[j]:
                rows[j].append((f + t, {k: np.array(v[j], copy=True) if k != "reports" else v[j] for k, v in d.items()}))
    g.close()
    return rows, steps


@pytest.fixture(scope="module")
def lock48(capi, defs, cases):
    logs, edits, recs = cases
    return run_lockstep(capi, defs, logs, recs, list(range(N_SEQ)), stages=True)


def test_lockstep_matches_one_shim_per_sequence(defs, cases, lock48):
    logs, edits, recs = cases
    rows, _ = lock48
    seen = dict(gate=0, stale_next=0, no_imu=0, ran=0)
    seen["idle"] = len({len(l["time"]) for l in logs}) > 1
    worst = 0.0
    for i, rr in enumerate(rows):
        r = recs[i]
        for k, d in rr:
            code = r["code"][k]
            assert d["status"] == code, (i, k, d["status"], code)
            if code >= defs.SEQ_RAN:
                seen["ran"] += 1
                assert d["results"]["iters"] == r["iters"][k] and d["results"]["flags"] == r["flags"][k], (i, k)
                if not r["map_replaced"][k] and k + 1 < len(r["code"]) and r["code"][k + 1] >= defs.SEQ_RAN:
                    seen["stale_next"] += 1  # the next step runs this unit on the legacy path
            seen["gate"] += code == defs.SEQ_SKIPPED
            seen["no_imu"] += len(pkg("synth").log_scan(logs[i], k)["imu"]) == 0
            for key in ("global_state", "filter_state", "filter_cov"):
                diff = np.abs(d[key] - r[key][k]).max()
                worst = max(worst, diff)
                assert diff <= STATE_TOL, (i, k, key, diff)
    for case, n in seen.items():
        assert n, f"case {case} did not occur in the shim's record"
    print("worst |device - shim|", worst, seen)


def test_predict_stage_matches_the_host_state_predictor(defs, cases, lock48):
    """lins_seq_predict_kernel at equal inputs: the device's prior against kalman_filter.hpp's predict from the same state,
    covariance, last IMU sample and samples."""
    logs, edits, recs = cases
    synth = pkg("synth")
    _, steps = lock48
    imu_last = [recs[i]["handover"]["imu_last"].copy() for i in range(N_SEQ)]
    n_checked = n_samples = 0
    for st in steps:
        status = st["after"]["status"]
        for j in range(N_SEQ):
            if status[j] == defs.SEQ_IDLE:
                continue
            rows = st["scans"][j]["imu"]
            hs, hc, hi = synth.host_predict(st["state"]["filter_state"][j], st["state"]["filter_cov"][j], imu_last[j], rows)
            for dev, host in ((st["ieskf"]["prior_state"][j], hs), (st["ieskf"]["prior_cov"][j], hc)):
                tol = PREDICT_RTOL * (np.abs(host) + 1e-3 * np.abs(host).max())
                assert (np.abs(dev - host) <= tol).all(), (j, np.abs(dev - host).max())
                if len(rows) == 0:
                    assert np.array_equal(dev, host)  # (no sample: the state is untouched)
            imu_last[j] = hi
            n_checked += 1
            n_samples += len(rows)
    assert n_checked > 500 and n_samples > 20000


def test_ieskf_stage_matches_the_single_scan_seam_bit_for_bit(capi, defs, cases, lock48):
    """Each step's IESKF, fed with the device's own prior, map and 1-NN cloud to lins_gpu_set_map (+ a refresh that fails
    the guard, for a stale index) and lins_gpu_ieskf: state, covariance, iterations, flags and the last iteration's
    correspondence IDs are bit-identical."""
    logs, edits, recs = cases
    _, steps = lock48
    g = capi.LinsGpu()
    ident = np.zeros(19)
    ident[9] = 1.0
    n_checked = n_stale = 0
    for st in steps:
        status, m, ie = st["after"]["status"], st["maps"], st["ieskf"]
        for j in range(N_SEQ):
            if status[j] < defs.SEQ_RAN:
                continue
            if m["stale"][j]:  # the seam's own way to a stale index: set the old cloud, then a refresh below the guard
                g.set_map(m["surf_tree"][j], m["corner_tree"][j])
                s_out, c_out, replaced = g.update_map(m["surf_map"][j], m["corner_map"][j], ident)
                assert not replaced
                for a, b in ((s_out, m["surf_map"][j]), (c_out, m["corner_map"][j])):  # (the identity pose moves no point)
                    assert all(np.array_equal(a[f], b[f]) for f in ("x", "y", "z", "intensity"))
                n_stale += 1
            else:
                g.set_map(m["surf_map"][j], m["corner_map"][j])
            sc_ = st["scans"][j]
            so, co, rep = g.ieskf(sc_["surf_flat"], sc_["corner_sharp"], ie["prior_state"][j], ie["prior_cov"][j])
            si, ci = g.download_indices(len(sc_["surf_flat"]), len(sc_["corner_sharp"]))
            res = st["after"]["results"][j]
            assert (rep.iters, rep.converged | rep.diverged << 1 | rep.has_nan << 2) == (res["iters"], res["flags"]), j
            assert np.array_equal(so, ie["state_out"][j]) and np.array_equal(co, ie["cov_out"][j]), j
            assert np.array_equal(si, ie["surf_ind"][j]) and np.array_equal(ci, ie["corner_ind"][j]), j
            n_checked += 1
    g.close()
    assert n_checked > 500 and n_stale >= 1, (n_checked, n_stale)


def _same(a, b):
    for key in ("global_state", "filter_state", "filter_cov", "status"):
        if not np.array_equal(a[key], b[key]):
            return key
    if a["status"] >= 2 and not (np.array_equal(a["results"]["pose"], b["results"]["pose"]) and a["results"]["iters"] == b["results"]["iters"]):
        return "results"
    return None


def test_outputs_do_not_depend_on_the_other_sequences(capi, defs, cases, lock48):
    logs, edits, recs = cases
    full, _ = lock48
    rng = np.random.default_rng(3)
    for order in (list(rng.permutation(N_SEQ)), [1], list(range(4, 11))):
        order = [int(i) for i in order]
        part, _ = run_lockstep(capi, defs, logs, recs, order)
        for j, i in enumerate(order):
            assert [k for k, _ in part[j]] == [k for k, _ in full[i]]
            for (k, d), (_, e) in zip(part[j], full[i]):
                assert _same(d, e) is None, (i, k, _same(d, e))


def test_300_sequences_share_ctas_across_the_legacy_and_indexed_paths(capi, defs, cases, lock48, monkeypatch, capfd):
    """S = 300 (the VLP-16 logs tiled: a 64-ring unit's query tile leaves room for one unit per CTA only): several resident
    units per CTA, so the guard-cut sequence's stale step runs on the legacy path next to indexed units in the same CTA.
    Every output, correspondence IDs included, is bit-identical to the S = 48 run."""
    logs, edits, recs = cases
    full, steps48 = lock48
    guard_seq = next(s for s, (case, _) in edits.items() if case == "guard")
    assert any(st["maps"]["stale"][guard_seq] and st["after"]["status"][guard_seq] >= defs.SEQ_RAN for st in steps48)
    vlp = [i for i in range(N_SEQ) if logs[i]["lidar"] == 0]
    assert guard_seq in vlp
    order = [vlp[j % len(vlp)] for j in range(300)]
    monkeypatch.setenv("LINS_VERBOSE", "1")
    capfd.readouterr()
    rows, steps = run_lockstep(capi, defs, logs, recs, order, stages=True)
    err = capfd.readouterr().err
    slots = [int(x) for x in re.findall(r"\[lins_gpu\] mode 0: .* slots (\d+)", err)]
    assert slots and min(slots[:5]) >= 2, slots[:5]  # (the first steps run every sequence: several units per CTA)
    for j, i in enumerate(order):
        assert [k for k, _ in rows[j]] == [k for k, _ in full[i]]
        for (k, d), (_, e) in zip(rows[j], full[i]):
            assert _same(d, e) is None, (j, k, _same(d, e))
    for st, st48 in zip(steps, steps48):
        for j, i in enumerate(order):
            if st["after"]["status"][j] >= defs.SEQ_RAN:
                assert st["maps"]["stale"][j] == st48["maps"]["stale"][i]
                assert np.array_equal(st["ieskf"]["surf_ind"][j], st48["ieskf"]["surf_ind"][i]), (j, i)
                assert np.array_equal(st["ieskf"]["corner_ind"][j], st48["ieskf"]["corner_ind"][i]), (j, i)


def test_icp_fallback_matches_the_shim(capi, defs, cases):
    """Divergence of every running scan: the residual blow-up branch (StateEstimator.hpp:566-570), forced through
    lidar_scale as in test_gpu_parity.py, for the shim's context and the device alike (no edit of a feature log made the
    IESKF diverge with the shipped parameters).  Every step then runs the estimateTransform fallback of every sequence,
    the guard-cut one on its stale 1-NN index too."""
    logs, edits, recs = cases
    prm = defs.LinsParams.shipped(lidar_scale=1e9)
    synth = pkg("synth")
    pick = [0, 1, 2, 4, 5, 11]
    recs2 = {i: synth.replay_feature_log(logs[i], params=prm) for i in pick}
    assert all(r["handover_index"] == 1 for r in recs2.values())
    rows, _ = run_lockstep(capi, defs, logs, [recs2.get(i) for i in range(N_SEQ)], pick, params=prm)
    n_icp = 0
    for j, i in enumerate(pick):
        r = recs2[i]
        for k, d in rows[j]:
            code = r["code"][k]
            assert d["status"] == code, (i, k, d["status"], code)
            n_icp += code == defs.SEQ_ICP
            if code >= defs.SEQ_RAN:
                assert d["results"]["iters"] == r["iters"][k] and d["results"]["flags"] == r["flags"][k], (i, k)
            for key in ("global_state", "filter_state", "filter_cov"):
                diff = np.abs(d[key] - r[key][k]).max()
                assert diff <= STATE_TOL, (i, k, key, diff)
    assert n_icp >= 20, n_icp


def test_nonzero_reset_variances_match_the_shim(capi, defs, cases):
    """reset(1) with non-zero INIT_POS_STD / INIT_ATT_STD, on the shim's filter and in lins_seq_params alike."""
    logs, edits, recs = cases
    pos, att = (0.1, 0.2, 0.3), (0.5, 1.0, 2.0)
    synth = pkg("synth")
    pick = [1, 5, 6, 12]
    recs2 = {i: synth.replay_feature_log(logs[i], init_std=pos + att) for i in pick}
    rows, _ = run_lockstep(capi, defs, logs, [recs2.get(i) for i in range(N_SEQ)], pick,
                           seq_params=defs.LinsSeqParams.shipped(init_pos_std=pos, init_att_std=att))
    n = 0
    for j, i in enumerate(pick):
        r = recs2[i]
        for k, d in rows[j]:
            assert d["status"] == r["code"][k], (i, k)
            for key in ("global_state", "filter_state", "filter_cov"):
                diff = np.abs(d[key] - r[key][k]).max()
                assert diff <= STATE_TOL, (i, k, key, diff)
            if d["status"] >= defs.SEQ_RAN:
                n += 1
                P = d["filter_cov"].reshape(18, 18)
                assert np.allclose(np.diag(P)[:3], np.square(pos)), np.diag(P)[:3]
    assert n > 40


def test_bad_input_is_rejected_and_the_context_stays_usable(capi, defs, cases):
    logs, edits, recs = cases
    g = capi.LinsGpu()
    L = g.L
    d = defs.LinsSeqStepDesc()
    d.n_seq = 1
    assert L.lins_gpu_seq_step(g.h, d) == -3  # before seq_begin: LINS_E_NOMAP
    assert L.lins_gpu_seq_download(g.h, None, None, None, None, None, None) == -3
    bd = defs.LinsSeqBeginDesc()
    assert L.lins_gpu_seq_begin(g.h, defs.LinsSeqParams.shipped(), bd) == -1  # n_seq = 0
    h = recs[10]["handover"]
    ho = dict(h, surf_map_off=[0, len(h["surf_map"])], corner_map_off=[0, len(h["corner_map"])])
    for k in ("filter_state", "filter_cov", "global_state", "imu_last"):
        ho[k] = h[k][None]
    g.seq_begin(defs.LinsSeqParams.shipped(), ho)
    synth = pkg("synth")
    s = synth.log_scan(logs[10], 2)
    step = dict(imu=s["imu"], imu_off=[0, len(s["imu"])], **{c: s[c] for c in defs.Batch.FIELDS},
                **{c + "_off": [0, len(s[c])] for c in defs.Batch.FIELDS})
    for bad in (dict(imu_off=[1, len(s["imu"])]), dict(surf_flat_off=[5, 3]), dict(point_format=7)):
        with pytest.raises(capi.LinsError):
            g.seq_step(dict(step, **bad))
    g.seq_step(step)
    d = g.seq_download()
    assert d["status"][0] == recs[10]["code"][2]
    assert np.abs(d["filter_state"][0] - recs[10]["filter_state"][2]).max() <= STATE_TOL
