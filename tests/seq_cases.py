"""Feature logs for the sequence-mode tests: seeded simulated drives, some of them edited so that every case the device
chain branches on occurs (tests/test_gpu_seq.py asserts that each one does in the shim's own record)."""
import numpy as np

from conftest import pkg

synth = pkg("synth")

N_SCANS = 22        # scans per full-length log (the hand-over is after scan 1: 20 steps)
GATE_SURF = 8       # surfLessFlat <= 10 fails the processScan gate (StateEstimator.hpp:436-440)
GUARD_SURF = 15     # 10 < surfLessFlat < 20 passes the gate but fails the map refresh guard (:1156-1157)


def _edit(log, k, fn):
    scans = [synth.log_scan(log, i) for i in range(len(log["time"]))]
    fn(scans[k])
    return synth.make_log(scans, log["lidar"])


def cut(field, n):
    def f(s):
        s[field] = s[field][:n].copy()
    return f


def no_imu(s):
    s["imu"] = np.zeros((0, 7))


def case_logs(n_seq=48):
    """n_seq logs: seeds 100.., every sixth a 64-ring drive, some shorter than the others, and the edits of `plan`.
    Returns (logs, edits) with edits = {sequence: (case, scan)}."""
    logs, edits = [], {}
    plan = {0: ("gate", 6, cut("surf_less_flat", GATE_SURF)), 1: ("guard", 7, cut("surf_less_flat", GUARD_SURF)),
            2: ("no_imu", 5, no_imu), 3: ("no_imu", 9, no_imu)}
    for s in range(n_seq):
        dense = s % 6 == 5
        n = N_SCANS - (s % 5 == 4) * (3 + s % 7)
        log = synth.feature_log("config4" if dense else "config3", seed=100 + s, n_scans=n)
        if s in plan:
            case, k, fn = plan[s]
            log = _edit(log, k, fn)
            edits[s] = (case, k)
        logs.append(log)
    return logs, edits
