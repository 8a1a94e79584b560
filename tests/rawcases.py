"""Raw logs for the sequence-mode tests of lins_gpu_seq_step_raw — TEST INFRASTRUCTURE.

A raw log is a simulated drive as the LiDAR driver publishes it (synth.raw_log).  Its host reference is copyPointCloud's
NaN removal in numpy, a fresh host ImageProjection per sweep (projcases.host_projection), which gives a pcl log, and the
shim replaying that pcl log (synth.replay_pcl_log).  `case_logs` edits some sweeps so that the first-scan gate, the
processScan gate, a scan without IMU rows, an empty sweep, non-finite points at the sweep's ends and in its middle, and an
entirely non-finite sweep occur (the tests assert each in the shim's own record).
"""
import numpy as np

import pclcases as pc
import projcases as pj
from conftest import pkg

synth = pkg("synth")


def finite(sweep):
    """pcl::removeNaNFromPointCloud: the points whose x, y and z are finite, in firing order."""
    a = np.asarray(sweep, np.float32).reshape(-1, 4)
    return a[np.isfinite(a[:, :3]).all(1)]


def model_of(defs, log):
    return defs.LinsLidarModel.dense64() if int(log["lidar"]) == 1 else defs.LinsLidarModel.vlp16()


def host_scan(defs, sweep, model):
    """cloudHandler on the host: the removal, then a fresh ImageProjection (a scan dict as pcl logs hold them)."""
    a = finite(sweep)
    p = pj.host_projection(defs, defs.make_points(a[:, :3], a[:, 3]), model)
    return {k: p[k] for k in ("seg", "ground", "col", "range", "start_ring", "end_ring", "ori")}


def pcl_of(defs, log):
    """The host-projected pcl log of a raw log."""
    m = model_of(defs, log)
    out = {k: log[k] for k in ("lidar", "line_num", "time", "imu", "imu_off", "imu_last")}
    out["scans"] = [host_scan(defs, s, m) for s in log["sweeps"]]
    return out


def _truncate(defs, log, k, want):
    """The shortest prefix of sweep k (a multiple of 40 points) whose host features reach `want(ncl, nsl)`."""
    m = model_of(defs, log)
    sw = log["sweeps"][k]
    for n in range(40, len(sw), 40):
        if want(*pc.counts(defs, host_scan(defs, sw[:n], m))):
            return sw[:n].copy()
    raise AssertionError("no prefix of the sweep reaches the case")


def case_logs(defs, lidar, n_seq=12, n_scans=14, gpu=None):
    """n_seq raw logs of one lidar (0: VLP-16 config3 drives, 1: 64 x 1024 config4 drives; seeds 300.., some shorter) and
    the edits {log: (case, scan)}.  With gpu, a drive where a tie between equal curvatures decides a pick on the host pcl
    log (pclcases.tie_decided) is replaced by the next seed's, so the device's features equal the shim's."""
    config = "config4" if lidar == 1 else "config3"
    logs, edits, skipped = [], {}, 0
    for s in range(n_seq):
        n = n_scans - (s % 5 == 4) * (3 + s % 4)
        for t in range(8):
            log = synth.raw_log(config, seed=300 + s + 1000 * t, n_scans=n)
            if gpu is None or not pc.tie_decided(gpu, defs, pcl_of(defs, log)):
                break
            skipped += 1
        logs.append(log)
    sw = logs[0]["sweeps"]
    sw[6] = _truncate(defs, logs[0], 6, lambda ncl, nsl: ncl <= 5 or nsl <= 10)            # processScan gate (:436-440)
    edits[0] = ("gate", 6)
    lg = logs[1]
    o = lg["imu_off"]
    lg["imu"] = np.concatenate([lg["imu"][: o[5]], lg["imu"][o[6]:]])
    lg["imu_off"] = np.concatenate([o[:6], o[6:] - (o[6] - o[5])]).astype(np.int32)              # scan 5 without IMU rows
    edits[1] = ("no_imu", 5)
    logs[2]["sweeps"][0] = _truncate(defs, logs[2], 0, lambda ncl, nsl: ncl < 10 or nsl < 100)   # first-scan gate
    edits[2] = ("first_gate", 0)
    logs[3]["sweeps"][8] = np.zeros((0, 4), np.float32)                                          # a present empty sweep
    edits[3] = ("empty", 8)
    a = logs[5]["sweeps"][3].copy()                                                              # non-finite points
    n = len(a)
    a[0, 0] = np.nan
    a[n - 2, 0] = np.inf
    a[n - 1, 1] = -np.inf
    a[n // 3: n // 3 + 40: 3, 2] = np.nan
    a[n // 2: n // 2 + 40: 5, 1] = np.inf
    logs[5]["sweeps"][3] = a
    edits[5] = ("nonfinite", 3)
    a = logs[6]["sweeps"][7].copy()
    a[:, 0] = np.nan
    logs[6]["sweeps"][7] = a                                                                     # entirely non-finite
    edits[6] = ("all_nonfinite", 7)
    if gpu is not None:
        for s in range(7):
            assert not pc.tie_decided(gpu, defs, pcl_of(defs, logs[s]))
    edits["tie_skipped"] = skipped
    return logs, edits
