"""Pcl logs for the sequence-mode tests of lins_gpu_seq_step_pcl: seeded simulated drives as processPCL receives them
(segmented cloud + cloud_info per scan), some with edited segmented clouds so that the processScan gate, the map-refresh
guard, the first-scan gate and a scan without IMU rows occur (the tests assert each in the shim's own record)."""
import numpy as np

import featcases as fc
from conftest import pkg

synth = pkg("synth")
LINES = 64  # every log of a run shares line_num: VLP-16 scans carry 48 empty rings (no visited sextant)


def pad(scan, line_num=LINES):
    s = dict(scan)
    k = len(scan["start_ring"])
    s["start_ring"] = np.concatenate([scan["start_ring"], np.zeros(line_num - k, np.int32)])
    s["end_ring"] = np.concatenate([scan["end_ring"], np.zeros(line_num - k, np.int32)])
    return s


def cut(scan, a, b):
    """Points [a, b) of a scan as one ring (LeGO-LOAM's layout: start = first + 4, end = last - 6)."""
    s = {k: np.asarray(scan[k])[a:b].copy() for k in ("seg", "ground", "col", "range")}
    s["start_ring"] = np.zeros(len(scan["start_ring"]), np.int32)
    s["end_ring"] = np.zeros(len(scan["start_ring"]), np.int32)
    s["start_ring"][0], s["end_ring"][0] = 4, (b - a) - 6
    s["ori"] = scan["ori"].copy()
    return s


def counts(defs, scan):
    h = fc.host_features(defs, scan, len(scan["start_ring"]))
    return len(h["corner_less_sharp"]), len(h["surf_less_flat"])


def _find_cut(defs, scan, want):
    for length in range(40, 1500, 20):
        for a in range(0, len(scan["seg"]) - length, 97):
            c = cut(scan, a, a + length)
            if want(*counts(defs, c)):
                return c
    raise AssertionError("no cut of the scan reaches the case")


def tie_decided(gpu, defs, log):
    """Scans of the log where the device's clouds differ from the host FeatureExtractor's.  Each must be one where equal
    curvatures decide a pick (the reference's std::sort leaves their order unspecified): there the device equals
    tests/pyfront.py, which keeps equal curvatures in array order, and the host's libstdc++ std::sort does not."""
    import pyfront
    dev = gpu.extract_features(log["scans"], line_num=log["line_num"], undist=True)
    out = []
    for k, s in enumerate(log["scans"]):
        h = fc.host_features(defs, s, log["line_num"])
        if all(fc.same_bits(dev[k][n], h[n]) for n in fc.NAMES + ("undist",)):
            continue
        p = pyfront.extract_features(s["seg"], s, lm=pyfront.Lidar(line_num=log["line_num"]))
        pm = dict(surf_flat="flat", corner_sharp="sharp", surf_less_flat="less_flat", corner_less_sharp="less_sharp", undist="undist")
        assert p["sort_ties"] > 0 and all(fc.same_bits(dev[k][n], p[pm[n]]) for n in pm), k
        out.append(k)
    return out


def case_logs(defs, n_seq=12, n_scans=14, gpu=None):
    """n_seq pcl logs (seeds 200.., every sixth a 64-ring drive, some shorter) and the edits: {sequence: (case, scan)}.
    With gpu, a drive with a scan where a tie between equal curvatures decides a pick (tie_decided) is replaced by the
    next seed's, so the device's features equal the host's on every scan of every log (the shim and step_ex comparisons
    need that); the number of drives skipped so is returned as edits["tie_skipped"]."""
    logs, edits, skipped = [], {}, 0
    for s in range(n_seq):
        dense = s % 6 == 5
        n = n_scans - (s % 5 == 4) * (3 + s % 4)
        for t in range(8):
            log = synth.pcl_log("config4" if dense else "config3", seed=200 + s + 1000 * t, n_scans=n)
            log["scans"] = [pad(x) for x in log["scans"]]
            log["line_num"] = LINES
            if gpu is None or not tie_decided(gpu, defs, log):
                break
            skipped += 1
        logs.append(log)
    sc = logs[0]["scans"]
    sc[6] = _find_cut(defs, sc[6], lambda ncl, nsl: ncl <= 5 or nsl <= 10)                  # processScan gate (:436-440)
    edits[0] = ("gate", 6)
    sc = logs[1]["scans"]
    sc[7] = _find_cut(defs, sc[7], lambda ncl, nsl: ncl > 5 and 10 < nsl < 20)              # passes the gate, fails the refresh guard
    edits[1] = ("guard", 7)
    lg = logs[2]
    o = lg["imu_off"]
    lg["imu"] = np.concatenate([lg["imu"][: o[5]], lg["imu"][o[6]:]])
    lg["imu_off"] = np.concatenate([o[:6], o[6:] - (o[6] - o[5])]).astype(np.int32)                  # scan 5 without IMU rows
    edits[2] = ("no_imu", 5)
    logs[3]["scans"][0] = cut(logs[3]["scans"][0], 0, 400)                                            # first-scan gate
    edits[3] = ("first_gate", 0)
    if gpu is not None:
        for s in range(4):
            assert not tie_decided(gpu, defs, logs[s])
    edits["tie_skipped"] = skipped
    return logs, edits


def feature_log(defs, log):
    """The pcl log with every scan's features extracted on the host (FeatureExtractor): a feature log for seq_step_ex."""
    scans = []
    o = log["imu_off"]
    for k, s in enumerate(log["scans"]):
        h = fc.host_features(defs, s, log["line_num"])
        d = dict(imu=log["imu"][o[k]:o[k + 1]], imu_last=log["imu_last"][k], time=log["time"][k])
        for name in fc.NAMES:
            d[name] = pkg("capi")._points_from_xyzi(h[name])
        scans.append(d)
    return synth.make_log(scans, log["lidar"])
