"""Feature extraction on the device against the host FeatureExtractor, and sequence mode fed segmented clouds
(lins_gpu_seq_step_pcl) against the features-in step (lins_gpu_seq_step_ex).

    python tools/feat_bench.py [--scans 1000] [--seqs 132,1000] [--steps 8] [--out DIR]

Prints one JSON line:
  - extract_ms_per_1000: CUDA-event time of the extraction kernel per 1000 scans, VLP-16 (config3) and 64 x 1024 (config4);
  - host_extract_ms_per_scan: FeatureExtractor::run in C++ (no Python in the loop) on one thread, and
    host_scans_per_s_all_cores: the same on one std::thread per core of this machine;
  - per S: step_ms of seq_step_pcl and of seq_step_ex (features uploaded, extraction not counted), the extraction kernel's
    share of the pcl step, and the H2D bytes per step of both inputs (from the sizes uploaded);
  - the card's name and power limit.
Every scan is a simulated sweep through the host image projection; S slots cycle through a pool of them.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=1000)
    ap.add_argument("--pool", type=int, default=64, help="distinct simulated sweeps the batches cycle through")
    ap.add_argument("--seqs", default="132,1000")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import importlib

    import featcases as fc

    capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
    defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
    synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
    synth.build()
    res = {}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        res["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    except OSError:
        res["gpu"] = "unknown"
    g = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
    pools = {}
    for name, config in (("vlp16", "config3"), ("dense64", "config4")):
        pools[name] = [fc.segmented(synth, defs, config, 5000 + i) for i in range(a.pool)]
    # ---- extraction kernel per 1000 scans ----
    res["extract_ms_per_1000"] = {}
    for name, pool in pools.items():
        scans = [pool[i % len(pool)][0] for i in range(a.scans)]
        ln = pool[0][1]
        g.extract_features(scans, line_num=ln)  # warm-up
        ms = []
        for _ in range(3):
            g.extract_features(scans, line_num=ln)
            ms.append(g.extract_ms())
        res["extract_ms_per_1000"][name] = round(float(np.median(ms)) * 1000.0 / a.scans, 3)
        res.setdefault("points_per_scan", {})[name] = int(np.mean([len(p[0]["seg"]) for p in pool]))
    # ---- host FeatureExtractor::run in C++ threads (tools/synth lins_features_host_bench): one thread, then every core ----
    L = fc._lib(defs)
    L.lins_features_host_bench.restype = C.c_double
    L.lins_features_host_bench.argtypes = [C.c_void_p, C.c_int, C.c_int]
    res["host_extract_ms_per_scan"], res["host_scans_per_s_all_cores"] = {}, {}
    nthr = os.cpu_count() or 1
    res["host_cores"] = nthr
    for name, pool in pools.items():
        keep = {}
        d = capi.LinsGpu._pcl_desc([p[0] for p in pool], pool[0][1], keep)
        L.lins_features_host_bench(C.byref(d), 1, 1)  # warm-up
        t1 = L.lins_features_host_bench(C.byref(d), 1, 2)
        res["host_extract_ms_per_scan"][name] = round(t1 * 1000.0 / (2 * len(pool)), 3)
        reps = 4 * nthr
        tn = L.lins_features_host_bench(C.byref(d), nthr, reps)
        res["host_scans_per_s_all_cores"][name] = round(reps * len(pool) / tn, 1)
    # ---- sequence mode: segmented clouds in vs features in ----
    res["seq"] = {}
    pool = pools["vlp16"]
    feats = g.extract_features([p[0] for p in pool], line_num=16)
    si = lambda S: np.tile(np.array([0, 0, 9.81, 0, 0, 0.0]), (S, 1))  # noqa: E731
    for S in [int(v) for v in a.seqs.split(",")]:
        out = {}
        for mode in ("pcl", "ex"):
            h = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
            h.seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(), S)
            times, ext, h2d = [], [], []
            for t in range(a.steps):
                idx = [(s * 7 + t) % len(pool) for s in range(S)]
                imu = dict(imu=np.zeros((1, 7)), imu_off=np.zeros(S + 1, np.int32))
                sim = si(S)
                if mode == "pcl":  # (the descriptor is built before the clock starts: the timed call is the C entry point)
                    keep = dict((k, np.ascontiguousarray(v)) for k, v in imu.items())
                    d = defs.LinsSeqPclDesc()
                    d.pcl = capi.LinsGpu._pcl_desc([pool[i][0] for i in idx], 16, keep)
                    d.n_seq, d.imu, d.imu_off = S, keep["imu"].ctypes.data, keep["imu_off"].ctypes.data
                    fp = defs.LinsFeatureParams.shipped()
                    n = int(keep["cloud_off"][-1])
                    h2d.append(n * (16 + 1 + 4 + 4) + S * (2 * 16 * 4 + 12) + (S + 1) * 4 * 4)
                    h.sync()
                    t0 = time.perf_counter()
                    rc = h.L.lins_gpu_seq_step_pcl(h.h, C.byref(d), C.byref(fp), sim.ctypes.data)
                    times.append(time.perf_counter() - t0)
                    assert rc == 0, rc
                    ext.append(h.extract_ms())
                else:
                    d = dict(imu)
                    for k in fc.NAMES:
                        clouds = [capi._points_from_xyzi(feats[i][k]) for i in idx]
                        d[k] = np.concatenate(clouds)
                        d[k + "_off"] = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
                    h2d.append(sum(16 * len(d[k]) + 4 * (S + 1) for k in fc.NAMES))
                    sd = defs.LinsSeqStepDesc()
                    sd.n_seq, sd.imu, sd.imu_off = S, d["imu"].ctypes.data, d["imu_off"].ctypes.data
                    for k in fc.NAMES:
                        setattr(sd, k, d[k].ctypes.data)
                        setattr(sd, k + "_off", d[k + "_off"].ctypes.data)
                    h.sync()
                    t0 = time.perf_counter()
                    rc = h.L.lins_gpu_seq_step_ex(h.h, C.byref(sd), sim.ctypes.data)
                    times.append(time.perf_counter() - t0)
                    assert rc == 0, rc
            w = slice(2, None)  # the first two steps initialise every slot
            out[mode] = dict(step_ms=round(float(np.median(times[w])) * 1000, 3), h2d_bytes_per_step=int(np.median(h2d)))
            if mode == "pcl":
                out[mode]["extract_kernel_ms"] = round(float(np.median(ext[w])), 3)
            del h
        res["seq"][str(S)] = out
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "feat_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
