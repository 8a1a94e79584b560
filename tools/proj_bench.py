"""Image projection on the device (lins_gpu_project_scans) against the host ImageProjection::process.

    python tools/proj_bench.py [--scans 1000] [--pool 64] [--out DIR]

Prints one JSON line:
  - project_ms_per_1000: CUDA-event time of the projection kernel per 1000 sweeps in one batch, VLP-16 (config3) and
    64 x 1024 (config4), and call_ms_per_1000: the whole lins_gpu_project_scans call from host buffers to host buffers
    (upload, kernel, read-back of the used prefixes), host wall clock;
  - host_project_ms_per_scan: ImageProjection::process in C++ (no Python in the loop) on one thread, and
    host_scans_per_s: the same on 1 and 16 std::threads (one ImageProjection each);
  - h2d_bytes_per_1000: what the batch uploads (16-B records + offsets), and points_per_sweep;
  - the card's name and power limit.
The batches cycle through a pool of simulated raw sweeps.
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
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import importlib

    import featcases as fc
    import projcases as pc

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
        pools[name] = [pc.raw_sweep(synth, defs, config, 5000 + i) for i in range(a.pool)]
    # ---- projection kernel per 1000 sweeps ----
    res["project_ms_per_1000"], res["points_per_sweep"], res["h2d_bytes_per_1000"] = {}, {}, {}
    for name, pool in pools.items():
        raws = [pool[i % len(pool)][0] for i in range(a.scans)]
        m = pool[0][1]
        g.project_scans(raws, model=m)  # warm-up
        ms = []
        for _ in range(3):
            g.project_scans(raws, model=m)
            ms.append(g.project_ms())
        res["project_ms_per_1000"][name] = round(float(np.median(ms)) * 1000.0 / a.scans, 3)
        # the C entry point with its buffers prepared beforehand
        keep = {}
        d = capi.LinsGpu._raw_desc(raws, 0, keep)
        total, n, L = int(keep["cloud_off"][-1]), len(raws), m.line_num
        outs = [np.zeros(total, defs.POINT_DTYPE), np.zeros(total, np.uint8), np.zeros(total, np.uint32), np.zeros(total, np.float32),
                np.zeros(total, defs.POINT_DTYPE), np.zeros((n, L), np.int32), np.zeros((n, L), np.int32), np.zeros((n, 3), np.float32),
                np.zeros((n, 2), np.int32)]
        wall = []
        for _ in range(4):
            t0 = time.perf_counter()
            rc = g.L.lins_gpu_project_scans(g.h, C.byref(m), C.byref(d), *[o.ctypes.data for o in outs])
            wall.append(time.perf_counter() - t0)
            assert rc == 0, rc
        res.setdefault("call_ms_per_1000", {})[name] = round(float(np.median(wall[1:])) * 1000.0 * 1000.0 / a.scans, 3)
        npts = sum(len(r) for r in raws)
        res["points_per_sweep"][name] = int(npts / a.scans)
        res["h2d_bytes_per_1000"][name] = int((16 * npts + 4 * (a.scans + 1)) * 1000 / a.scans)
    # ---- host ImageProjection::process in C++ threads (tools/synth lins_projection_host_bench) ----
    L = fc._lib(defs)
    L.lins_projection_host_bench.restype = C.c_double
    L.lins_projection_host_bench.argtypes = [C.c_void_p, C.POINTER(defs.LinsLidarModel), C.c_int, C.c_int]
    res["host_project_ms_per_scan"], res["host_scans_per_s"] = {}, {}
    res["host_cores"] = os.cpu_count() or 1
    for name, pool in pools.items():
        keep = {}
        d = capi.LinsGpu._raw_desc([p[0] for p in pool], 0, keep)
        m = pool[0][1]
        L.lins_projection_host_bench(C.byref(d), C.byref(m), 1, 1)  # warm-up
        t1 = L.lins_projection_host_bench(C.byref(d), C.byref(m), 1, 2)
        res["host_project_ms_per_scan"][name] = round(t1 * 1000.0 / (2 * len(pool)), 3)
        res["host_scans_per_s"][name] = {}
        for nthr in (1, 16):
            reps = 4 * nthr
            tn = L.lins_projection_host_bench(C.byref(d), C.byref(m), nthr, reps)
            res["host_scans_per_s"][name][str(nthr)] = round(reps * len(pool) / tn, 1)
        res.setdefault("device_scans_per_s", {})[name] = round(1000.0 * 1000.0 / res["project_ms_per_1000"][name], 1)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "proj_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
