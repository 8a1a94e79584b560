#!/usr/bin/env python
"""tools/globalmap_bench.py [--slots 1,132,1000] [--seed 6] [--long-trips 15]

The mapping node's global map (lins_gpu_mappers_global_map, DESIGN.md §4.15) on tools/loops_bench.py's drifted
out-and-back drive, copied into every slot with loop closure enabled (no closure is run: the global map reads the store,
whatever moved its poses):

- the call's time at each M: CUDA events around it on the library's stream, and a host clock around the call (which ends
  in a synchronisation); median of 5 calls after one warm-up call;
- gathered and output points per slot, the number of device passes (the library's rule: slots in order while a pass
  stays within LINS_GLOBAL_MAP_PASS_POINTS), and the device memory the first call adds (its grow-only scratch plus the
  results, from cudaMemGetInfo before and after), with the results' own bytes;
- a long single drive (--long-trips round trips of the same road, >= 1000 key frames) at M = 1.
M = 1000 is skipped when the slots' host key-frame stores would not fit in a quarter of the host's MemAvailable (the
host is shared; a slot's need is its host store's bytes after the M = 1 run rounded up to whole 1 MiB chunks, plus one
chunk for the chunks' unused tails), or their device stores in the free device memory.
Prints one JSON line with the GPU's name and power limit."""
import argparse
import importlib
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
import mapper_drive  # noqa: E402
from loops_bench import drive  # noqa: E402


def long_drive(seed, trips):
    """trips out-and-back runs of 36 scans 0.5 m apart over the same road (odometry without drift)"""
    xs, yaws = [], []
    for r in range(trips):
        xs += [-9.0 + 0.5 * k for k in range(36)] + [-9.0 + 0.5 * (35 - k) - 0.25 for k in range(1, 36)]
        yaws += [0.0] * 36 + [math.pi] * 35
    poses = [(x, 0.3 * math.sin(0.15 * k), 1.5, yaw) for k, (x, yaw) in enumerate(zip(xs, yaws))]
    scans, truth = synth.generate_map_drive(np.array(poses), seed=seed)
    ev, t = [], 100.0
    for (corner, surf, outlier), T in zip(scans, truth):
        odo = T.astype(np.float64)
        ev.append((t, mapper_drive.odometry_quat(odo), (odo[3], odo[4], odo[5]), corner, surf, outlier))
        t += 0.5
    return ev


def run(ev, M, stream):
    g = capi.LinsGpu(stream=stream.cuda_stream)
    g.mappers_open(M)
    g.mappers_loops(np.ones(M, np.uint8))
    reps = None
    for e in ev:
        reps = g.mappers_step([e] * M)
    return g, reps


def passes(points):
    n, cur = 0, 0
    for p in points:
        if p == 0:
            continue
        if n == 0 or cur + p > defs.GLOBAL_MAP_PASS_POINTS:
            n, cur = n + 1, 0
        cur += p
    return n


def measure(g, M, stream):
    mask = np.ones(M, np.uint8)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    reps = g.mappers_global_map(mask)  # (warm-up; grows the scratch)
    free1 = torch.cuda.mem_get_info()[0]
    dev_ms, host_ms = [], []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        t0 = time.perf_counter()
        reps = g.mappers_global_map(mask)
        host_ms.append((time.perf_counter() - t0) * 1e3)
        b.record(stream)
        b.synchronize()
        dev_ms.append(a.elapsed_time(b))
    pts = [r.n_points for r in reps]
    return dict(call_ms_device_median=float(np.median(dev_ms)), call_ms_host_median=float(np.median(host_ms)),
                key_frames=int(np.mean([r.n_key_frames for r in reps])), key_poses=int(np.mean([r.n_key_poses for r in reps])),
                gathered_points_per_slot=float(np.mean(pts)), output_points_per_slot=float(np.mean([r.n_map for r in reps])),
                unfiltered=int(sum(r.unfiltered for r in reps)), passes=passes(pts),
                device_bytes_added_by_first_call=int(free0 - free1), result_bytes=int(16 * sum(r.n_map for r in reps)))


CHUNK = 1 << 20  # the host store's chunk (lins_ctx.hpp: kKfChunkBytes)


def host_need_per_slot(g):
    """pinned bytes one slot of run g needs: its host store's bytes in whole chunks, plus one chunk of unused tails"""
    return (-(-int(g.mappers_store_bytes()[1][0]) // CHUNK) + 1) * CHUNK


def mem_available():
    """MemAvailable of /proc/meminfo in bytes"""
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("no MemAvailable in /proc/meminfo")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="1,132,1000")
    ap.add_argument("--seed", type=int, default=6)
    ap.add_argument("--long-trips", type=int, default=15)
    a = ap.parse_args()
    stream = torch.cuda.Stream()
    ev = drive(a.seed)
    res = {"what": "lins_gpu_mappers_global_map, tools/loops_bench.py's drifted out-and-back drive in every slot",
           "pass_points": defs.GLOBAL_MAP_PASS_POINTS}
    store = host = None  # per slot: the device memory a run adds, the host store's pinned bytes
    res["host_mem_available"] = mem_available()
    for M in [int(x) for x in a.slots.split(",")]:
        if store is not None and (M * host > 0.25 * mem_available() or M * store > 0.8 * torch.cuda.mem_get_info()[0]):
            res[f"M={M}"] = "skipped: the store does not fit"
            continue
        free0 = torch.cuda.mem_get_info()[0]
        g, reps = run(ev, M, stream)
        if store is None:
            store = (free0 - torch.cuda.mem_get_info()[0]) / M
            host = host_need_per_slot(g)
        res[f"M={M}"] = measure(g, M, stream)
        del g
    g, reps = run(long_drive(a.seed, a.long_trips), 1, stream)
    res["long_drive_M=1"] = measure(g, 1, stream)
    res["long_drive_M=1"]["key_frames_stored"] = reps[0].n_keyframes
    res["device"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
