#!/usr/bin/env python
"""tools/loop_store_bench.py [--trips 15] [--seed 6] [--every 100] [--big-slots auto]

The key-frame stores of slots with loop closure (DESIGN.md §4.14) on a long drive: tools/globalmap_bench.py's
long_drive (--trips out-and-back runs of one road, 71 key frames each; >= 1000 key frames at the default), copied into
every slot with loop closure enabled (no closure is run: the stores' sizes do not depend on the poses).

- M = 1: the device and host store bytes (lins_gpu_mappers_store_bytes) every --every key frames, the run's pinned
  reserve, and the mapping step's median time over the last 100 steps;
- a run at a large M (--big-slots; auto: the smallest M at which the whole store at 32 bytes per DS point, every key
  frame in the map and the body frame on the device, would exceed the card's memory), when its host stores fit in a
  quarter of the host's MemAvailable (the host is shared): the same bytes per slot, the device memory the run holds
  (cudaMemGetInfo before and after) and the step's median time.
Prints one JSON line with the GPU's name and power limit."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
from globalmap_bench import CHUNK, long_drive, mem_available  # noqa: E402

import torch  # noqa: E402  (cudaMemGetInfo)


def run(ev, M, every=None):
    g = capi.LinsGpu()
    g.mappers_open(M)
    g.mappers_loops(np.ones(M, np.uint8))
    curve, step_ms, pts = [], [], 0
    for e in ev:
        t0 = time.perf_counter()
        reps = g.mappers_step([e] * M)
        step_ms.append((time.perf_counter() - t0) * 1e3)
        r = reps[0]
        if r.processed and r.keyframe_saved:
            pts += r.n_corner_ds + r.n_surf_ds + r.n_outlier_ds
            if every and r.n_keyframes % every == 0:
                dev, host, res = g.mappers_store_bytes()
                curve.append(dict(key_frames=r.n_keyframes, device_bytes=int(dev[0]), host_bytes=int(host[0]), host_reserved=res,
                                  two_copy_device_bytes=32 * pts))
    dev, host, res = g.mappers_store_bytes()
    return g, dict(key_frames=int(reps[0].n_keyframes), device_bytes_per_slot=int(dev[0]), host_bytes_per_slot=int(host[0]),
                   host_reserved=res, two_copy_device_bytes_per_slot=32 * pts, step_ms_median_last_100=float(np.median(step_ms[-100:])),
                   curve=curve)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trips", type=int, default=15)
    ap.add_argument("--seed", type=int, default=6)
    ap.add_argument("--every", type=int, default=100)
    ap.add_argument("--big-slots", default="auto")
    a = ap.parse_args()
    ev = long_drive(a.seed, a.trips)
    res = {"what": "key-frame store bytes of loop-closure slots, tools/globalmap_bench.py's long drive in every slot"}
    g, one = run(ev, 1, a.every)
    del g
    res["M=1"] = one
    total = torch.cuda.mem_get_info()[1]
    M = int(total // one["two_copy_device_bytes_per_slot"]) + 1 if a.big_slots == "auto" else int(a.big_slots)
    need, cap = M * (-(-one["host_bytes_per_slot"] // CHUNK) + 1) * CHUNK, mem_available() // 4  # (whole chunks, one for tails)
    big = dict(slots=M, two_copy_device_bytes=M * one["two_copy_device_bytes_per_slot"], device_total=total, host_bytes_needed=need,
               host_cap=cap)
    if need > cap:
        big["skipped"] = "the host stores exceed a quarter of MemAvailable"
    else:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        g, r = run(ev, M)
        r.pop("curve")
        big.update(r, device_bytes_held_by_run=int(free0 - torch.cuda.mem_get_info()[0]))
        del g
    res[f"M={M}"] = big
    res["device"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
