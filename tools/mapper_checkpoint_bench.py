#!/usr/bin/env python
"""tools/mapper_checkpoint_bench.py [--slots 1,132,1000] [--seed 6] [--long-trips 15] [--reps 3]

Saving and loading mapping nodes (lins_gpu_mappers_save / _load, DESIGN.md §4.16), every slot masked:

- plain: tools/loops_bench.py's drifted out-and-back drive in every slot without loop closure, saved with a full
  50-key-frame window (the store: the window and the newest key frame);
- loops: the same drive with loop closure enabled and close_loops ticked on the way back, so that slots hold loop
  factors (the store: every key frame, saved in the body frame);
- long: tools/globalmap_bench.py's long drive (>= 1000 key frames) with loop closure enabled (no closure run), at M = 1.

Per case: the blob bytes per slot; save wall time (host clock around a call that ends in its one synchronisation,
median of --reps); load wall time into a fresh run of a new context (the store's buffers are allocated then) and into
the same run after lins_gpu_mappers_reset (the store's buffers are reused), median of --reps each, with the host
phases of lins_gpu_mappers_load_phase_ms (validation, allocation, staging, device, bookkeeping); the device split of one
load (torch.profiler: the H2D copy and the two kernels); the launches per call; the device memory a fresh load adds.
Prints one JSON line with the GPU's name and power limit."""
import argparse
import importlib
import json
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
from globalmap_bench import long_drive  # noqa: E402
from loops_bench import drive  # noqa: E402

PHASES = ("validation", "allocation", "staging", "device", "bookkeeping")


def source(ev, M, loops, close=True):
    g = capi.LinsGpu()
    g.mappers_open(M)
    mask = np.ones(M, np.uint8)
    if loops:
        g.mappers_loops(mask)
    reps = None
    for k, e in enumerate(ev):
        reps = g.mappers_step([e] * M)
        if loops and close and k >= 50 and k % 2 == 0:  # the loop thread, ticked on the way back (every 1 s of stamps)
            g.mappers_close_loops(mask)
    return g, reps


def timed(f):
    t0 = time.perf_counter()
    out = f()
    return (time.perf_counter() - t0) * 1e3, out


def device_split(M, blobs):
    """one load into a fresh run under torch.profiler: device time of the H2D copies and of each kernel (ms)"""
    g = capi.LinsGpu()
    g.mappers_open(M)
    mask = np.ones(M, np.uint8)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        g.mappers_load(mask, blobs)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = "h2d" if "HtoD" in ev.name else ev.name
        out[name] = out.get(name, 0.0) + ev.time_range.elapsed_us() / 1e3
    return {k: round(v, 4) for k, v in out.items()}


def measure(g, M, reps_n):
    mask = np.ones(M, np.uint8)
    save_ms = []
    for _ in range(reps_n):
        n0 = g.launch_count()
        ms, blobs = timed(lambda: g.mappers_save(mask))
        save_launches = g.launch_count() - n0
        save_ms.append(ms)
    sizes = [len(b) for b in blobs]
    fresh, reuse, ph_fresh, ph_reuse, added = [], [], [], [], None
    for _ in range(reps_n):
        h = capi.LinsGpu()
        h.mappers_open(M)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        n0 = h.launch_count()
        ms, _ = timed(lambda: h.mappers_load(mask, blobs))
        load_launches = h.launch_count() - n0
        added = free0 - torch.cuda.mem_get_info()[0]
        fresh.append(ms)
        ph_fresh.append(h.mappers_load_phase_ms())
        h.mappers_reset(mask)
        ms, _ = timed(lambda: h.mappers_load(mask, blobs))
        reuse.append(ms)
        ph_reuse.append(h.mappers_load_phase_ms())
        assert h.mappers_save(mask) == blobs
        del h
    med = lambda v: round(float(np.median(v)), 3)  # noqa: E731
    phases = lambda rows: {p: med([r[i] for r in rows]) for i, p in enumerate(PHASES)}  # noqa: E731
    return dict(bytes_per_slot_mean=float(np.mean(sizes)), bytes_total=int(sum(sizes)), save_ms_median=med(save_ms),
                load_fresh_ms_median=med(fresh), load_fresh_phases_ms=phases(ph_fresh), load_reuse_ms_median=med(reuse),
                load_reuse_phases_ms=phases(ph_reuse), device_split_fresh_load_ms=device_split(M, blobs),
                launches_save=int(save_launches), launches_load=int(load_launches), device_bytes_added_by_fresh_load=int(added))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="1,132,1000")
    ap.add_argument("--seed", type=int, default=6)
    ap.add_argument("--long-trips", type=int, default=15)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    ev = drive(a.seed)
    res = {"what": "lins_gpu_mappers_save / _load of every slot, tools/loops_bench.py's drifted out-and-back drive in every slot"}
    for loops in (False, True):
        for M in [int(x) for x in a.slots.split(",")]:
            g, reps = source(ev, M, loops)
            row = measure(g, M, a.reps)
            row["key_frames"] = reps[0].n_keyframes
            row["window"] = reps[0].window_len
            res[f"{'loops' if loops else 'plain'}_M={M}"] = row
            del g
    g, reps = source(long_drive(a.seed, a.long_trips), 1, True, close=False)  # (no closure: as globalmap_bench.py runs it)
    row = measure(g, 1, a.reps)
    row["key_frames"] = reps[0].n_keyframes
    res["long_M=1"] = row
    res["device"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
