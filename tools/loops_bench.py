#!/usr/bin/env python
"""tools/loops_bench.py [--slots 1,132,1000] [--seed 6]

Loop closure of the mapping node (lins_gpu_mappers_close_loops, DESIGN.md §4.14) on a synthetic out-and-back drive
whose odometry drifts, copied into every slot, so that every slot has a candidate when the drive has come back:

- close_loops: the call's time (host clock around a call that ends in its one synchronisation) at each M, with every
  slot holding a candidate, and the ICP iterations it ran (mean / max over the slots);
- the mapping step (lins_gpu_mappers_step) of M enabled slots against M plain slots over the same drive, median over the
  steps at a full 50-key-frame window;
- the host cost of a key-frame save once a slot has a loop factor (the Gauss-Newton solve of the key-pose graph and
  correctPoses): the single mapper's step time after its first closure minus a plain mapper's at the same step, against
  the key-frame count;
- the key-frame stores' bytes after the drive, from lins_gpu_mappers_store_bytes: an enabled slot's device store (the
  window and the newest key frame in the map frame, as a plain slot's) and its host store (every key frame's three DS
  clouds in the body frame, 16 B per point, in pinned host memory), per slot and per key frame, and the run's pinned
  slabs.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mapper_drive  # noqa: E402


def drive(seed, n_out=36, yaw_bias=2e-3, x_bias=0.02):
    xs = [-9.0 + 0.5 * k for k in range(n_out)] + [-9.0 + 0.5 * (n_out - 1 - k) - 0.25 for k in range(1, n_out)]
    poses = [(x, 0.3 * math.sin(0.15 * k), 1.5, 0.0 if k < n_out else math.pi) for k, x in enumerate(xs)]
    scans, _ = synth.generate_map_drive(np.array(poses), seed=seed)
    ev, t = [], 100.0
    for k, ((corner, surf, outlier), T) in enumerate(zip(scans, _)):
        odo = T.astype(np.float64) + k * np.array([0, yaw_bias, 0, x_bias, 0, 0])
        ev.append((t, mapper_drive.odometry_quat(odo), (odo[3], odo[4], odo[5]), corner, surf, outlier))
        t += 0.5
    return ev


def lockstep(ev, M, loops):
    g = capi.LinsGpu()
    g.mappers_open(M)
    if loops:
        g.mappers_loops(np.ones(M, np.uint8))
    step_ms, reps = [], None
    for e in ev:
        t0 = time.perf_counter()
        reps = g.mappers_step([e] * M)
        step_ms.append(((time.perf_counter() - t0) * 1e3, reps[0].window_len))
    return g, step_ms, reps


def single(ev, loops):
    g = capi.LinsGpu()
    g.mapper_reset()
    if loops:
        g.mapper_loops()
    out, tick, closed, first = [], None, False, None
    for e in ev:
        t0 = time.perf_counter()
        rep = g.mapper_step(*e)
        ms = (time.perf_counter() - t0) * 1e3
        out.append((ms, rep.keyframe_saved, rep.n_keyframes, closed))
        if loops and (tick is None or e[0] - tick >= 1.0):
            tick = e[0]
            lr = g.mapper_close_loop()
            if lr.accepted and not closed:
                closed, first = True, len(out)
    return out, first


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="1,132,1000")
    ap.add_argument("--seed", type=int, default=6)
    a = ap.parse_args()
    ev = drive(a.seed)
    res = {"what": "lins_gpu_mappers_close_loops / mappers_step with loop closure, synthetic drifted out-and-back drive in every slot"}
    for M in [int(x) for x in a.slots.split(",")]:
        g, en, reps = lockstep(ev, M, True)
        row = {"mapping_step_ms_enabled_full_window_median": float(np.median([ms for ms, w in en if w == 50] or [np.nan]))}
        if M <= 132:
            _, pl, _ = lockstep(ev, M, False)
            row["mapping_step_ms_plain_full_window_median"] = float(np.median([ms for ms, w in pl if w == 50] or [np.nan]))
        mask = np.ones(M, np.uint8)
        calls = []
        for _ in range(3):
            t0 = time.perf_counter()
            lrs = g.mappers_close_loops(mask)
            calls.append((time.perf_counter() - t0) * 1e3)
        it = np.array([lr.icp_iters for lr in lrs])
        row.update(close_loops_ms=calls, with_candidate=int(sum(lr.closest_history_frame_id >= 0 for lr in lrs)),
                   icp_iters_mean=float(it.mean()), icp_iters_max=int(it.max()), n_source_mean=float(np.mean([lr.n_source for lr in lrs])),
                   n_history_ds_mean=float(np.mean([lr.n_history_ds for lr in lrs])), accepted=int(sum(lr.accepted for lr in lrs)))
        nk = reps[0].n_keyframes
        dev, host, reserved = g.mappers_store_bytes()
        row.update(store_device_bytes_per_slot=int(dev[0]), store_host_bytes_per_slot=int(host[0]),
                   store_host_bytes_per_key_frame=round(int(host[0]) / max(nk, 1), 1), store_host_reserved_bytes=reserved)
        row["key_frames"] = nk
        res[f"M={M}"] = row
        del g
    en, first = single(ev, True)
    pl, _ = single(ev, False)
    res["host_save_after_closure"] = [{"key_frames": e[2], "extra_ms": round(e[0] - p[0], 3)} for e, p in zip(en, pl) if e[3] and e[1]]
    res["first_closure_at_event"] = first
    res["device"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
