"""Sequence mode with per-slot rigs and tunings: what lins_gpu_seq_configure and lins_gpu_seq_tune cost a step.

    python tools/config_bench.py [--slots 132,1000] [--warmup 3] [--steps 20] [--out DIR]

S slots of simulated VLP-16 drives (config3) through lins_gpu_seq_step_raw, in five cases that take the same steps,
their order rotating from step to step:
  (a) unconfigured: every slot reads the run's values;
  (b) defaults: every slot configured with the run's own values (the same doubles: the same results);
  (c) mixed: the slots configured with three rigs in turn (scan periods 0.1, 0.05 and 0.075, other thresholds, extrinsic,
      noise, stds and biases);
  (d) tuned: every slot tuned with the run's own lins_params and no IMU misalignment (the same results as (a); the step
      adds the IMU rotation's launch);
  (e) tuned_mixed: the slots tuned with three tunings in turn (NUM_ITER 30 / 12 / 5, ICP_FREQ 1 / 2 / 3, gates 25 / 1 / 400,
      LIDAR_STD, LIDAR_SCALE, misalignments 0 / 3 / -2.5 degrees): a different workload, not an overhead.
Each context first steps every slot's largest sweep and restarts (so the timed steps do not reallocate), then configures.
After --warmup steps it prints per S and case the step's device time (the library's CUDA events: projection kernel +
extraction kernel + the four seq_phase_ms phases), the host wall time around the call (which ends with a stream
synchronisation; the descriptors are built beforehand), the kernel launches per step (lins_gpu_launch_count), whether
(a), (b) and (d) agree bit for bit, and the card's name and power limit.
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


def rigs(defs):
    S = defs.LinsSlotConfig.shipped
    return [S(scan_period=0.1, edge_threshold=0.6, surf_threshold=0.4, imu_lidar_extrinsic_angle=2.5, acc_n=60000.0, init_pos_std=(0.01, 0.01, 0.02)),
            S(scan_period=0.05, edge_threshold=0.35, surf_threshold=0.7, imu_lidar_extrinsic_angle=-1.5, gyr_n=0.08, init_ba=(0.02, -0.05, 0.01)),
            S(scan_period=0.075, edge_threshold=0.8, surf_threshold=0.2, imu_lidar_extrinsic_angle=4.0, acc_w=250.0, init_att_std=(0.02, 0.03, 0.05))]


def tunings(defs):
    T = defs.LinsSlotTuning.shipped
    return [T(num_iter=30, icp_freq=1, nearest_feature_search_sq_dist=25.0, lidar_std=0.01, lidar_scale=1.0, imu_misalign_angle=0.0),
            T(num_iter=12, icp_freq=2, nearest_feature_search_sq_dist=1.0, lidar_std=0.05, lidar_scale=0.5, imu_misalign_angle=3.0),
            T(num_iter=5, icp_freq=3, nearest_feature_search_sq_dist=400.0, lidar_std=0.002, lidar_scale=2.0, imu_misalign_angle=-2.5)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="132,1000")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import importlib

    capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
    defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
    synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
    synth.build()
    res = {}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    n_steps = a.warmup + a.steps
    fp = defs.LinsFeatureParams.shipped()
    model = defs.LinsLidarModel.vlp16()
    pool = [synth.raw_log("config3", seed=7100 + i, n_scans=n_steps) for i in range(16)]
    seq_prm, init = defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped()
    cases = ("unconfigured", "defaults", "mixed", "tuned", "tuned_mixed")
    for S in (int(v) for v in a.slots.split(",")):
        drive = [pool[s % len(pool)] for s in range(S)]
        ctx = {}
        for c in cases:
            g = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
            g.seq_open(seq_prm, init, S)
            big = [max(d["sweeps"], key=len) for d in drive]
            g.seq_step_raw(dict(imu=np.zeros((0, 7)), imu_off=np.zeros(S + 1, np.int32), sweeps=big), model=model, scan_imu=np.zeros((S, 6)))
            g.seq_restart(np.ones(S, np.uint8))
            if c == "defaults":
                g.seq_configure(np.ones(S, np.uint8), [defs.LinsSlotConfig.shipped()] * S)
            elif c == "mixed":
                g.seq_configure(np.ones(S, np.uint8), [rigs(defs)[s % 3] for s in range(S)])
            elif c == "tuned":
                p = defs.LinsParams.shipped()
                g.seq_tune(np.ones(S, np.uint8), [defs.LinsSlotTuning.shipped(num_iter=p.num_iter, icp_freq=p.icp_freq, lidar_std=p.lidar_std,
                                                                               nearest_feature_search_sq_dist=p.nearest_feature_search_sq_dist,
                                                                               lidar_scale=p.lidar_scale, imu_misalign_angle=0.0)] * S)
            elif c == "tuned_mixed":
                g.seq_tune(np.ones(S, np.uint8), [tunings(defs)[s % 3] for s in range(S)])
            ctx[c] = g
        ms, dev, launches = {c: [] for c in cases}, {c: [] for c in cases}, {c: [] for c in cases}
        for t in range(n_steps):
            keep = {}
            rows = [d["imu"][d["imu_off"][t]:d["imu_off"][t + 1]] for d in drive]
            keep["imu"] = np.ascontiguousarray(np.concatenate(rows), np.float64)
            keep["imu_off"] = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
            keep["scan_imu"] = np.ascontiguousarray(np.stack([d["imu_last"][t] for d in drive]), np.float64)
            desc = defs.LinsSeqRawDesc()
            desc.n_seq, desc.imu, desc.imu_off = S, keep["imu"].ctypes.data, keep["imu_off"].ctypes.data
            desc.raw = capi.LinsGpu._raw_desc([d["sweeps"][t] for d in drive], 0, keep)
            order = cases[t % len(cases):] + cases[:t % len(cases)]
            for c in order:
                g = ctx[c]
                n0 = g.launch_count()
                t0 = time.perf_counter()
                g._ck(g.L.lins_gpu_seq_step_raw(g.h, C.byref(desc), C.byref(model), C.byref(fp), keep["scan_imu"].ctypes.data))
                g._ck(g.L.lins_gpu_sync(g.h))
                dt = (time.perf_counter() - t0) * 1000.0
                if t >= a.warmup:
                    ms[c].append(dt)
                    dev[c].append(g.project_ms() + g.extract_ms() + float(np.sum(g.seq_phase_ms())))
                    launches[c].append(g.launch_count() - n0)
        snap = {c: ctx[c].seq_download() for c in cases}
        keys = ("global_state", "filter_state", "filter_cov", "status")
        same = all(snap["unconfigured"][k].tobytes() == snap["defaults"][k].tobytes() for k in keys)
        same_tuned = all(snap["unconfigured"][k].tobytes() == snap["tuned"][k].tobytes() for k in keys)
        res[f"S{S}"] = dict(device_ms={c: round(float(np.median(dev[c])), 3) for c in cases},
                            device_ms_range={c: [round(float(np.min(dev[c])), 3), round(float(np.max(dev[c])), 3)] for c in cases},
                            wall_ms={c: round(float(np.median(ms[c])), 3) for c in cases},
                            wall_ms_range={c: [round(float(np.min(ms[c])), 3), round(float(np.max(ms[c])), 3)] for c in cases},
                            launches_per_step={c: sorted(set(launches[c])) for c in cases},
                            statuses={c: np.bincount(snap[c]["status"], minlength=7).tolist() for c in cases},
                            defaults_equal_unconfigured=bool(same), tuned_equal_unconfigured=bool(same_tuned))
        for g in ctx.values():
            g.close()
        print(f"S{S}", json.dumps(res[f"S{S}"]), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "config_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
