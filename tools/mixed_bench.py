"""Sequence mode over two sensors at once: one context with lins_gpu_seq_step_raw_mixed against a context per sensor.

    python tools/mixed_bench.py [--slots 132,1000] [--warmup 3] [--steps 3] [--out DIR]

S slots, half of them driving simulated VLP-16 drives (config3) and half 64 x 1024 drives (config4), the two sensors in
alternating slots.  Two arms take the same steps, alternating which goes first:
  (a) mixed: one context of S slots, one lins_gpu_seq_step_raw_mixed call per step (each slot projected with its sensor's
      model);
  (b) split: what a run needs without it, a context per sensor of S / 2 slots each, one lins_gpu_seq_step_raw per context,
      one after the other.
A context's buffers only grow, and a step whose point total exceeds every earlier one reallocates all of its per-point
buffers, pinned staging included.  The totals of these drives grow at every step, so before the first step each context
takes one step of every slot's largest sweep and then restarts all its slots (lins_gpu_seq_restart): the timed steps
then measure the step, not the reallocation.  --no-presize skips that.  After --warmup steps (the slots initialise) it
prints per S: the wall time per step of each arm (host clock, every call
ending with a stream synchronisation; descriptors are built beforehand), the projection and extraction kernel times and
seq_phase_ms (for (b) the two contexts' sum), whether the two arms' final global states agree bit for bit, with the
card's name and power limit.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="132,1000")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--no-presize", action="store_true", help="no step of the largest sweeps before the first step")
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
    models = [defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()]
    logs = [[synth.raw_log("config3", seed=7000 + i, n_scans=n_steps) for i in range(16)],
            [synth.raw_log("config4", seed=7000 + i, n_scans=n_steps) for i in range(8)]]
    init = defs.LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0))
    for S in (int(v) for v in a.slots.split(",")):
        # slot s runs sensor s % 2, drive (s // 2) % pool; the split arm's context k holds the slots of sensor k in order
        of = np.array([s % 2 for s in range(S)], np.int32)
        drive = [logs[s % 2][(s // 2) % len(logs[s % 2])] for s in range(S)]
        halves = [np.flatnonzero(of == k) for k in (0, 1)]
        mixed = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
        mixed.seq_open(defs.LinsSeqParams.shipped(), init, S)
        split = []
        for h in halves:
            g = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
            g.seq_open(defs.LinsSeqParams.shipped(), init, len(h))
            split.append(g)
        wall, kern = {"mixed": [], "split": []}, {"mixed": [], "split": []}
        keep_t = {}
        tab = capi.LinsGpu.models_table(models, of, keep_t)
        if not a.no_presize:
            big = [max(drive[s]["sweeps"], key=len) for s in range(S)]
            si = np.zeros((S, 6))
            step = dict(imu=np.zeros((0, 7)), imu_off=np.zeros(S + 1, np.int32), sweeps=big)
            mixed.seq_step_raw_mixed(step, models, of, scan_imu=si)
            for g, h, m in zip(split, halves, models):
                g.seq_step_raw(dict(imu=step["imu"], imu_off=np.zeros(len(h) + 1, np.int32), sweeps=[big[s] for s in h]), model=m,
                               scan_imu=si[h])
            for g in [mixed] + split:
                g.seq_restart(np.ones(g._seq_n, np.uint8))
        for t in range(n_steps):
            def desc(slots, keep):
                rows = [drive[s]["imu"][drive[s]["imu_off"][t]:drive[s]["imu_off"][t + 1]] for s in slots]
                keep["imu"] = np.ascontiguousarray(np.concatenate(rows), np.float64)
                keep["imu_off"] = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
                keep["scan_imu"] = np.ascontiguousarray(np.stack([drive[s]["imu_last"][t] for s in slots]), np.float64)
                d = defs.LinsSeqRawDesc()
                d.n_seq, d.imu, d.imu_off = len(slots), keep["imu"].ctypes.data, keep["imu_off"].ctypes.data
                d.raw = capi.LinsGpu._raw_desc([drive[s]["sweeps"][t] for s in slots], 0, keep)
                return d

            km = {}
            dm = desc(range(S), km)
            ks = [{}, {}]
            ds = [desc(h, k) for h, k in zip(halves, ks)]

            def run_mixed():
                g = mixed
                t0 = time.perf_counter()
                g._ck(g.L.lins_gpu_seq_step_raw_mixed(g.h, C.byref(dm), C.byref(tab), C.byref(fp), km["scan_imu"].ctypes.data))
                g._ck(g.L.lins_gpu_sync(g.h))
                return time.perf_counter() - t0

            def run_split():
                t0 = time.perf_counter()
                for g, d, k, m in zip(split, ds, ks, models):
                    g._ck(g.L.lins_gpu_seq_step_raw(g.h, C.byref(d), C.byref(m), C.byref(fp), k["scan_imu"].ctypes.data))
                    g._ck(g.L.lins_gpu_sync(g.h))
                return time.perf_counter() - t0

            for fn in ((run_mixed, run_split) if t % 2 == 0 else (run_split, run_mixed)):
                w = fn()
                arm = "mixed" if fn is run_mixed else "split"
                if t >= a.warmup:
                    wall[arm].append(w)
                    cs = [mixed] if arm == "mixed" else split
                    kern[arm].append(np.sum([[g.project_ms(), g.extract_ms()] + [float(v) for v in g.seq_phase_ms()] for g in cs], 0))
        st = mixed.seq_download()["status"]
        gs = mixed.seq_download()["global_state"]
        same = all(gs[h].tobytes() == g.seq_download()["global_state"].tobytes() for h, g in zip(halves, split))
        res[f"S{S}"] = dict(
            presized=not a.no_presize,
            points_per_step=int(km["cloud_off"][-1]),
            step_ms={p: round(float(np.median(wall[p])) * 1000.0, 2) for p in wall},
            step_ms_all={p: [round(w * 1000.0, 2) for w in wall[p]] for p in wall},
            project_ms={p: round(float(np.median([k[0] for k in kern[p]])), 3) for p in kern},
            extract_ms={p: round(float(np.median([k[1] for k in kern[p]])), 3) for p in kern},
            seq_phase_ms={p: [round(float(np.median([k[2 + i] for k in kern[p]])), 3) for i in range(4)] for p in kern},
            statuses=np.bincount(st, minlength=7).tolist(),
            mixed_equals_split=bool(same))
        for g in [mixed] + split:
            g.close()
        print(f"S{S}", json.dumps(res[f"S{S}"]), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "mixed_bench%s.json" % ("_no_presize" if a.no_presize else "")), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
