"""Lockstep mapping nodes (lins_gpu_mappers_step) against the same drives on single mappers stepped one after another.

M slots tile a few distinct seeded drives (tests/mapper_drive.make_drive: different seeds, and each slot starts its drive
a few scans later than the previous slot of the same drive).  Every slot is stepped until its window holds 50 key frames,
then `--steps` steps are timed after `--warmup` more:
  - lockstep: CUDA events on the context's stream around each lins_gpu_mappers_step call (the call ends in its
    synchronisation; the stop event also covers the key-frame transform it queues after it), the host clock around the
    call, and cycles/s = M / wall per step;
  - serial: the same events through one single-mapper context per slot (lins_gpu_mapper_step), one after another, for
    all slots at M <= 132 and for the first `--sample` slots at larger M (the per-step figures are then scaled by
    M / sample, and the output says so).
The card's name and power limit are read in the same run.  --profile prints the kernels and the host calls of one
lockstep step at the largest M (torch.profiler).

    python tools/mappers_bench.py [--slots 32,132,1000] [--steps 8] [--warmup 2] [--drives 4] [--sample 32] [--profile]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

FILL = 56  # steps until every slot's window holds 50 key frames (one key frame per cycle on these drives)
PHASES = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="32,132,1000")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--drives", type=int, default=4, help="distinct seeded drives the slots tile")
    ap.add_argument("--sample", type=int, default=32, help="serial single mappers timed when M > 132")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    import mapper_drive
    from mapping_bench import _pkg, card

    capi, synth = _pkg("capi"), _pkg("synth")
    synth.build()
    n_ev = FILL + PHASES + a.warmup + a.steps
    n_out = n_ev // 2 + 2
    drives = [[e[1:7] for e in mapper_drive.make_drive(synth, n_out=n_out, seed=11 + i, stall_at=-1) if e[0] == "odom" and e[-1] >= 0]
              for i in range(a.drives)]
    assert all(len(d) >= n_ev for d in drives)
    stream = torch.cuda.current_stream()

    def event(s, k):  # slot s's event at step k
        return drives[s % a.drives][k + (s // a.drives) % PHASES]

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        h0 = time.perf_counter()
        out = fn()
        h1 = time.perf_counter()
        e1.record(stream)
        e1.synchronize()
        return out, e0.elapsed_time(e1), 1e3 * (h1 - h0)

    results = []
    for M in [int(x) for x in a.slots.split(",")]:
        g = capi.LinsGpu(stream=stream.cuda_stream)
        g.mappers_open(M)
        dev, wall = [], []
        for k in range(FILL + a.warmup + a.steps):
            reps, d_ms, h_ms = timed(lambda: g.mappers_step([event(s, k) for s in range(M)]))
            if k >= FILL + a.warmup:
                assert all(r.processed and r.window_len == 50 for r in reps), "a window is not full"
                dev.append(d_ms); wall.append(h_ms)
        if a.profile and M == max(int(x) for x in a.slots.split(",")):
            from torch.profiler import ProfilerActivity, profile

            k = FILL + a.warmup + a.steps  # (one more full-window step)
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                g.mappers_step([event(s, k) for s in range(M)])
                torch.cuda.synchronize()
            for key in ("cuda_time_total", "self_cpu_time_total"):  # device kernels; host calls (CUDA runtime included)
                print(prof.key_averages().table(sort_by=key, row_limit=12), file=sys.stderr)
        g.close()
        n_ser = M if M <= 132 else min(a.sample, M)
        singles = [capi.LinsGpu(stream=stream.cuda_stream) for _ in range(n_ser)]
        for s in singles:
            s.mapper_reset()
        sdev, swall = [], []
        for k in range(FILL + a.warmup + a.steps):
            tot_d = tot_h = 0.0
            for i, s in enumerate(singles):
                rep, d_ms, h_ms = timed(lambda: s.mapper_step(*event(i, k)))
                tot_d += d_ms; tot_h += h_ms
            if k >= FILL + a.warmup:
                sdev.append(tot_d * M / n_ser); swall.append(tot_h * M / n_ser)
        for s in singles:
            s.close()
        lock_wall = float(np.median(wall))
        ser_wall = float(np.median(swall))
        results.append(dict(slots=M, lockstep_device_ms=round(float(np.median(dev)), 3), lockstep_wall_ms=round(lock_wall, 3),
                            lockstep_cycles_per_s=round(M / lock_wall * 1e3, 1), serial_device_ms=round(float(np.median(sdev)), 3),
                            serial_wall_ms=round(ser_wall, 3), serial_cycles_per_s=round(M / ser_wall * 1e3, 1),
                            serial_measured_slots=n_ser, speedup_wall=round(ser_wall / lock_wall, 2)))
        print(json.dumps(results[-1]), file=sys.stderr)
    print(json.dumps(dict(card=card(), drives=a.drives, steps=a.steps, window=50, results=results)))


if __name__ == "__main__":
    main()
