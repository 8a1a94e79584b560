"""Device time of the mapping node's cycle (lins_gpu_mapper_step) at a full 50-key-frame window.

Drives the mapper over a synthetic out-and-back drive (tests' generator: tools/synth, seeded) long enough to fill the
window, then times the cycles after it is full with CUDA events on the context's stream and the host clock around each
call (every call ends in a device synchronisation).  The phase split times the pieces of a steady-state cycle on the
same stream, each over many repetitions: the local map's VoxelGrids (corner 0.2 m, surf 0.4 m on the window's
concatenated clouds, sizes taken from the cycle), the scan's four VoxelGrids, and the scan-to-map loop
(lins_gpu_map_set + lins_gpu_scan2map on the cycle's DS clouds; the public entries add their H2D of those clouds).  The
card's name and power limit are read in the same run and printed with the numbers.

    python tools/mapping_bench.py [--cycles 30] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _pkg(name):
    import importlib

    return importlib.import_module("lins---lidar-inertial-slam_b200." + name)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cycles", type=int, default=30, help="timed cycles after the window is full")
    ap.add_argument("--reps", type=int, default=20, help="repetitions of each phase")
    a = ap.parse_args()
    import torch
    import mapper_drive
    import mapperref

    capi, synth, defs = _pkg("capi"), _pkg("synth"), _pkg("ctypes_defs")
    synth.build()
    n_out = (60 + a.cycles) // 2 + 2
    ev = [e for e in mapper_drive.make_drive(synth, n_out=n_out, stall_at=-1) if e[0] == "odom" and e[-1] >= 0]
    stream = torch.cuda.current_stream()
    g = capi.LinsGpu(stream=stream.cuda_stream)
    g.mapper_reset()
    host_ms, dev_ms, last = [], [], None
    for e in ev:
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(stream)
        h0 = time.perf_counter()
        rep = g.mapper_step(*e[1:7])
        h1 = time.perf_counter()
        t.record(stream)
        t.synchronize()
        if rep.window_len == 50 and rep.processed:
            host_ms.append(1e3 * (h1 - h0)); dev_ms.append(s.elapsed_time(t))
            last = rep
    assert last is not None and len(host_ms) >= 5, "the drive did not fill the window"
    poses, window, clouds = g.mapper_download(last)

    def timed(fn):
        fn()
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(stream)
        h0 = time.perf_counter()
        for _ in range(a.reps):
            fn()
        h1 = time.perf_counter()
        t.record(stream); t.synchronize()
        return s.elapsed_time(t) / a.reps, 1e3 * (h1 - h0) / a.reps

    # the window's concatenated clouds are not exported: rebuild same-size clouds from the map DS (the VoxelGrid's cost
    # follows the point count)
    ncat = [len(clouds["corner_ds"]) * 50, (len(clouds["surf_ds"]) + len(clouds["outlier_ds"])) * 50]
    rng = np.random.default_rng(1)
    cat_c = np.repeat(clouds["map_corner_ds"], max(1, ncat[0] // max(1, len(clouds["map_corner_ds"]))), 0)[: ncat[0]]
    cat_s = np.repeat(clouds["map_surf_ds"], max(1, ncat[1] // max(1, len(clouds["map_surf_ds"]))), 0)[: ncat[1]]
    P = lambda x: mapperref.to_points(np.asarray(x, np.float32) + rng.normal(0, 0.05, x.shape).astype(np.float32), defs.POINT_DTYPE)  # noqa: E731
    cat_c, cat_s = P(cat_c), P(cat_s)
    sc, ss, so = (P(clouds[k]) for k in ("corner_ds", "surf_ds", "outlier_ds"))
    phases = {}
    phases["local_map_voxelgrids"] = timed(lambda: (g.voxel_grid(cat_c, 0.2), g.voxel_grid(cat_s, 0.4)))
    phases["scan_voxelgrids"] = timed(lambda: (g.voxel_grid(sc, 0.2), g.voxel_grid(ss, 0.4), g.voxel_grid(so, 0.4), g.voxel_grid(ss, 0.4)))
    mc, ms = (mapperref.to_points(clouds[k], defs.POINT_DTYPE) for k in ("map_corner_ds", "map_surf_ds"))
    qc, qs = (mapperref.to_points(clouds[k], defs.POINT_DTYPE) for k in ("corner_ds", "surf_total_ds"))
    phases["scan_to_map"] = timed(lambda: (g.map_set(mc, ms), g.scan2map(qc, qs, last.transform_guess)))
    out = dict(card=card(), window=int(last.window_len), keyframes=int(last.n_keyframes), cycles=len(dev_ms),
               cycle_device_ms_median=float(np.median(dev_ms)), cycle_host_ms_median=float(np.median(host_ms)),
               cycle_device_ms_p90=float(np.percentile(dev_ms, 90)),
               local_map_points=[len(cat_c), len(cat_s)], map_ds=[int(last.n_map_corner_ds), int(last.n_map_surf_ds)],
               scan_points=[len(e) for e in ev[-1][4:7]], scan_ds=[int(last.n_corner_ds), int(last.n_surf_total_ds)],
               phases_device_ms={k: round(v[0], 4) for k, v in phases.items()},
               phases_host_ms={k: round(v[1], 4) for k, v in phases.items()})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
