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

    python tools/proj_bench.py --seq [--slots 132,1000] [--warmup 3] [--steps 3] [--out DIR]

Sequence mode from the raw sweep instead: S slots (VLP-16 and 64 x 1024, each S of --slots) opened with
lins_gpu_seq_open run simulated drives (slot s drives log s % pool).  Two contexts take the same steps, alternating which
goes first: lins_gpu_seq_step_raw, and the chain it replaces (lins_gpu_project_scans to host buffers, compaction of the
segmented clouds to dense CSR in numpy, lins_gpu_seq_step_pcl).  After --warmup steps (the slots initialise) it prints, per
lidar and S: the wall time per step of both (host clock, each call ends with a stream synchronisation; descriptors are
built beforehand), the projection and extraction kernel times and seq_phase_ms of each, and the H2D bytes per step
(point records, per-point cloud_info, offsets, ring indices, orientations, IMU rows), with the card's name and power
limit.
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
    ap.add_argument("--seq", action="store_true", help="sequence mode: lins_gpu_seq_step_raw against the host round trip")
    ap.add_argument("--slots", default="132,1000")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
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
    if a.seq:
        seq_mode(a, res, capi, defs, synth)
        return emit(a, res, "proj_bench_seq.json")
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
    emit(a, res, "proj_bench.json")


def emit(a, res, fname):
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, fname), "w") as f:
            f.write(line + "\n")


def seq_mode(a, res, capi, defs, synth):
    n_steps = a.warmup + a.steps
    fp = defs.LinsFeatureParams.shipped()
    for name, config, n_logs in (("vlp16", "config3", 16), ("dense64", "config4", 8)):
        logs = [synth.raw_log(config, seed=7000 + i, n_scans=n_steps) for i in range(n_logs)]
        model = defs.LinsLidarModel.dense64() if logs[0]["lidar"] == 1 else defs.LinsLidarModel.vlp16()
        L = model.line_num
        for S in (int(v) for v in a.slots.split(",")):
            ctx = {}
            for path in ("raw", "chain"):
                ctx[path] = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
                ctx[path].seq_open(defs.LinsSeqParams.shipped(), defs.LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0)), S)
            wall, kern, h2d = {"raw": [], "chain": []}, {"raw": [], "chain": []}, {}
            for t in range(n_steps):
                # the step's input, built before any clock starts
                keep = {}
                rows = [logs[s % n_logs]["imu"][logs[s % n_logs]["imu_off"][t]:logs[s % n_logs]["imu_off"][t + 1]] for s in range(S)]
                keep["imu"] = np.ascontiguousarray(np.concatenate(rows), np.float64)
                keep["imu_off"] = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
                scan_imu = np.ascontiguousarray(np.stack([logs[s % n_logs]["imu_last"][t] for s in range(S)]), np.float64)
                d = defs.LinsSeqRawDesc()
                d.n_seq, d.imu, d.imu_off = S, keep["imu"].ctypes.data, keep["imu_off"].ctypes.data
                d.raw = capi.LinsGpu._raw_desc([logs[s % n_logs]["sweeps"][t] for s in range(S)], 0, keep)
                total = int(keep["cloud_off"][-1])
                outs = [np.zeros(total, defs.POINT_DTYPE), np.zeros(total, np.uint8), np.zeros(total, np.uint32), np.zeros(total, np.float32),
                        np.zeros(total, defs.POINT_DTYPE), np.zeros((S, L), np.int32), np.zeros((S, L), np.int32), np.zeros((S, 3), np.float32),
                        np.zeros((S, 2), np.int32)]
                imu_bytes = keep["imu"].nbytes + keep["imu_off"].nbytes + scan_imu.nbytes

                def run_raw():
                    g = ctx["raw"]
                    t0 = time.perf_counter()
                    g._ck(g.L.lins_gpu_seq_step_raw(g.h, C.byref(d), C.byref(model), C.byref(fp), scan_imu.ctypes.data))
                    g._ck(g.L.lins_gpu_sync(g.h))
                    return time.perf_counter() - t0

                def run_chain():
                    g = ctx["chain"]
                    t0 = time.perf_counter()
                    g._ck(g.L.lins_gpu_project_scans(g.h, C.byref(model), C.byref(d.raw), *[o.ctypes.data for o in outs]))
                    cnt, off = outs[8][:, 0], keep["cloud_off"]
                    idx = np.repeat(off[:-1], cnt) + (np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt))  # dense CSR
                    pk = dict(cloud=outs[0][idx], ground=outs[1][idx], col=outs[2][idx], range=outs[3][idx],
                              off=np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32))
                    pd = defs.LinsSeqPclDesc()
                    pd.n_seq, pd.imu, pd.imu_off = S, d.imu, d.imu_off
                    p = pd.pcl
                    p.n_scans, p.line_num, p.point_format = S, L, 0
                    p.cloud, p.cloud_off = pk["cloud"].ctypes.data, pk["off"].ctypes.data
                    p.ground_flag, p.col_ind, p.range = pk["ground"].ctypes.data, pk["col"].ctypes.data, pk["range"].ctypes.data
                    p.start_ring_index, p.end_ring_index, p.orientation = outs[5].ctypes.data, outs[6].ctypes.data, outs[7].ctypes.data
                    pd.pcl = p
                    g._ck(g.L.lins_gpu_seq_step_pcl(g.h, C.byref(pd), C.byref(fp), scan_imu.ctypes.data))
                    g._ck(g.L.lins_gpu_sync(g.h))
                    dt = time.perf_counter() - t0
                    h2d["chain"] = int(16 * total + 4 * (S + 1) + (16 + 1 + 4 + 4) * len(idx) + 4 * (S + 1) + 8 * S * L + 12 * S + imu_bytes)
                    return dt

                order = (run_raw, run_chain) if t % 2 == 0 else (run_chain, run_raw)
                for fn in order:
                    w = fn()
                    path = "raw" if fn is run_raw else "chain"
                    if t >= a.warmup:
                        g = ctx[path]
                        wall[path].append(w)
                        kern[path].append([g.project_ms(), g.extract_ms()] + [float(v) for v in g.seq_phase_ms()])
                h2d["raw"] = int(16 * total + 4 * (S + 1) + imu_bytes)
                del outs
            key = f"{name}_S{S}"
            res[key] = dict(
                points_per_step=total,
                step_ms={p: round(float(np.median(wall[p])) * 1000.0, 2) for p in wall},
                step_ms_all={p: [round(w * 1000.0, 2) for w in wall[p]] for p in wall},
                project_ms={p: round(float(np.median([k[0] for k in kern[p]])), 3) for p in kern},
                extract_ms={p: round(float(np.median([k[1] for k in kern[p]])), 3) for p in kern},
                seq_phase_ms={p: [round(float(np.median([k[2 + i] for k in kern[p]])), 3) for i in range(4)] for p in kern},
                h2d_bytes_per_step=h2d,
                statuses=np.bincount(ctx["raw"].seq_download()["status"], minlength=7).tolist())
            for g in ctx.values():
                g.close()
            print(key, json.dumps(res[key]), flush=True)


if __name__ == "__main__":
    main()
