"""Sequence mode from sensor_msgs/PointCloud2 messages: device decode against host decode (DESIGN.md §4.8).

    python tools/cloud2_bench.py [--slots 132,1000] [--steps-set 32,22] [--warmup 3] [--steps 3] [--out DIR]

For VLP-16 (config3) and 64 x 1024 (config4) simulated drives, each S of --slots and each point_step of --steps-set
(32: the Velodyne driver's PointXYZIR; 22: x, y, z, intensity, ring u16, time f32), S slots opened with
lins_gpu_seq_open run the drives (slot s drives log s % pool) in three contexts that take the same steps, the arms in a
rotating order so that none always runs first:
  (a) pageable: lins_gpu_seq_step_cloud2 on the step's messages as they lie in one pageable buffer (whole PointCloud2
      messages back to back, as in an uncompressed bag chunk; data_off points at each message's data field, so the
      library uploads the bytes from the first data field to the last, headers in between included);
  (b) registered: the same from a buffer page-locked once with lins_gpu_host_register (one DMA, no host pass);
  (c) host: decode_pointcloud2 of every message in C++ threads (tools/synth/lins_bag.cpp lins_bag_decode_cloud2_many,
      --threads, default the core count) into packed 16-B records, then lins_gpu_seq_step_raw with LINS_POINTS_PACKED16.
After --warmup steps (the slots initialise), per shape, S and point_step it prints: the wall time per step of each arm
(host clock; each call ends in a stream synchronisation; buffers are built before any clock starts), the decode kernel's
CUDA-event time (a, b), the host decode's share of (c), the projection and extraction kernel times, and the H2D bytes per
step.  gather_ms is what tools/run_bags.py (bag_replay.py) adds to (b) per step: copying the S data fields out of their
bags into its one registered buffer.  Also the card's name and power limit.  The three arms' sequence states are checked
to be bit-identical after every step.
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
import cloud2cases as cc  # noqa: E402

LAYOUT = {32: "velodyne32", 22: "ring_time22"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="132,1000")
    ap.add_argument("--steps-set", default="32,22", help="point_step values (32, 22)")
    ap.add_argument("--shapes", default="vlp16,dense64")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import importlib

    capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
    defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
    synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
    synth.build()
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tools", "synth"), "liblins_bag.so"])
    bag = cc.baglib()
    bag.lins_bag_decode_cloud2_many.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    res = {"host_threads": a.threads}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        res["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    except OSError:
        res["gpu"] = "unknown"
    n_steps = a.warmup + a.steps
    fp = defs.LinsFeatureParams.shipped()
    init = defs.LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0))
    shapes = {"vlp16": ("config3", 16), "dense64": ("config4", 8)}
    for name in a.shapes.split(","):
        config, n_logs = shapes[name]
        logs = [synth.raw_log(config, seed=7000 + i, n_scans=n_steps) for i in range(n_logs)]
        model = defs.LinsLidarModel.dense64() if logs[0]["lidar"] == 1 else defs.LinsLidarModel.vlp16()
        for ps in (int(v) for v in a.steps_set.split(",")):
            # every message of the pool, encoded once: (bytes, index)
            msgs = [[cc.message(LAYOUT[ps], l["sweeps"][t], seq=t)[0] for t in range(n_steps)] for l in logs]
            idx = [[cc.bag_tool.index_pointcloud2(m) for m in ms] for ms in msgs]
            for S in (int(v) for v in a.slots.split(",")):
                run_one(a, res, capi, defs, bag, logs, msgs, idx, model, fp, init, name, ps, S, n_steps)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "cloud2_bench.json"), "w") as f:
            f.write(line + "\n")


def run_one(a, res, capi, defs, bag, logs, msgs, idx, model, fp, init, name, ps, S, n_steps):
    n_logs = len(logs)
    arms = ("pageable", "registered", "host")
    ctx = {}
    for arm in arms:
        ctx[arm] = capi.LinsGpu(defs.LinsParams.shipped(), device=0)
        ctx[arm].seq_open(defs.LinsSeqParams.shipped(), init, S)
    lib = capi.lib()
    reg_buf, gather_buf = None, None
    wall = {k: [] for k in arms}
    kern = {k: [] for k in arms}
    host_ms, gather_ms, h2d = [], [], {}
    try:
        for t in range(n_steps):
            # the step's input, built before any clock starts
            sl = [s % n_logs for s in range(S)]
            rows = [logs[l]["imu"][logs[l]["imu_off"][t]:logs[l]["imu_off"][t + 1]] for l in sl]
            imu = np.ascontiguousarray(np.concatenate(rows), np.float64)
            imu_off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
            scan_imu = np.ascontiguousarray(np.stack([logs[l]["imu_last"][t] for l in sl]), np.float64)
            step_msgs = [msgs[l][t] for l in sl]
            ixs = [idx[l][t] for l in sl]
            msg_off = np.concatenate([[0], np.cumsum([len(m) for m in step_msgs])]).astype(np.int64)
            blob = np.frombuffer(b"".join(step_msgs), np.uint8)
            starts = msg_off[:-1] + np.array([ix["data_start"] for ix in ixs], np.int64)
            data_off = np.concatenate([starts, [starts[-1] + ixs[-1]["data_len"]]]).astype(np.int64)
            lays = (defs.LinsCloud2Layout * S)(*[cc.layout_of(defs, ix) for ix in ixs])
            if reg_buf is None or len(reg_buf) < len(blob):
                if reg_buf is not None:
                    lib.lins_gpu_host_unregister(reg_buf.ctypes.data)
                reg_buf = np.empty(int(len(blob) * 1.25), np.uint8)
                assert lib.lins_gpu_host_register(reg_buf.ctypes.data, reg_buf.nbytes) == 0
            reg_buf[: len(blob)] = blob
            # bag_replay's gather: the S data fields copied into one registered buffer (timed on its own)
            field_bytes = sum(ix["data_len"] for ix in ixs)
            if gather_buf is None or len(gather_buf) < field_bytes:
                gather_buf = np.empty(int(field_bytes * 1.25), np.uint8)
            t0 = time.perf_counter()
            o = 0
            for m, ix in zip(step_msgs, ixs):
                gather_buf[o: o + ix["data_len"]] = np.frombuffer(m, np.uint8, ix["data_len"], ix["data_start"])
                o += ix["data_len"]
            g_ms = (time.perf_counter() - t0) * 1000.0
            counts = np.array([ix["width"] * ix["height"] for ix in ixs], np.int64)
            out_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
            packed = np.zeros((max(int(out_off[-1]), 1), 4), np.float32)

            def seq_desc(base):
                d = defs.LinsSeqCloud2Desc()
                d.n_seq, d.imu, d.imu_off = S, imu.ctypes.data, imu_off.ctypes.data
                c2 = d.cloud2
                c2.n_scans, c2.data, c2.data_off, c2.layouts = S, base, data_off.ctypes.data, C.cast(lays, C.c_void_p)
                d.cloud2 = c2
                return d

            d_page, d_reg = seq_desc(blob.ctypes.data), seq_desc(reg_buf.ctypes.data)

            def run_cloud2(arm, d):
                g = ctx[arm]
                t0 = time.perf_counter()
                g._ck(g.L.lins_gpu_seq_step_cloud2(g.h, C.byref(d), C.byref(model), C.byref(fp), scan_imu.ctypes.data))
                g._ck(g.L.lins_gpu_sync(g.h))
                return time.perf_counter() - t0, None

            def run_host():
                g = ctx["host"]
                t0 = time.perf_counter()
                assert bag.lins_bag_decode_cloud2_many(blob.ctypes.data, msg_off.ctypes.data, S, packed.ctypes.data, out_off.ctypes.data, a.threads) == 0
                t1 = time.perf_counter()
                d = defs.LinsSeqRawDesc()
                d.n_seq, d.imu, d.imu_off = S, imu.ctypes.data, imu_off.ctypes.data
                r = d.raw
                r.n_scans, r.cloud, r.cloud_off, r.point_format = S, packed.ctypes.data, out_off.ctypes.data, 1
                d.raw = r
                g._ck(g.L.lins_gpu_seq_step_raw(g.h, C.byref(d), C.byref(model), C.byref(fp), scan_imu.ctypes.data))
                g._ck(g.L.lins_gpu_sync(g.h))
                return time.perf_counter() - t0, (t1 - t0) * 1000.0

            runs = {"pageable": lambda: run_cloud2("pageable", d_page), "registered": lambda: run_cloud2("registered", d_reg), "host": run_host}
            order = [arms[(t + k) % 3] for k in range(3)]
            for arm in order:
                w, hm = runs[arm]()
                if t >= a.warmup:
                    g = ctx[arm]
                    wall[arm].append(w)
                    kern[arm].append([g.decode_ms() if arm != "host" else 0.0, g.project_ms(), g.extract_ms()])
                    if hm is not None:
                        host_ms.append(hm)
            if t >= a.warmup:
                gather_ms.append(g_ms)
            snaps = [ctx[arm].seq_download() for arm in arms]
            for sn in snaps[1:]:
                for k in ("global_state", "filter_state", "filter_cov", "status"):
                    assert sn[k].tobytes() == snaps[0][k].tobytes(), (name, ps, S, t, k)
            aux = imu.nbytes + imu_off.nbytes + scan_imu.nbytes
            h2d["pageable"] = h2d["registered"] = int(data_off[-1] - data_off[0] + 48 * S + 2 * 4 * (S + 1) + aux)
            h2d["host"] = int(16 * int(out_off[-1]) + 4 * (S + 1) + aux)
            res_pts = int(out_off[-1])
    finally:
        if reg_buf is not None:
            lib.lins_gpu_host_unregister(reg_buf.ctypes.data)
        for g in ctx.values():
            g.close()
    key = f"{name}_ps{ps}_S{S}"
    med = lambda v: round(float(np.median(v)), 3)  # noqa: E731
    res[key] = dict(
        points_per_step=res_pts,
        step_ms={k: round(float(np.median(wall[k])) * 1000.0, 2) for k in arms},
        step_ms_all={k: [round(w * 1000.0, 2) for w in wall[k]] for k in arms},
        decode_kernel_ms={k: med([x[0] for x in kern[k]]) for k in ("pageable", "registered")},
        host_decode_ms=med(host_ms),
        gather_ms=med(gather_ms),
        project_ms={k: med([x[1] for x in kern[k]]) for k in arms},
        extract_ms={k: med([x[2] for x in kern[k]]) for k in arms},
        h2d_bytes_per_step=h2d,
        statuses=np.bincount(snaps[0]["status"], minlength=7).tolist())
    print(key, json.dumps(res[key]), flush=True)


if __name__ == "__main__":
    main()
