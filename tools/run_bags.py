#!/usr/bin/env python
"""tools/run_bags.py BAG... [--slots S] [--lidar /velodyne_points] [--imu /imu/data] [--max-scans N] [--lidar-model 0|1] [--out DIR]

Replays many ROS1 bags through sequence mode in lockstep (bag_replay.py): every bag is scheduled as tools/run_bag.py
schedules one, the bags are queued through S slots, and each scan's sensor_msgs/PointCloud2 message is decoded on the
device (lins_gpu_seq_step_cloud2).  Prints a summary line and the trajectory per bag, like run_bag.py; with --out, writes
DIR/<bag name>.npz (stamps, status, scan_status, global_est, iters, flags per scan)."""
import argparse, importlib, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
ap = argparse.ArgumentParser()
ap.add_argument("bags", nargs="+"); ap.add_argument("--slots", type=int, default=0, help="slots (0 = one per bag)")
ap.add_argument("--lidar", default="/velodyne_points"); ap.add_argument("--imu", default="/imu/data")
ap.add_argument("--max-scans", type=int, default=0); ap.add_argument("--lidar-model", type=int, default=0); ap.add_argument("--out")
a = ap.parse_args()
br = importlib.import_module("lins---lidar-inertial-slam_b200.bag_replay")
defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
recs = [br.Recording(p, a.lidar, a.imu, a.max_scans) for p in a.bags]
model = defs.LinsLidarModel.dense64() if a.lidar_model == 1 else defs.LinsLidarModel.vlp16()
outs = br.replay(recs, a.slots or len(recs), model=model)
np.set_printoptions(precision=4, suppress=True)
for p, o in zip(a.bags, outs):
    print(p, br.summary(o))
    for k, (st, g) in enumerate(zip(o["status"], o["global_est"])):
        print(k, int(st), g)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        np.savez(os.path.join(a.out, os.path.splitext(os.path.basename(p))[0] + ".npz"),
                 **{k: o[k] for k in ("stamps", "status", "scan_status", "global_est", "iters", "flags")})
