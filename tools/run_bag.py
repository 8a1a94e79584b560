#!/usr/bin/env python
"""tools/run_bag.py BAG [--lidar /velodyne_points] [--imu /imu/data] [--max-scans N] [--lidar-model 0|1] [--map [--loops [--global-map]] [--out DIR]]

BASELINE.json configs[1] runner (GPU box): replays a ROS1 bag through the restated front end (image projection, feature
extraction, IMU propagation) and the GPU IESKF update, prints the trajectory.  With --map, every odometry output (what
LinsFusion::publishTopics hands the mapping node: globalStateYZX_ and the YZX clouds) also runs one cycle of the device
mapper (lins_gpu_mapper_step), and DIR/odometry.txt, DIR/mapped.txt and DIR/integrated.txt receive three trajectories,
one line per published scan: stamp, then x y z qx qy qz qw of the odometry, resp. the processed flag and
transformAftMapped (rx ry rz tx ty tz, the mapping node's YZX frame), resp. x y z qx qy qz qw of transform_fusion_node's
pose (/integrated_to_init in /camera_init: the odometry corrected by the last processed cycle before the scan,
lins_gpu_mapper_fuse).  --loops also closes loops (the loop thread ticked after a cycle whenever the stamp has advanced
>= 1 s since its last tick), and mapped.txt then holds the final, corrected key poses (stamp, x y z roll pitch yaw).
--global-map (with --loops) also writes DIR/global_map.pcd after the last cycle: the mapping node's global map
(publishGlobalMap, lins_gpu_mapper_global_map) as a binary PCD of x y z intensity in /camera_init.  The replayed IMU messages are not fed to the mapper's roll / pitch queue (the
front end reads their rates and accelerations only), so transformUpdate runs without the IMU blend.  Uncompressed and lz4-compressed bags
are read directly; for bz2 run `python tools/bag_tool.py decompress IN.bag OUT.bag` first."""
import argparse, importlib, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
ap = argparse.ArgumentParser()
ap.add_argument("bag"); ap.add_argument("--lidar", default="/velodyne_points"); ap.add_argument("--imu", default="/imu/data")
ap.add_argument("--max-scans", type=int, default=0); ap.add_argument("--lidar-model", type=int, default=0)
ap.add_argument("--map", action="store_true", help="run the mapping node's cycle after every odometry output")
ap.add_argument("--loops", action="store_true", help="with --map: close loops; mapped.txt then holds the corrected key poses")
ap.add_argument("--global-map", action="store_true", help="with --loops: write DIR/global_map.pcd after the last cycle")
ap.add_argument("--out", default=".", help="with --map: directory for odometry.txt, mapped.txt and integrated.txt")
a = ap.parse_args()
if a.loops and not a.map:
    ap.error("--loops needs --map")
if a.global_map and not a.loops:
    ap.error("--global-map needs --loops: the global map reads the key frames loop closure keeps")
synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
out = synth.run_bag(a.bag, a.lidar, a.imu, a.max_scans, a.lidar_model)
print("scans", len(out["status"]), "IESKF updates", len(out["iters"]), "mean iterations %.2f" % (out["iters"].mean() if len(out["iters"]) else 0), "diverged", int(((out["flags"] & 2) != 0).sum()))
np.set_printoptions(precision=4, suppress=True)
for k, (st, g) in enumerate(zip(out["status"], out["global_est"])):
    print(k, int(st), g)
if a.map:
    capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
    g = capi.LinsGpu()
    g.mapper_reset()
    if a.loops:
        g.mapper_loops()
    tick, last_processed = None, None
    os.makedirs(a.out, exist_ok=True)
    files = [os.path.join(a.out, f) for f in ("odometry.txt", "mapped.txt", "integrated.txt")]
    with open(files[0], "w") as fo, open(files[1], "w") as fm, open(files[2], "w") as fi:
        for m in out["map_inputs"]:
            fused = g.mapper_fuse(m["time"], m["quat"], m["pos"])  # (the fusion node sees the odometry before the cycle ends)
            rep = g.mapper_step(m["time"], m["quat"], m["pos"], m["corner"], m["surf"], m["outlier"])
            fo.write("%.9f %s\n" % (m["time"], " ".join("%.9g" % v for v in list(m["pos"]) + list(m["quat"]))))
            if rep.processed:
                last_processed = rep
            if a.loops and last_processed is not None and (tick is None or m["time"] - tick >= 1.0):  # the 1 Hz loop thread
                tick = m["time"]
                g.mapper_close_loop()
            if not a.loops:
                fm.write("%.9f %d %s\n" % (m["time"], rep.processed, " ".join("%.9g" % v for v in rep.transform_aft_mapped)))
            fi.write("%.9f %s\n" % (m["time"], " ".join("%.9g" % v for v in fused.row())))
            last = rep
        if a.loops and last_processed is not None:  # the final, loop-corrected key poses: stamp, x y z roll pitch yaw
            for k in g.mapper_download(last_processed)[0]:
                fm.write("%.9f %s\n" % (k[6], " ".join("%.9g" % v for v in k[:6])))
    if a.global_map:
        pcd = importlib.import_module("lins---lidar-inertial-slam_b200.pcd")
        grep = g.mapper_global_map()
        path = os.path.join(a.out, "global_map.pcd")
        pcd.write_pcd(path, g.mapper_global_map_download(grep)[1])
        print("global map:", grep.n_map, "points from", grep.n_key_frames, "key frames" + (" (unfiltered)" if grep.unfiltered else "") + ";", path)
    print("mapper:", len(out["map_inputs"]), "odometry outputs,", last.n_keyframes if out["map_inputs"] else 0, "key frames;",
          "trajectories in", ", ".join(files[:2]), "and", files[2])
