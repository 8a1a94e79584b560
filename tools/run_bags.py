#!/usr/bin/env python
"""tools/run_bags.py BAG... [--slots S] [--lidar /velodyne_points] [--imu /imu/data] [--max-scans N] [--lidar-model M] [--map [--loops [--global-map]]]
                   [--config a.yaml[,b.yaml,...] [--tune]] [--checkpoint-every N DIR] [--resume DIR] [--out DIR]

Replays many ROS1 bags through sequence mode in lockstep (bag_replay.py): every bag is scheduled as tools/run_bag.py
schedules one, the bags are queued through S slots, and each scan's sensor_msgs/PointCloud2 message is decoded on the
device (lins_gpu_seq_step_cloud2).  --lidar-model is 0 (VLP-16) or 1 (64 x 1024) for every bag, or a comma-separated list
with one value per bag (e.g. 0,1,1,0): bags of different sensors then run in one context, each slot projected with its
bag's model (lins_gpu_seq_step_cloud2_mixed).  Prints a summary line and the trajectory per bag, like run_bag.py; with
--out, writes DIR/<bag name>.npz (stamps, status, scan_status, global_est, iters, flags per scan).  With --map, each
bag's mapping node runs on what its estimator publishes, in lockstep on the device (lins_gpu_seq_map_step), and
DIR/<bag name>.odometry.txt, DIR/<bag name>.mapped.txt and DIR/<bag name>.integrated.txt (DIR: --out, default .)
receive the three trajectories in tools/run_bag.py --map's line format; like run_bag.py --map, the bags' IMU orientation
is not fed to the mappers.  --loops also closes each bag's loops (bag_replay.replay(loops=True): the loop thread ticked
when the bag's stamp has advanced >= 1 s), and <bag name>.mapped.txt then holds the final, corrected key poses (stamp,
x y z roll pitch yaw per key frame); it cannot be combined with --checkpoint-every or --resume.  --global-map (with
--loops) also writes each bag's global map when the bag ends (bag_replay.replay(global_map=True)) to
DIR/<bag name>.global_map.pcd, a binary PCD of x y z intensity in /camera_init.
--config a.yaml[,b.yaml,...] takes LINS config files (exp_port.yaml, OpenCV YAML): one for every bag or one per bag.
Each bag's slot is configured with its file's rig (scan period, feature thresholds, extrinsic, IMU noise, init stds and
biases); the files must agree on the keys every slot shares (num_iter, icp_freq, nearest_feature_search_sq_dist,
lidar_std, lidar_scale), which set the context's parameters.  With --tune as well, each bag's slot also takes its file's
tuning (those shared keys) and imu_misalign_angle (lins_gpu_seq_tune: its IMU values are rotated into the vehicle frame as
LinsFusion::imuCallback does), so the files may differ in any key; the first file's tuning sets the context's parameters.
--checkpoint-every N DIR writes a checkpoint of the replay into DIR after every N-th step (every occupied slot saved by
lins_gpu_seq_save, and the driver's state); --resume DIR continues a replay of the same bags and options from the
checkpoint in DIR, in a new context, with the outputs an uninterrupted replay would give."""
import argparse, importlib, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def lidar_models(spec, n_bags):
    """The --lidar-model value as one LinsLidarModel (a single value) or a list with one per bag (a comma-separated list,
    which must have n_bags entries)."""
    defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
    presets = {"0": defs.LinsLidarModel.vlp16, "1": defs.LinsLidarModel.dense64}
    vals = [v.strip() for v in str(spec).split(",")]
    bad = [v for v in vals if v not in presets]
    if bad:
        raise ValueError(f"--lidar-model: {bad[0]!r} is not 0 (VLP-16) or 1 (64 x 1024)")
    if len(vals) == 1:
        return presets[vals[0]]()
    if len(vals) != n_bags:
        raise ValueError(f"--lidar-model lists {len(vals)} models for {n_bags} bags")
    return [presets[v]() for v in vals]


def bag_configs(spec, n_bags):
    """(LinsParams of the context, one LinsSlotConfig per bag) from the --config value: one file for every bag or a
    comma-separated list with one per bag.  ValueError for a count mismatch or files whose shared keys disagree."""
    rc = importlib.import_module("lins---lidar-inertial-slam_b200.rig_config")
    paths = [v.strip() for v in str(spec).split(",")]
    if len(paths) not in (1, n_bags):
        raise ValueError(f"--config lists {len(paths)} files for {n_bags} bags")
    loaded = [rc.load_rig(p) for p in paths]
    shared = loaded[0][1]
    for p, (_, sh) in zip(paths, loaded):
        bad = [k for k in rc.SHARED_KEYS if sh[k] != shared[k]]
        if bad:
            raise ValueError(f"--config: {p} and {paths[0]} disagree on {', '.join(bad)}, which every slot of a run shares")
    cfgs = [rc.slot_config(r) for r, _ in loaded]
    if len(cfgs) == 1:
        cfgs = cfgs * n_bags
    return rc.lins_params(shared), cfgs


def bag_tunings(spec, n_bags):
    """(LinsParams of the context, one LinsSlotConfig and one LinsSlotTuning per bag) from the --config value with --tune:
    each file gives its bag's rig and tuning (rig_config.load_config), and the files may differ in any key.  ValueError
    for a count mismatch."""
    rc = importlib.import_module("lins---lidar-inertial-slam_b200.rig_config")
    paths = [v.strip() for v in str(spec).split(",")]
    if len(paths) not in (1, n_bags):
        raise ValueError(f"--config lists {len(paths)} files for {n_bags} bags")
    loaded = [rc.load_config(p) for p in paths]
    if len(loaded) == 1:
        loaded = loaded * n_bags
    return rc.lins_params(loaded[0][1]), [rc.slot_config(r) for r, _ in loaded], [rc.slot_tuning(t) for _, t in loaded]


def write_map(o, out_dir, name, loops=False):
    """<name>.odometry.txt, <name>.mapped.txt and <name>.integrated.txt of one replayed bag, one line per published scan as
    tools/run_bag.py --map writes odometry.txt, mapped.txt and integrated.txt: stamp, then x y z qx qy qz qw of the
    odometry, resp. the processed flag and transformAftMapped, resp. x y z qx qy qz qw of the fused pose.  loops: mapped.txt
    holds the final (loop-corrected) key poses instead, one line per key frame: stamp, x y z roll pitch yaw."""
    os.makedirs(out_dir, exist_ok=True)
    files = [os.path.join(out_dir, name + ext) for ext in (".odometry.txt", ".mapped.txt", ".integrated.txt")]
    with open(files[0], "w") as fo, open(files[1], "w") as fm, open(files[2], "w") as fi:
        for t, od, pr, aft, fu in zip(o["map_time"], o["map_odom"], o["map_processed"], o["map_aft_mapped"], o["map_fused"]):
            fo.write("%.9f %s\n" % (t, " ".join("%.9g" % v for v in od)))
            if not loops:
                fm.write("%.9f %d %s\n" % (t, pr, " ".join("%.9g" % v for v in aft)))
            fi.write("%.9f %s\n" % (t, " ".join("%.9g" % v for v in fu)))
        if loops:
            for k in o["key_poses"]:
                fm.write("%.9f %s\n" % (k[6], " ".join("%.9g" % v for v in k[:6])))
    print("mapper:", len(o["map_time"]), "odometry outputs,", len(o["key_poses"]), "key frames;", "trajectories in",
          ", ".join(files[:2]), "and", files[2])


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("bags", nargs="+"); ap.add_argument("--slots", type=int, default=0, help="slots (0 = one per bag)")
    ap.add_argument("--lidar", default="/velodyne_points"); ap.add_argument("--imu", default="/imu/data")
    ap.add_argument("--max-scans", type=int, default=0)
    ap.add_argument("--lidar-model", default="0", help="0 | 1 for every bag, or one per bag: 0,1,...")
    ap.add_argument("--map", action="store_true", help="run each bag's mapping node on what its estimator publishes")
    ap.add_argument("--loops", action="store_true", help="with --map: close loops (mapped.txt: the corrected key poses)")
    ap.add_argument("--global-map", action="store_true", help="with --loops: write DIR/<bag name>.global_map.pcd")
    ap.add_argument("--config", help="LINS config file(s): one for every bag, or one per bag: a.yaml,b.yaml,...")
    ap.add_argument("--tune", action="store_true", help="with --config: each bag also takes its file's tuning and IMU misalignment")
    ap.add_argument("--checkpoint-every", nargs=2, metavar=("N", "DIR"), help="write a checkpoint into DIR after every N-th step")
    ap.add_argument("--resume", metavar="DIR", help="continue from the checkpoint in DIR")
    ap.add_argument("--out")
    a = ap.parse_args(argv)
    try:
        every, ck_dir = (None, None)
        if a.checkpoint_every:
            if not a.checkpoint_every[0].isdigit() or int(a.checkpoint_every[0]) < 1:
                raise ValueError(f"--checkpoint-every: {a.checkpoint_every[0]!r} is not a step count >= 1")
            every, ck_dir = int(a.checkpoint_every[0]), a.checkpoint_every[1]
        if a.loops and not a.map:
            raise ValueError("--loops needs --map")
        if a.global_map and not a.loops:
            raise ValueError("--global-map needs --loops: the global map reads the key frames loop closure keeps")
        if a.loops and (a.checkpoint_every or a.resume):
            raise ValueError("--loops cannot be combined with --checkpoint-every / --resume: a slot with loop closure is not saved")
        model = lidar_models(a.lidar_model, len(a.bags))
        if a.tune and not a.config:
            raise ValueError("--tune takes the tuning from the --config files")
        tunes = [None] * len(a.bags)
        if a.tune:
            prm, cfgs, tunes = bag_tunings(a.config, len(a.bags))
        else:
            prm, cfgs = bag_configs(a.config, len(a.bags)) if a.config else (None, [None] * len(a.bags))
    except ValueError as e:
        ap.error(str(e))
    br = importlib.import_module("lins---lidar-inertial-slam_b200.bag_replay")
    capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
    recs = [br.Recording(p, a.lidar, a.imu, a.max_scans, config=c, tuning=t) for p, c, t in zip(a.bags, cfgs, tunes)]
    outs = br.replay(recs, a.slots or len(recs), model=model, map=a.map, gpu=capi.LinsGpu(prm) if prm is not None else None,
                     checkpoint=ck_dir, checkpoint_every=every, resume=a.resume, loops=a.loops,
                     global_map=a.global_map)
    np.set_printoptions(precision=4, suppress=True)
    for p, o in zip(a.bags, outs):
        print(p, br.summary(o))
        for k, (st, g) in enumerate(zip(o["status"], o["global_est"])):
            print(k, int(st), g)
        if a.map:
            write_map(o, a.out or ".", os.path.splitext(os.path.basename(p))[0], a.loops)
        if a.global_map:
            pcd = importlib.import_module("lins---lidar-inertial-slam_b200.pcd")
            path = os.path.join(a.out or ".", os.path.splitext(os.path.basename(p))[0] + ".global_map.pcd")
            pcd.write_pcd(path, o["global_map"])
            print("global map:", len(o["global_map"]), "points from", len(o["global_map_keys"]), "key frames;", path)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            np.savez(os.path.join(a.out, os.path.splitext(os.path.basename(p))[0] + ".npz"),
                     **{k: o[k] for k in ("stamps", "status", "scan_status", "global_est", "iters", "flags")})


if __name__ == "__main__":
    main()
