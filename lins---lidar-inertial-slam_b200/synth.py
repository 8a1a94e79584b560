"""ctypes binding of tools/synth/liblins_synth.so — the synthetic scan-pair generator (inputs only).

The generator runs the product's own host-side CPU stages (image projection, feature extraction, IMU
propagation; all stay on the CPU per BASELINE.json north_star) over a seeded ray-cast world and returns a
:class:`Batch` of independent (scan pair, prior) units in the C-ABI's ``lins_batch_desc`` layout.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .ctypes_defs import Batch, LinsBatchDesc, LinsPclDesc, LinsRawDesc, POINT_DTYPE

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_DIR = os.path.join(_ROOT, "tools", "synth")
_LIB = None


class SynthCfg(C.Structure):
    _fields_ = [
        ("lidar", C.c_int32),
        ("world", C.c_int32),
        ("fixed_motion", C.c_int32),
        ("stress_queries", C.c_int32),
        ("v_max", C.c_double),
        ("w_max", C.c_double),
        ("range_noise", C.c_double),
        ("prior_vel_sigma", C.c_double),
    ]


def build():
    subprocess.check_call(["make", "-s", "-C", _DIR])


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_DIR, "liblins_synth.so")
        if not os.path.exists(path):
            build()
        L = C.CDLL(path)
        L.lins_synth_batch_create.restype = C.c_void_p
        L.lins_synth_batch_create.argtypes = [C.POINTER(SynthCfg), C.c_uint64, C.c_int, C.c_int]
        L.lins_synth_batch_destroy.argtypes = [C.c_void_p]
        L.lins_synth_batch_desc.argtypes = [C.c_void_p, C.POINTER(LinsBatchDesc)]
        L.lins_synth_batch_truth.restype = C.POINTER(C.c_double)
        L.lins_synth_batch_truth.argtypes = [C.c_void_p]
        L.lins_synth_batch_new_less.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        _LIB = L
    return _LIB


# BASELINE.json configs -> generator settings
CONFIGS = {
    # configs[0] "single synthetic VLP-16 scan ... correctness gate" (SURVEY.md §8(d) config 1a)
    "config1": dict(lidar=0, world=0, fixed_motion=1, stress_queries=0, v_max=10.0, w_max=0.3, range_noise=0.01,
                    prior_vel_sigma=0.05),
    # config 1b: the literal "~2k surf + 500 edge feats" as queries
    "config1b": dict(lidar=0, world=0, fixed_motion=1, stress_queries=1, v_max=10.0, w_max=0.3, range_noise=0.01,
                     prior_vel_sigma=0.05),
    # configs[2] "synthetic 1000-scan sequence, flat-ground map" / configs[4] (8000 scans)
    "config3": dict(lidar=0, world=1, fixed_motion=0, stress_queries=0, v_max=10.0, w_max=0.3, range_noise=0.01,
                    prior_vel_sigma=0.05),
    # configs[3] "synthetic 64-ring (64x1024) dense scan"
    "config4": dict(lidar=1, world=0, fixed_motion=0, stress_queries=0, v_max=10.0, w_max=0.3, range_noise=0.01,
                    prior_vel_sigma=0.05),
}


def _copy(ptr, n, dtype):
    if n == 0:
        return np.zeros(0, dtype)
    buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=n).copy()


def generate(config="config3", n=1, seed0=1, threads=None, **overrides):
    """n independent units, seeds seed0..seed0+n-1."""
    L = lib()
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    threads = threads or min(os.cpu_count() or 1, 32)
    h = L.lins_synth_batch_create(C.byref(cfg), seed0, n, threads)
    try:
        d = LinsBatchDesc()
        L.lins_synth_batch_desc(h, C.byref(d))
        clouds, offsets = {}, {}
        for k in Batch.FIELDS:
            off = _copy(getattr(d, k + "_off"), n + 1, np.int32)
            offsets[k] = off
            clouds[k] = _copy(getattr(d, k), int(off[-1]), POINT_DTYPE)
        state = _copy(d.state_in, n * 19, np.float64)
        cov = _copy(d.cov_in, n * 324, np.float64)
        truth = np.ctypeslib.as_array(L.lins_synth_batch_truth(h), shape=(n * 7,)).copy()
        extra = {}
        for which, name in ((0, "new_surf_less_flat"), (1, "new_corner_less_sharp")):
            p, o = C.c_void_p(), C.c_void_p()
            L.lins_synth_batch_new_less(h, which, C.byref(p), C.byref(o))
            off = _copy(o.value, n + 1, np.int32)
            extra[name] = _copy(p.value, int(off[-1]), POINT_DTYPE)
            extra[name + "_off"] = off
        return Batch(clouds, offsets, state, cov, truth, extra)
    finally:
        L.lins_synth_batch_destroy(h)


# ---- offline sequence driver (tools/synth/lins_sequence.cpp): the C++ StateEstimator shim on a synthetic drive ----
_SEQ = None


def seq_lib():
    global _SEQ
    if _SEQ is None:
        path = os.path.join(_DIR, "liblins_seq.so")
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", _DIR, "seq"])
        L = C.CDLL(path)
        L.lins_seq_run.restype = C.c_void_p
        L.lins_seq_run.argtypes = [C.POINTER(SynthCfg), C.c_uint64, C.c_int, C.c_int]
        L.lins_seq_destroy.argtypes = [C.c_void_p]
        L.lins_seq_num_units.argtypes = [C.c_void_p]
        L.lins_seq_num_scans.argtypes = [C.c_void_p]
        L.lins_seq_desc.argtypes = [C.c_void_p, C.POINTER(LinsBatchDesc)]
        L.lins_seq_array.restype = C.POINTER(C.c_double)
        L.lins_seq_array.argtypes = [C.c_void_p, C.c_int]
        L.lins_seq_ints.restype = C.POINTER(C.c_int32)
        L.lins_seq_ints.argtypes = [C.c_void_p, C.c_int]
        L.lins_seq_write_bag.argtypes = [C.POINTER(SynthCfg), C.c_uint64, C.c_int, C.c_char_p, C.c_char_p, C.c_char_p]
        L.lins_seq_run_bag.restype = C.c_void_p
        L.lins_seq_run_bag.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.lins_seq_write_bag_period.argtypes = [C.POINTER(SynthCfg), C.c_uint64, C.c_int, C.c_char_p, C.c_char_p, C.c_char_p, C.c_double]
        L.lins_seq_run_bag_rig.restype = C.c_void_p
        L.lins_seq_run_bag_rig.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int)]
        L.lins_seq_run_bag_tuned.restype = C.c_void_p
        L.lins_seq_run_bag_tuned.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
        L.lins_host_align_imu.argtypes = [C.c_double, C.c_void_p, C.c_void_p]
        L.lins_seq_map_count.argtypes = [C.c_void_p]
        L.lins_seq_map_array.restype = C.POINTER(C.c_double)
        L.lins_seq_map_array.argtypes = [C.c_void_p, C.c_int]
        L.lins_seq_map_cloud.restype = C.c_void_p
        L.lins_seq_map_cloud.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        _SEQ = L
    return _SEQ


def _seq_record(L, h):
    n, ns = L.lins_seq_num_units(h), L.lins_seq_num_scans(h)
    d = LinsBatchDesc()
    L.lins_seq_desc(h, C.byref(d))
    clouds, offsets = {}, {}
    for k in Batch.FIELDS:
        off = _copy(getattr(d, k + "_off"), n + 1, np.int32)
        offsets[k] = off
        clouds[k] = _copy(getattr(d, k), int(off[-1]), POINT_DTYPE)
    arr = lambda which, cnt: np.ctypeslib.as_array(L.lins_seq_array(h, which), shape=(cnt,)).copy() if cnt else np.zeros(0)  # noqa: E731
    ints = lambda which, cnt: np.ctypeslib.as_array(L.lins_seq_ints(h, which), shape=(cnt,)).copy() if cnt else np.zeros(0, np.int32)  # noqa: E731
    units = Batch(clouds, offsets, _copy(d.state_in, n * 19, np.float64), _copy(d.cov_in, n * 324, np.float64), arr(1, n * 7)) if n else None
    return dict(units=units, state_out=arr(0, n * 19).reshape(-1, 19), iters=ints(0, n), flags=ints(1, n), scan_index=ints(2, n),
                status=ints(3, ns), global_est=arr(2, ns * 7).reshape(-1, 7), global_true=arr(3, ns * 7).reshape(-1, 7),
                map_inputs=_map_inputs(L, h))


def _map_inputs(L, h):
    """What the estimator published for the mapping node after each scan (LinsFusion::publishTopics): per published scan
    the stamp, the odometry (YZX position + quaternion x, y, z, w of globalStateYZX_) and the YZX less-sharp, less-flat and
    outlier clouds."""
    m = L.lins_seq_map_count(h)
    time = _copy(C.cast(L.lins_seq_map_array(h, 0), C.c_void_p).value, m, np.float64)
    odom = _copy(C.cast(L.lins_seq_map_array(h, 1), C.c_void_p).value, 7 * m, np.float64).reshape(-1, 7)
    clouds = []
    for which in range(3):
        o = C.c_void_p()
        p = L.lins_seq_map_cloud(h, which, C.byref(o))
        off = _copy(o.value, m + 1, np.int32)
        pts = _copy(p, int(off[-1]), POINT_DTYPE)
        clouds.append([pts[off[k]:off[k + 1]] for k in range(m)])
    return [dict(time=float(time[k]), quat=odom[k, 3:], pos=odom[k, :3], corner=clouds[0][k], surf=clouds[1][k], outlier=clouds[2][k])
            for k in range(m)]


def write_sequence_bag(path, config="config3", seed=1, n_scans=12, lidar_topic="/velodyne_points", imu_topic="/imu/data", scan_period=None,
                       **overrides):
    """The synthetic drive of run_sequence written as a ROS1 bag (raw sweeps + IMU): no GPU needed.  scan_period: the
    sweep's duration in seconds (None: the lidar's 0.1 s); the IMU keeps 40 samples per sweep."""
    L = seq_lib()
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    rc = L.lins_seq_write_bag_period(C.byref(cfg), seed, n_scans, path.encode(), lidar_topic.encode(), imu_topic.encode(),
                                     float(scan_period or 0.0))
    if rc != 0:
        raise RuntimeError(f"lins_seq_write_bag failed with {rc}")


RIG_ORDER = ("scan_period", "edge_threshold", "surf_threshold", "imu_lidar_extrinsic_angle", "acc_n", "gyr_n", "acc_w", "gyr_w",
             "init_pos_std", "init_vel_std", "init_att_std", "init_acc_std", "init_gyr_std", "init_ba", "init_bw")


def rig_array(rig):
    """A rig dict (rig_config.RIG_KEYS: scalars and 3-vectors) as the 29 doubles lins_seq_run_bag_rig takes."""
    return np.array([v for k in RIG_ORDER for v in np.atleast_1d(np.asarray(rig[k], np.float64))], np.float64)


TUNING_ORDER = ("num_iter", "icp_freq", "nearest_feature_search_sq_dist", "lidar_std", "lidar_scale", "imu_misalign_angle")


def run_bag(path, lidar_topic="/velodyne_points", imu_topic="/imu/data", max_scans=0, lidar_model=0, device=0, rig=None, tuning=None):
    """BASELINE.json configs[1] runner: replay a ROS1 bag (sensor_msgs/PointCloud2 + sensor_msgs/Imu) through image
    projection, feature extraction and the GPU IESKF update, the way LinsFusion does (Estimator.cpp:123-284).  rig: the
    robot's exp_port.yaml values (a dict as rig_config.load_rig returns) for the StateEstimator's EstimatorParams; None =
    the shipped values with zero INIT_BA / INIT_BW.  tuning: the estimator's tuning and IMU misalignment (a dict as
    rig_config.load_config returns): EstimatorParams::gpu takes the tuning, and every IMU sample is rotated by
    alignIMUtoVehicle as imuCallback does; None = the shipped tuning and no rotation."""
    L = seq_lib()
    err = C.c_int(0)
    r = rig_array(rig) if rig is not None else None
    if r is not None and len(r) != 29:
        raise ValueError(f"a rig has 29 values, got {len(r)}")
    t = np.array([float(tuning[k]) for k in TUNING_ORDER], np.float64) if tuning is not None else None
    h = L.lins_seq_run_bag_tuned(path.encode(), lidar_topic.encode(), imu_topic.encode(), max_scans, lidar_model, device,
                                 None if r is None else r.ctypes.data, None if t is None else t.ctypes.data, C.byref(err))
    if not h:
        raise RuntimeError(f"lins_seq_run_bag failed with {err.value}")
    try:
        return _seq_record(L, h)
    finally:
        L.lins_seq_destroy(h)


def host_align_imu(angle, v):
    """The shim's alignIMUtoVehicle of one 3-vector (lins_host_align_imu): R^T v, R = rpy2R((0, 0, deg2rad(angle)))."""
    a = np.ascontiguousarray(v, np.float64)
    out = np.zeros(3)
    seq_lib().lins_host_align_imu(float(angle), a.ctypes.data, out.ctypes.data)
    return out


def run_sequence(config="config3", seed=1, n_scans=12, device=0, **overrides):
    """Drive fusion::StateEstimator (GPU hot path) over a synthetic sequence.  Returns the recorded performIESKF
    units as a Batch plus the shim's outputs."""
    L = seq_lib()
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    h = L.lins_seq_run(C.byref(cfg), seed, n_scans, device)
    try:
        return _seq_record(L, h)
    finally:
        L.lins_seq_destroy(h)


# ---- feature logs (tools/synth/lins_sequence.cpp): per scan the IMU calls and the four feature clouds ----------------
class FeatureLogDesc(C.Structure):
    _fields_ = [("n_scans", C.c_int32), ("time", C.c_void_p), ("imu", C.c_void_p), ("imu_off", C.c_void_p),
                ("imu_last", C.c_void_p), ("clouds", C.c_void_p * 4), ("offs", C.c_void_p * 4)]


def _flog_lib():
    L = seq_lib()
    if not hasattr(L, "_flog"):
        L.lins_flog_create.restype = C.c_void_p
        L.lins_flog_create.argtypes = [C.POINTER(SynthCfg), C.c_uint64, C.c_int]
        L.lins_flog_destroy.argtypes = [C.c_void_p]
        L.lins_flog_desc.argtypes = [C.c_void_p, C.POINTER(FeatureLogDesc)]
        L.lins_flog_replay.restype = C.c_void_p
        L.lins_flog_replay.argtypes = [C.POINTER(FeatureLogDesc), C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.lins_host_predict.argtypes = [C.c_void_p] * 4 + [C.c_int]
        L.lins_replay_destroy.argtypes = [C.c_void_p]
        L.lins_replay_handover.argtypes = [C.c_void_p]
        L.lins_replay_ints.restype = C.POINTER(C.c_int32)
        L.lins_replay_ints.argtypes = [C.c_void_p, C.c_int]
        L.lins_replay_doubles.restype = C.POINTER(C.c_double)
        L.lins_replay_doubles.argtypes = [C.c_void_p, C.c_int]
        L.lins_replay_handover_cloud.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L._flog = True
    return L


def feature_log(config="config3", seed=1, n_scans=12, **overrides):
    """A simulated drive through the front end only (image projection + feature extraction; no GPU): dict with time (n),
    imu (k x 7: dt, acc, gyr) + imu_off (n + 1), imu_last (n x 6) and the four feature clouds (Batch.FIELDS) with their
    offsets (<name>_off).  Edit it freely, then replay it with replay_feature_log or sequence mode."""
    L = _flog_lib()
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    h = L.lins_flog_create(C.byref(cfg), seed, n_scans)
    try:
        d = FeatureLogDesc()
        L.lins_flog_desc(h, C.byref(d))
        n = d.n_scans
        log = dict(lidar=kw["lidar"], time=_copy(d.time, n, np.float64), imu_off=_copy(d.imu_off, n + 1, np.int32),
                   imu_last=_copy(d.imu_last, n * 6, np.float64).reshape(n, 6))
        log["imu"] = _copy(d.imu, int(log["imu_off"][-1]) * 7, np.float64).reshape(-1, 7)
        for j, k in enumerate(Batch.FIELDS):
            log[k + "_off"] = _copy(d.offs[j], n + 1, np.int32)
            log[k] = _copy(d.clouds[j], int(log[k + "_off"][-1]), POINT_DTYPE)
        return log
    finally:
        L.lins_flog_destroy(h)


def log_scan(log, k):
    """Scan k of a feature log: its IMU rows and its four clouds."""
    o = log["imu_off"]
    out = dict(imu=log["imu"][o[k]:o[k + 1]], imu_last=log["imu_last"][k], time=log["time"][k])
    for f in Batch.FIELDS:
        out[f] = log[f][log[f + "_off"][k]:log[f + "_off"][k + 1]]
    return out


def make_log(scans, lidar=0):
    """Reassemble a feature log from a list of log_scan dicts (the way tests edit one)."""
    log = dict(lidar=lidar, time=np.array([s["time"] for s in scans], np.float64), imu_last=np.array([s["imu_last"] for s in scans], np.float64).reshape(-1, 6))
    log["imu"] = np.ascontiguousarray(np.concatenate([np.asarray(s["imu"], np.float64).reshape(-1, 7) for s in scans]))
    log["imu_off"] = np.concatenate([[0], np.cumsum([len(s["imu"]) for s in scans])]).astype(np.int32)
    for f in Batch.FIELDS:
        log[f] = np.ascontiguousarray(np.concatenate([s[f] for s in scans])) if scans else np.zeros(0, POINT_DTYPE)
        log[f + "_off"] = np.concatenate([[0], np.cumsum([len(s[f]) for s in scans])]).astype(np.int32)
    return log


def replay_feature_log(log, device=0, params=None, init_std=None):
    """Replay a feature log through one C++ StateEstimator shim (processImu + processFeatures per scan).  Returns per scan
    code (LINS_SEQ_*: 0 before the hand-over), iters, flags, map_replaced, est_status, global_state / filter_state /
    lin_state (n x 19) and filter_cov (n x 324) after the scan, plus `handover`: the scan index after which the shim first
    ran and its state then, as lins_gpu_seq_begin takes it.  init_code: the code an opened sequence-mode slot gets for
    the scan (LINS_SEQ_INIT_WAIT / FIRST / SECOND while initialising, else code); icp_pose (n x 7: t, q xyzw), icp_iters,
    icp_converged: the second scan's estimateTransform result where init_code is LINS_SEQ_SECOND, else zero.  params: the shim context's LinsParams (None = shipped);
    init_std: INIT_POS_STD (3) + INIT_ATT_STD (3, degrees) of its filter (None = zero).  scan_s: wall seconds per scan."""
    L = _flog_lib()
    n = len(log["time"])
    keep = {k: np.ascontiguousarray(log[k]) for k in ("time", "imu", "imu_off", "imu_last")}
    d = FeatureLogDesc()
    d.n_scans = n
    for k, v in keep.items():
        setattr(d, k, v.ctypes.data)
    for j, k in enumerate(Batch.FIELDS):
        keep[k], keep[k + "_off"] = np.ascontiguousarray(log[k]), np.ascontiguousarray(log[k + "_off"], dtype=np.int32)
        d.clouds[j], d.offs[j] = keep[k].ctypes.data, keep[k + "_off"].ctypes.data
    std = None if init_std is None else np.ascontiguousarray(init_std, dtype=np.float64)
    h = L.lins_flog_replay(C.byref(d), int(log.get("lidar", 0)), device, C.cast(C.byref(params), C.c_void_p) if params is not None else None,
                           None if std is None else std.ctypes.data)
    return _replay_record(L, h, n)


def _replay_record(L, h, n):
    """Read (and free) a replay record of lins_flog_replay / lins_plog_replay."""
    try:
        ints = lambda w: np.ctypeslib.as_array(L.lins_replay_ints(h, w), shape=(n,)).copy()  # noqa: E731
        dbl = lambda w, cnt: np.ctypeslib.as_array(L.lins_replay_doubles(h, w), shape=(cnt,)).copy()  # noqa: E731
        rec = dict(code=ints(0), iters=ints(1), flags=ints(2), map_replaced=ints(3), est_status=ints(4),
                   global_state=dbl(0, n * 19).reshape(n, 19), filter_state=dbl(1, n * 19).reshape(n, 19),
                   filter_cov=dbl(2, n * 324).reshape(n, 324), lin_state=dbl(3, n * 19).reshape(n, 19), scan_s=dbl(8, n),
                   init_code=ints(5), icp_pose=dbl(9, n * 7).reshape(n, 7), icp_iters=ints(6), icp_converged=ints(7))
        k = L.lins_replay_handover(h)
        rec["handover_index"] = k
        if k >= 0:
            ho = dict(filter_state=dbl(4, 19), global_state=dbl(5, 19), filter_cov=dbl(6, 324), imu_last=dbl(7, 6))
            for which, name in ((0, "surf_map"), (1, "corner_map")):
                p = C.c_void_p()
                cnt = L.lins_replay_handover_cloud(h, which, C.byref(p))
                ho[name] = _copy(p.value, cnt, POINT_DTYPE)
            rec["handover"] = ho
        return rec
    finally:
        L.lins_replay_destroy(h)


# ---- pcl logs: the same drives as processPCL receives them (segmented cloud + cloud_info per scan) ---------------------
class PclLogDesc(C.Structure):
    _fields_ = [("n_scans", C.c_int32), ("time", C.c_void_p), ("imu", C.c_void_p), ("imu_off", C.c_void_p),
                ("imu_last", C.c_void_p), ("pcl", LinsPclDesc)]


def _plog_lib():
    L = _flog_lib()
    if not hasattr(L, "_plog"):
        L.lins_plog_desc.argtypes = [C.c_void_p, C.POINTER(PclLogDesc)]
        L.lins_plog_replay.restype = C.c_void_p
        L.lins_plog_replay.argtypes = [C.POINTER(PclLogDesc), C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L._plog = True
    return L


def pcl_log(config="config3", seed=1, n_scans=12, **overrides):
    """The drive of feature_log(config, seed, n_scans) as processPCL receives it: dict with lidar, line_num, time, imu +
    imu_off, imu_last (as in a feature log) and scans: one dict per scan with seg (m x 4 float32 x, y, z, intensity), ground,
    col, range, start_ring / end_ring (line_num) and ori (start, end, diff).  Edit the scans freely, then replay the log
    with replay_pcl_log or sequence mode (LinsGpu.seq_step_pcl)."""
    L = _plog_lib()
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    h = L.lins_flog_create(C.byref(cfg), seed, n_scans)
    try:
        d = PclLogDesc()
        L.lins_plog_desc(h, C.byref(d))
        n, p = d.n_scans, d.pcl
        ln = p.line_num
        log = dict(lidar=kw["lidar"], line_num=ln, time=_copy(d.time, n, np.float64), imu_off=_copy(d.imu_off, n + 1, np.int32),
                   imu_last=_copy(d.imu_last, n * 6, np.float64).reshape(n, 6))
        log["imu"] = _copy(d.imu, int(log["imu_off"][-1]) * 7, np.float64).reshape(-1, 7)
        off = _copy(p.cloud_off, n + 1, np.int32)
        tot = int(off[-1])
        pts = _copy(p.cloud, tot, POINT_DTYPE)
        xyzi = np.stack([pts["x"], pts["y"], pts["z"], pts["intensity"]], 1).astype(np.float32)
        ground, col, rng = _copy(p.ground_flag, tot, np.uint8), _copy(p.col_ind, tot, np.uint32), _copy(p.range, tot, np.float32)
        sr, er = _copy(p.start_ring_index, n * ln, np.int32).reshape(n, ln), _copy(p.end_ring_index, n * ln, np.int32).reshape(n, ln)
        ori = _copy(p.orientation, n * 3, np.float32).reshape(n, 3)
        log["scans"] = [dict(seg=xyzi[off[k]:off[k + 1]].copy(), ground=ground[off[k]:off[k + 1]].copy(), col=col[off[k]:off[k + 1]].copy(),
                             range=rng[off[k]:off[k + 1]].copy(), start_ring=sr[k].copy(), end_ring=er[k].copy(), ori=ori[k].copy()) for k in range(n)]
        return log
    finally:
        L.lins_flog_destroy(h)


def raw_log(config="config3", seed=1, n_scans=12, **overrides):
    """The drive of feature_log(config, seed, n_scans) as the LiDAR driver publishes it: dict with lidar, line_num, time,
    imu + imu_off, imu_last (as in a feature log) and sweeps: one raw sweep per scan (m x 4 float32 x, y, z, intensity,
    firing order).  Run through sequence mode with LinsGpu.seq_step_raw; the host reference projects each sweep (after
    dropping its non-finite points) into a pcl log for replay_pcl_log."""
    L = _plog_lib()
    if not hasattr(L, "_rlog"):
        L.lins_flog_raw.argtypes = [C.c_void_p, C.c_void_p]
        L._rlog = True
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    h = L.lins_flog_create(C.byref(cfg), seed, n_scans)
    try:
        d = PclLogDesc()
        L.lins_plog_desc(h, C.byref(d))
        r = LinsRawDesc()
        L.lins_flog_raw(h, C.byref(r))
        n = d.n_scans
        log = dict(lidar=kw["lidar"], line_num=d.pcl.line_num, time=_copy(d.time, n, np.float64), imu_off=_copy(d.imu_off, n + 1, np.int32),
                   imu_last=_copy(d.imu_last, n * 6, np.float64).reshape(n, 6))
        log["imu"] = _copy(d.imu, int(log["imu_off"][-1]) * 7, np.float64).reshape(-1, 7)
        off = _copy(r.cloud_off, n + 1, np.int32)
        pts = _copy(r.cloud, int(off[-1]), POINT_DTYPE)
        xyzi = np.stack([pts["x"], pts["y"], pts["z"], pts["intensity"]], 1).astype(np.float32)
        log["sweeps"] = [xyzi[off[k]:off[k + 1]].copy() for k in range(n)]
        return log
    finally:
        L.lins_flog_destroy(h)


def replay_pcl_log(log, device=0, params=None, init_std=None):
    """Replay a pcl log through one C++ StateEstimator shim: processImu for every IMU row, then processPCL with the scan's
    segmented cloud and cloud_info (the shim's host FeatureExtractor runs).  The record of replay_feature_log."""
    L = _plog_lib()
    n = len(log["time"])
    scans = log["scans"]
    keep = {k: np.ascontiguousarray(log[k]) for k in ("time", "imu", "imu_off", "imu_last")}
    d = PclLogDesc()
    d.n_scans = n
    for k, v in keep.items():
        setattr(d, k, v.ctypes.data)
    off = np.concatenate([[0], np.cumsum([len(s["seg"]) for s in scans])]).astype(np.int32)
    pts = np.zeros(max(int(off[-1]), 1), POINT_DTYPE)
    xyzi = np.concatenate([np.asarray(s["seg"], np.float32).reshape(-1, 4) for s in scans])
    pts["x"][:len(xyzi)], pts["y"][:len(xyzi)], pts["z"][:len(xyzi)], pts["intensity"][:len(xyzi)] = xyzi.T
    pts["pad0"] = 1.0
    cat = lambda k, t: np.ascontiguousarray(np.concatenate([np.asarray(s[k], t).reshape(-1) for s in scans] + [np.zeros(1, t)]))  # noqa: E731
    keep.update(cloud=pts, cloud_off=off, ground=cat("ground", np.uint8), col=cat("col", np.uint32), range=cat("range", np.float32),
                sr=cat("start_ring", np.int32), er=cat("end_ring", np.int32), ori=cat("ori", np.float32))
    p = d.pcl
    p.n_scans, p.line_num, p.point_format = n, int(log["line_num"]), 0
    p.cloud, p.cloud_off, p.ground_flag, p.col_ind, p.range = (keep[k].ctypes.data for k in ("cloud", "cloud_off", "ground", "col", "range"))
    p.start_ring_index, p.end_ring_index, p.orientation = keep["sr"].ctypes.data, keep["er"].ctypes.data, keep["ori"].ctypes.data
    d.pcl = p
    std = None if init_std is None else np.ascontiguousarray(init_std, dtype=np.float64)
    h = L.lins_plog_replay(C.byref(d), int(log.get("lidar", 0)), device, C.cast(C.byref(params), C.c_void_p) if params is not None else None,
                           None if std is None else std.ctypes.data)
    return _replay_record(L, h, n)


def host_predict(state, cov, imu_last, rows):
    """kalman_filter.hpp StatePredictor::predict over `rows` (k x 7) from (state, cov, imu_last): returns the three after."""
    L = _flog_lib()
    s, c, i = (np.array(a, np.float64).ravel().copy() for a in (state, cov, imu_last))
    r = np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, 7)
    L.lins_host_predict(s.ctypes.data, c.ctypes.data, i.ctypes.data, r.ctypes.data, len(r))
    return s, c, i


# ---- row F2: scan-to-map units (tools/synth/lins_synth.cpp: lins_synth_map_unit_create) -------------------------------
class MapUnit:
    """One scan2MapOptimization input: map clouds, the newest scan's (down-sampled) features, true / guessed transform."""

    def __init__(self, corner_map, surf_map, corner_last, surf_last, truth, guess):
        self.corner_map, self.surf_map, self.corner_last, self.surf_last = corner_map, surf_map, corner_last, surf_last
        self.truth, self.guess = truth, guess


def generate_map_unit(config="config3", seed=1, n_keyframes=20, sigma_t=0.1, sigma_r=0.01, **overrides):
    L = lib()
    L.lins_synth_map_unit_create.restype = C.c_void_p
    L.lins_synth_map_unit_create.argtypes = [C.POINTER(SynthCfg), C.c_uint64, C.c_int, C.c_double, C.c_double]
    L.lins_synth_map_unit_destroy.argtypes = [C.c_void_p]
    L.lins_synth_map_unit_cloud.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.lins_synth_map_unit_transforms.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    h = L.lins_synth_map_unit_create(C.byref(cfg), seed, n_keyframes, sigma_t, sigma_r)
    try:
        clouds = []
        for which in range(4):
            p = C.c_void_p()
            n = L.lins_synth_map_unit_cloud(h, which, C.byref(p))
            clouds.append(_copy(p.value, n, POINT_DTYPE))
        truth, guess = np.zeros(6, np.float32), np.zeros(6, np.float32)
        L.lins_synth_map_unit_transforms(h, truth.ctypes.data_as(C.c_void_p), guess.ctypes.data_as(C.c_void_p))
        return MapUnit(*clouds, truth, guess)
    finally:
        L.lins_synth_map_unit_destroy(h)


# ---- the mapping node's input along a drive (tools/synth/lins_synth.cpp: lins_synth_map_drive_create) ----------------
def generate_map_drive(poses_xyzyaw, config="config3", seed=1, **overrides):
    """One sweep at each sensor pose (rows x, y, z, yaw in the world) through the product's CPU front end: per scan the YZX
    less-sharp corners, less-flat surfs and outliers the estimator publishes, and the true pose as the mapping node's
    transform (rx, ry, rz, tx, ty, tz).  Returns (list of (corner, surf, outlier) POINT_DTYPE triples, truth (n, 6) f32)."""
    L = lib()
    L.lins_synth_map_drive_create.restype = C.c_void_p
    L.lins_synth_map_drive_create.argtypes = [C.POINTER(SynthCfg), C.c_uint64, C.c_int, C.c_void_p]
    L.lins_synth_map_drive_destroy.argtypes = [C.c_void_p]
    L.lins_synth_map_drive_cloud.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    L.lins_synth_map_drive_truth.argtypes = [C.c_void_p, C.c_void_p]
    kw = dict(CONFIGS[config])
    kw.update(overrides)
    cfg = SynthCfg(**kw)
    P = np.ascontiguousarray(poses_xyzyaw, np.float64).reshape(-1, 4)
    h = L.lins_synth_map_drive_create(C.byref(cfg), seed, len(P), P.ctypes.data_as(C.c_void_p))
    try:
        scans = []
        for k in range(len(P)):
            trip = []
            for which in range(3):
                p = C.c_void_p()
                n = L.lins_synth_map_drive_cloud(h, k, which, C.byref(p))
                trip.append(_copy(p.value, n, POINT_DTYPE))
            scans.append(tuple(trip))
        truth = np.zeros((len(P), 6), np.float32)
        L.lins_synth_map_drive_truth(h, truth.ctypes.data_as(C.c_void_p))
        return scans, truth
    finally:
        L.lins_synth_map_drive_destroy(h)
