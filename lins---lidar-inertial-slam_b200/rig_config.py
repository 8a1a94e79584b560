"""A robot's LINS configuration (exp_port.yaml, OpenCV's YAML format) as sequence mode takes it.

LINS reads its parameters with cv::FileStorage: a `%YAML:1.0` file of `key: value` lines and `!!opencv-matrix` blocks
(rows, cols, dt, data: [...]).  read_opencv_yaml parses that subset.  load_rig splits a file into the values that
describe one recording's sensors (RIG_KEYS: they go into a slot's lins_slot_config) and the estimator's tuning
(SHARED_KEYS: the context's lins_params); it reads imu_misalign_angle but does not apply it.  load_config splits a file into
the rig and the tuning (TUNING_KEYS: SHARED_KEYS and imu_misalign_angle), which a slot takes with lins_gpu_seq_tune: its
own tuning, and alignIMUtoVehicle (Estimator.cpp:124-135, 286-292) on its IMU values.  misalign_R / align_imu restate that
rotation on the host, in the same f64 expression the library and the shim evaluate.
"""
import math
import re
import warnings

from .ctypes_defs import LinsParams, LinsSlotConfig, LinsSlotTuning

SCALAR_RIG = ("scan_period", "edge_threshold", "surf_threshold", "imu_lidar_extrinsic_angle", "acc_n", "gyr_n", "acc_w", "gyr_w")
VECTOR_RIG = ("init_pos_std", "init_vel_std", "init_att_std", "init_acc_std", "init_gyr_std", "init_ba", "init_bw")
RIG_KEYS = SCALAR_RIG + VECTOR_RIG
SHARED_KEYS = ("num_iter", "icp_freq", "nearest_feature_search_sq_dist", "lidar_std", "lidar_scale")
TUNING_KEYS = SHARED_KEYS + ("imu_misalign_angle",)


def _scalar(text):
    t = text.strip()
    if len(t) >= 2 and t[0] == t[-1] == '"':
        return t[1:-1]
    try:
        return int(t)
    except ValueError:
        pass
    try:
        return float(t)
    except ValueError:
        return t


def read_opencv_yaml(path):
    """{key: value} of an OpenCV YAML file: numbers as int / float, quoted strings as str, matrices as a list of floats
    (row-major, rows * cols of them)."""
    with open(path) as f:
        lines = f.read().splitlines()
    if not lines or not lines[0].startswith("%YAML"):
        raise ValueError(f"{path}: not an OpenCV YAML file (no %YAML header)")
    out, i = {}, 1
    while i < len(lines):
        line = lines[i].split("#", 1)[0].rstrip()
        i += 1
        m = re.match(r"^([A-Za-z_]\w*)\s*:\s*(.*)$", line)
        if not m:
            continue
        key, rest = m.group(1), m.group(2).strip()
        if rest != "!!opencv-matrix":
            out[key] = _scalar(rest)
            continue
        fields = {}
        while i < len(lines) and (lines[i].startswith((" ", "\t")) or not lines[i].strip()):
            body = lines[i].split("#", 1)[0].strip()
            i += 1
            fm = re.match(r"^(\w+)\s*:\s*(.*)$", body)
            if not fm:
                continue
            name, val = fm.group(1), fm.group(2)
            if name == "data":
                while "]" not in val and i < len(lines):  # a data list may run over several lines
                    val += " " + lines[i].split("#", 1)[0].strip()
                    i += 1
                val = [float(v) for v in val.strip().strip("[]").replace(",", " ").split()]
            fields[name] = val
        try:
            rows, cols, data = int(fields["rows"]), int(fields["cols"]), fields["data"]
        except KeyError as e:
            raise ValueError(f"{path}: matrix {key} has no {e.args[0]}") from None
        if len(data) != rows * cols:
            raise ValueError(f"{path}: matrix {key} is {rows} x {cols} with {len(data)} values")
        out[key] = data
    return out


def _rig_of(y, path):
    rig = {}
    for k in SCALAR_RIG:
        rig[k] = float(y[k])
    for k in VECTOR_RIG:
        v = y[k]
        if not isinstance(v, list) or len(v) != 3:
            raise ValueError(f"{path}: {k} must be a 3 x 1 matrix")
        rig[k] = tuple(float(x) for x in v)
    return rig


def _read(path, keys):
    y = read_opencv_yaml(path)
    missing = [k for k in RIG_KEYS + keys if k not in y]
    if missing:
        raise ValueError(f"{path}: missing {', '.join(missing)}")
    return y, _rig_of(y, path)


def load_rig(path):
    """(rig, shared): rig = {RIG_KEYS: float or 3 floats}, shared = {SHARED_KEYS: number}.  A missing key is a
    ValueError; a non-zero imu_misalign_angle gives a warning, since it is not applied."""
    y, rig = _read(path, SHARED_KEYS)
    if float(y.get("imu_misalign_angle", 0.0)) != 0.0:
        warnings.warn(f"{path}: imu_misalign_angle = {y['imu_misalign_angle']} is not applied (alignIMUtoVehicle is not run)")
    shared = {k: y[k] for k in SHARED_KEYS}
    return rig, shared


def load_config(path):
    """(rig, tuning): rig as load_rig's, tuning = {TUNING_KEYS: number}: every value of the file the odometry reads.  A
    missing key (imu_misalign_angle included) is a ValueError."""
    y, rig = _read(path, TUNING_KEYS)
    tuning = {k: y[k] for k in TUNING_KEYS}
    for k in ("num_iter", "icp_freq"):
        if float(tuning[k]) != int(tuning[k]):
            raise ValueError(f"{path}: {k} must be an integer")
    return rig, tuning


def slot_tuning(tuning):
    """The LinsSlotTuning of a tuning (load_config's)."""
    return LinsSlotTuning.shipped(**{k: (int(tuning[k]) if k in ("num_iter", "icp_freq") else float(tuning[k])) for k in TUNING_KEYS})


def misalign_R(angle):
    """alignIMUtoVehicle's R = rpy2R((0, 0, deg2rad(angle))) = Rz Ry Rx (math_utils.h:164-182) as 3 rows, with Python's
    libm math.cos / math.sin and each product entry summed (a0 b0 + a1 b1) + a2 b2, as the library builds it."""
    y, p, r = angle * math.pi / 180.0, 0.0, 0.0
    Rz = ((math.cos(y), -math.sin(y), 0.0), (math.sin(y), math.cos(y), 0.0), (0.0, 0.0, 1.0))
    Ry = ((math.cos(p), 0.0, math.sin(p)), (0.0, 1.0, 0.0), (-math.sin(p), 0.0, math.cos(p)))
    Rx = ((1.0, 0.0, 0.0), (0.0, math.cos(r), -math.sin(r)), (0.0, math.sin(r), math.cos(r)))

    def mul(A, B):
        return tuple(tuple((A[i][0] * B[0][j] + A[i][1] * B[1][j]) + A[i][2] * B[2][j] for j in range(3)) for i in range(3))
    return mul(mul(Rz, Ry), Rx)


def align_imu(R, v):
    """R^T v of one IMU vector (alignIMUtoVehicle), out_j = (R_0j v_0 + R_1j v_1) + R_2j v_2 in f64."""
    x, y, z = (float(c) for c in v)
    return tuple((R[0][j] * x + R[1][j] * y) + R[2][j] * z for j in range(3))


def slot_config(rig):
    """The LinsSlotConfig of a rig (the IMU noise as StatePredictor::setNoise computes it from acc_n .. gyr_w)."""
    return LinsSlotConfig.shipped(**rig)


def lins_params(shared, scan_period=0.1):
    """The context's LinsParams from the shared keys (scan_period: the context's, read by unconfigured slots)."""
    return LinsParams.shipped(num_iter=int(shared["num_iter"]), icp_freq=int(shared["icp_freq"]),
                              nearest_feature_search_sq_dist=float(shared["nearest_feature_search_sq_dist"]),
                              lidar_std=float(shared["lidar_std"]), lidar_scale=float(shared["lidar_scale"]), scan_period=scan_period)
