"""A robot's LINS configuration (exp_port.yaml, OpenCV's YAML format) as sequence mode takes it.

LINS reads its parameters with cv::FileStorage: a `%YAML:1.0` file of `key: value` lines and `!!opencv-matrix` blocks
(rows, cols, dt, data: [...]).  read_opencv_yaml parses that subset.  load_rig splits a file into the values that
describe one recording's sensors (RIG_KEYS: they go into a slot's lins_slot_config) and the estimator's tuning
(SHARED_KEYS: every slot of a context shares them, in its lins_params).  imu_misalign_angle is read but not applied:
neither bag_replay nor the shim's run_bag runs alignIMUtoVehicle (Estimator.cpp:124-135, 286-292).
"""
import re
import warnings

from .ctypes_defs import LinsParams, LinsSlotConfig

SCALAR_RIG = ("scan_period", "edge_threshold", "surf_threshold", "imu_lidar_extrinsic_angle", "acc_n", "gyr_n", "acc_w", "gyr_w")
VECTOR_RIG = ("init_pos_std", "init_vel_std", "init_att_std", "init_acc_std", "init_gyr_std", "init_ba", "init_bw")
RIG_KEYS = SCALAR_RIG + VECTOR_RIG
SHARED_KEYS = ("num_iter", "icp_freq", "nearest_feature_search_sq_dist", "lidar_std", "lidar_scale")


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


def load_rig(path):
    """(rig, shared): rig = {RIG_KEYS: float or 3 floats}, shared = {SHARED_KEYS: number}.  A missing key is a
    ValueError; a non-zero imu_misalign_angle gives a warning, since it is not applied."""
    y = read_opencv_yaml(path)
    missing = [k for k in RIG_KEYS + SHARED_KEYS if k not in y]
    if missing:
        raise ValueError(f"{path}: missing {', '.join(missing)}")
    rig = {}
    for k in SCALAR_RIG:
        rig[k] = float(y[k])
    for k in VECTOR_RIG:
        v = y[k]
        if not isinstance(v, list) or len(v) != 3:
            raise ValueError(f"{path}: {k} must be a 3 x 1 matrix")
        rig[k] = tuple(float(x) for x in v)
    if float(y.get("imu_misalign_angle", 0.0)) != 0.0:
        warnings.warn(f"{path}: imu_misalign_angle = {y['imu_misalign_angle']} is not applied (alignIMUtoVehicle is not run)")
    shared = {k: y[k] for k in SHARED_KEYS}
    return rig, shared


def slot_config(rig):
    """The LinsSlotConfig of a rig (the IMU noise as StatePredictor::setNoise computes it from acc_n .. gyr_w)."""
    return LinsSlotConfig.shipped(**rig)


def lins_params(shared, scan_period=0.1):
    """The context's LinsParams from the shared keys (scan_period: the context's, read by unconfigured slots)."""
    return LinsParams.shipped(num_iter=int(shared["num_iter"]), icp_freq=int(shared["icp_freq"]),
                              nearest_feature_search_sq_dist=float(shared["nearest_feature_search_sq_dist"]),
                              lidar_std=float(shared["lidar_std"]), lidar_scale=float(shared["lidar_scale"]), scan_period=scan_period)
