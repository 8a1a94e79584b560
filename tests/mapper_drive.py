"""A synthetic drive for the mapping node's cycle: sensor poses out and back along a road of the seeded world, the
estimator's clouds at each pose (synth.generate_map_drive), odometry messages with a slow drift, IMU roll / pitch
messages, and the schedule the mapper tests need (interval skips, a stall in the cycle where the window first fills, an
empty and then a wrapped IMU queue, a return past the start more than 30 s later).  sparse_first > 0 thins the first
scans' clouds so that the map of their key frame fails the 10 / 100 gate.""" 
import math

import numpy as np

SCAN_PERIOD = 0.1


def set_rpy(roll, pitch, yaw):
    """tf::Quaternion::setRPY -> (x, y, z, w)."""
    hr, hp, hy = roll * 0.5, pitch * 0.5, yaw * 0.5
    cr, sr, cp, sp, cy, sy = math.cos(hr), math.sin(hr), math.cos(hp), math.sin(hp), math.cos(hy), math.sin(hy)
    return (sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy)


def odometry_quat(T):
    """The odometry orientation whose laserOdometryHandler conversion gives transformSum[0:3] = T[0:3]: the estimator
    publishes (-q.y, -q.z, q.x, q.w) of setRPY(T[2], -T[0], -T[1])."""
    qx, qy, qz, qw = set_rpy(float(T[2]), -float(T[0]), -float(T[1]))
    return (-qy, -qz, qx, qw)


def make_drive(synth, n_out=36, step=0.5, dt=0.5, seed=4, stall_at=50, sparse_first=0):
    """Returns a list of events: ("imu", t, roll, pitch) and ("odom", t, quat, pos, corner, surf, outlier, tag)."""
    xs = [-9.0 + step * k for k in range(n_out)] + [-9.0 + step * (n_out - 1 - k) - 0.25 for k in range(1, n_out)]
    poses = []
    for k, x in enumerate(xs):
        if k == stall_at:
            poses.append(poses[-1])  # no motion: no key frame in the cycle where the window first fills
        yaw = 0.0 if k < n_out else math.pi
        poses.append((x, 0.3 * math.sin(0.15 * k), 1.5, yaw))
    scans, truth = synth.generate_map_drive(np.array(poses), seed=seed)
    rng = np.random.default_rng(seed)
    events, t = [], 100.0
    drift = np.zeros(6)
    for k, (trip, T) in enumerate(zip(scans, truth)):
        corner, surf, outlier = trip
        if k < sparse_first:  # the first key frames' clouds: a map below the 10 / 100 gate
            corner, surf, outlier = corner[:6], surf[:40], outlier[:5]
        drift += np.array([2e-4, 5e-4, 1e-4, 0.01, 0.0, 0.005]) * rng.standard_normal(6)
        odo = T.astype(np.float64) + drift
        if k >= 20:  # the IMU starts late: the queue is empty for the first cycles
            n_imu = 30 if k % 3 else 12  # 60 Hz, and some cycles lag the scan
            horizon = t + (0.3 if k % 3 else -0.05)
            for j in range(n_imu):
                ti = horizon - (n_imu - 1 - j) / 60.0
                events.append(("imu", ti, float(T[2] + 1e-3 * rng.standard_normal()), float(T[0] + 1e-3 * rng.standard_normal())))
        events.append(("odom", t, odometry_quat(odo), (odo[3], odo[4], odo[5]), corner, surf, outlier, k))
        if k % 7 == 3:  # a message 0.1 s later: skipped by the 0.3 s interval
            events.append(("odom", t + SCAN_PERIOD, odometry_quat(odo), (odo[3], odo[4], odo[5]), corner, surf, outlier, -1))
        t += dt
    return events
