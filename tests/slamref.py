"""A numpy restatement of LinsFusion::publishTopics as sequence mode's publish step runs it — TEST INFRASTRUCTURE.

publishes(): performStateEstimation publishes after every scan of an estimator that was initialised before the scan
(Estimator.cpp:254-284).  yzx_pose(): globalStateYZX_ of updatePointCloud (StateEstimator.hpp:1116-1161), Q * rn and
Q * qbn * Q^-1 with Q = Q_xyz_to_yzx, in f64 in the order of the Eigen expressions.  Publisher: per slot what scan_last_
holds (the YZX clouds and pose, written only by updatePointCloud; a first scan swaps in a scan that never ran it), so a
test can drive the host composition of the publish step: download the maps and state, apply the rule, feed the mappers.
"""
import numpy as np

FUSION_INIT, FUSION_FIRST_SCAN, FUSION_RUNNING = 0, 1, 3
IDLE, SKIPPED, RAN, ICP, INIT_WAIT, FIRST, SECOND = 0, 1, 2, 3, 4, 5, 6
ACCEPTED = (SECOND, RAN, ICP)
Q_XYZ_TO_YZX = np.array([0.5, 0.5, 0.5, -0.5])  # x y z w: R2Quat of the permutation (y, z, x) <- (x, y, z)


def publishes(fusion_before, code):
    return code != IDLE and fusion_before != FUSION_INIT


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _qmul(a, b):  # x y z w, Eigen's term order
    x = a[..., 3] * b[..., 0] + a[..., 0] * b[..., 3] + a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1]
    y = a[..., 3] * b[..., 1] + a[..., 1] * b[..., 3] + a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2]
    z = a[..., 3] * b[..., 2] + a[..., 2] * b[..., 3] + a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]
    w = a[..., 3] * b[..., 3] - a[..., 0] * b[..., 0] - a[..., 1] * b[..., 1] - a[..., 2] * b[..., 2]
    return np.stack([x, y, z, w], -1)


def yzx_pose(rn, qbn):
    """(..., 3) positions and (..., 4) quaternions x y z w -> (..., 7): YZX position, quaternion x y z w."""
    rn, qbn = np.asarray(rn, np.float64), np.asarray(qbn, np.float64)
    q = np.broadcast_to(Q_XYZ_TO_YZX, qbn.shape)
    qv = q[..., :3]
    t = _cross(qv, rn) * 2.0
    pos = (rn + t * q[..., 3:4]) + _cross(qv, t)
    n = (((q[..., 0] * q[..., 0] + q[..., 1] * q[..., 1]) + q[..., 2] * q[..., 2]) + q[..., 3] * q[..., 3])[..., None]
    qi = np.concatenate([-qv / n, q[..., 3:4] / n], -1)
    return np.concatenate([pos, _qmul(_qmul(q, qbn), qi)], -1)


def to_yzx(xyzi):
    """(n, 4) x y z intensity -> (n, 4) y z x intensity."""
    a = np.asarray(xyzi, np.float32).reshape(-1, 4)
    return np.ascontiguousarray(a[:, [1, 2, 0, 3]])


EMPTY = np.zeros((0, 4), np.float32)


class Publisher:
    """scan_last_'s YZX clouds and globalStateYZX_ of n slots' estimators (fresh: no clouds, the identity pose)."""

    def __init__(self, n):
        self.clouds = [(EMPTY, EMPTY, EMPTY)] * n
        self.pose = [np.array([0.0, 0, 0, 0, 0, 0, 1])] * n

    def restart(self, s):
        self.clouds[s] = (EMPTY, EMPTY, EMPTY)
        self.pose[s] = np.array([0.0, 0, 0, 0, 0, 0, 1])

    def step(self, s, fusion_before, code, global_state=None, corner=None, surf=None, outlier=None):
        """One scan of slot s (code: LINS_SEQ_*; for an accepted scan its global state row (19) and the XYZ less-sharp,
        less-flat (the new maps) and outlier clouds as (n, 4) arrays).  Returns (pose (7), corner, surf, outlier) when
        the slot publishes, else None."""
        if code == FIRST:
            self.clouds[s] = (EMPTY, EMPTY, EMPTY)
        elif code in ACCEPTED:
            self.clouds[s] = (to_yzx(corner), to_yzx(surf), to_yzx(outlier))
            g = np.asarray(global_state, np.float64)
            self.pose[s] = yzx_pose(g[0:3], g[6:10])
        if not publishes(fusion_before, code):
            return None
        return (self.pose[s].copy(),) + self.clouds[s]
