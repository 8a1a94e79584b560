"""CPU oracle of the mapping node's cycle (lidar_mapping_node.cpp run() :1806-1855 without loop closure): test
infrastructure, no product code.  The scan-to-map loop is the existing C++ oracle (oracle/lins_map_oracle.hpp through
oracle_binding.MapOracle); everything around it is restated here: its own pcl::VoxelGrid, the window of key-frame ids
(:1204-1246), transformPointCloud (:609-652), transformAssociateToMap (:411-536), transformUpdate (:538-577),
saveKeyFramesAndFactor (:1654-1765) with tf's getRPY and gtsam's Rot3::RzRyRx / xyz(), and detectLoopClosure's
candidate (:1043-1067).

f32 arithmetic is numpy float32 (IEEE, no contraction); sin / cos / asin / atan2 / sqrt of floats are libm's f32
functions, the overloads the reference's float arguments select."""
import collections
import ctypes
import ctypes.util
import math

import numpy as np

F = np.float32
WINDOW, LEAF_CORNER, LEAF_SURF, INTERVAL, KEY_DIST = 50, 0.2, 0.4, 0.3, 0.3
IMU_QUE = 200
INT32_MAX = (1 << 31) - 1

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
for _fn, _n in (("sinf", 1), ("cosf", 1), ("asinf", 1), ("sqrtf", 1), ("atan2f", 2)):
    getattr(_libm, _fn).restype = ctypes.c_float
    getattr(_libm, _fn).argtypes = [ctypes.c_float] * _n


def sinf(v): return F(_libm.sinf(float(F(v))))
def cosf(v): return F(_libm.cosf(float(F(v))))
def asinf(v): return F(_libm.asinf(float(F(v))))
def sqrtf(v): return F(_libm.sqrtf(float(F(v))))
def atan2f(y, x): return F(_libm.atan2f(float(F(y)), float(F(x))))


class TooBig(Exception):
    """div_x * div_y * div_z > INT32_MAX (PCL's 'Leaf size is too small' case), or a box bound floor(min / max * inv)
    at or beyond 2^62 in magnitude, inf included."""


def voxel_grid(pts, leaf):
    """pcl::VoxelGrid<PointXYZI>: (n, >=4) float32 rows (x, y, z, intensity) -> (m, 4) centroids.  Same semantics as
    tests/pyfront.voxel_grid (f32 sums in input order per voxel, ascending voxel index), vectorised by rank within the
    voxel so that 10^6 points stay fast: the k-th points of all voxels are added in one step, in order k = 0, 1, ..."""
    p = np.asarray(pts, F)
    if p.size == 0:
        return np.zeros((0, 4), F)
    p = p.reshape(len(p), -1)[:, :4]
    fin = np.isfinite(p[:, :3]).all(1)
    if not fin.any():
        return np.zeros((0, 4), F)
    inv = F(1.0) / F(leaf)
    q = p[fin]
    with np.errstate(over="ignore"):
        lo, hi = np.floor(q[:, :3].min(0) * inv), np.floor(q[:, :3].max(0) * inv)
    if not (np.abs(lo) < F(2.0 ** 62)).all() or not (np.abs(hi) < F(2.0 ** 62)).all():
        raise TooBig((lo, hi))  # (no exact int64 box: an overflow to inf, or 2^62 voxels from the origin)
    min_b, max_b = lo.astype(np.int64), hi.astype(np.int64)
    div = max_b - min_b + 1
    if float(div[0]) * float(div[1]) * float(div[2]) > INT32_MAX:
        raise TooBig(div)
    mul = np.array([1, div[0], div[0] * div[1]], np.int64)
    ijk = (np.floor(q[:, :3] * inv) - min_b.astype(F)).astype(np.int64)
    key = ijk @ mul
    order = np.argsort(key, kind="stable")
    ks, qs = key[order], q[order]
    head = np.r_[True, ks[1:] != ks[:-1]]
    vid = np.cumsum(head) - 1
    start = np.flatnonzero(head)
    cnt = np.diff(np.r_[start, len(ks)])
    rank = np.arange(len(ks)) - start[vid]
    by_rank = np.argsort(rank, kind="stable")
    bounds = np.r_[0, np.cumsum(np.bincount(rank))]
    acc = np.zeros((len(start), 4), F)
    for r in range(len(bounds) - 1):
        sel = by_rank[bounds[r]:bounds[r + 1]]
        acc[vid[sel]] = (acc[vid[sel]] + qs[sel]).astype(F)
    return (acc / cnt.astype(F)[:, None]).astype(F)


def get_rpy(qx, qy, qz, qw):
    """tf::Matrix3x3(tf::Quaternion(qx, qy, qz, qw)).getRPY(roll, pitch, yaw) in f64."""
    d = qx * qx + qy * qy + qz * qz + qw * qw
    s = 2.0 / d
    xs, ys, zs = qx * s, qy * s, qz * s
    wx, wy, wz = qw * xs, qw * ys, qw * zs
    xx, xy, xz = qx * xs, qx * ys, qx * zs
    yy, yz, zz = qy * ys, qy * zs, qz * zs
    m00, m10, m20, m21, m22 = 1.0 - (yy + zz), xy + wz, xz - wy, yz + wx, 1.0 - (xx + yy)
    if abs(m20) >= 1:
        delta = math.atan2(m21, m22)
        return delta, (math.pi / 2 if m20 < 0 else -math.pi / 2), 0.0
    pitch = -math.asin(m20)
    c = math.cos(pitch)
    return math.atan2(m21 / c, m22 / c), pitch, math.atan2(m10 / c, m00 / c)


def rot3_rzryrx(x, y, z):
    """gtsam Rot3::RzRyRx(x, y, z) = Rz(z) Ry(y) Rx(x)."""
    cx, sx, cy, sy, cz, sz = math.cos(x), math.sin(x), math.cos(y), math.sin(y), math.cos(z), math.sin(z)
    return [[cy * cz, -cx * sz + sx * sy * cz, sx * sz + cx * sy * cz],
            [cy * sz, cx * cz + sx * sy * sz, -sx * cz + cx * sy * sz],
            [-sy, sx * cy, cx * cy]]


def _mm(A, B):
    return [[A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


def rot3_xyz(A):
    """gtsam Rot3::xyz() through RQ: (x, y, z) with A = Rz(z) Ry(y) Rx(x); roll() = x, pitch() = y, yaw() = z."""
    x = -math.atan2(-A[2][1], A[2][2])
    c, s = math.cos(-x), math.sin(-x)
    B = _mm(A, [[1, 0, 0], [0, c, -s], [0, s, c]])
    y = -math.atan2(B[2][0], B[2][2])
    c, s = math.cos(-y), math.sin(-y)
    Cm = _mm(B, [[c, 0, s], [0, 1, 0], [-s, 0, c]])
    z = -math.atan2(-Cm[1][0], Cm[1][1])
    return x, y, z


def transform_cloud(p4, pose):
    """transformPointCloud (:624-652) with updateTransformPointCloudSinCos (:609-622); pose = (x, y, z, roll, pitch, yaw)."""
    x, y, z, roll, pitch, yaw = (F(v) for v in pose[:6])
    cr, sr, cp, sp, cy, sy = cosf(roll), sinf(roll), cosf(pitch), sinf(pitch), cosf(yaw), sinf(yaw)
    p = np.asarray(p4, F)
    with np.errstate(all="ignore"):
        x1 = cy * p[:, 0] - sy * p[:, 1]
        y1 = sy * p[:, 0] + cy * p[:, 1]
        z1 = p[:, 2]
        y2 = cr * y1 - sr * z1
        z2 = sr * y1 + cr * z1
        out = np.stack([cp * x1 + sp * z2 + x, y2 + y, -sp * x1 + cp * z2 + z, p[:, 3]], 1)
    return out.astype(F)


def extract_window(window, latest, num_poses):
    """The deque bookkeeping of extractSurroundingKeyFrames (:1204-1240) on key-frame ids; latest = [latestFrameID]."""
    if num_poses == 0:
        return
    if len(window) < WINDOW:
        window.clear()
        for i in range(num_poses - 1, -1, -1):
            window.appendleft(i)
            if len(window) >= WINDOW:
                break
    elif latest[0] != num_poses - 1:
        window.popleft()
        latest[0] = num_poses - 1
        window.append(latest[0])


def to_points(a4, dtype):
    """(n, 4) float32 -> the C-ABI's point records."""
    out = np.zeros(len(a4), dtype)
    for k, name in enumerate(("x", "y", "z", "intensity")):
        out[name] = a4[:, k]
    return out


def xyzi(points):
    a = np.asarray(points)
    if a.dtype.names:
        return np.stack([a["x"], a["y"], a["z"], a["intensity"]], 1).astype(F)
    return np.asarray(a, F).reshape(len(a), -1)[:, :4]


class MappingOracle:
    """One mapping node.  step() returns a dict shaped like lins_mapper_report, and keeps the cycle's clouds."""

    def __init__(self, map_oracle, point_dtype, scan_period=0.1):
        self.mo, self.dtype, self.scan_period = map_oracle, point_dtype, scan_period
        z = lambda: np.zeros(6, F)  # noqa: E731
        self.Sum, self.Incre, self.Tobe, self.Bef, self.Aft, self.Last = z(), z(), z(), z(), z(), z()
        self.imu_time, self.imu_roll, self.imu_pitch = np.zeros(IMU_QUE), np.zeros(IMU_QUE, F), np.zeros(IMU_QUE, F)
        self.imu_front, self.imu_last = 0, -1
        self.time_last = -1.0
        self.latest = [0]
        self.prev_pos = np.zeros(3, F)
        self.window = collections.deque()
        self.poses = []  # (x, y, z, roll, pitch, yaw) f32 + time
        self.frames = []  # per key frame: (corner, surf, outlier) in the map frame
        self.clouds = {}

    def imu(self, t, roll, pitch):
        self.imu_last = (self.imu_last + 1) % IMU_QUE
        self.imu_time[self.imu_last] = t
        self.imu_roll[self.imu_last] = F(roll)
        self.imu_pitch[self.imu_last] = F(pitch)

    def associate_to_map(self):  # :411-536
        S, Bf, A, I, T = self.Sum, self.Bef, self.Aft, self.Incre, self.Tobe
        x1 = cosf(S[1]) * (Bf[3] - S[3]) - sinf(S[1]) * (Bf[5] - S[5])
        y1 = Bf[4] - S[4]
        z1 = sinf(S[1]) * (Bf[3] - S[3]) + cosf(S[1]) * (Bf[5] - S[5])
        x2 = x1
        y2 = cosf(S[0]) * y1 + sinf(S[0]) * z1
        z2 = -sinf(S[0]) * y1 + cosf(S[0]) * z1
        I[3] = cosf(S[2]) * x2 + sinf(S[2]) * y2
        I[4] = -sinf(S[2]) * x2 + cosf(S[2]) * y2
        I[5] = z2
        sbcx, cbcx, sbcy, cbcy, sbcz, cbcz = sinf(S[0]), cosf(S[0]), sinf(S[1]), cosf(S[1]), sinf(S[2]), cosf(S[2])
        sblx, cblx, sbly, cbly, sblz, cblz = sinf(Bf[0]), cosf(Bf[0]), sinf(Bf[1]), cosf(Bf[1]), sinf(Bf[2]), cosf(Bf[2])
        salx, calx, saly, caly, salz, calz = sinf(A[0]), cosf(A[0]), sinf(A[1]), cosf(A[1]), sinf(A[2]), cosf(A[2])
        srx = (-sbcx * (salx * sblx + calx * cblx * salz * sblz + calx * calz * cblx * cblz)
               - cbcx * sbcy * (calx * calz * (cbly * sblz - cblz * sblx * sbly) - calx * salz * (cbly * cblz + sblx * sbly * sblz) + cblx * salx * sbly)
               - cbcx * cbcy * (calx * salz * (cblz * sbly - cbly * sblx * sblz) - calx * calz * (sbly * sblz + cbly * cblz * sblx) + cblx * cbly * salx))
        T[0] = -asinf(srx)
        srycrx = (sbcx * (cblx * cblz * (caly * salz - calz * salx * saly) - cblx * sblz * (caly * calz + salx * saly * salz) + calx * saly * sblx)
                  - cbcx * cbcy * ((caly * calz + salx * saly * salz) * (cblz * sbly - cbly * sblx * sblz)
                                   + (caly * salz - calz * salx * saly) * (sbly * sblz + cbly * cblz * sblx) - calx * cblx * cbly * saly)
                  + cbcx * sbcy * ((caly * calz + salx * saly * salz) * (cbly * cblz + sblx * sbly * sblz)
                                   + (caly * salz - calz * salx * saly) * (cbly * sblz - cblz * sblx * sbly) + calx * cblx * saly * sbly))
        crycrx = (sbcx * (cblx * sblz * (calz * saly - caly * salx * salz) - cblx * cblz * (saly * salz + caly * calz * salx) + calx * caly * sblx)
                  + cbcx * cbcy * ((saly * salz + caly * calz * salx) * (sbly * sblz + cbly * cblz * sblx)
                                   + (calz * saly - caly * salx * salz) * (cblz * sbly - cbly * sblx * sblz) + calx * caly * cblx * cbly)
                  - cbcx * sbcy * ((saly * salz + caly * calz * salx) * (cbly * sblz - cblz * sblx * sbly)
                                   + (calz * saly - caly * salx * salz) * (cbly * cblz + sblx * sbly * sblz) - calx * caly * cblx * sbly))
        T[1] = atan2f(srycrx / cosf(T[0]), crycrx / cosf(T[0]))
        srzcrx = ((cbcz * sbcy - cbcy * sbcx * sbcz) * (calx * salz * (cblz * sbly - cbly * sblx * sblz) - calx * calz * (sbly * sblz + cbly * cblz * sblx) + cblx * cbly * salx)
                  - (cbcy * cbcz + sbcx * sbcy * sbcz) * (calx * calz * (cbly * sblz - cblz * sblx * sbly) - calx * salz * (cbly * cblz + sblx * sbly * sblz) + cblx * salx * sbly)
                  + cbcx * sbcz * (salx * sblx + calx * cblx * salz * sblz + calx * calz * cblx * cblz))
        crzcrx = ((cbcy * sbcz - cbcz * sbcx * sbcy) * (calx * calz * (cbly * sblz - cblz * sblx * sbly) - calx * salz * (cbly * cblz + sblx * sbly * sblz) + cblx * salx * sbly)
                  - (sbcy * sbcz + cbcy * cbcz * sbcx) * (calx * salz * (cblz * sbly - cbly * sblx * sblz) - calx * calz * (sbly * sblz + cbly * cblz * sblx) + cblx * cbly * salx)
                  + cbcx * cbcz * (salx * sblx + calx * cblx * salz * sblz + calx * calz * cblx * cblz))
        T[2] = atan2f(srzcrx / cosf(T[0]), crzcrx / cosf(T[0]))
        x1 = cosf(T[2]) * I[3] - sinf(T[2]) * I[4]
        y1 = sinf(T[2]) * I[3] + cosf(T[2]) * I[4]
        z1 = I[5]
        x2 = x1
        y2 = cosf(T[0]) * y1 - sinf(T[0]) * z1
        z2 = sinf(T[0]) * y1 + cosf(T[0]) * z1
        T[3] = A[3] - (cosf(T[1]) * x2 + sinf(T[1]) * z2)
        T[4] = A[4] - y2
        T[5] = A[5] - (-sinf(T[1]) * x2 + cosf(T[1]) * z2)

    def transform_update(self, t):  # :538-577
        T, sp = self.Tobe, self.scan_period
        if self.imu_last >= 0:
            while self.imu_front != self.imu_last:
                if t + sp < self.imu_time[self.imu_front]:
                    break
                self.imu_front = (self.imu_front + 1) % IMU_QUE
            f = self.imu_front
            if t + sp > self.imu_time[f]:
                rl, pl = self.imu_roll[f], self.imu_pitch[f]
            else:
                b = (f + IMU_QUE - 1) % IMU_QUE
                den = self.imu_time[f] - self.imu_time[b]
                rf = F((t + sp - self.imu_time[b]) / den)
                rb = F((self.imu_time[f] - t - sp) / den)
                rl = F(self.imu_roll[f] * rf + self.imu_roll[b] * rb)
                pl = F(self.imu_pitch[f] * rf + self.imu_pitch[b] * rb)
            T[0] = F(0.998 * float(T[0]) + 0.002 * float(pl))
            T[2] = F(0.998 * float(T[2]) + 0.002 * float(rl))
        self.Bef[:] = self.Sum
        self.Aft[:] = T

    def step(self, t, quat, pos, corner, surf, outlier):
        r = dict(processed=0, skipped_interval=0, keyframe_saved=0, loop_candidate=-1, map_skipped=0)
        roll, pitch, yaw = get_rpy(quat[2], -quat[0], -quat[1], quat[3])
        self.Sum[:] = (F(-pitch), F(-yaw), F(roll), F(pos[0]), F(pos[1]), F(pos[2]))
        if not (t - self.time_last >= INTERVAL):
            r["skipped_interval"] = 1
            return r
        self.time_last = t
        self.associate_to_map()
        r["transform_guess"] = self.Tobe.copy()
        n = len(self.poses)
        extract_window(self.window, self.latest, n)
        if n:
            cm = np.concatenate([self.frames[i][0] for i in self.window])
            sm = np.concatenate([c for i in self.window for c in self.frames[i][1:]])
            map_c, map_s = voxel_grid(cm, LEAF_CORNER), voxel_grid(sm, LEAF_SURF)
        else:
            map_c = map_s = np.zeros((0, 4), F)
        cds, sds, ods = voxel_grid(xyzi(corner), LEAF_CORNER), voxel_grid(xyzi(surf), LEAF_SURF), voxel_grid(xyzi(outlier), LEAF_SURF)
        tds = voxel_grid(np.concatenate([sds, ods]), LEAF_SURF)
        self.clouds = dict(map_corner_ds=map_c, map_surf_ds=map_s, corner_ds=cds, surf_ds=sds, outlier_ds=ods, surf_total_ds=tds)
        if len(map_c) > 10 and len(map_s) > 100:  # :1636
            self.mo.set_map(to_points(map_c, self.dtype), to_points(map_s, self.dtype))
            T, rep = self.mo.scan2map(to_points(cds, self.dtype), to_points(tds, self.dtype), self.Tobe)
            self.Tobe[:] = T
            r["map"] = rep
            self.transform_update(t)
        else:
            r["map_skipped"] = 1
        self.save_key_frame(t, r)
        r.update(processed=1, n_keyframes=len(self.poses), window=list(self.window), transform_aft_mapped=self.Aft.copy())
        return r

    def save_key_frame(self, t, r):  # :1654-1765
        cur = self.Aft[3:6].copy()
        d = self.prev_pos - cur
        save = not (float(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])) < KEY_DIST)
        if not save and self.poses:
            return
        self.prev_pos = cur
        first = not self.poses
        P = self.Tobe if first else self.Aft
        if first:
            self.Last[:] = self.Tobe
        x, y, z = rot3_xyz(rot3_rzryrx(float(P[2]), float(P[0]), float(P[1])))
        pose = np.array([P[3], P[4], P[5], F(y), F(z), F(x)], F)  # translation (y, z, x); roll = pitch(), ...
        self.add_key_frame(pose, t)
        if len(self.poses) > 1:
            self.Aft[:] = pose[[3, 4, 5, 0, 1, 2]]
            self.Last[:] = self.Aft
            self.Tobe[:] = self.Aft
        r["keyframe_saved"] = 1
        best = None
        for i, (q, qt) in enumerate(self.poses):
            e = q[:3] - cur
            d2 = F(F(e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
            if d2 < F(25.0) and abs(qt - t) > 30.0 and (best is None or d2 < best):
                best, r["loop_candidate"] = d2, i

    def add_key_frame(self, pose, t):
        c = self.clouds
        self.poses.append((pose, t))
        self.frames.append(tuple(transform_cloud(c[k], pose) for k in ("corner_ds", "surf_ds", "outlier_ds")))

    def adopt(self, aft, last_pose=None):
        """Re-anchor on another implementation's transformAftMapped and newest key pose (f32 values within the LM
        tolerance of this oracle's), so that the next cycle's inputs are bit-identical on both sides."""
        self.Aft[:] = aft
        if last_pose is not None:
            pose = np.asarray(last_pose[:6], F)
            t = self.poses[-1][1]
            self.poses.pop(); self.frames.pop()
            self.add_key_frame(pose, t)
            self.prev_pos = np.asarray(pose[:3], F).copy() if len(self.poses) > 1 else self.prev_pos
