"""An independent numpy / scipy restatement of the mapping node's loop closure (lidar_mapping_node.cpp
detectLoopClosure :1043-1112, performLoopClosure :1114-1186, correctPoses :1767-1795) and of the key-pose graph the
library solves in place of iSAM2 (DESIGN.md §4.14).

Rotation exponentials and logarithms come from scipy's Rotation, the 1-NN from scipy's cKDTree (its candidates
re-ranked by the f32 distance the library computes, ties to the lower index) or, exactly, by brute force (nn1_exact),
the rigid transform from Umeyama's SVD (or Horn's quaternion, for stability checks),
and the graph's solve is a dense Gauss-Newton with central-difference Jacobians, so none of it shares
code with the library's kernels or its host solver."""
import math

import numpy as np
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

import mapperref

F = np.float32
HISTORY = 25
FITNESS = F(0.3)
MAX_ITER = 100
ODOM_VAR = np.array([1e-6, 1e-6, 1e-6, 1e-8, 1e-8, 1e-6])


# ---- pcl's Euler helpers, f32 (pcl/common/eigen.hpp, taken on trust) -------------------------------------------------
def pcl_transformation(x, y, z, roll, pitch, yaw):
    """pcl::getTransformation -> 3 x 4 float32."""
    A, B, C, D, E, Fs = mapperref.cosf(yaw), mapperref.sinf(yaw), mapperref.cosf(pitch), mapperref.sinf(pitch), mapperref.cosf(roll), mapperref.sinf(roll)
    DE, DF = F(D * E), F(D * Fs)
    return np.array([[A * C, A * DF - B * E, B * Fs + A * DE, x], [B * C, A * E + B * DF, B * DE - A * Fs, y], [-D, C * Fs, C * E, z]], F)


def pcl_euler(t):
    """pcl::getTranslationAndEulerAngles of a 3 x 4 float32: x, y, z, roll, pitch, yaw."""
    return (F(t[0, 3]), F(t[1, 3]), F(t[2, 3]), mapperref.atan2f(t[2, 1], t[2, 2]), mapperref.asinf(-t[2, 0]), mapperref.atan2f(t[1, 0], t[0, 0]))


def affine_mul(a, b):
    c = np.zeros((3, 4), F)
    for r in range(3):
        for k in range(4):
            s = F(F(F(a[r, 0] * b[0, k]) + F(a[r, 1] * b[1, k])) + F(a[r, 2] * b[2, k]))
            c[r, k] = F(s + a[r, 3]) if k == 3 else s
    return c


# ---- gtsam Pose3 (default build: EXPMAP retraction and local coordinates, taken on trust) --------------------------
def pose3(roll, pitch, yaw, x, y, z):
    """Pose3(Rot3::RzRyRx(roll, pitch, yaw), Point3(x, y, z)) as a 4 x 4 float64."""
    T = np.eye(4)
    T[:3, :3] = Rotation.from_euler("xyz", [roll, pitch, yaw]).as_matrix()  # extrinsic x, y, z = Rz Ry Rx
    T[:3, 3] = (x, y, z)
    return T


def between(a, b):
    return np.linalg.inv(a) @ b


def _V(w):
    th = np.linalg.norm(w)
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-10:
        return np.eye(3) + W / 2
    return np.eye(3) + (1 - math.cos(th)) / th ** 2 * W + (th - math.sin(th)) / th ** 3 * W @ W


def expmap(xi):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(xi[:3]).as_matrix()
    T[:3, 3] = _V(xi[:3]) @ xi[3:]
    return T


def logmap(T):
    w = Rotation.from_matrix(T[:3, :3]).as_rotvec()
    return np.concatenate([w, np.linalg.solve(_V(w), T[:3, 3])])


def factor_error(f, x):
    a, b, z, _ = f
    return logmap(between(z, x[a])) if b < 0 else logmap(between(z, between(x[a], x[b])))


def gn_solve(factors, x0, iters=100, tol=1e-10):
    """Dense Gauss-Newton on the keys (right retraction by expmap) to the fixed point."""
    x = [np.array(p) for p in x0]
    n = len(x)
    for _ in range(iters):
        H, g = np.zeros((6 * n, 6 * n)), np.zeros(6 * n)
        for f in factors:
            keys = [f[0]] if f[1] < 0 else [f[0], f[1]]
            e = factor_error(f, x)
            w = 1.0 / np.asarray(f[3])
            J = {}
            for k in keys:
                Jk = np.zeros((6, 6))
                for j in range(6):
                    d = np.zeros(6); d[j] = 1e-6
                    xp, xm = list(x), list(x)
                    xp[k], xm[k] = x[k] @ expmap(d), x[k] @ expmap(-d)
                    Jk[:, j] = (factor_error(f, xp) - factor_error(f, xm)) / 2e-6
                J[k] = Jk
            for k in keys:
                g[6 * k:6 * k + 6] += J[k].T @ (w * e)
                for l in keys:
                    H[6 * k:6 * k + 6, 6 * l:6 * l + 6] += J[k].T @ (w[:, None] * J[l])
        d = np.linalg.solve(H, -g)
        x = [x[i] @ expmap(d[6 * i:6 * i + 6]) for i in range(n)]
        if np.abs(d).max() < tol:
            break
    return x


def graph_cost(factors, x):
    return sum(float(np.sum(factor_error(f, x) ** 2 / np.asarray(f[3]))) for f in factors)


# ---- ICP: pcl::IterativeClosestPoint<PointXYZI, PointXYZI> as performLoopClosure sets it (:1127-1138) ---------------
def keep_mask(w):
    """(int)intensity >= 0 on x86: NaN and values outside (-1, 2^31) truncate to a negative int."""
    w = np.asarray(w, F)
    with np.errstate(invalid="ignore"):
        return (w > F(-1)) & (w < F(2147483648.0))


def xf(T, p):
    """transformCloud on f32 points: rows summed left to right."""
    T = np.asarray(T, F)
    o = np.empty_like(p)
    for r in range(3):
        o[:, r] = ((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3]
    o[:, 3] = p[:, 3]
    return o


def nn1(tree, tgt, p):
    """Exact f32 1-NN: cKDTree's candidates re-ranked by ((dx^2 + dy^2) + dz^2) in f32, ties to the lower index."""
    k = min(8, len(tgt))
    _, idx = tree.query(p[:, :3].astype(np.float64), k=k)
    idx = np.asarray(idx).reshape(len(p), k)
    d = np.full((len(p), k), np.inf, F)
    for j in range(k):
        q = tgt[idx[:, j]]
        dx, dy, dz = q[:, 0] - p[:, 0], q[:, 1] - p[:, 1], q[:, 2] - p[:, 2]
        d[:, j] = (dx * dx + dy * dy) + dz * dz
    order = np.lexsort((idx, d), axis=1)[:, 0]
    rows = np.arange(len(p))
    return idx[rows, order], d[rows, order]


def nn1_exact(tgt, p, chunk=1 << 22):
    """Brute-force exact f32 1-NN of every point of p over all of tgt: ((dx^2 + dy^2) + dz^2) in f32, ties to the lower
    target index, a distance that is not below FLT_MAX never taken (as the device's strict d < best from FLT_MAX).
    -> (idx (-1: none), d (FLT_MAX: none), gap: sqrt(second best) - sqrt(best) in f64 (inf with fewer than two))."""
    n, m = len(p), len(tgt)
    idx, d, gap = np.full(n, -1, np.int64), np.full(n, F(np.finfo(F).max), F), np.full(n, np.inf)
    if m == 0 or n == 0:
        return idx, d, gap
    q = np.asarray(tgt, F)[:, :3]
    step = max(1, chunk // m)
    for a in range(0, n, step):
        s = np.asarray(p[a:a + step, :3], F)
        dx, dy, dz = (q[None, :, k] - s[:, None, k] for k in range(3))
        with np.errstate(over="ignore", invalid="ignore"):
            dd = (dx * dx + dy * dy) + dz * dz
            dd = np.where(dd < np.finfo(F).max, dd, F(np.inf))
        i = np.argmin(dd, axis=1)  # (the first of equal minima: the lower index)
        rows = np.arange(len(s))
        b = dd[rows, i]
        ok = np.isfinite(b)
        idx[a:a + step] = np.where(ok, i, -1)
        d[a:a + step] = np.where(ok, b, F(np.finfo(F).max))
        if m > 1:
            dd[rows, i] = np.inf
            b2 = dd.min(1).astype(np.float64)
            with np.errstate(invalid="ignore"):
                gap[a:a + step] = np.where(ok, np.sqrt(b2) - np.sqrt(b.astype(np.float64)), np.inf)
    return idx, d, gap


def umeyama(s, t):
    ms, mt = s.mean(0), t.mean(0)
    Sg = (t - mt).T @ (s - ms) / len(s)
    U, _, Vt = np.linalg.svd(Sg)
    D = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        D[2, 2] = -1
    R = U @ D @ Vt
    return R, mt - R @ ms


def horn(s, t, reverse=False):
    """The same optimum by Horn's quaternion (numpy.linalg.eigh of the 4 x 4 form) on the one-pass cross-covariance
    sum s t^T - n ms mt^T, summed in reverse point order: a second solver and summation order for stability checks."""
    if reverse:
        s, t = s[::-1], t[::-1]
    n = len(s)
    ms, mt = np.sum(s, 0) / n, np.sum(t, 0) / n
    H = np.einsum("ij,ik->jk", s, t) - n * np.outer(ms, mt)
    (Sxx, Sxy, Sxz), (Syx, Syy, Syz), (Szx, Szy, Szz) = H
    N = np.array([[Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx],
                  [Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz],
                  [Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy],
                  [Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz]])
    w, x, y, z = np.linalg.eigh(N)[1][:, -1]
    R = Rotation.from_quat([x, y, z, w]).as_matrix()
    return R, mt - R @ ms


def icp(src, tgt, exact=False, solver="svd", reverse=False, trace=False):
    """-> dict(iters, converged, n_corr0, fitness, final (4 x 4 f32), corr0 (first iteration's 1-NN indices)).
    exact: the 1-NN by nn1_exact (else cKDTree's 8 nearest re-ranked, which can miss the f32 nearest among more than 8
    near-equidistant targets); solver "svd" (Umeyama) or "horn"; reverse: the sums in reverse point order.  trace: also
    "trace", per iteration dict(n_corr, mse, cos (the rotation criterion's cos_angle), tsq (the translation
    criterion's squared norm), gap (per used correspondence: sqrt(second best) - sqrt(best) f32 distance, exact only),
    near_limit (the distinct 1-NN distances within 1 m^2 of the 1e4 m^2 correspondence limit)),
    and "stop": "ncorr" (fewer than 3 correspondences), "cap", "transform" or "mse"."""
    src = np.asarray(src, F)[keep_mask(np.asarray(src, F)[:, 3])]
    tgt = np.asarray(tgt, F)
    out = dict(iters=0, converged=0, n_corr0=0, n_source=len(src), fitness=np.finfo(np.float64).max, final=np.eye(4, dtype=F), corr0=None,
               trace=[], stop="ncorr")
    if len(tgt) == 0 or len(src) == 0:
        return out
    if exact:
        nn = lambda p: nn1_exact(tgt, p)  # noqa: E731
    else:
        tree = cKDTree(tgt[:, :3].astype(np.float64))
        nn = lambda p: nn1(tree, tgt, p) + (None,)  # noqa: E731
    fin = np.eye(4, dtype=F)[:3]
    cur = src.copy()
    prev_mse = np.finfo(np.float64).max
    it = 0
    while True:
        idx, d, gap = nn(cur)
        ok = (idx >= 0) & (d <= F(1e4))
        if it == 0:
            out["n_corr0"], out["corr0"] = int(ok.sum()), np.where(ok, idx, -1)
        found = d[idx >= 0]
        rec = dict(n_corr=int(ok.sum()), gap=None if gap is None else gap[ok], near_limit=np.unique(found[np.abs(found.astype(np.float64) - 1e4) < 1.0]))
        if trace:
            out["trace"].append(rec)
        if ok.sum() < 3:
            out["converged"], out["stop"] = 0, "ncorr"
            break
        s64, t64 = cur[ok, :3].astype(np.float64), tgt[idx[ok], :3].astype(np.float64)
        R, t = umeyama(s64, t64) if solver == "svd" else horn(s64, t64, reverse)
        T = np.concatenate([R, t[:, None]], 1).astype(F)
        cur = xf(T, cur)
        nf = np.zeros((3, 4), F)
        for r in range(3):
            for k in range(4):
                s = F(F(F(T[r, 0] * fin[0, k]) + F(T[r, 1] * fin[1, k])) + F(T[r, 2] * fin[2, k]))
                nf[r, k] = F(s + T[r, 3]) if k == 3 else s
        fin = nf
        it += 1
        cos_angle = 0.5 * float(F(F(F(T[0, 0] + T[1, 1]) + T[2, 2]) - F(1)))
        tsq = float(F(F(F(T[0, 3] * T[0, 3]) + F(T[1, 3] * T[1, 3])) + F(T[2, 3] * T[2, 3])))
        dk = d[ok].astype(np.float64)
        mse = float(np.sum(dk[::-1] if reverse else dk)) / ok.sum()
        rec.update(mse=mse, prev_mse=prev_mse, cos=cos_angle, tsq=tsq)
        stop = "cap" if it >= MAX_ITER else "transform" if (cos_angle >= 0.99999 and tsq <= 1e-6) else \
            "mse" if (abs(mse - prev_mse) < 1e-12 or abs(mse - prev_mse) / prev_mse < 1e-6) else None
        if stop:
            out["converged"], out["stop"] = 1, stop
            break
        prev_mse = mse
    out["iters"] = it
    out["final"] = np.concatenate([fin, np.array([[0, 0, 0, 1]], F)])
    idx, d, _ = nn(xf(fin, src))
    d = d[idx >= 0].astype(np.float64)
    out["fitness"] = float(np.sum(d[::-1] if reverse else d)) / len(d) if len(d) else np.finfo(np.float64).max
    return out


def fitness_of(final, src, tgt):
    """getFitnessScore of a given final transform: the mean exact f32 1-NN distance of the kept source under it"""
    src = np.asarray(src, F)[keep_mask(np.asarray(src, F)[:, 3])]
    idx, d, _ = nn1_exact(np.asarray(tgt, F), xf(np.asarray(final, F)[:3], src))
    d = d[idx >= 0].astype(np.float64)
    return float(np.sum(d)) / len(d) if len(d) else np.finfo(np.float64).max


# ---- detectLoopClosure's inputs and the loop factor ------------------------------------------------------------------
def candidate(poses, cur, time):
    """The nearest key pose within 5 m of cur whose time differs by > 30 s (poses: n x 7), else -1."""
    best, c = None, -1
    for i, q in enumerate(poses):
        e = np.asarray(q[:3], F) - np.asarray(cur, F)
        d2 = F(F(e[0] * e[0] + e[1] * e[1]) + e[2] * e[2])
        if d2 < F(25.0) and abs(q[6] - time) > 30.0 and (best is None or d2 < best):
            best, c = d2, i
    return c


def loop_clouds(poses, frames, closest):
    """Source (latest corner + surf in the map frame) and the history sub-map's VoxelGrid; frames[i] = body-frame
    (corner, surf) DS clouds of key frame i."""
    latest = len(poses) - 1
    tf = lambda i, k: mapperref.transform_cloud(frames[i][k], poses[i][:6])  # noqa: E731
    src = np.concatenate([tf(latest, 0), tf(latest, 1)])
    hist = [tf(j, k) for j in range(max(0, closest - HISTORY), min(latest, closest + HISTORY) + 1) for k in (0, 1)]
    return src, mapperref.voxel_grid(np.concatenate(hist), mapperref.LEAF_SURF)


def loop_factor(final, latest_pose, closest_pose):
    """poseFrom.between(poseTo) of :1156-1170 (4 x 4 float64) from ICP's final transform and the two key poses."""
    x, y, z, roll, pitch, yaw = pcl_euler(np.asarray(final, F)[:3])
    cl = pcl_transformation(z, x, y, yaw, roll, pitch)
    k = latest_pose
    tw = pcl_transformation(F(k[2]), F(k[0]), F(k[1]), F(k[5]), F(k[3]), F(k[4]))
    x, y, z, roll, pitch, yaw = pcl_euler(affine_mul(cl, tw))
    frm = pose3(float(roll), float(pitch), float(yaw), float(x), float(y), float(z))
    c = closest_pose
    to = pose3(float(F(c[5])), float(F(c[3])), float(F(c[4])), float(F(c[2])), float(F(c[0])), float(F(c[1])))
    return between(frm, to)


def key_pose_of(T):
    """A key pose's six f32 fields from an estimate (translation (y, z, x), roll = pitch(), pitch = yaw(), yaw = roll())."""
    x, y, z = mapperref.rot3_xyz(T[:3, :3].tolist())
    return np.array([T[1, 3], T[2, 3], T[0, 3], y, z, x], F)


def pose_of_key(k):
    """The Pose3 of a key pose (pclPointTogtsamPose3 :1188-1193)."""
    return pose3(float(F(k[5])), float(F(k[3])), float(F(k[4])), float(F(k[2])), float(F(k[0])), float(F(k[1])))


# ---- the mapping node with loop closure enabled ----------------------------------------------------------------------
def _pose_of_T(T):
    """Pose3(Rot3::RzRyRx(T[2], T[0], T[1]), Point3(T[5], T[3], T[4])) of a transform row (:1676-1704)."""
    return pose3(float(T[2]), float(T[0]), float(T[1]), float(T[5]), float(T[3]), float(T[4]))


class LoopMappingOracle(mapperref.MappingOracle):
    """mapperref.MappingOracle with loopClosureEnableFlag's graph: the prior and chain factors of every save, the loop
    factors close() adds, the estimate of each save (the inserted pose without a loop factor, else gn_solve of the
    graph), correctPoses at the end of a processed cycle after a closure (every key pose from the estimate of the last
    save, each key frame's map-frame clouds re-transformed from its body-frame ones, the window cleared)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.graph, self.est, self.n_loop, self.closed = [], [], 0, False
        self.body = []  # per key frame: (corner, surf, outlier) DS clouds in the body frame
        self.cur, self.time = np.zeros(3, F), 0.0
        self.corrected = []  # per processed cycle: whether correctPoses ran, and whether the cycle saved a key frame

    def step(self, t, quat, pos, corner, surf, outlier):
        self.time = t
        r = super().step(t, quat, pos, corner, surf, outlier)
        if r["processed"]:
            r["corrected"] = self.closed
            if self.closed:
                for i, E in enumerate(self.est):
                    pose = key_pose_of(E)
                    self.poses[i] = (pose, self.poses[i][1])
                    self.frames[i] = tuple(mapperref.transform_cloud(c, pose) for c in self.body[i])
                self.window.clear()
                self.closed = False
        return r

    def save_key_frame(self, t, r):  # :1654-1765 with the graph
        cur = self.Aft[3:6].copy()
        self.cur = cur
        d = self.prev_pos - cur
        save = not (float(mapperref.sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])) < mapperref.KEY_DIST)
        if not save and self.poses:
            return
        self.prev_pos = cur
        first = not self.poses
        P = self.Tobe if first else self.Aft
        R = mapperref.rot3_rzryrx(float(P[2]), float(P[0]), float(P[1]))
        ins = np.eye(4)
        ins[:3, :3], ins[:3, 3] = R, (float(P[5]), float(P[3]), float(P[4]))
        n = len(self.poses)
        if first:
            self.graph, self.est = [(0, -1, ins, ODOM_VAR)], []
            self.Last[:] = self.Tobe
        else:
            self.graph.append((n - 1, n, between(_pose_of_T(self.Last), ins), ODOM_VAR))
        self.est.append(ins)
        if self.n_loop:
            self.est = gn_solve(self.graph, self.est)
            pose = key_pose_of(self.est[-1])
        else:
            x, y, z = mapperref.rot3_xyz(R)
            pose = np.array([P[3], P[4], P[5], F(y), F(z), F(x)], F)
        self.add_key_frame(pose, t)
        if len(self.poses) > 1:
            self.Aft[:] = pose[[3, 4, 5, 0, 1, 2]]
            self.Last[:] = self.Aft
            self.Tobe[:] = self.Aft
        r["keyframe_saved"] = 1
        r["loop_candidate"] = candidate(self.poses7(), cur, t)

    def add_key_frame(self, pose, t):
        super().add_key_frame(pose, t)
        self.body.append(tuple(self.clouds[k] for k in ("corner_ds", "surf_ds", "outlier_ds")))

    def adopt(self, aft, last_pose=None):
        if last_pose is not None:
            self.body.pop()
        super().adopt(aft, last_pose)

    def poses7(self):
        return np.array([list(p) + [t] for p, t in self.poses]) if self.poses else np.zeros((0, 7))

    def close(self, use=None):
        """performLoopClosure: dict(closest, latest, icp result, accepted, factor).  use = (final, fitness) of another
        implementation's ICP (checked against this one's by the caller) anchors the loop factor on it."""
        out = dict(closest=-1, latest=-1, accepted=0)
        if not self.poses:
            return out
        P = self.poses7()
        c = candidate(P, self.cur, self.time)
        if c < 0:
            return out
        src, tgt = loop_clouds(P, self.body, c)
        ref = icp(src, tgt)
        out.update(closest=c, latest=len(P) - 1, icp=ref, n_history=len(tgt))
        final, fitness = (ref["final"], ref["fitness"]) if use is None else use
        if not (ref["converged"] and not fitness > float(FITNESS)):
            return out
        z = loop_factor(np.asarray(final, F), P[-1], P[c])
        noise = float(F(fitness))
        self.graph.append((len(P) - 1, c, z, np.full(6, noise)))
        self.n_loop += 1
        self.closed = True
        out.update(accepted=1, factor=z, noise=noise)
        return out
