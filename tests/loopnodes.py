"""Mapping nodes built to order for the loop-closure tests: a mapper blob (csrc/cuda/lins_mapper_blob.hpp, the loop flag
set) that lins_gpu_mapper(s)_load takes into a fresh slot, so that close_loops runs on exactly the designed key poses
and clouds, and the catalogue of scenes tests/test_loopnodes_cpu.py and tests/test_gpu_loop_nodes.py share.

A node's key frame holds body-frame corner, surf and outlier clouds ((m, 4) float32 x, y, z, intensity); the map-frame
clouds are mapperref.transform_cloud of them, which the device's transform reproduces bit for bit, so every reference
is computed from the node itself (reference()).  With zero rotation and dyadic coordinates that transform is exact, and
a history voxel holding one point outputs that point, in ascending voxel order: the hand-made thresholds and ties
below rely on both."""
import math
import struct

import numpy as np

import loopref

F = np.float32

HEADER, N_SEC = 192, 9
K_SCALARS, K_MAPPER, K_POSES, K_WINDOW, K_KEYFRAMES, K_KFCLOUDS, K_LOOP, K_FACTORS, K_EST = range(N_SEC)
MAGIC, VERSION, F_LOOPS = 0x5250414D534E494C, 1, 1
IMU_QUEUE, WINDOW = 200, 50
MAPPER_REC = 4 * (36 + 2 * IMU_QUEUE + 3) + 8 * (IMU_QUEUE + 1) + 3 * 4
IMU_LAST_OFF = 4 * (36 + 2 * IMU_QUEUE) + 8 * IMU_QUEUE + 4  # imuPointerLast in MapperRec
FACTOR, EST = 8 + 18 * 8, 12 * 8
CPU_LOOP_STATE = 304  # the loop-state size of the CPU suite's blob validator build (test_mapper_checkpoint_cpu.py)


def _a16(x):
    return (x + 15) & ~15


class Node:
    """poses: (n, 7) x, y, z, roll, pitch, yaw (f32 fields) and time; clouds[i] = (corner, surf, outlier) body frame;
    cur / time: the Scalars close_loops reads (default: the newest key pose's position and stamp)."""

    def __init__(self, poses, clouds, cur=None, time=None):
        self.poses = np.asarray(poses, np.float64).reshape(-1, 7)
        self.clouds = [tuple(np.asarray(c, F).reshape(-1, 4) for c in kf) for kf in clouds]
        assert len(self.clouds) == len(self.poses)
        last = self.poses[-1] if len(self.poses) else np.zeros(7)
        self.cur = np.asarray(last[:3] if cur is None else cur, F)
        self.time = float(last[6] if time is None else time)


def template(blob):
    """(sizes (4 x uint32), MapperRec bytes, loop-state bytes) of a blob a fresh enabled slot saved"""
    b = bytes(blob)
    sizes = struct.unpack_from("<4I", b, 16)
    sec = [struct.unpack_from("<2Q", b, 48 + 16 * k) for k in range(N_SEC)]
    return sizes, b[sec[K_MAPPER][0]:sec[K_MAPPER][0] + MAPPER_REC], b[sec[K_LOOP][0]:sec[K_LOOP][0] + sizes[0]]


def cpu_template():
    """zeros with valid IMU pointers (front 0, last -1), for the CPU suite's validator build"""
    m = bytearray(MAPPER_REC)
    struct.pack_into("<i", m, IMU_LAST_OFF, -1)
    return (CPU_LOOP_STATE, IMU_QUEUE, WINDOW, FACTOR), bytes(m), bytes(CPU_LOOP_STATE)


def _rec_pose3(T):
    return T[:3, :3].astype(np.float64).tobytes() + T[:3, 3].astype(np.float64).tobytes()


def blob(node, tmpl):
    """The mapper blob of node with loop closure: every key frame stored, an empty window, the graph mapper_loops_save
    builds (the prior on key 0, then chain factors between consecutive key poses with the odometry variances), an
    estimate per key pose, no loop factor.  tmpl: template() of a fresh enabled slot's blob, or cpu_template().  (A NaN
    key-pose field enters the graph as 0: the validator refuses a non-finite graph, and close_loops does not read it.)"""
    sizes, mrec, lstate = tmpl
    n = len(node.poses)
    keys = [loopref.pose_of_key(p) for p in np.nan_to_num(node.poses)]
    factors = [(0, -1, keys[0])] if n else []
    factors += [(i - 1, i, loopref.between(keys[i - 1], keys[i])) for i in range(1, n)]
    kf = b"".join(struct.pack("<4i", i, *(len(c) for c in node.clouds[i])) for i in range(n))
    pts = b"".join(np.ascontiguousarray(c, F).tobytes() for kf_ in node.clouds for c in kf_)
    poses = b"".join(struct.pack("<6fd", *(F(v) for v in p[:6]), float(p[6])) for p in node.poses)
    fac = b"".join(struct.pack("<2i", a, b) + _rec_pose3(z) + np.asarray(loopref.ODOM_VAR, np.float64).tobytes() for a, b, z in factors)
    est = b"".join(_rec_pose3(k) for k in keys)
    scal = struct.pack("<7i3fd", n, 0, n, len(factors), n, 0, 0, *node.cur.tolist(), node.time)
    body = [scal, mrec, poses, b"", kf, pts, lstate, fac, est]
    sec, o = [], _a16(HEADER)
    for s in body:
        sec.append((o, len(s)))
        o = _a16(o + len(s))
    out = bytearray(o)
    struct.pack_into("<QII4III Q", out, 0, MAGIC, VERSION, F_LOOPS, *sizes, N_SEC, 0, o)
    for k, (off, nb) in enumerate(sec):
        struct.pack_into("<2Q", out, 48 + 16 * k, off, nb)
        out[off:off + nb] = body[k]
    return bytes(out)


def reference(node, solver="svd", reverse=False):
    """loopref on the node: dict(closest, latest, n_history, icp (with trace), src, tgt)"""
    out = dict(closest=-1, latest=-1)
    if not len(node.poses):
        return out
    c = loopref.candidate(node.poses, node.cur, node.time)
    if c < 0:
        return out
    src, tgt = loopref.loop_clouds(node.poses, [kf[:2] for kf in node.clouds], c)
    ref = loopref.icp(src, tgt, exact=True, solver=solver, reverse=reverse, trace=True)
    out.update(closest=c, latest=len(node.poses) - 1, n_history=len(tgt), icp=ref, src=src, tgt=tgt, scale=scale(src, tgt))
    return out


def scale(*clouds):
    """max |coordinate| over the finite coordinates of the clouds (the scale of the translation tolerances)"""
    m = [np.abs(c[:, :3][np.isfinite(c[:, :3])]).max(initial=0.0) for c in clouds if len(c)]
    return float(max(m, default=0.0))


# ---- scene building blocks ---------------------------------------------------------------------------------------------
def lattice(nx, ny, nz, origin=(0.0, 0.0, 0.0), step=1.0, w=1.0):
    """one point per 0.4 m voxel at origin + 0.25 + step * (i, j, k), x fastest: ascending voxel order is this order"""
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    p = np.stack([i.ravel(), j.ravel(), k.ravel()], 1) * step + 0.25 + np.asarray(origin)
    return np.concatenate([p, np.full((len(p), 1), w)], 1).astype(F)


def moved(p, rot=(0.0, 0.0, 0.0), t=(0.0, 0.0, 0.0), about=None):
    """rotation vector rot about `about` (default: the points' mean), then + t; intensities kept"""
    p = np.asarray(p, F)
    c = p[:, :3].astype(np.float64).mean(0) if about is None else np.asarray(about, np.float64)
    R = loopref.Rotation.from_rotvec(rot).as_matrix()
    q = (p[:, :3] - c) @ R.T + c + np.asarray(t)
    return np.concatenate([q, p[:, 3:4]], 1).astype(F)


def _M(pose):
    """the rotation of transformPointCloud for a key pose: Ry(pitch) Rx(roll) Rz(yaw)"""
    r, p, y = (float(F(v)) for v in pose[3:6])
    Rz = np.array([[math.cos(y), -math.sin(y), 0], [math.sin(y), math.cos(y), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, math.cos(r), -math.sin(r)], [0, math.sin(r), math.cos(r)]])
    Ry = np.array([[math.cos(p), 0, math.sin(p)], [0, 1, 0], [-math.sin(p), 0, math.cos(p)]])
    return Ry @ Rx @ Rz


def body_of(world, pose):
    """map-frame points into the body frame of a key pose (f64, rounded to f32); exact for zero rotation and
    translations that keep the coordinates' bits"""
    world = np.asarray(world, F)
    if not len(world):
        return world.reshape(0, 4)
    if not np.any(np.asarray(pose[3:6], np.float64)):
        q = world[:, :3] - np.asarray(pose[:3], F)
    else:
        q = (world[:, :3].astype(np.float64) - np.asarray(pose[:3], np.float64).astype(F)) @ _M(pose)
    return np.concatenate([q, world[:, 3:4]], 1).astype(F)


E = np.zeros((0, 4), F)


def loop_node(cands, src, latest=(0.0, 0.0, 0.0, 0, 0, 0), t_latest=100.0, pad=None, split=3, cur=None, time=None):
    """cands: [(pose7, world cloud)] first, far empty padding key frames (100 m apart) so that the newest key frame lies
    beyond the history window, then the newest key frame at `latest` holding the map-frame cloud src.  Clouds go into
    the body frame of their pose, the first 1/split of each into corner, the rest into surf."""
    poses, clouds = [], []

    def add(pose7, world):
        b = body_of(world, pose7)
        k = len(b) // split
        poses.append(list(pose7))
        clouds.append((b[:k], b[k:], E))

    for pose7, world in cands:
        add(pose7, world)
    # (by default the newest key frame lies past every candidate's history window, closest + 25)
    n_pad = 25 if pad is None else pad
    for i in range(n_pad):
        add((1000.0 + 100.0 * i, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0 + i), E)
    add(tuple(latest) + (t_latest,), src)
    return Node(poses, clouds, cur=cur, time=time)


def simple(hist, src, off=(0.0, 0.0, 0.0), **k):
    """history `hist` in the candidate key frame 0 at off (stamp 0), source `src` in the newest key frame at off (stamp
    100); both clouds given relative to off"""
    o = np.asarray(off, np.float64)
    sh = lambda c: np.concatenate([np.asarray(c, F)[:, :3] + o.astype(F), np.asarray(c, F)[:, 3:4]], 1).astype(F) if len(c) else E  # noqa: E731
    pose = tuple(o) + (0.0, 0.0, 0.0)
    return loop_node([(pose + (0.0,), sh(hist))], sh(src), latest=pose, **k)


def intens(p, w):
    p = np.array(p, F)
    p[:, 3] = np.resize(np.asarray(w, F), len(p))
    return p


# ---- the scenes --------------------------------------------------------------------------------------------------------
class Scene:
    """kind: "parity" (every field against the oracle), "tie" (the same, with exact 1-NN ties by construction),
    "degenerate" (properties: a proper rotation, no NaN, the oracle's optimum of the objective) or "factor_only" (the
    candidate, counts and decisions, and the loop factor on the device's own final transform); expect: what the CPU
    suite checks the oracle reaches (closest, stop, accepted, n_source, n_corr0, n_history; at_limit: the only 1-NN
    distances allowed within 1 m^2 of the correspondence limit; last_target_used: the history's last target is a first
    correspondence)."""

    def __init__(self, name, node, kind="parity", **expect):
        self.name, self.node, self.kind, self.expect = name, node, kind, expect


W = lattice(6, 5, 3)                               # 90 points, 6 x 5 x 3 m
SHIFT = dict(rot=(0.004, -0.006, 0.01), t=(0.11, -0.07, 0.05))


def _lifted(n_lift, h, seed):
    """a block's top layer copy, moved; n_lift of its points lifted h off it (their nearest target is the one below)"""
    base = lattice(12, 12, 3)
    src = moved(base, **SHIFT)
    rng = np.random.default_rng(seed)
    top = np.flatnonzero(base[:, 2] > 2.0)
    pick = rng.choice(top, n_lift, replace=False)
    src[pick, 2] += F(h)
    return base, src


def scenes():
    S = []
    nx = float(np.nextafter(F(5), F(0)))
    wsrc = moved(W, **SHIFT)
    # candidate edges: d^2 exactly 25 and |dt| exactly 30 (neither a candidate), just below / above, an equal-distance
    # tie (the lower id), a NaN key pose (never a candidate), no key poses
    S.append(Scene("cand_at_edges", loop_node([((3.0, 4.0, 0, 0, 0, 0, 0.0), W), ((0.0, 0, 0, 0, 0, 0, 70.0), W)], wsrc), closest=-1))
    S.append(Scene("cand_d2_below", loop_node([((nx, 0, 0, 0, 0, 0, 0.0), W)], wsrc), closest=0, stop="transform"))
    t_above = float(np.nextafter(30.0, 31.0))
    S.append(Scene("cand_dt_above", loop_node([((0.0, 0, 0, 0, 0, 0, 0.0), W)], wsrc, t_latest=t_above), closest=0, stop="transform"))
    S.append(Scene("cand_equal_distance", loop_node([((2.0, 0, 0, 0, 0, 0, 0.0), W), ((-2.0, 0, 0, 0, 0, 0, 1.0), W)], wsrc), closest=0, stop="transform"))
    S.append(Scene("cand_nan_pose", loop_node([((math.nan, 0, 0, 0, 0, 0, 0.0), E), ((1.0, 0, 0, 0, 0, 0, 1.0), W)], wsrc), closest=1, stop="transform"))
    S.append(Scene("cand_no_poses", Node(np.zeros((0, 7)), []), closest=-1))
    # source edges
    S.append(Scene("src_empty", simple(W, E), closest=0, stop="ncorr", n_source=0))
    wi = intens(wsrc, [-1.0, float(np.nextafter(F(-1), F(0))), 2147483520.0, 2.0 ** 31, math.nan, math.inf, -math.inf, 0.0, 7.0])
    S.append(Scene("src_intensity", simple(W, wi), closest=0, stop="transform", n_source=40))
    for n, stop in ((1, "ncorr"), (2, "ncorr"), (3, "transform")):
        S.append(Scene(f"src_{n}", simple(W, wsrc[[0, 17, 44][:n]]), closest=0, stop=stop, n_source=n))
    big = lattice(16, 16, 14)
    bsrc = moved(big, **SHIFT)
    for n in (127, 128, 129):
        S.append(Scene(f"src_{n}", simple(big, bsrc[:n]), closest=0, stop="transform", n_source=n))
    # (the last 3000: their nearest targets run to the end of the 3584, across three full tiles and a partial one)
    S.append(Scene("src_3000", simple(big, bsrc[-3000:]), closest=0, stop="transform", n_source=3000))
    # history edges
    S.append(Scene("hist_beyond_100m", simple(lattice(4, 4, 2, origin=(150.0, 0, 0)), wsrc), closest=0, stop="ncorr", n_corr0=0))
    far2 = np.concatenate([lattice(4, 4, 2, origin=(150.0, 0, 0)), W[[0, 1]]])
    S.append(Scene("hist_two_within", simple(far2, np.concatenate([W[[0, 1]], lattice(3, 3, 1, origin=(-150.0, 0, 0))])), closest=0, stop="ncorr",
                   n_corr0=2))
    # d = 10000 exactly (kept) for two sources symmetric about the pins, and 10000 + 2^-10 (the next f32) for a third
    cl = lattice(4, 3, 2, origin=(150.0, 200.0, 0))
    tg = np.concatenate([np.array([[100.0, 0, 0, 1], [200.0, 0, 0, 1]], F), cl])
    sr = np.concatenate([np.array([[0.0, 0, 0, 1], [300.0, 0, 0, 1], [0.0, -0.03125, 0, 1]], F), cl])
    S.append(Scene("hist_corr_at_1e4", simple(tg, sr), closest=0, stop="transform", n_corr0=len(cl) + 2, accepted=0,
                   at_limit=(1e4, 1e4 + 2.0 ** -10)))
    # the sources are the moved copies of the prefix's last 200 targets, so that target n - 1 is a nearest neighbour: the
    # last of a full tile (1024), or alone in a partial last tile (1025, 2049)
    hsrc = moved(lattice(16, 16, 9), **SHIFT)
    for n in (0, 1023, 1024, 1025, 2049):
        S.append(Scene(f"hist_{n}", simple(lattice(16, 16, 9)[:n], hsrc[max(0, n - 200):max(n, 200)]), closest=0,
                       stop="ncorr" if n == 0 else "transform", n_history=n, last_target_used=n > 0))
    # an exact tie between targets 1023 and 1024 (the two tiles' edges): the lower index must win
    grid = lattice(11, 11, 9)
    mid = (grid[1023] + grid[1024]) / F(2)
    pins = grid[[0, 10, 110, 900]]
    S.append(Scene("hist_tie_tiles", simple(grid, np.concatenate([pins, mid[None]])), kind="tie", closest=0))
    # a history window clipped at both ends (newest key frame inside it) and one partly outside the device store
    S.append(Scene("hist_clipped", loop_node([((0.0, 0, 0, 0, 0, 0, 0.0), W[:45])] + [((40.0 + i, 0, 0, 0, 0, 0, 1.0 + i), W[45:]) for i in range(3)],
                                             wsrc, pad=5), closest=0))
    parts = [((-20.0 - 10 * i, 0, 0, 0, 0, 0, float(i)), W[10 * i:10 * i + 10]) for i in range(5)]
    parts.append(((0.0, 0, 0, 0, 0, 0, 5.0), W[50:]))
    S.append(Scene("hist_over_51_keyframes", loop_node(parts, wsrc, pad=54), closest=5, stop="transform"))
    # stop criteria: a noiseless moved copy (the transform criterion)
    S.append(Scene("stop_transform", simple(lattice(8, 8, 4), moved(lattice(8, 8, 4), rot=(0.0, 0.0, 0.02), t=(0.1, -0.05, 0.03))),
                   closest=0, stop="transform", accepted=1))
    # fitness: a share of the source lifted off the block's top, about 0.2 (accepted) and 0.4 (rejected)
    b, s = _lifted(43, math.sqrt(2.0), 1)
    S.append(Scene("fit_accept", simple(b, s), closest=0, accepted=1))
    b, s = _lifted(104, math.sqrt(2.0), 2)
    S.append(Scene("fit_reject", simple(b, s), closest=0, accepted=0))
    # degenerate geometry
    one = np.repeat(np.array([[2.3, 1.6, 0.9, 1.0]], F), 12, 0)
    S.append(Scene("deg_one_position", simple(W, one), kind="degenerate", closest=0))
    line = lattice(30, 1, 1)
    S.append(Scene("deg_collinear", simple(line, moved(line[3:25], t=(0.1, 0.06, -0.04))), kind="degenerate", closest=0))
    # far from the origin
    # (at 20 km the f32 rounding of the coordinates is the noise that leaves the relative-MSE criterion to stop it)
    for name, off, stop in (("far_1km", (1000.0, -250.0, 12.0), "transform"), ("far_20km", (20000.0, 5000.0, -30.0), "mse")):
        S.append(Scene(name, simple(lattice(8, 8, 4), moved(lattice(8, 8, 4), rot=(0.0, 0.0, 0.02), t=(0.1, -0.05, 0.03)), off=off),
                       closest=0, stop=stop, accepted=1))
    S += factor_scenes()
    return S


def _blob_world(seed, n=260, ext=(9.0, 7.0, 4.0)):
    """an irregular cloud, one point per voxel"""
    rng = np.random.default_rng(seed)
    p = rng.uniform(0, 1, (4 * n, 3)) * ext
    p = p[np.unique(np.floor(p / 0.8).astype(np.int64) @ [1, 1000, 1000000], return_index=True)[1]][:n]
    return np.concatenate([p, np.ones((len(p), 1))], 1).astype(F)


def factor_scene(name, pose0, dpose, corr, seed, kind="parity"):
    """key frame 0 at pose0 sees the world; the newest key frame, at pose0 + dpose (stored), saw it from a pose whose
    rotation differs by the rotation vector corr about the world's centre: ICP's correction"""
    w = _blob_world(seed)
    c = np.asarray(pose0[:3], np.float64)
    world = np.concatenate([w[:, :3] + c.astype(F), w[:, 3:]], 1).astype(F)
    p_l = tuple(np.asarray(pose0[:6], np.float64) + np.asarray(dpose))
    seen = moved(world, rot=corr, about=world[:, :3].astype(np.float64).mean(0))
    b0 = body_of(world, pose0)
    bl = body_of(seen, p_l)
    k0, kl = len(b0) // 3, len(bl) // 3
    poses = [tuple(pose0[:6]) + (0.0,)] + [(c[0] + 1000.0 + 100.0 * i, c[1], c[2], 0, 0, 0, 1.0 + i) for i in range(26)] + [p_l + (100.0,)]
    clouds = [(b0[:k0], b0[k0:], E)] + [(E, E, E)] * 26 + [(bl[:kl], bl[kl:], E)]
    return Scene(name, Node(poses, clouds), kind=kind, closest=0, accepted=1, factor=True)


def factor_scenes():
    return [
        factor_scene("factor_yaw_pi_1km", (1000.0, -700.0, 30.0, 0.3, -0.25, 3.1, 0.0), (0.5, -0.4, 0.1, -0.02, 0.01, 0.08), (0.0, 0.01, 0.05), 12),
        factor_scene("factor_yaw_minus_pi", (-120.0, 64.0, -3.0, -0.28, 0.3, -3.12, 0.0), (1.0, 0.5, 0.0, 0.0, 0.0, -0.05), (0.02, -0.02, -0.1), 12),
        factor_scene("factor_corr_0_2", (3.0, 2.0, 0.5, 0.1, 0.05, 0.7, 0.0), (0.2, 0.3, 0.0, 0.0, 0.0, 0.0), (0.0, 0.0, 0.2), 13),
        # 10 km out, the f32 rounding of the rotated key frames leaves the ICP's last relative-MSE steps without margin:
        # its iteration count and final transform (to decimetres: 1e-4 rad about an origin 10 km away) are not
        # determined, only its decisions; the factor is pinned on the device's own final transform
        factor_scene("factor_yaw_pi_10km", (9000.0, -4000.0, 30.0, 0.3, -0.25, 3.1, 0.0), (0.5, -0.4, 0.1, -0.02, 0.01, 0.08), (0.0, 0.01, 0.05), 14,
                     kind="factor_only"),
    ]


def toobig_scene():
    """a history body cloud with points at the origin and at (1000, 1000, 1000): more than 2^31 voxels at 0.4 m"""
    return Scene("toobig", simple(np.array([[0.0, 0, 0, 1], [1000.0, 1000.0, 1000.0, 1]], F), moved(W, **SHIFT)), closest=0)
