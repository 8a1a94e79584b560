"""Adversarial clouds for the mapping node's segmented VoxelGrid and its scan-to-map gate (lins_mapper.cu,
lins_mappers.cu): test infrastructure, no product code, no GPU.

A case is one slot's scan: (corner, surf, outlier) POINT_DTYPE clouds, filtered at 0.2 / 0.4 / 0.4 m, with the outcome
a mapping cycle on them must have ("ok", or "toobig": LINS_E_TOOBIG).  Intensities are finite except in the one case
named "nan_intensity", whose centroids are compared by NaN-ness there.  The episodes and the lockstep step plan of
tests/test_gpu_mappers_scale.py are built here too, so that tests/test_vgcases_cpu.py can check on the host what they
claim to reach: every listed processed-slot count P, a round of more than 600 k points, and the 10 / 11 / 100 / 101
map-gate counts."""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
_defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
F = np.float32
POINT_DTYPE = _defs.POINT_DTYPE
LEAVES = (0.2, 0.4, 0.4)  # corner, surf, outlier
INT32_MAX = (1 << 31) - 1


def pts(xyz, intensity=None):
    """POINT_DTYPE cloud of (n, 3) coordinates taken as f32 as they are; intensities default to 0, 1, 2, ... mod 16."""
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    inten = np.arange(len(xyz)) % 16 if intensity is None else intensity
    return _defs.make_points(xyz, np.asarray(inten, F))


def empty():
    return pts(np.zeros((0, 3)))


class Case:
    def __init__(self, name, corner, surf, outlier, expect="ok"):
        self.name, self.clouds, self.expect = name, (corner, surf, outlier), expect


def _blob(rng, n, lo=-6.0, hi=6.0, center=(0.0, 0.0, 0.0)):
    return rng.uniform(lo, hi, (n, 3)) + np.asarray(center)


def _faces(leaf):
    """Coordinates on the voxel faces k * leaf (f32) and their nextafter neighbours, both signs, -0.0 and +0.0."""
    out = [F(-0.0), F(0.0)]
    for k in (1, 2, 3, 7, 10, 25, 49):
        for s in (1, -1):
            v = F(s * k * F(leaf))
            out += [v, np.nextafter(v, F(np.inf)), np.nextafter(v, F(-np.inf))]
    return np.array(out, F)


def _face_cloud(leaf):
    f = _faces(leaf)
    xyz = np.stack([f, np.roll(f, 1), np.roll(f, 5)], 1)  # every axis sees every face value
    return np.concatenate([xyz, xyz[:, [2, 0, 1]]])


def far_pair():
    """Two points 2^31 voxels from the origin along x at 0.2 m: one int32-clamped bound gives div_x = 1 and one key."""
    return np.array([[5e8 + 64, 0.0, 0.0], [5e8, 51.2, 0.0]], F)


def int32_extent(extra):
    """A 1 x 1 x (INT32_MAX + extra) voxel box at 0.2 m along x, found by search over f32 coordinates: x floors to -126
    - extra at one end and to 2^31 - 128 (the largest f32 integer below 2^31) at the other, with points near that end
    whose keys lie next to 2^31 - 1 (the f32 differences to the low floor round up to 2^31)."""
    inv = F(1.0) / F(0.2)

    def find(target, start):
        x = F(start)
        for _ in range(1 << 16):
            b = np.floor(x * inv)
            if b == target:
                return x
            x = np.nextafter(x, F(np.inf) if b < target else F(-np.inf))
        raise AssertionError(target)

    lo = find(-126 - extra, (-126 - extra + 0.5) * 0.2)
    hi = find(F(2.0 ** 31 - 128), (2.0 ** 31 - 128 + 0.5) * 0.2)
    xs = [lo, hi, np.nextafter(hi, F(-np.inf)), find(F(2.0 ** 31 - 256), (2.0 ** 31 - 256 + 0.5) * 0.2), F(0.1), F(-3.3)]
    return np.array([[x, 0.05, 0.05] for x in xs], F)


def extent_box(div, leaf=0.2):
    """Corners of a div^3-voxel box at `leaf`, from floor 0 to floor div - 1 on every axis, plus a few inner points."""
    inv = F(1.0) / F(leaf)
    hi = F((div - 1 + 0.5) * leaf)
    assert np.floor(hi * inv) == div - 1 and np.floor(F(0.5 * leaf) * inv) == 0
    c = np.array([[a, b, d] for a in (F(0.5 * leaf), hi) for b in (F(0.5 * leaf), hi) for d in (F(0.5 * leaf), hi)], F)
    return np.concatenate([c, c[:3] * F(0.5)])


def gate_grid(n, z=0.0, spacing=1.5, origin=(2.0, -3.0)):
    """n points on a z plane, `spacing` m apart: each its own voxel at 0.2 and 0.4 m before and after any rigid motion,
    and no point has a neighbour within the 1 m of the scan-to-map searches (the LM loop selects nothing)."""
    w = int(np.ceil(np.sqrt(n)))
    k = np.arange(n)
    return np.stack([origin[0] + spacing * (k % w), origin[1] + spacing * (k // w), np.full(n, z)], 1)


def catalogue(seed=17):
    rng = np.random.default_rng(seed)
    small = lambda n=40: pts(_blob(rng, n))  # noqa: E731
    cs = []
    add = lambda *a, **k: cs.append(Case(*a, **k))  # noqa: E731
    # empty clouds, each one alone and all three
    add("empty_corner", empty(), small(), small())
    add("empty_surf", small(), empty(), small())
    add("empty_outlier", small(), small(), empty())
    add("empty_all", empty(), empty(), empty())
    add("one_point", pts([[1.25, -0.5, 0.3]]), pts([[0.0, 0.0, 0.0]]), pts([[-7.0, 2.0, 1.0]]))
    for n in (31, 32, 33):
        add(f"n{n}", small(n), small(n), small(n))
    nan, inf = np.nan, np.inf
    add("all_nonfinite", pts([[nan, 0, 0], [0, nan, 0], [0, 0, nan]]), pts([[inf, 0, 0], [0, -inf, 0], [nan, inf, -inf]]),
        pts([[0, 0, inf]] * 5))
    ends = []
    for n in (3, 34, 70):
        a = _blob(rng, n)
        a[0, 0], a[-1, 2] = nan, -inf
        ends.append(pts(a))
    add("nonfinite_ends", *ends)
    add("voxel_faces", pts(_face_cloud(0.2)), pts(_face_cloud(0.4)), pts(np.concatenate([_face_cloud(0.2), _face_cloud(0.4)])))
    dense = rng.uniform(0.401, 0.599, (700, 3))
    dup = np.repeat(_blob(rng, 5), 40, axis=0)
    add("dense_voxel", pts(np.concatenate([dense, dup]), rng.uniform(0, 255, 900)), pts(dense[:300], rng.uniform(0, 255, 300)),
        pts(np.concatenate([dup, dup])))
    for off in (1e4, 1e5, 1e6, 4e6):
        c = (off, -0.5 * off, 0.25 * off)
        add(f"offset_{off:.0e}", pts(_blob(rng, 60, -3, 3, c)), pts(_blob(rng, 200, -5, 5, c)), pts(_blob(rng, 30, -5, 5, c)))
    add("extent_1290", pts(extent_box(1290)), small(), small())
    add("extent_1291", pts(extent_box(1291)), small(), small(), expect="toobig")
    add("int32_extent", pts(int32_extent(0)), small(), small())
    add("int32_extent_plus1", pts(int32_extent(1)), small(), small(), expect="toobig")
    add("far_coordinate", pts(far_pair()), small(), small())
    add("overflow_inf", small(), pts([[1.0, 2.0, 3.0], [-3e38, 0.0, 0.0]]), small(), expect="toobig")
    add("beyond_2p62", pts([[1e18, 0.0, 0.0], [1e18, 0.0, 0.0]]), small(), small(), expect="toobig")
    ni = rng.uniform(0, 10, 120)
    ni[::7] = nan
    add("nan_intensity", pts(_blob(rng, 120), ni), small(), small())
    # the map gate: the key frame's clouds come back as the next cycle's map, n_corner / n_surf points after DS
    for nc, ns in ((10, 100), (11, 100), (10, 101), (11, 101)):
        g = gate_grid(ns, z=-1.0)
        add(f"gate_{nc}_{ns}", pts(gate_grid(nc, z=2.0, origin=(-8.0, 5.0))), pts(g[: ns - ns // 3]), pts(g[ns - ns // 3:]))
    # after gate_11_101: a map that passes the gate and a scan with no corner query (none, or none finite)
    c = cs[-1].clouds
    add("nocorner_after_gate", empty(), c[1], c[2])
    add("nancorner_after_gate", pts(np.full((7, 3), np.nan)), c[1], c[2])
    return {c.name: c for c in cs}


def big_case(rng, n_corner, n_surf, n_outlier, name):
    return Case(name, pts(_blob(rng, n_corner, -30, 30)), pts(_blob(rng, n_surf, -40, 40)), pts(_blob(rng, n_outlier, -40, 40)))


# ---- episodes and the lockstep step plan -----------------------------------------------------------------------
GATE_POSE = ((0.0, 0.0, 0.0871557, 0.9961947), (3.5, -1.25, 0.75))  # 10 degrees of yaw and a translation
ZERO_POSE = ((0.0, 0.0, 0.0, 1.0), (0.0, 0.0, 0.0))
P_TARGETS = (1, 2, 3, 5, 8, 9, 25, 26, 51, 52, 102, 103, 128, 129, 160)
M_SLOTS = 160
BIG_ROUND = 600_000


class Episode:
    """Cycles (case names) of one drive between two resets, at one odometry pose."""

    def __init__(self, cases, pose):
        self.cases, self.pose = tuple(cases), pose


def episode_queue(cat, slot):
    """Slot s's endless queue of episodes: 1 to 3 cycles, the cases in a slot-dependent rotation; the gate cases run two
    cycles at GATE_POSE (the second cycle's map is the first's clouds; after gate_11_101 the second cycle may have no
    corner query), the toobig ones one cycle."""
    ok = [n for n, c in cat.items() if c.expect == "ok" and not n.startswith("gate_") and not n.endswith("_after_gate")]
    bad = [n for n, c in cat.items() if c.expect == "toobig"]
    gates = [[n] * 2 for n in cat if n.startswith("gate_")] + [["gate_11_101", n] for n in cat if n.endswith("_after_gate")]
    k = slot * 7
    while True:
        r = k % 11
        if r == 3:
            yield Episode(gates[(slot // 2 + k) % len(gates)], GATE_POSE)
        elif r == 8 and slot % 5 == 1:
            yield Episode([bad[(k // 11 + slot) % len(bad)]], ZERO_POSE)
        else:
            n = 1 + k % 3
            name = ok[(k + slot) % len(ok)]
            yield Episode([name] * n if k % 2 else [name, ok[(k + 3) % len(ok)]][:n], ZERO_POSE)
        k += 1


def step_plan(m=M_SLOTS):
    """[(processed slots, interval-skipped slots, big)]: per step which slots run a cycle and which send an odometry
    message 0.1 s after their last one; the others are absent.  One step per P of P_TARGETS (slot 0 and slot m - 1 are
    processed next to absent or skipped neighbours), and the big-round step (big = True: its processed slots run the
    big clouds of big_step_cases)."""
    plan = []
    for j, P in enumerate(P_TARGETS):
        if P == m:
            proc = list(range(m))
        elif j % 2 == 0:  # spread out, the first slot included
            proc = sorted({(i * m) // P for i in range(P)})
        else:  # a run at the end, the last slot included
            proc = list(range(m - P, m))
        assert len(proc) == P
        rest = [s for s in range(m) if s not in set(proc)]
        plan.append((proc, rest[::3], False))
        if j == 6:
            plan.append((BIG_SLOTS, [], True))
    return plan


BIG_SLOTS = [0, 1, 2, 5, 6, 9, 12, 13, 14, 159]  # big clouds in 0, 2, 6, 12, 14; tiny / empty / non-finite ones between


def big_step_cases(cat, seed=5):
    rng = np.random.default_rng(seed)
    big = iter(big_case(rng, 20_000, 90_000, 15_000, f"big{i}") for i in range(5))
    filler = iter(cat[n] for n in ("n31", "empty_all", "all_nonfinite", "one_point", "nonfinite_ends"))
    return {s: (next(big) if i % 2 == 0 else next(filler)) for i, s in enumerate(BIG_SLOTS)}


class Step:
    """One step of the plan.  reset: the slots reset before it; fail: {slot: event} of the slots whose cycle must fail
    the whole step with LINS_E_TOOBIG, tried first together with `events` (None: no such attempt); events: {slot:
    ("run" | "skip", event)} of the step that succeeds, event = (time, quat, pos, corner, surf, outlier)."""

    def __init__(self, reset, fail, events, big):
        self.reset, self.fail, self.events, self.big = reset, fail, events, big

    @property
    def P(self):
        return sum(1 for k, _ in self.events.values() if k == "run")

    def round1_points(self):
        """Points of the step's first VoxelGrid round when every processed slot starts an episode (no local map)."""
        return sum(sum(len(c) for c in ev[3:]) for k, ev in self.events.values() if k == "run")


def schedule(cat, m=M_SLOTS):
    """The steps of step_plan with every slot's episodes: a slot whose episode is done (or that starts the big round)
    is reset and starts its next one; a toobig episode is tried once in a failing attempt and then dropped."""
    queues = [episode_queue(cat, s) for s in range(m)]
    cur = [None] * m  # [episode, next cycle, last time]
    big = big_step_cases(cat)
    t0 = 100.0
    steps = []
    for proc, skip, is_big in step_plan(m):
        reset, fail, events = set(), {}, {}

        def start(s, ep):
            reset.add(s)
            cur[s] = [ep, 0, cur[s][2] if cur[s] else t0 + s]

        for s in proc:
            if is_big:
                start(s, Episode([big[s]], ZERO_POSE))
            elif cur[s] is None or cur[s][1] >= len(cur[s][0].cases):
                ep = next(queues[s])
                if cat[ep.cases[0]].expect == "toobig":
                    start(s, ep)
                    q, p = ep.pose
                    fail[s] = (cur[s][2] + 1.0, q, p) + cat[ep.cases[0]].clouds
                    ep = next(queues[s])
                start(s, ep)
            ep, k, t = cur[s]
            case = ep.cases[k] if isinstance(ep.cases[k], Case) else cat[ep.cases[k]]
            cur[s][1], cur[s][2] = k + 1, t + 1.0
            events[s] = ("run", (t + 1.0, ep.pose[0], ep.pose[1]) + case.clouds)
        for s in skip:
            if cur[s] is not None and cur[s][1] > 0:  # (a fresh episode's first message is always processed)
                ep, k, t = cur[s]
                case = ep.cases[k - 1] if isinstance(ep.cases[k - 1], Case) else cat[ep.cases[k - 1]]
                events[s] = ("skip", (t + 0.1, ep.pose[0], ep.pose[1]) + case.clouds)
        steps.append(Step(reset, fail or None, events, is_big))
    return steps
