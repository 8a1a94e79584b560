"""Seeded scene builders for row F2's 5-NN, fits and LM loop (lins_map.cuh), each asserting that it contains the edge it
is named after, so that a case cannot silently stop exercising it.  Nothing here needs a GPU; the grid checks use the
numpy model of the device grid in mapref.py (f32 emulation of the former cell rule, the exact rule, grid_hash and the
bucket count).

A case is a MapCase: the corner / surf map clouds and feature clouds (POINT_DTYPE), the transform of the pass and
`facts`, the counts the builder verified (straddling pairs, colliding buckets, cross-slice ties, ...)."""
import importlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mapref  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
_defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")
F = np.float32


def pts(xyz):
    """POINT_DTYPE cloud of (n, 3) coordinates, taken as f32 as they are."""
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    return _defs.make_points(xyz, np.zeros(len(xyz), F))


class MapCase:
    def __init__(self, name, corner_map, surf_map, corner_q, surf_q, T=None, **facts):
        self.name = name
        self.corner_map, self.surf_map = pts(corner_map), pts(surf_map)
        self.corner_q, self.surf_q = pts(corner_q), pts(surf_q)
        self.T = np.zeros(6, F) if T is None else np.asarray(T, F).copy()
        self.facts = facts

    def __repr__(self):
        return f"MapCase({self.name})"

    def clouds(self):
        return self.corner_map, self.surf_map, self.corner_q, self.surf_q


def _ulps(v, n, up):
    out, x = [], F(v)
    for _ in range(n):
        x = np.nextafter(x, F(np.inf) if up else F(-np.inf), dtype=F)
        out.append(x)
    return out


# ---- straddling pairs: f32 distance < 1, former cells two apart -----------------------------------------------------
def straddle_pair(o, k):
    """(lo, hi) f32 coordinates on one axis with origin o: hi - lo < 1 in f32 (and (hi - lo)^2 < 1), exact cells k - 1 and
    k, but the f32 differences floor to k - 1 and k + 1.  None if this (o, k) has none near o + k."""
    o = F(o)
    oo = np.array([o, 0, 0], F)
    cells = lambda v, rule: rule(np.stack([v, np.zeros_like(v), np.zeros_like(v)], -1).reshape(-1, 3), oo)[:, 0].reshape(v.shape)
    lo = np.array(_ulps(F(o + F(k)), 80, False), F)
    lo = lo[(cells(lo, mapref.cell_f32) == k - 1) & (cells(lo, mapref.cell_exact) == k - 1)]
    if len(lo) == 0:
        return None
    hi = (lo + F(1)).astype(F)[:, None]
    steps = [hi]
    for _ in range(80):
        steps.append(np.nextafter(steps[-1], F(-np.inf), dtype=F))
    hi = np.concatenate(steps[1:], 1)  # (lo, 80): hi below lo + 1
    dx = (hi - lo[:, None]).astype(F)
    ok = ((dx * dx).astype(F) < F(1)) & (cells(hi, mapref.cell_f32) == k + 1) & (cells(hi, mapref.cell_exact) == k)
    if not ok.any():
        return None
    i, j = np.argwhere(ok)[0]
    return lo[i], hi[i, j]


def straddle_pair_for(rng, k, tries=400):
    """A negative origin o and a straddling pair at offset k from it (they exist where |o + k| is small: there the
    coordinates resolve finer than the difference does)."""
    for _ in range(tries):
        o = F(-rng.uniform(0.05, 2 * k))
        p = straddle_pair(o, k)
        if p is not None:
            return o, p
    raise AssertionError(f"no straddling pair at offset {k}")


def worked_example():
    """The pair of DESIGN.md §4.4: origin -50, query x = 14 - 3 * 2^-20, map point x = 15 - 2^-18."""
    o, q, m = F(-50), F(14 - 3 * 2.0 ** -20), F(15 - 2.0 ** -18)
    return o, q, m


def _group(axis, normal, q_a, m_a, cn, ct, corner):
    """Five map points around a query that straddles along `axis`: four close ones, the straddler fifth.  Surf: all on
    the plane normal-coordinate = cn through the query; corner: near a line along `axis`, the query 0.01 m off it."""
    third = 3 - axis - normal
    def p(a, n, t):
        v = [0.0, 0.0, 0.0]
        v[axis], v[normal], v[third] = a, n, t
        return v
    q = p(q_a, cn, ct)
    if corner:  # four points on a line 0.01 m beside the query, the straddler level with it: not all on one line
        near = [p(F(q_a + d), F(cn + 0.01), ct) for d in (-0.3, -0.15, 0.15, 0.3)]
    else:
        near = [p(F(q_a + 0.3), cn, F(ct + 0.2)), p(F(q_a - 0.2), cn, F(ct + 0.3)),
                p(q_a, cn, F(ct - 0.25)), p(F(q_a + 0.1), cn, F(ct - 0.1))]
    return np.array(q, F), np.array(near + [p(m_a, cn, ct)], F)


def _check_straddles(mp, q, T, nb=None):
    """For every query: the reference's fifth neighbour is within 1 m, lies two former (f32) cells away on some axis
    and within one exact cell on every axis, and its bucket is not among the former block's.  Returns the count."""
    mp, qm = mapref.xyz(mp), mapref.associate_to_map(q, T)
    o = mapref.grid_origin(mp)
    nb = nb or mapref.n_buckets(len(mp))
    idx, dist = mapref.knn5(mp, qm)
    assert (dist[:, 4] < 1).all(), dist[:, 4]
    m5 = mp[idx[:, 4]]
    cq, cm = mapref.cell_f32(qm, o), mapref.cell_f32(m5, o)
    assert (np.abs(cm - cq) == 2).any(1).all(), "a query lost its straddling neighbour"
    assert (np.abs(mapref.cell_exact(m5, o) - mapref.cell_exact(qm, o)) <= 1).all()
    blocks = mapref.block_buckets(cq, nb)
    missed = mapref.grid_hash(cm) & np.uint64(nb - 1)
    assert not (blocks == missed[:, None]).any(1).any(), "a straddler's bucket is scanned anyway"
    return len(q)


def straddle_case(axis, above, corner, k, seed):
    """One straddling query (the neighbour above or below it along `axis`) in a corner or surf cloud, origin negative,
    the pair at offset k from it; the other cloud is a few far points."""
    rng = np.random.default_rng(seed)
    o, (lo, hi) = straddle_pair_for(rng, k)
    q_a, m_a = (lo, hi) if above else (hi, lo)
    normal = (axis + 1 + int(rng.integers(0, 2))) % 3
    origin = np.array([F(-rng.uniform(1, 30)) for _ in range(3)], F)
    origin[axis] = o
    for _ in range(200):
        cn, ct = (F(origin[(axis + j) % 3] + rng.uniform(3, 40)) for j in (1, 2))
        if normal != (axis + 1) % 3:
            cn, ct = ct, cn
        qv, grp = _group(axis, normal, q_a, m_a, cn, ct, corner)
        mp = np.concatenate([origin[None], grp])
        try:
            _check_straddles(mp, qv[None], np.zeros(6, F))
        except AssertionError:
            continue
        other = origin[None] + np.array([[0, 0, 0], [200, 0, 0], [0, 200, 0]], F)
        name = f"straddle-{'xyz'[axis]}-{'above' if above else 'below'}-{'corner' if corner else 'surf'}-2^{int(np.log2(k))}"
        if corner:
            return MapCase(name, mp, other, qv[None], np.zeros((0, 3), F), straddling_pairs=1)
        return MapCase(name, other, mp, np.zeros((0, 3), F), qv[None], straddling_pairs=1)
    raise AssertionError("no placement whose straddler's bucket stays outside the block")


def worked_example_case():
    o, q_a, m_a = worked_example()
    origin = np.array([o, -20, -10], F)
    for seed in range(100):
        rng = np.random.default_rng(seed)
        cn, ct = F(-20 + rng.uniform(3, 30)), F(-10 + rng.uniform(3, 30))
        qv, grp = _group(0, 1, q_a, m_a, cn, ct, False)
        mp = np.concatenate([origin[None], grp])
        try:
            _check_straddles(mp, qv[None], np.zeros(6, F))
        except AssertionError:
            continue
        return MapCase("worked-example", origin[None] + np.array([[0, 0, 0], [200, 0, 0]], F), mp, np.zeros((0, 3), F), qv[None],
                       straddling_pairs=1)
    raise AssertionError("worked example: no placement")


def straddle_cases():
    out = [worked_example_case()]
    seed = 100
    for axis in range(3):
        for above in (True, False):
            for corner in (False, True):
                for e in range(3, 11):
                    out.append(straddle_case(axis, above, corner, 2 ** e, seed))
                    seed += 1
    return out


def straddle_scene(seed=7, copies=6):
    """One scene for scan2map: every query straddles (each axis, both directions, corner and surf, an offset of 8..64
    per axis), with one origin for both clouds; the queries lie on their planes / beside their lines, so the first LM
    step is ~0 and the loop stops after one iteration."""
    rng = np.random.default_rng(seed)
    origin = np.zeros(3, F)
    pairs = {}
    for axis in range(3):  # an origin per axis with a straddling pair at an offset of 8..64
        while axis not in pairs:
            e = int(rng.integers(3, 7))
            o = F(-rng.uniform(0.05, 2 * 2 ** e))
            p = straddle_pair(o, 2 ** e)
            if p is not None:
                origin[axis], pairs[axis] = o, (e, p)
    n_groups = copies * 3 * 2  # per cloud
    nb = mapref.n_buckets(1 + 5 * n_groups)
    groups = {True: [], False: []}  # corner?
    slot = 0
    for rep in range(copies):
        for axis in range(3):
            normal = (axis + 1) % 3
            e, (lo, hi) = pairs[axis]
            for above in (True, False):
                for corner in (False, True):
                    q_a, m_a = (lo, hi) if above else (hi, lo)
                    while True:  # each straddle axis has its own region of the other two axes, 4 m between groups
                        base = F(100 + 80 * axis)
                        cn = F(origin[normal] + base + 4 * (slot % 16))
                        ct = F(origin[3 - axis - normal] + base + 4 * (slot // 16 % 16))
                        slot += 1
                        g = _group(axis, normal, q_a, m_a, cn, ct, corner)
                        try:  # (the group alone, with the scene's origin and bucket count)
                            _check_straddles(np.concatenate([origin[None], g[1]]), g[0][None], np.zeros(6, F), nb)
                        except AssertionError:
                            continue
                        groups[corner].append(g)
                        break
    out = {}
    for corner in (True, False):
        q = np.stack([g[0] for g in groups[corner]])
        mp = np.concatenate([origin[None]] + [g[1] for g in groups[corner]])
        out[corner] = (mp, q)
    n_c = _check_straddles(out[True][0], out[True][1], np.zeros(6, F))
    n_s = _check_straddles(out[False][0], out[False][1], np.zeros(6, F))
    assert len(out[False][0]) > 100 and len(out[True][0]) > 10 and n_c + n_s >= 50
    return MapCase("straddle-scene", out[True][0], out[False][0], out[True][1], out[False][1], straddling_pairs=n_c + n_s)


# ---- boundary-snapped fuzz, far maps ----------------------------------------------------------------------------------
def boundary_fuzz(seed, n_map=3000, n_q=1500):
    """Map points and queries within a few ulps of origin + k for many k, origins of mixed sign and magnitude."""
    rng = np.random.default_rng(seed)
    scale = [1, 50, 3000, 60000][seed % 4]
    origin = np.array([F(rng.uniform(-scale, scale)) for _ in range(3)], F)
    span = 12.0

    def snapped(n):
        k = rng.integers(1, int(span), (n, 3)).astype(np.float64)
        v = (origin.astype(np.float64) + k).astype(F)
        steps = rng.integers(-4, 5, (n, 3))
        for _ in range(4):
            mv = steps != 0
            v = np.where(mv, np.nextafter(v, np.where(steps > 0, F(np.inf), F(-np.inf)), dtype=F), v)
            steps = steps - np.sign(steps)
        free = rng.random((n, 3)) < 0.4  # some coordinates anywhere in the cell
        return np.where(free, (origin + rng.uniform(0, span, (n, 3))).astype(F), v)

    mp = np.concatenate([origin[None], snapped(n_map)])
    q = snapped(n_q)
    return MapCase(f"boundary-fuzz-{seed}", mp[: n_map // 3], mp, q[: n_q // 3], q)


def translated(case, off):
    """The same scene moved by `off` (3-vector), T's translation moved with it (the feature clouds stay)."""
    off = np.asarray(off, np.float64)
    mv = lambda c: (mapref.xyz(c).astype(np.float64) + off).astype(F)
    T = case.T.astype(np.float64).copy()
    T[3:] += off
    return MapCase(f"{case.name}+{off.tolist()}", mv(case.corner_map), mv(case.surf_map), mapref.xyz(case.corner_q),
                   mapref.xyz(case.surf_q), T.astype(F), **case.facts)


def plane_scene(seed, n_planes=12, n_q=1200, extent=20.0):
    """Planes and lines with noise: a generic scene whose queries are mostly accepted (the base of the far scenes)."""
    rng = np.random.default_rng(seed)
    surf, corner = [], []
    for _ in range(n_planes):
        nrm = rng.normal(size=3); nrm /= np.linalg.norm(nrm)
        c = rng.uniform(-extent, extent, 3)
        u = np.cross(nrm, [1, 0, 0] if abs(nrm[0]) < 0.9 else [0, 1, 0]); u /= np.linalg.norm(u)
        v = np.cross(nrm, u)
        ab = rng.uniform(-4, 4, (400, 2))
        surf.append(c + ab[:, :1] * u + ab[:, 1:] * v + rng.normal(0, 0.01, (400, 1)) * nrm)
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        corner.append(c + rng.uniform(-3, 3, (60, 1)) * d + rng.normal(0, 0.01, (60, 3)))
    surf, corner = np.concatenate(surf).astype(F), np.concatenate(corner).astype(F)
    sq = surf[rng.integers(0, len(surf), n_q)] + rng.normal(0, 0.05, (n_q, 3)).astype(F)
    cq = corner[rng.integers(0, len(corner), n_q // 4)] + rng.normal(0, 0.05, (n_q // 4, 3)).astype(F)
    T = np.array([0.01, -0.02, 0.015, 0.1, -0.05, 0.08], F)
    return MapCase(f"planes-{seed}", corner, surf, cq, sq, T)


FAR_OFFSETS = [[s * d if a == i else 0.0 for i in range(3)] for d in (1e3, 1e4, 6e4) for a in range(3) for s in (1, -1)]


def far_cases(base):
    """The scene translated by +-1e3, +-1e4 and +-6e4 m on each axis (the f32 ulp is ~4 mm at 6e4 m)."""
    return [translated(base, o) for o in FAR_OFFSETS]


# ---- hash collisions ------------------------------------------------------------------------------------------------
def collision_case(seed, n_cells=40, per_cell=100):
    """Distinct occupied cells found by search to share one bucket, so that the bucket a query block scans holds
    thousands of points of other cells; plus queries whose 27-cell block has cells that share a bucket."""
    rng = np.random.default_rng(seed)
    n_map = 1 + (n_cells - 1) * per_cell + 2 * 400
    nb = mapref.n_buckets(n_map)
    origin = np.array([-3.5, -7.25, -1.0], F)
    cand = rng.integers(2, 400, (400000, 3))
    h = mapref.grid_hash(cand) & np.uint64(nb - 1)
    # the query cell: one whose bucket many candidate cells share
    vals, counts = np.unique(h, return_counts=True)
    b0 = vals[np.argmax(counts)]
    cells = np.unique(cand[h == b0], axis=0)
    assert len(cells) > n_cells, len(cells)
    home, others = cells[0], cells[1:n_cells]
    pts_ = [origin[None]]
    for c in others:  # points of other cells in the home bucket
        pts_.append((origin + c + rng.uniform(0.05, 0.95, (per_cell, 3))).astype(F))
    home_pts = (origin + home + rng.uniform(0.05, 0.95, (400, 3))).astype(F)
    q_home = (origin + home + rng.uniform(0.2, 0.8, (200, 3))).astype(F)
    # a block with internal collisions: search a cell whose 27 block buckets repeat
    blk = mapref.block_buckets(cand[:20000], nb)
    dup = np.array([len(np.unique(r)) < 27 for r in blk])
    assert dup.any()
    cdup = cand[:20000][np.argmax(dup)]
    dup_pts = (origin + cdup + rng.uniform(-0.9, 1.9, (400, 3))).astype(F)
    q_dup = (origin + cdup + rng.uniform(0.0, 1.0, (200, 3))).astype(F)
    mp = np.concatenate(pts_ + [home_pts, dup_pts])
    assert len(mp) == n_map and mapref.n_buckets(len(mp)) == nb
    o = mapref.grid_origin(mp)
    assert np.array_equal(o, origin)
    hb = mapref.grid_hash(mapref.cell_exact(mp, o)) & np.uint64(nb - 1)
    in_home = int((hb == b0).sum()) - 400 - int((mapref.cell_exact(dup_pts, o) == home).all(1).sum())
    assert in_home >= 1000, in_home  # thousands of points of other cells share the home bucket
    n_dup_blocks = int(sum(len(np.unique(r)) < 27 for r in mapref.block_buckets(mapref.cell_exact(q_dup, o), nb)))
    assert n_dup_blocks > 0
    q = np.concatenate([q_home, q_dup])
    return MapCase(f"collisions-{seed}", mp[:500], mp, q[::4], q, colliding_cells=len(others) + 1, colliding_points=in_home,
                   blocks_with_shared_buckets=n_dup_blocks)


# ---- ties -----------------------------------------------------------------------------------------------------------
def copies_case(k, seed=0):
    """k copies of one point (k up to 8) among random points: the whole 5-NN is ties."""
    rng = np.random.default_rng(seed + k)
    base = F([1.25, -2.5, 0.75])
    other = rng.uniform(-10, 10, (300, 3)).astype(F)
    pos = rng.choice(len(other) + k, k, replace=False)
    mp = np.insert(other, np.sort(pos) - np.arange(k), base, axis=0)
    q = np.concatenate([base[None], (base + rng.normal(0, 0.05, (40, 3))).astype(F)])
    idx, dist = mapref.knn5(mp, q)
    assert (dist[0, : min(k, 5)] == 0).all()
    return MapCase(f"copies-{k}", mp, mp, q, q, tied_copies=k)


def lattice_case(seed=0):
    """Queries at lattice centres: 6 / 8 / 12 equidistant lattice points."""
    g = np.arange(-3, 4, dtype=F) * F(0.5)
    mp = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(F) + F(0.125)
    rng = np.random.default_rng(seed)
    mp = mp[rng.permutation(len(mp))]
    inner = mp[(np.abs(mp - F(0.125)) <= F(1.0)).all(1)][:20]
    q = np.concatenate([inner, inner + F(0.25), inner + np.array([0.25, 0.25, 0], F)]).astype(F)
    idx, dist = mapref.knn5(mp, q)
    assert (dist[:, 3] == dist[:, 4]).sum() >= 40  # the fifth ties the fourth: the lower index decides
    return MapCase("lattice", mp, mp, q, q)


def slice_ties_case(n_map=64 * 256, seed=0):
    """For the brute-force kernel: a map of 64 x 256 points (64 slices of 256 with few queries) with exact duplicates
    placed in different slices, some on the two sides of a slice boundary."""
    rng = np.random.default_rng(seed)
    mp = rng.uniform(-40, 40, (n_map, 3)).astype(F)
    slice_len = n_map // 64
    src = rng.choice(n_map, 200, replace=False)
    ties = 0
    for j, s in enumerate(src):
        if j < 60:  # the two sides of a slice boundary
            b = slice_len * int(rng.integers(1, 64))
            a, c = b - 1, b
        else:
            a, c = rng.choice(n_map, 2, replace=False)
        mp[a] = mp[s]
        mp[c] = mp[s]
    q = np.concatenate([mp[src] + rng.normal(0, 0.02, (len(src), 3)).astype(F), mp[src]]).astype(F)
    idx, dist = mapref.knn5(mp, q)
    for r in range(len(q)):  # equal distances whose indices lie in different slices
        for a in range(5):
            for b in range(a + 1, 5):
                if idx[r, a] >= 0 and idx[r, b] >= 0 and dist[r, a] == dist[r, b] and idx[r, a] // slice_len != idx[r, b] // slice_len:
                    ties += 1
    assert ties >= 100, ties
    return MapCase("slice-ties", mp[:2000], mp, q[:64], q, cross_slice_ties=ties)


# ---- sparse and non-finite ---------------------------------------------------------------------------------------------
def sparse_cases(seed=0):
    rng = np.random.default_rng(seed)
    out = []
    cen = F([0.5, -0.25, 1.0])
    for n in range(7):
        mp = (cen + rng.uniform(-0.5, 0.5, (n, 3))).astype(F)
        q = (cen + rng.uniform(-0.6, 0.6, (16, 3))).astype(F)
        out.append(MapCase(f"map-of-{n}", mp, mp, q, q))
    surf = (cen + rng.uniform(-2, 2, (300, 3))).astype(F)
    out.append(MapCase("empty-corner-map", np.zeros((0, 3), F), surf, (cen + rng.uniform(-1, 1, (20, 3))).astype(F), surf[:50]))
    # fewer than five points in the query's block: four close points, the rest > 2 m away
    mp = np.concatenate([(cen + rng.uniform(-0.3, 0.3, (4, 3))).astype(F), (cen + F(5) + rng.uniform(0, 1, (30, 3))).astype(F)])
    out.append(MapCase("four-in-block", mp, mp, cen[None], cen[None]))
    # the fifth distance exactly 1.0f and the float just below it
    q = F([0.0, 3.0, 4.0])  # (x = 0: 1 - 2^-24 is exact there)
    near = [q + F([0.1, 0, 0]), q + F([0, 0.1, 0]), q + F([0, 0, 0.1]), q - F([0.1, 0, 0])]
    at1 = q + F([1.0, 0, 0])
    below = None
    for dy in (2.0 ** -12, 2.0 ** -12 + 2.0 ** -30, 3 * 2.0 ** -13):
        cand = np.array([q[0] + F(1 - 2.0 ** -24), q[1] + F(dy), q[2]], F)
        if mapref.sqdist(q, cand) == np.nextafter(F(1), F(0), dtype=F):
            below = cand
            break
    assert below is not None and mapref.sqdist(q, at1) == F(1)
    for nm, p5 in (("fifth-at-1", at1), ("fifth-below-1", below)):
        mp = np.array(near + [p5], F)
        out.append(MapCase(nm, mp, mp, q[None], q[None]))
    return out


def nonfinite_case(seed=0):
    """NaN and +-inf in map points and queries; queries at 1e30 and beyond 2^31 m from the origin (saturated cells)."""
    rng = np.random.default_rng(seed)
    mp = rng.uniform(-5, 5, (600, 3)).astype(F)
    bad = rng.choice(len(mp), 40, replace=False)
    vals = np.array([np.nan, np.inf, -np.inf], F)
    mp[bad, rng.integers(0, 3, 40)] = vals[rng.integers(0, 3, 40)]
    q = (mp[rng.integers(0, len(mp), 100)] + rng.normal(0, 0.1, (100, 3))).astype(F)
    extra = []
    for v in (np.nan, np.inf, -np.inf, 1e30, -1e30, 2.0 ** 31 + 4096, -(2.0 ** 31) - 4096, 3e9, 3e38):
        for a in range(3):
            p = np.array([0.5, 0.5, 0.5], F)
            p[a] = F(v)
            extra.append(p)
    q = np.concatenate([q, np.array(extra, F)])
    o = mapref.grid_origin(mp)
    sat = mapref.cell_exact(q, o)
    assert ((sat == mapref.INT_MAX) | (sat == mapref.INT_MIN)).any()
    return MapCase("non-finite", mp, mp, q, q)


# ---- degenerate fits ----------------------------------------------------------------------------------------------------
def degenerate_fit_case():
    """Five identical neighbours; five axis-aligned collinear surf neighbours (the QR fails); an isotropic corner
    covariance; a corner query at the centroid of its line; a surf query at the origin."""
    groups, qs = [], []
    c1 = F([3.0, 4.0, 5.0])  # five identical
    groups.append(np.repeat(c1[None], 5, 0)); qs.append(c1 + F([0.1, 0, 0]))
    c2 = F([10.0, 4.0, 5.0])  # collinear along x
    groups.append(np.array([c2 + F([d, 0, 0]) for d in (-0.4, -0.2, 0.0, 0.2, 0.4)], F)); qs.append(c2 + F([0, 0.05, 0]))
    c3 = F([3.0, 12.0, 5.0])  # regular tetrahedron + centre: isotropic covariance
    tet = F(0.3) * np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1], [0, 0, 0]], F)
    groups.append((c3 + tet).astype(F)); qs.append(c3)
    c4 = F([10.0, 12.0, 5.0])  # the query at the centroid of its line
    groups.append(np.array([c4 + F([d, 0, 0]) for d in (-0.4, -0.2, 0.0, 0.2, 0.4)], F)); qs.append(c4)
    c5 = F([0.0, 0.0, 0.0])  # a surf query at the origin, on a plane through it
    groups.append(np.array([[0.3, 0, 0], [0, 0.3, 0], [-0.3, 0, 0], [0, -0.3, 0], [0.2, 0.2, 0]], F)); qs.append(c5)
    mp = np.concatenate(groups)
    q = np.array(qs, F)
    idx, dist = mapref.knn5(mp, q)
    assert (dist[:, 4] < 1).all() and all(set(idx[i] // 5) == {i} for i in range(len(q)))
    return MapCase("degenerate-fits", mp, mp, q, q)


def corridor_scene(seed=3, n_map=6000, n_q=1500):
    """Two parallel walls (y = +-2) and the ground (z = -1.5) along x, nothing across x: the LM system has no constraint
    along the corridor, so iteration 0 finds eigenvalues < 100 (isDegenerate)."""
    rng = np.random.default_rng(seed)

    def sample(n):
        x = rng.uniform(-30, 30, n)
        w = rng.integers(0, 3, n)
        a = rng.uniform(-2, 2, n)
        b = rng.uniform(-1.5, 1.5, n)
        y = np.where(w == 0, 2.0, np.where(w == 1, -2.0, a))
        z = np.where(w == 2, -1.5, b)
        return np.stack([x, y, z], 1).astype(F)

    surf = sample(n_map)
    edges = np.stack([rng.uniform(-30, 30, 400), np.where(rng.random(400) < 0.5, 2.0, -2.0), np.full(400, -1.5)], 1).astype(F)
    sq, cq = sample(n_q), edges[rng.integers(0, 400, 100)] + np.array([rng.uniform(-0.1, 0.1), 0, 0], F)
    T = np.array([0.004, -0.003, 0.01, 0.25, 0.08, -0.06], F)
    return MapCase("corridor", edges, surf, cq.astype(F), sq, T)


def ground_only_scene(seed=4, n_map=3000, n_q=800):
    """All surf points on the plane z = -1.5 (corners on two lines in it): the 6 x 6 system has zero columns, its QR
    fails and the step is X = 0."""
    rng = np.random.default_rng(seed)
    g = lambda n: np.stack([rng.uniform(-20, 20, n), rng.uniform(-20, 20, n), np.full(n, -1.5)], 1).astype(F)
    edges = np.stack([rng.uniform(-20, 20, 200), np.where(rng.random(200) < 0.5, 3.0, -3.0), np.full(200, -1.5)], 1).astype(F)
    T = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.2], F)
    return MapCase("ground-only", edges, g(n_map), edges[:30], g(n_q), T)


def all_pass_cases():
    """Every case of this module that a single associate pass is compared on."""
    base = plane_scene(1)
    return (straddle_cases() + [straddle_scene()] + [boundary_fuzz(s) for s in range(4)] + [base] + far_cases(base)
            + [collision_case(0), collision_case(1)] + [copies_case(k) for k in range(1, 9)] + [lattice_case(), slice_ties_case()]
            + sparse_cases() + [nonfinite_case(), degenerate_fit_case(), corridor_scene(), ground_only_scene()])
