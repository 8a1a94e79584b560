"""Independent numpy / scipy restatement of the mapping node's exact 5-NN (row F2, lidar_mapping_node.cpp:1371-1372,
:1479-1480: nearestKSearch(k = 5) on the map clouds) and of the grid the device searches it with (lins_map.cuh).

The 5-NN as the reference defines it:
  * f32 ((dx*dx)+dy*dy)+dz*dz between the query, taken to the map frame by pointAssociateToMap in f32, and each point;
  * ascending (distance, index): among equal distances the lower index wins;
  * index -1 and distance +inf where fewer than five points remain; NaN and +inf distances are never taken.
sin / cos of the transform come from libm's sinf / cosf (the host side of lins_map.cu and the oracle use libm), not
from np.sin on float32, which may differ by an ulp.

Large inputs are pruned with a float64 cKDTree at radius 1 + 1e-3: an f32 distance < 1 implies a true distance
< 1 + 1e-6, so every neighbour the 1 m gate can accept is among the candidates, whose exact f32 distances are then
recomputed.  A pruned search is exact for the points whose fifth distance is < 1; for the others it reports only the
candidates it saw.

This module deliberately imports nothing of the oracle, the library or the reference."""
import ctypes
import ctypes.util

import numpy as np
from scipy.spatial import cKDTree

F = np.float32
PRUNE_RADIUS = 1.0 + 1e-3

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
for _fn in ("sinf", "cosf"):
    getattr(_libm, _fn).restype = ctypes.c_float
    getattr(_libm, _fn).argtypes = [ctypes.c_float]


def sinf(v):
    return F(_libm.sinf(float(F(v))))


def cosf(v):
    return F(_libm.cosf(float(F(v))))


def xyz(cloud):
    """(n, 3) float32 of a POINT_DTYPE cloud or an (n, >=3) array."""
    a = np.asarray(cloud)
    if a.dtype.names:
        return np.stack([a["x"], a["y"], a["z"]], 1).astype(F)
    a = np.asarray(a, F)
    return (a if a.ndim == 2 else a.reshape(len(a), -1))[:, :3].copy()


def associate_to_map(p, T):
    """pointAssociateToMap (:594-608), every operation rounded to f32 in the reference's order."""
    T = np.asarray(T, F)
    cR, sR, cP, sP, cY, sY = cosf(T[0]), sinf(T[0]), cosf(T[1]), sinf(T[1]), cosf(T[2]), sinf(T[2])
    p = xyz(p)
    with np.errstate(over="ignore", invalid="ignore"):
        x1 = cY * p[:, 0] - sY * p[:, 1]
        y1 = sY * p[:, 0] + cY * p[:, 1]
        z1 = p[:, 2]
        y2 = cR * y1 - sR * z1
        z2 = sR * y1 + cR * z1
        return np.stack([(cP * x1 + sP * z2) + T[3], y2 + T[4], (-sP * x1 + cP * z2) + T[5]], 1).astype(F)


def sqdist(q, m):
    """f32 ((dx*dx)+dy*dy)+dz*dz, broadcasting; NaN where an input is NaN."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = (q - m).astype(F)
        return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(F)


def _select(r, j, d, n_q):
    """From candidate triples (query row, map index, f32 distance): the five smallest (distance, index) per row."""
    idx = np.full((n_q, 5), -1, np.int32)
    dist = np.full((n_q, 5), np.inf, F)
    ok = d < np.inf  # (NaN compares false too)
    r, j, d = r[ok], j[ok], d[ok]
    o = np.lexsort((j, d, r))
    r, j, d = r[o], j[o], d[o]
    rank = np.arange(len(r)) - np.searchsorted(r, r, side="left")
    k = rank < 5
    idx[r[k], rank[k]] = j[k]
    dist[r[k], rank[k]] = d[k]
    return idx, dist


def knn5_brute(mp, q, chunk_elems=1 << 24):
    """Exact 5-NN of every query (rows of q, map frame) among the map points mp: (idx int32 (n, 5), dist f32 (n, 5))."""
    mp, q = xyz(mp), xyz(q)
    n_q, n_m = len(q), len(mp)
    if n_m == 0 or n_q == 0:
        return np.full((n_q, 5), -1, np.int32), np.full((n_q, 5), np.inf, F)
    idx, dist = [], []
    step = max(1, chunk_elems // n_m)
    for a in range(0, n_q, step):
        D = sqdist(q[a:a + step, None, :], mp[None, :, :])
        D = np.where(D < np.inf, D, F(np.inf))
        k = min(5, n_m)
        thr = np.partition(D, k - 1, axis=1)[:, k - 1]
        r, j = np.nonzero((D <= thr[:, None]) & (D < np.inf))  # every key that can be among the five, ties included
        i5, d5 = _select(r, j.astype(np.int64), D[r, j], len(D))
        idx.append(i5); dist.append(d5)
    return np.concatenate(idx), np.concatenate(dist)


def knn5_pruned(mp, q):
    """5-NN through a float64 cKDTree at radius 1 + 1e-3; exact wherever the fifth distance is < 1."""
    mp, q = xyz(mp), xyz(q)
    n_q = len(q)
    fm = np.flatnonzero(np.isfinite(mp).all(1))
    fq = np.flatnonzero(np.isfinite(q).all(1))
    if len(fm) == 0 or len(fq) == 0:
        return np.full((n_q, 5), -1, np.int32), np.full((n_q, 5), np.inf, F)
    tm = cKDTree(mp[fm].astype(np.float64))
    tq = cKDTree(q[fq].astype(np.float64))
    pairs = tq.sparse_distance_matrix(tm, PRUNE_RADIUS, output_type="ndarray")
    r, j = fq[pairs["i"]], fm[pairs["j"]]
    return _select(r, j, sqdist(q[r], mp[j]), n_q)


def knn5(mp, q, prune=None):
    """Exact 5-NN; prune=None prunes when the brute-force work would exceed ~2e9 distances."""
    n = len(xyz(mp)) * len(xyz(q))
    if prune is None:
        prune = n > 2_000_000_000
    return knn5_pruned(mp, q) if prune else knn5_brute(mp, q)


def associate_knn(corner_map, surf_map, corner_q, surf_q, T, prune=None):
    """The five neighbour indices / distances of one cornerOptimization + surfOptimization pass at transform T."""
    out = {}
    for name, mp, q in (("corner", corner_map, corner_q), ("surf", surf_map, surf_q)):
        out[name + "_knn"], out[name + "_dist"] = knn5(mp, associate_to_map(q, T), prune)
    return out


# ---- the device grid (lins_map.cuh: grid_cell, grid_hash; lins_map.cu: map_grid_origin, map_fill_table) ------------
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1


def grid_origin(mp):
    """The finite minimum per axis (|v| < 1e30), 0 on an axis without one."""
    mp = xyz(mp)
    o = np.zeros(3, F)
    for k in range(3):
        v = mp[:, k]
        v = v[np.isfinite(v) & (np.abs(v) < F(1e30))]
        if len(v):
            o[k] = v.min()
    return o


def n_buckets(n):
    nb = 4096
    while nb < 2 * n and nb < (1 << 24):
        nb <<= 1
    return nb


def _sat_floor(v):
    """floor, saturated to int32, NaN -> 0 (the device's float -> int conversions)."""
    with np.errstate(invalid="ignore"):
        f = np.floor(np.asarray(v, np.float64))
        f = np.where(np.isnan(f), 0.0, np.clip(f, INT_MIN, INT_MAX))
    return f.astype(np.int64)


def cell_f32(p, o):
    """The former rule: floorf of the f32 difference x - ox."""
    with np.errstate(over="ignore", invalid="ignore"):
        return _sat_floor((xyz(p) - np.asarray(o, F)).astype(F))


def cell_exact(p, o):
    """The device's rule: floor of the difference taken in f64."""
    with np.errstate(over="ignore", invalid="ignore"):
        return _sat_floor(xyz(p).astype(np.float64) - np.asarray(o, F).astype(np.float64))


def grid_hash(c):
    """((ix * 73856093) ^ (iy * 19349663) ^ (iz * 83492791)) in uint32 of (n, 3) int cells."""
    c = (np.asarray(c, np.int64) & 0xFFFFFFFF).astype(np.uint64)
    h = (c[..., 0] * np.uint64(73856093)) ^ (c[..., 1] * np.uint64(19349663)) ^ (c[..., 2] * np.uint64(83492791))
    return (h & np.uint64(0xFFFFFFFF)).astype(np.uint64)


BLOCK = np.array([(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)], np.int64)


def block_buckets(cell, nb):
    """The buckets a query in `cell` scans: its 3 x 3 x 3 block, neighbour arithmetic wrapping in uint32."""
    return grid_hash((np.asarray(cell, np.int64)[..., None, :] + BLOCK) & 0xFFFFFFFF) & np.uint64(nb - 1)
