"""Segmented scans for the feature-extraction tests — TEST INFRASTRUCTURE.

Simulated sweeps go through the product's host image projection (tools/synth lins_frontend_run) to give what processPCL
receives: the segmented cloud and cloud_info.  `host_features` runs the host FeatureExtractor
(csrc/host/feature_extraction.hpp, through tools/synth lins_features_host) on any such scan, hand-built ones included.
Scans are dicts: seg (m x 4 float32 x, y, z, intensity), ground (u8), col (u32), range (f32), start_ring / end_ring
(line_num int32), ori (3 float32: start, end, diff).
"""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
NAMES = ("surf_flat", "corner_sharp", "surf_less_flat", "corner_less_sharp")
LIDARS = {0: (16, 1800), 1: (64, 1024)}  # lins_frontend_run lidar_model -> (line_num, scan_num)

_L = None


def _lib(defs):
    global _L
    if _L is None:
        L = C.CDLL(os.path.join(ROOT, "tools", "synth", "liblins_synth.so"))
        vp = C.c_void_p
        L.lins_synth_raw_sweep.argtypes = [vp, C.c_uint64, vp, C.c_int]
        L.lins_frontend_run.argtypes = [vp, C.c_int, C.c_int, C.c_int] + [vp] * 13 + [vp]
        L.lins_features_host.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp] + [vp] * 6
        _L = L
    return _L


def _x4(a, k=None):
    return np.stack([a["x"], a["y"], a["z"], a["intensity"]], 1).astype(F)[:k]


def _pts(defs, xyzi):
    xyzi = np.asarray(xyzi, F).reshape(-1, 4)
    p = np.zeros(max(len(xyzi), 1), defs.POINT_DTYPE)
    p["x"][: len(xyzi)], p["y"][: len(xyzi)], p["z"][: len(xyzi)], p["intensity"][: len(xyzi)] = xyzi.T
    p["pad0"] = 1.0
    return p


def segmented(synth, defs, config, seed):
    """One simulated sweep of synth.CONFIGS[config] through the host image projection: a scan dict + line_num."""
    L = _lib(defs)
    cfg = synth.SynthCfg(**synth.CONFIGS[config])
    model = int(synth.CONFIGS[config]["lidar"])
    line_num, scan_num = LIDARS[model]
    cap = line_num * scan_num
    raw = np.zeros(cap, defs.POINT_DTYPE)
    n = L.lins_synth_raw_sweep(C.byref(cfg), seed, defs.ptr(raw), cap)
    P = lambda: np.zeros(cap, defs.POINT_DTYPE)  # noqa: E731
    seg, outl, und, a, b, c, d = P(), P(), P(), P(), P(), P(), P()
    sr, er, ori = np.zeros(line_num, np.int32), np.zeros(line_num, np.int32), np.zeros(3, F)
    ground, col, rng, cnt = np.zeros(cap, np.uint8), np.zeros(cap, np.uint32), np.zeros(cap, F), np.zeros(6, np.int32)
    rc = L.lins_frontend_run(defs.ptr(raw), n, model, cap, *[defs.ptr(v) for v in (seg, outl, sr, er, ori, ground, col, rng, und, a, b, c, d, cnt)])
    assert rc == 0
    m = int(cnt[0])
    return dict(seg=_x4(seg, m), ground=ground[:m].copy(), col=col[:m].copy(), range=rng[:m].copy(), start_ring=sr, end_ring=er, ori=ori), line_num


def host_features(defs, scan, line_num, edge=0.5, surf=0.5, angle=0.0, scan_period=0.1):
    """FeatureExtractor::run on the scan: dict of the four clouds (k x 4 float32) and undist."""
    L = _lib(defs)
    n = len(scan["seg"])
    seg = _pts(defs, scan["seg"])
    A = lambda v, t: np.ascontiguousarray(np.asarray(v, t).reshape(-1) if n or t != F else np.zeros(1, t))  # noqa: E731
    ground, col, rng = A(scan["ground"], np.uint8), A(scan["col"], np.uint32), A(scan["range"], F)
    sr, er, ori = A(scan["start_ring"], np.int32), A(scan["end_ring"], np.int32), A(scan["ori"], F)
    assert len(sr) == line_num and len(er) == line_num
    prm = np.array([edge, surf, angle, scan_period], np.float64)
    outs = [np.zeros(max(n, 1), defs.POINT_DTYPE) for _ in range(5)]
    cnt = np.zeros(4, np.int32)
    g1, c1, r1 = (np.zeros(1, t) if n == 0 else v for v, t in ((ground, np.uint8), (col, np.uint32), (rng, F)))
    L.lins_features_host(defs.ptr(seg), n, line_num, defs.ptr(sr), defs.ptr(er), defs.ptr(ori), defs.ptr(g1), defs.ptr(c1), defs.ptr(r1),
                         defs.ptr(prm), *[defs.ptr(o) for o in outs], defs.ptr(cnt))
    res = {k: _x4(outs[1 + i], int(cnt[i])) for i, k in enumerate(NAMES)}
    res["undist"] = _x4(outs[0], n)
    return res


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, F), np.ascontiguousarray(b, F)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- hand-built scans -------------------------------------------------------------------------------------------------
def ring_scan(rings, line_num=None, ori=None):
    """A scan from per-ring lists of (x, y, z, range, col, ground) rows, concatenated ring after ring with the LeGO-LOAM
    cloud_info layout (startRingIndex = first point + 4, endRingIndex = last point - 6, i.e. 10 points of gap between rings)
    unless `abut` rows are given in ranges.  intensity = ring index (image projection's ring + col / 10000 truncates to it)."""
    line_num = line_num or len(rings)
    seg, ground, col, rng, sr, er = [], [], [], [], np.zeros(line_num, np.int32), np.zeros(line_num, np.int32)
    for i in range(line_num):
        rows = rings[i] if i < len(rings) else []
        sr[i] = len(seg) - 1 + 5
        for (x, y, z, r, c, g) in rows:
            seg.append((x, y, z, i + c / 10000.0))
            rng.append(r); col.append(c); ground.append(g)
        er[i] = len(seg) - 1 - 5
    seg = np.asarray(seg, F).reshape(-1, 4)
    if ori is None:
        ori = _orientation(seg)
    return dict(seg=seg, ground=np.asarray(ground, np.uint8), col=np.asarray(col, np.uint32), range=np.asarray(rng, F),
                start_ring=sr, end_ring=er, ori=np.asarray(ori, F))


def _orientation(seg):
    import math
    if len(seg) < 2:
        return (0.0, 2 * math.pi, 2 * math.pi)
    start = -math.atan2(float(seg[0, 1]), float(seg[0, 0]))
    end = -math.atan2(float(seg[-1, 1]), float(seg[-2, 0])) + 2 * math.pi
    if end - start > 3 * math.pi:
        end -= 2 * math.pi
    elif end - start < math.pi:
        end += 2 * math.pi
    return (F(start), F(end), F(F(end) - F(start)))


def sweep_ring(n, radius, z, ground=0, rng=None, col0=0, noise=0.0, bumps=(), a0=-3.141592653589793):
    """n points of one ring sweeping a full turn clockwise (ori increasing), range = radius (+ noise), with optional
    (index, extra range) bumps that make corners."""
    import math
    rows = []
    for k in range(n):
        a = a0 + (k + 0.25) * 2 * math.pi / n
        r = radius + (rng.normal(0, noise) if rng is not None and noise else 0.0)
        for (bi, br) in bumps:
            if k == bi:
                r += br
        # ori = -atan2(y, x) = a  ->  y = -sin(a)
        rows.append((r * math.cos(a), -r * math.sin(a), z, r, col0 + k, ground))
    return rows
