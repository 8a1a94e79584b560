"""GPU suite: lins_gpu_extract_features (csrc/cuda/lins_features.cu) against the host FeatureExtractor
(csrc/host/feature_extraction.hpp) bit for bit — the four clouds, the de-skewed cloud and the counts — on simulated sweeps
in one batch, permuted, alone, and on hand-built scans that reach each corner of the extraction; against tests/pyfront.py
where equal curvatures decide a pick.  Invalid input returns its code and leaves the next call's result unchanged."""
import ctypes as C
import math

import numpy as np
import pytest

import featcases as fc
import pyfront

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu(capi, defs):
    return capi.LinsGpu(defs.LinsParams.shipped(), device=0)


def _pad_rings(scan, line_num):
    """The same scan with line_num rings: the extra rings are empty (start = end = 0: no visited sextant)."""
    s = dict(scan)
    k = len(scan["start_ring"])
    s["start_ring"] = np.concatenate([scan["start_ring"], np.zeros(line_num - k, np.int32)])
    s["end_ring"] = np.concatenate([scan["end_ring"], np.zeros(line_num - k, np.int32)])
    return s


def _check(defs, dev, scans, line_num, **kw):
    for i, s in enumerate(scans):
        h = fc.host_features(defs, s, line_num, **kw)
        for k in fc.NAMES + ("undist",):
            assert fc.same_bits(dev[i][k], h[k]), f"scan {i}: {k} differs ({len(dev[i][k])} vs {len(h[k])} points)"


@pytest.fixture(scope="module")
def sweeps(synth, defs):
    scans = []
    for config, seeds in (("config3", range(100, 180)), ("config1", range(200, 270)), ("config4", range(300, 355))):
        for seed in seeds:
            s, ln = fc.segmented(synth, defs, config, seed)
            scans.append(_pad_rings(s, 64))
    return scans


def test_batch_of_sweeps_matches_host(gpu, defs, sweeps):
    assert len(sweeps) >= 200
    dev = gpu.extract_features(sweeps, line_num=64, undist=True)
    _check(defs, dev, sweeps, 64)
    assert sum(len(d["corner_sharp"]) for d in dev) > 1000 and sum(len(d["surf_less_flat"]) for d in dev) > 100000
    ms = gpu.extract_ms()
    assert ms > 0


def test_permuted_and_single_scans(gpu, defs, sweeps):
    ref = gpu.extract_features(sweeps, line_num=64, undist=True)
    perm = np.random.default_rng(5).permutation(len(sweeps))
    dev = gpu.extract_features([sweeps[i] for i in perm], line_num=64, undist=True)
    for j, i in enumerate(perm):
        for k in fc.NAMES + ("undist",):
            assert fc.same_bits(dev[j][k], ref[i][k])
    for i in (0, 90, len(sweeps) - 1):
        one = gpu.extract_features([sweeps[i]], line_num=64, undist=True)[0]
        for k in fc.NAMES + ("undist",):
            assert fc.same_bits(one[k], ref[i][k])


def _rng_ring(rng, n, radius, z, ground, col0=0, bumps=()):
    return fc.sweep_ring(n, radius, z, ground=ground, rng=rng, col0=col0, noise=0.02, bumps=bumps)


def _scene(name):
    rng = np.random.default_rng(sum(name.encode()))
    if name == "empty":
        return fc.ring_scan([[], []]), {}
    if name == "tiny":  # fewer than 11 points: no curvature is computed
        return fc.ring_scan([_rng_ring(rng, 8, 5.0, -1.0, 1)]), {}
    if name == "empty_and_short_rings":
        return fc.ring_scan([[], _rng_ring(rng, 14, 6.0, -1.0, 1), [], _rng_ring(rng, 300, 7.0, 0.5, 0), _rng_ring(rng, 9, 8.0, 1.0, 0)]), {}
    if name == "ring0_default_entry":  # point 0 is ground: the (value 0, ind 0) entries of ring 0 pick it as flat
        return fc.ring_scan([_rng_ring(rng, 400, 6.0, -1.5, 1), _rng_ring(rng, 400, 7.0, 0.0, 0)]), {}
    if name == "many_corners":  # > 20 corner candidates in one sextant
        bumps = [(k, 0.1) for k in range(10, 1800, 8)]
        return fc.ring_scan([fc.sweep_ring(1800, 6.0, 0.0, rng=rng, noise=0.005, bumps=bumps)]), {}
    if name == "column_jump":  # column indices jump by > 10 every 7 points: suppression stops there
        rows = _rng_ring(rng, 420, 6.0, -1.0, 1)
        rows = [(x, y, z, r, c + 20 * (k // 7), g) for k, (x, y, z, r, c, g) in enumerate(rows)]
        return fc.ring_scan([rows, _rng_ring(rng, 420, 8.0, 0.3, 0, bumps=[(k, 0.1) for k in range(5, 420, 9)])]), {}
    if name == "abutting_rings":  # no gap: a corner 3 points before ring 0's end suppresses ring 1's first candidates
        return abutting_scene(0), {}
    if name == "fourth_flat":  # the 4th flat point of sextant 0 sits next to sextant 1: suppressing it would change a pick
        return fourth_flat_scene(8), {}
    if name == "wrap_half_passed":  # orientations wrap through +-pi: halfPassed is set half-way
        return fc.ring_scan([fc.sweep_ring(500, 6.0, -1.0, ground=1, rng=rng, noise=0.02, a0=-math.pi / 2),
                             fc.sweep_ring(500, 9.0, 0.5, ground=0, rng=rng, noise=0.02, a0=-math.pi / 2, bumps=[(250, 0.1)])]), {}
    if name == "extrinsic_angle":
        return fc.ring_scan([_rng_ring(rng, 500, 6.0, -1.0, 1), _rng_ring(rng, 500, 9.0, 0.5, 0, bumps=[(77, 0.1)])]), dict(angle=17.5)
    if name == "negative_voxels":  # all coordinates negative; one voxel of hundreds of points
        rows = []
        for k in range(700):
            x, y = -3.05 - 0.0001 * (k % 13), -4.07 - 0.0001 * (k % 7)
            rows.append((x, y, -1.13, 5.0 + rng.normal(0, 0.01), k, 1 if k % 3 else 0))
        return fc.ring_scan([rows], ori=(-2.0, 4.0, 6.0)), {}
    raise KeyError(name)


SCENES = ["empty", "tiny", "empty_and_short_rings", "ring0_default_entry", "many_corners", "column_jump", "abutting_rings",
          "fourth_flat", "wrap_half_passed", "extrinsic_angle", "negative_voxels"]


def abutting_scene(seed):
    """Three rings with no gap (visited ranges [5, 239], [240, 479], [480, 713]) and continuous column indices: ring 0's
    corner at 237 suppresses 238..242, which covers ring 1's bumps at 241 / 242."""
    rng = np.random.default_rng(seed)
    a = fc.sweep_ring(240, 6.0, -1.0, ground=0, rng=rng, noise=0.003, bumps=[(237, 0.1)])
    b = fc.sweep_ring(240, 6.0, -0.9, ground=0, rng=rng, noise=0.003, col0=240, bumps=[(1, 0.1), (2, 0.1)])
    c = fc.sweep_ring(240, 7.0, 0.2, ground=1, rng=rng, noise=0.02, col0=480)
    s = fc.ring_scan([a, b, c])
    s["start_ring"] = np.array([5, 240, 480], np.int32)
    s["end_ring"] = np.array([240, 480, 714], np.int32)
    return s


def fourth_flat_scene(seed):
    """A ground ring whose ranges are nearly constant over points 60..113, around the boundary of sextants 0 and 1 (102):
    the lowest curvatures of both sextants meet there."""
    rng = np.random.default_rng(seed)
    rows = fc.sweep_ring(600, 6.0, -1.2, ground=1, rng=rng, noise=0.02)
    rows = [(x, y, z, (6.0 + rng.normal(0, 1e-4)) if 60 <= k < 114 else r, c, g) for k, (x, y, z, r, c, g) in enumerate(rows)]
    return fc.ring_scan([rows])


@pytest.mark.parametrize("name", SCENES)
def test_hand_built_scene_matches_host(gpu, defs, name):
    scan, kw = _scene(name)
    ln = len(scan["start_ring"])
    fp = defs.LinsFeatureParams.shipped(imu_lidar_extrinsic_angle=kw.get("angle", 0.0))
    dev = gpu.extract_features([scan], line_num=ln, params=fp, undist=True)
    _check(defs, dev, [scan], ln, **kw)
    # the scene reaches its condition (read from the device's clouds, which _check found equal to the host's)
    h = dev[0]
    if name == "many_corners":
        assert len(h["corner_less_sharp"]) == 120 and len(h["corner_sharp"]) == 12
    if name == "ring0_default_entry":
        assert any(fc.same_bits(p[:3], scan["seg"][0, :3]) for p in h["surf_flat"])
    if name == "negative_voxels":
        assert (scan["seg"][:, :3] < 0).all() and len(h["surf_less_flat"]) == 1


def test_constant_range_ties_match_pyfront(gpu, defs):
    """A ring of constant range: every curvature of its sextants ties, and the tie decides the flat picks.  The device
    keeps equal curvatures in array order — pyfront's stable order."""
    rows = fc.sweep_ring(600, 6.0, -1.2, ground=1)
    rows2 = fc.sweep_ring(600, 9.0, 0.4, ground=0, bumps=[(k, 0.1) for k in range(7, 600, 10)])
    scan = fc.ring_scan([rows, rows2])
    lm = pyfront.Lidar(line_num=2)
    ref = pyfront.extract_features(scan["seg"], scan, lm=lm)
    assert ref["sort_ties"] > 500
    dev = gpu.extract_features([scan], line_num=2, undist=True)[0]
    for dk, pk in (("surf_flat", "flat"), ("corner_sharp", "sharp"), ("surf_less_flat", "less_flat"), ("corner_less_sharp", "less_sharp"), ("undist", "undist")):
        assert fc.same_bits(dev[dk], ref[pk]), dk
    assert len(dev["surf_flat"]) == 24


def test_ring_capacity_both_sides(gpu, capi, defs):
    cap = defs.FEAT_RING_CAP
    for span, ok in ((cap, True), (cap + 1, False)):
        n = span + 11
        rows = fc.sweep_ring(n, 6.0, -1.0, ground=1, rng=np.random.default_rng(span), noise=0.02, bumps=[(k, 0.1) for k in range(3, n, 40)])
        scan = fc.ring_scan([rows])
        scan["start_ring"] = np.array([5], np.int32)
        scan["end_ring"] = np.array([5 + span], np.int32)
        if ok:
            _check(defs, gpu.extract_features([scan], line_num=1, undist=True), [scan], 1)
        else:
            with pytest.raises(capi.LinsError, match="error -4"):
                gpu.extract_features([scan], line_num=1)


def test_invalid_input_changes_nothing(gpu, capi, defs, sweeps):
    good = sweeps[:3]
    ref = gpu.extract_features(good, line_num=64, undist=True)

    def bad(**edit):
        s = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in good[1].items()}
        for k, f in edit.items():
            f(s[k])
        return [good[0], s, good[2]]

    def setv(i, v):
        def f(a):
            a.reshape(-1)[i] = v
        return f

    cases = [bad(seg=setv(7, np.nan)), bad(seg=setv(2, np.inf)), bad(range=setv(40, np.inf)), bad(ori=setv(2, np.nan)),
             bad(start_ring=setv(0, -30)), bad(end_ring=setv(63, 10 ** 7))]
    for c in cases:
        with pytest.raises(capi.LinsError, match="error -1"):
            gpu.extract_features(c, line_num=64)
    for ln in (0, 129):
        with pytest.raises(capi.LinsError, match="error -1"):
            gpu.extract_features([], line_num=ln)
    # rings whose visited ranges overlap, or come out of order
    over = bad(start_ring=setv(1, int(good[1]["start_ring"][0]) + 20))
    with pytest.raises(capi.LinsError, match="error -1"):
        gpu.extract_features(over, line_num=64)
    # bad CSR offsets and NULL arrays, through the C entry point
    L = gpu.L

    def raw(edit):
        keep = {}
        d = capi.LinsGpu._pcl_desc(good, 64, keep)
        edit(d, keep)
        total = int(keep["cloud_off"][-1])
        outs = [np.zeros(total, defs.POINT_DTYPE) for _ in range(4)]
        counts = np.zeros((3, 4), np.int32)
        return L.lins_gpu_extract_features(gpu.h, C.byref(defs.LinsFeatureParams.shipped()), C.byref(d), *[o.ctypes.data for o in outs], None,
                                           counts.ctypes.data)

    def off(i, v):
        def f(d, keep):
            keep["cloud_off"][i] = v
        return f

    def null(field):
        def f(d, keep):
            setattr(d, field, None)
        return f

    edits = [off(0, 1), off(2, int(good[0]["seg"].shape[0]) - 1)] + [null(k) for k in (
        "cloud", "cloud_off", "ground_flag", "col_ind", "range", "start_ring_index", "end_ring_index", "orientation")]
    for e in edits:
        assert raw(e) == -1
    assert raw(lambda d, keep: None) == 0
    again = gpu.extract_features(good, line_num=64, undist=True)
    for a, b in zip(again, ref):
        for k in fc.NAMES + ("undist",):
            assert fc.same_bits(a[k], b[k])
