"""GPU suite: lins_gpu_project_scans (csrc/cuda/lins_projection.cu) against a fresh host ImageProjection per scan
(csrc/host/image_projection.hpp) bit for bit — segmented cloud, outlier cloud, ground flags, columns, ranges, ring
indices, orientations and counts — on simulated sweeps in one batch, permuted, alone and as packed 16-B records; on
hand-built scans that reach each corner of the projection and of the labelling; invalid input returns LINS_E_INVALID and
writes nothing; and the chain projection -> feature extraction equals the host front end."""
import ctypes as C
import math

import numpy as np
import pytest

import featcases as fc
import projcases as pc

pytestmark = pytest.mark.gpu

F = np.float32


@pytest.fixture(scope="module")
def gpu(capi, defs):
    return capi.LinsGpu(defs.LinsParams.shipped(), device=0)


def _same_ori(a, b):
    a, b = np.asarray(a, F), np.asarray(b, F)
    # a NaN orientation is NaN on both sides; its payload is the platform's (the GPU's NaN is canonical)
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and fc.same_bits(a[~nan], b[~nan])


def _check(defs, dev, raws, model):
    assert len(dev) == len(raws)
    for i, raw in enumerate(raws):
        h = pc.host_projection(defs, raw, model)
        d = dev[i]
        for k in ("seg", "outlier", "range"):
            assert fc.same_bits(d[k], h[k]), f"scan {i}: {k} differs ({len(d[k])} vs {len(h[k])})"
        for k in ("ground", "col", "start_ring", "end_ring"):
            assert np.array_equal(d[k], h[k]), f"scan {i}: {k} differs"
        assert _same_ori(d["ori"], h["ori"]), f"scan {i}: ori {d['ori']} vs {h['ori']}"


def _non_finite(raw, seed):
    r = raw.copy()
    rng = np.random.default_rng(seed)
    k = rng.choice(len(r), len(r) // 25, replace=False)
    for j, i in enumerate(k):
        if j % 3 == 0:
            r["x"][i] = r["y"][i] = r["z"][i] = np.nan
        else:
            r[("x", "y", "z")[j % 3]][i] = np.inf if j % 2 else -np.inf
    if seed % 2:
        r["x"][0] = r["y"][0] = r["z"][0] = np.nan
    return r


@pytest.fixture(scope="module")
def vlp_sweeps(synth, defs):
    raws = []
    for config, seeds in (("config3", range(100, 200)), ("config1", range(200, 300))):
        for seed in seeds:
            raw, m = pc.raw_sweep(synth, defs, config, seed)
            raws.append(_non_finite(raw, seed) if seed % 10 == 3 else raw)
    return raws, m


@pytest.fixture(scope="module")
def dense_sweeps(synth, defs):
    raws = []
    for seed in range(300, 340):
        raw, m = pc.raw_sweep(synth, defs, "config4", seed)
        raws.append(raw)
    return raws, m


def test_batch_of_sweeps_matches_host(gpu, defs, vlp_sweeps, dense_sweeps):
    for raws, m in (vlp_sweeps, dense_sweeps):
        dev = gpu.project_scans(raws, model=m)
        _check(defs, dev, raws, m)
        assert gpu.project_ms() > 0
        assert sum(len(d["seg"]) for d in dev) > 1000 * len(raws) and sum(len(d["outlier"]) for d in dev) > 0
        assert sum(int(d["ground"].sum()) for d in dev) > 100 * len(raws)
    assert len(vlp_sweeps[0]) + len(dense_sweeps[0]) >= 200


def test_permuted_single_and_packed(gpu, defs, vlp_sweeps, dense_sweeps):
    for raws, m in (vlp_sweeps, dense_sweeps):
        ref = gpu.project_scans(raws, model=m)
        perm = np.random.default_rng(7).permutation(len(raws))
        dev = gpu.project_scans([raws[i] for i in perm], model=m)
        for j, i in enumerate(perm):
            for k in ("seg", "outlier", "range", "ground", "col", "start_ring", "end_ring"):
                assert fc.same_bits(dev[j][k].view(np.uint8), ref[i][k].view(np.uint8)), k
            assert _same_ori(dev[j]["ori"], ref[i]["ori"])
        for i in (0, len(raws) // 2, len(raws) - 1):
            one = gpu.project_scans([raws[i]], model=m)[0]
            for k in ("seg", "outlier", "range", "ground", "col", "start_ring", "end_ring"):
                assert fc.same_bits(one[k].view(np.uint8), ref[i][k].view(np.uint8)), k
        packed = gpu.project_scans(raws, model=m, point_format=1)
        for a, b in zip(packed, ref):
            for k in ("seg", "outlier", "range", "ground", "col", "start_ring", "end_ring"):
                assert fc.same_bits(a[k].view(np.uint8), b[k].view(np.uint8)), k
            assert _same_ori(a["ori"], b["ori"])


# ---- hand-built scans ----------------------------------------------------------------------------------------------------
COL0_RANGE = 6.005  # the wrapped points' range: close enough to join the 6 m wall's segment, distinct from it


def _ground_image(defs, rows, cols, z=-1.5):
    """VLP-16 pixels on the plane z = -1.5 (rows below the horizon only)."""
    m = defs.LinsLidarModel.vlp16()
    img = np.full((16, 1800), np.nan)
    for r in rows:
        v = math.radians((r + 0.5) * 2.0 - 15.1)
        img[r, cols] = z / math.sin(v)
    return m, img


def _hand_scene(defs, name):
    m = defs.LinsLidarModel.vlp16()
    P = lambda *rows: np.asarray(rows, F).reshape(-1, 3)  # noqa: E731
    if name == "empty":
        return m, P()
    if name == "one_point":
        return m, P((5.0, 1.0, 0.2))
    if name == "two_points":
        return m, P((5.0, 1.0, 0.2), (4.0, -2.0, 0.1))
    if name in ("nan_first", "nan_last", "nan_inside"):
        rng = np.random.default_rng(3)
        _, img = _ground_image(defs, range(0, 6), np.arange(0, 1800, 3))
        img[8:12, 100:400] = 7.0 + rng.normal(0, 0.01, (4, 300))
        pts = pc.image_points(m, img)
        nan = np.full(3, np.nan, F)
        if name == "nan_first":
            pts = np.vstack([nan, pts])
        elif name == "nan_last":
            pts = np.vstack([pts, nan])
        else:
            pts[::7] = nan
        return m, pts
    if name == "outside_fan":  # points above the top row and below the bottom one, next to a wall
        img = np.full((16, 1800), np.nan)
        img[4:12, 500:600] = 6.0
        pts = pc.image_points(m, img)
        return m, np.vstack([pts, P((3.0, 0.5, 10.0), (3.0, 0.5, -10.0), (0.0, 2.0, 50.0), (1.0, 1.0, -1e6))])
    if name == "col_equals_scan_num":  # horizonAngle -90: colD == 1800, wrapped to column 0 (which nothing else fills)
        img = np.full((16, 1800), np.nan)
        img[4:12, 1:40] = 6.0
        img[4:12, 1760:1800] = 6.0
        pts = pc.image_points(m, img)
        rv = [math.radians((r + 0.5) * 2 - 15.1) for r in range(4, 12)]
        extra = [(-COL0_RANGE * math.cos(v), 0.0, COL0_RANGE * math.sin(v)) for v in rv]
        return m, np.vstack([pts, P(*extra)])
    if name == "shared_pixels":  # several points per pixel: the last one wins, the raw intensity is ignored
        img = np.full((16, 1800), np.nan)
        img[6:12, 200:300] = 5.0
        a = pc.image_points(m, img)
        img[6:12, 200:300] = 5.02
        b = pc.image_points(m, img)
        rows = np.empty((2 * len(a), 3), F)
        rows[0::2], rows[1::2] = a, b
        return m, rows
    if name == "all_ground":
        mm, img = _ground_image(defs, range(0, 6), np.arange(1800))
        return mm, pc.image_points(mm, img)
    if name == "ground_overwrite":  # rows 0 and 1 on the ground, row 2 empty: row 1 loses its ground mark (i = 1)
        mm, img = _ground_image(defs, (0, 1), np.arange(300, 500))
        _, img2 = _ground_image(defs, range(0, 6), np.arange(800, 900))
        img[np.isfinite(img2)] = img2[np.isfinite(img2)]
        return mm, pc.image_points(mm, img)
    raise KeyError(name)


HAND = ["empty", "one_point", "two_points", "nan_first", "nan_last", "nan_inside", "outside_fan", "col_equals_scan_num",
        "shared_pixels", "all_ground", "ground_overwrite"]


@pytest.mark.parametrize("name", HAND)
def test_hand_built_scan_matches_host(gpu, defs, name):
    m, pts = _hand_scene(defs, name)
    raw = defs.make_points(pts, np.arange(len(pts), dtype=F) * 3.5 + 100.0)  # the raw intensity must not matter
    dev = gpu.project_scans([raw], model=m)
    _check(defs, dev, [raw], m)
    d = dev[0]
    if name in ("empty", "one_point"):
        assert np.array_equal(d["ori"], np.zeros(3, F)) and len(d["seg"]) == 0
    if name in ("nan_first", "nan_last"):
        assert np.isnan(d["ori"][0] if name == "nan_first" else d["ori"][1])
    if name == "col_equals_scan_num":
        c0 = d["col"] == 0
        assert c0.sum() == 8 and np.allclose(d["range"][c0], COL0_RANGE, atol=1e-4)
    if name == "shared_pixels":
        assert len(d["seg"]) > 0 and np.allclose(d["range"], 5.02, atol=1e-4)
    if name == "all_ground":
        assert len(d["seg"]) > 0 and d["ground"].all() and len(d["outlier"]) == 0
    if name == "ground_overwrite":
        row = np.floor(d["seg"][:, 3]).astype(int)
        assert ((row == 1) & (d["ground"] == 0) & (d["col"] >= 300) & (d["col"] < 500)).sum() > 50


@pytest.mark.parametrize("name", pc.SCENES)
def test_labelling_scene_matches_host(gpu, defs, name):
    img, gsi = pc.scene(name)
    m = pc.model(defs, img.shape[0], img.shape[1], ground_scan_ind=gsi)
    pts = pc.image_points(m, img)
    dev = gpu.project_scans([pts], model=m)
    _check(defs, dev, [pts], m)
    d = dev[0]
    if name == "size30":
        assert len(d["seg"]) == 30
    if name in ("size29", "five_seed_row_only"):
        assert len(d["seg"]) == 0
    if name == "five_three_rows":
        assert len(d["seg"]) == 5


# ---- invalid input ---------------------------------------------------------------------------------------------------------
def test_invalid_input_writes_nothing(gpu, capi, defs, vlp_sweeps):
    raws = vlp_sweeps[0][:3]
    good = defs.LinsLidarModel.vlp16()
    L = gpu.L

    def call(model, edit=None):
        keep = {}
        d = capi.LinsGpu._raw_desc(raws, 0, keep)
        if edit:
            edit(d, keep)
        total, ln = int(keep["cloud_off"][-1]), max(model.line_num, 1)
        outs = dict(seg=np.full(total, 0x7f, defs.POINT_DTYPE), ground=np.full(total, 0xAB, np.uint8), col=np.full(total, 0xABCD, np.uint32),
                    range=np.full(total, -3.0, F), outl=np.full(total, 0x7f, defs.POINT_DTYPE), sr=np.full((3, ln), -77, np.int32),
                    er=np.full((3, ln), -77, np.int32), ori=np.full((3, 3), -5.0, F), counts=np.full((3, 2), -9, np.int32))
        before = {k: v.copy() for k, v in outs.items()}
        rc = L.lins_gpu_project_scans(gpu.h, C.byref(model), C.byref(d), *[outs[k].ctypes.data for k in ("seg", "ground", "col", "range", "outl", "sr", "er", "ori", "counts")])
        same = all(np.array_equal(outs[k].view(np.uint8), before[k].view(np.uint8)) for k in outs)
        return rc, same

    def mod(**kw):
        m = defs.LinsLidarModel(good.line_num, good.scan_num, good.ang_res_x, good.ang_res_y, good.ang_bottom, good.ground_scan_ind)
        for k, v in kw.items():
            setattr(m, k, v)
        return m

    bad_models = [mod(line_num=0), mod(line_num=129), mod(scan_num=1), mod(scan_num=defs.FEAT_RING_CAP + 1), mod(ang_res_x=0.0),
                  mod(ang_res_x=-0.2), mod(ang_res_x=float("nan")), mod(ang_res_y=float("inf")), mod(ang_res_y=0.0),
                  mod(ang_bottom=float("nan")), mod(ang_bottom=float("-inf")), mod(ground_scan_ind=-1), mod(ground_scan_ind=16)]
    for m in bad_models:
        assert call(m) == (-1, True)

    def off(i, v):
        def f(d, keep):
            keep["cloud_off"][i] = v
        return f

    def null(field):
        def f(d, keep):
            setattr(d, field, None)
        return f

    def fmt(d, keep):
        d.point_format = 5

    for e in (off(0, 1), off(2, int(len(raws[0])) - 1), null("cloud"), null("cloud_off"), fmt):
        assert call(good, e) == (-1, True)
    # the model's limits themselves are accepted
    for m in (mod(line_num=128, ground_scan_ind=127), mod(scan_num=2, ground_scan_ind=0), mod(scan_num=defs.FEAT_RING_CAP, line_num=1, ground_scan_ind=0)):
        rc, _ = call(m)
        assert rc == 0
    # NULL outputs
    keep = {}
    d = capi.LinsGpu._raw_desc(raws, 0, keep)
    assert L.lins_gpu_project_scans(gpu.h, C.byref(good), C.byref(d), *([None] * 9)) == -1
    again = gpu.project_scans(raws, model=good)
    _check(defs, again, raws, good)


# ---- chaining: projection -> feature extraction ---------------------------------------------------------------------------
def test_projection_then_extraction_equals_host_front_end(gpu, defs, vlp_sweeps, dense_sweeps):
    for (raws, m), ln in ((vlp_sweeps, 16), (dense_sweeps, 64)):
        # (sweeps with infinite coordinates can put them in the segmented cloud, which the extraction rejects)
        sel = [r for r in raws[:50] if np.isfinite(np.stack([r["x"], r["y"], r["z"]])).all()]
        proj = gpu.project_scans(sel, model=m)
        feats = gpu.extract_features(proj, line_num=ln, undist=True)
        for raw, p, f in zip(sel, proj, feats):
            h = fc.host_features(defs, pc.host_projection(defs, raw, m), ln)
            for k in fc.NAMES + ("undist",):
                assert fc.same_bits(f[k], h[k]), k
