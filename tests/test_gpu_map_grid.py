"""GPU suite, row F2: adversarial parity of the grid 5-NN, the brute-force 5-NN, the fits and the LM loop (lins_map.cuh)
against the CPU oracle and the independent restatement in tests/mapref.py, on the scenes of tests/mapcases.py:
straddling pairs (f32 distance < 1, cells that an f32 x - ox put two apart), boundary-snapped fuzz, far maps, hash
collisions, ties across brute-force slices, sparse and non-finite inputs, degenerate fits and degenerate LM steps.

Bar: masks and coefficients bit-exact against the oracle (where the oracle's coefficient is NaN the device's must be a
NaN as well: the host's default NaN and the device's canonical NaN have different bits), indices equal to mapref's for
every point whose fifth distance is < 1 (grid) or for every point (brute force), the LM report equal and the transform
within 1e-5 (plus two f32 ulps of its value: at 6e4 m the ulp is ~4 mm)."""
import contextlib
import os

import numpy as np
import pytest

import mapcases
import mapref

pytestmark = pytest.mark.gpu

T_TOL = 1e-5


@contextlib.contextmanager
def knn_mode(mode):
    """LINS_MAP_KNN=mode (None: unset) for the calls inside, restored afterwards."""
    old = os.environ.get("LINS_MAP_KNN")
    try:
        if mode is None:
            os.environ.pop("LINS_MAP_KNN", None)
        else:
            os.environ["LINS_MAP_KNN"] = mode
        yield
    finally:
        if old is None:
            os.environ.pop("LINS_MAP_KNN", None)
        else:
            os.environ["LINS_MAP_KNN"] = old


def same_pass(dev, ora, ctx, knn=True):
    """Masks equal, coefficients bit for bit (NaN where the oracle has NaN), indices equal if `knn`."""
    for name in ("corner", "surf"):
        assert np.array_equal(dev[name + "_mask"], ora[name + "_mask"]), f"{ctx} {name}_mask rows {np.flatnonzero(dev[name + '_mask'] != ora[name + '_mask'])[:8].tolist()}"
        a, b = dev[name + "_coeff"], ora[name + "_coeff"]
        nan = np.isnan(b)
        assert np.array_equal(np.isnan(a), nan), f"{ctx} {name}_coeff NaN pattern"
        assert np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan]), f"{ctx} {name}_coeff not bit-exact"
        if knn:
            assert np.array_equal(dev[name + "_knn"], ora[name + "_knn"]), f"{ctx} {name}_knn"


def grid_rows_ok(dev, ref, n_map, ctx):
    """Indices equal mapref's where its fifth distance is < 1; every index in range; none repeats within a row."""
    for name in ("corner", "surf"):
        g, r, d = dev[name + "_knn"], ref[name + "_knn"], ref[name + "_dist"]
        acc = d[:, 4] < 1
        assert np.array_equal(g[acc], r[acc]), f"{ctx} {name}: rows {np.flatnonzero((g != r).any(1) & acc)[:8].tolist()}"
        assert ((g >= -1) & (g < n_map[name])).all(), f"{ctx} {name}: index out of range"
        s = np.sort(g, 1)
        assert not ((s[:, 1:] == s[:, :-1]) & (s[:, 1:] >= 0)).any(), f"{ctx} {name}: repeated index"
        # a row the reference accepts nothing for is rejected by the device
        assert not dev[name + "_mask"][~acc].any(), f"{ctx} {name}: accepted without five neighbours within 1 m"


def _sizes(c):
    return {"corner": len(c.corner_map), "surf": len(c.surf_map)}


@pytest.fixture(scope="module")
def cases():
    return mapcases.all_pass_cases()


def test_grid_pass_matches_mapref_and_oracle_on_every_case(gpu, ob, cases):
    n_acc = 0
    for c in cases:
        gpu.map_set(c.corner_map, c.surf_map)
        with knn_mode("grid"):
            dev = gpu.map_associate(c.corner_q, c.surf_q, c.T)
        m = ob.MapOracle()
        m.set_map(c.corner_map, c.surf_map)
        same_pass(dev, m.associate(c.corner_q, c.surf_q, c.T), c.name, knn=False)
        ref = mapref.associate_knn(c.corner_map, c.surf_map, c.corner_q, c.surf_q, c.T)
        grid_rows_ok(dev, ref, _sizes(c), c.name)
        n_acc += int(dev["corner_mask"].sum() + dev["surf_mask"].sum())
    assert n_acc > 1000


def test_straddling_queries_are_accepted_by_the_grid(gpu, cases):
    """The worked example and every straddle case: the grid must find the neighbour two f32 cells away (mask 1)."""
    for c in cases:
        if not c.name.startswith(("straddle", "worked")):
            continue
        gpu.map_set(c.corner_map, c.surf_map)
        with knn_mode("grid"):
            dev = gpu.map_associate(c.corner_q, c.surf_q, c.T)
        assert dev["corner_mask"].all() and dev["surf_mask"].all(), c.name


def test_brute_force_pass_matches_mapref_for_every_point(gpu, ob, cases):
    """map_associate's default: exact for every point, rejected ones too — pins the merge of the map slices (the
    slice-ties case runs 64 slices with duplicates on both sides of slice boundaries)."""
    for c in cases:
        gpu.map_set(c.corner_map, c.surf_map)
        with knn_mode(None):
            dev = gpu.map_associate(c.corner_q, c.surf_q, c.T)
        ref = mapref.associate_knn(c.corner_map, c.surf_map, c.corner_q, c.surf_q, c.T, prune=False)
        for name in ("corner", "surf"):
            assert np.array_equal(dev[name + "_knn"], ref[name + "_knn"]), f"{c.name} {name}"


def _t_close(T, To):
    tol = T_TOL + 2 * np.spacing(np.abs(To).astype(np.float32)).astype(np.float64)
    return (np.abs(T.astype(np.float64) - To.astype(np.float64)) <= tol).all()


def _same_report(rep, ro, ctx):
    assert (rep.iters, rep.converged, rep.degenerate, rep.skipped) == (ro.iters, ro.converged, ro.degenerate, ro.skipped), \
        f"{ctx}: (iters, converged, degenerate, skipped) {(rep.iters, rep.converged, rep.degenerate, rep.skipped)} != {(ro.iters, ro.converged, ro.degenerate, ro.skipped)}"
    assert list(rep.n_sel) == list(ro.n_sel), f"{ctx}: n_sel {list(rep.n_sel)} != {list(ro.n_sel)}"
    assert np.allclose(list(rep.delta_r), list(ro.delta_r), rtol=1e-3, atol=1e-5), ctx
    assert np.allclose(list(rep.delta_t), list(ro.delta_t), rtol=1e-3, atol=1e-5), ctx


def test_scan2map_on_the_straddle_scene_and_far_scenes(gpu, ob):
    scenes = [mapcases.straddle_scene()] + mapcases.far_cases(mapcases.plane_scene(1))
    for c in scenes:
        gpu.map_set(c.corner_map, c.surf_map)
        m = ob.MapOracle()
        m.set_map(c.corner_map, c.surf_map)
        with knn_mode(None):  # scan2map's own default: the grid
            T, rep = gpu.scan2map(c.corner_q, c.surf_q, c.T)
        To, ro = m.scan2map(c.corner_q, c.surf_q, c.T)
        _same_report(rep, ro, c.name)
        assert _t_close(T, To), (c.name, T, To)
        if c.name == "straddle-scene":
            assert rep.n_sel[0] == c.facts["straddling_pairs"] >= 50


def test_degenerate_lm_step_and_failed_qr(capi, ob):
    g = capi.LinsGpu()
    for c, check in ((mapcases.corridor_scene(), lambda ro: ro.degenerate == 1 and ro.n_sel[0] >= 50),
                     (mapcases.ground_only_scene(), lambda ro: ro.n_sel[0] >= 50 and ro.delta_r[0] == 0 and ro.delta_t[0] == 0)):
        m = ob.MapOracle()
        m.set_map(c.corner_map, c.surf_map)
        To, ro = m.scan2map(c.corner_q, c.surf_q, c.T)
        assert check(ro), c.name  # the scene does reach the branch
        g.map_set(c.corner_map, c.surf_map)
        T, rep = g.scan2map(c.corner_q, c.surf_q, c.T)
        _same_report(rep, ro, c.name)
        assert _t_close(T, To), (c.name, T, To)


def test_report_over_a_call_sequence_on_a_fresh_context(capi, ob):
    """matP / isDegenerate persist across calls (members of the reference's node); the report's `degenerate` describes
    the call: 0 when its first pass selects < 50 points and no LM step runs."""
    g, m = capi.LinsGpu(), ob.MapOracle()
    cor, pl = mapcases.corridor_scene(), mapcases.plane_scene(2)
    few = mapcases.MapCase("few", mapref.xyz(cor.corner_map), mapref.xyz(cor.surf_map), mapref.xyz(cor.corner_q)[:5],
                           mapref.xyz(cor.surf_q)[:20], cor.T)
    tiny = mapcases.MapCase("tiny-map", mapref.xyz(pl.corner_map)[:10], mapref.xyz(pl.surf_map), mapref.xyz(pl.corner_q),
                            mapref.xyz(pl.surf_q), pl.T)
    seq = [("set", cor), ("call", cor), ("call", few), ("set", pl), ("call", pl), ("set", tiny), ("call", tiny),
           ("set", mapcases.plane_scene(3, n_planes=30)), ("call", None)]
    last_set = None
    degs = []
    for op, c in seq:
        if op == "set":
            g.map_set(c.corner_map, c.surf_map)
            m.set_map(c.corner_map, c.surf_map)
            last_set = c
            continue
        c = c or last_set
        T, rep = g.scan2map(c.corner_q, c.surf_q, c.T)
        To, ro = m.scan2map(c.corner_q, c.surf_q, c.T)
        _same_report(rep, ro, c.name)
        assert _t_close(T, To), (c.name, T, To)
        degs.append(rep.degenerate)
    assert degs[0] == 1 and degs[1] == 0  # (the second call selects < 50 points right after a degenerate one)


def _map_set_sequence():
    """200 k points, then 300, then an empty corner cloud, then 60 k with a shifted origin."""
    big = mapcases.plane_scene(5, n_planes=500, n_q=20000)
    small = mapcases.plane_scene(6, n_planes=1, n_q=200)
    small = mapcases.MapCase("300", mapref.xyz(small.corner_map)[:40], mapref.xyz(small.surf_map)[:300],
                             mapref.xyz(small.corner_q), mapref.xyz(small.surf_q), small.T)
    empty = mapcases.MapCase("empty-corner", np.zeros((0, 3), np.float32), mapref.xyz(small.surf_map), mapref.xyz(small.corner_q),
                             mapref.xyz(small.surf_q), small.T)
    shifted = mapcases.translated(mapcases.plane_scene(7, n_planes=150, n_q=5000), [-317.25, 1250.5, -40.0])
    assert len(big.surf_map) == 200_000 and len(shifted.surf_map) == 60_000
    return big, small, empty, shifted


def test_map_set_sequence_leaves_no_stale_grid(capi):
    """The sequence on one context: after each map_set the grid pass equals mapref's (stale bucket starts or counts would
    show as wrong or missing neighbours)."""
    g = capi.LinsGpu()
    for c in _map_set_sequence():
        g.map_set(c.corner_map, c.surf_map)
        with knn_mode("grid"):
            dev = g.map_associate(c.corner_q, c.surf_q, c.T)
        ref = mapref.associate_knn(c.corner_map, c.surf_map, c.corner_q, c.surf_q, c.T)
        grid_rows_ok(dev, ref, _sizes(c), c.name)
        assert (ref["surf_dist"][:, 4] < 1).sum() > len(c.surf_q) // 4, c.name


def test_scan2map_after_each_map_set_of_the_sequence(capi, ob):
    """scan2map after each map_set of the sequence, on one context, equals the oracle taken through the same sequence:
    the one-slot table's grids, fit blocks and loop state follow every change of the maps' sizes (the empty corner map
    fails the 10 / 100 gate; matP / isDegenerate persist across the calls)."""
    g, m = capi.LinsGpu(), ob.MapOracle()
    ran = []
    for c in _map_set_sequence():
        g.map_set(c.corner_map, c.surf_map)
        m.set_map(c.corner_map, c.surf_map)
        cq, sq = c.corner_q[:500], c.surf_q[:2000]  # (the oracle's 5-NN is brute force)
        T, rep = g.scan2map(cq, sq, c.T)
        To, ro = m.scan2map(cq, sq, c.T)
        _same_report(rep, ro, c.name)
        assert _t_close(T, To), (c.name, T, To)
        ran.append(not rep.skipped and rep.n_sel[0] >= 50)
    assert ran == [True, True, False, True]


def test_large_shape_grid_equals_mapref(gpu):
    """~150 k surf queries against a 300 k-point map."""
    c = mapcases.plane_scene(8, n_planes=750, n_q=150_000)
    assert len(c.surf_map) == 300_000
    gpu.map_set(c.corner_map, c.surf_map)
    with knn_mode("grid"):
        dev = gpu.map_associate(c.corner_q, c.surf_q, c.T)
    ref = mapref.associate_knn(c.corner_map, c.surf_map, c.corner_q, c.surf_q, c.T, prune=True)
    grid_rows_ok(dev, ref, _sizes(c), c.name)
    assert (ref["surf_dist"][:, 4] < 1).sum() > 100_000


def _to_scan_frame(p, T):
    """The inverse of pointAssociateToMap in f64: map-frame points -> the scan frame of transform T."""
    p = mapref.xyz(p).astype(np.float64) - np.asarray(T[3:], np.float64)
    r, pi, y = (float(v) for v in T[:3])
    x2 = np.cos(pi) * p[:, 0] - np.sin(pi) * p[:, 2]  # undo the pitch rotation
    z2 = np.sin(pi) * p[:, 0] + np.cos(pi) * p[:, 2]
    y1 = np.cos(r) * p[:, 1] + np.sin(r) * z2  # undo the roll
    z1 = -np.sin(r) * p[:, 1] + np.cos(r) * z2
    x = np.cos(y) * x2 + np.sin(y) * y1  # undo the yaw
    yy = -np.sin(y) * x2 + np.cos(y) * y1
    return np.stack([x, yy, z1], 1).astype(np.float32)


@pytest.mark.parametrize("T", [[3.1, -0.2, 3.14, 1200.0, -850.5, 30.25], [-3.13, 0.05, -3.1, -990.0, 1010.0, -4.0],
                               [0.3, 1.55, -1.6, 500.5, 750.25, -1000.0], [-0.4, -1.56, 3.141, -1500.0, -20.0, 950.0]])
def test_first_pass_far_from_identity(gpu, ob, T):
    """Roll, pitch and yaw near +-pi (and pitch near +-pi/2), translations of ~1e3 m: the first pass's libm sin / cos
    and f32 re-projection, bit-exact against the oracle; indices equal mapref's."""
    T = np.asarray(T, np.float32)
    base = mapcases.plane_scene(9)
    off = np.asarray(T[3:], np.float64)
    mp = mapcases.translated(base, off)
    cq = _to_scan_frame(mapref.xyz(base.corner_q).astype(np.float64) + off, T)
    sq = _to_scan_frame(mapref.xyz(base.surf_q).astype(np.float64) + off, T)
    c = mapcases.MapCase("far-T", mapref.xyz(mp.corner_map), mapref.xyz(mp.surf_map), cq, sq, T)
    gpu.map_set(c.corner_map, c.surf_map)
    m = ob.MapOracle()
    m.set_map(c.corner_map, c.surf_map)
    ora = m.associate(c.corner_q, c.surf_q, c.T)
    with knn_mode(None):
        dev = gpu.map_associate(c.corner_q, c.surf_q, c.T)
    same_pass(dev, ora, "brute")
    ref = mapref.associate_knn(c.corner_map, c.surf_map, c.corner_q, c.surf_q, c.T, prune=False)
    assert np.array_equal(dev["surf_knn"], ref["surf_knn"]) and np.array_equal(dev["corner_knn"], ref["corner_knn"])
    assert ora["surf_mask"].sum() > len(sq) // 2  # the queries do land on the map
    with knn_mode("grid"):
        dg = gpu.map_associate(c.corner_q, c.surf_q, c.T)
    same_pass(dg, ora, "grid", knn=False)
    grid_rows_ok(dg, ref, _sizes(c), "grid")
