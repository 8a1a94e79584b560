"""CPU suite, row F2: pins tests/mapref.py (the independent numpy / scipy restatement of the mapping node's exact 5-NN)
against the CPU oracle's brute force (oracle/lins_map_oracle.hpp knn5) on the golden unit, two synthetic map units and
every case of tests/mapcases.py, and checks that the cases contain what they are named after — including the two LM
scenes the GPU suite relies on: the corridor, whose iteration 0 is degenerate, and the ground-only scene, whose 6 x 6
QR fails."""
import os

import numpy as np
import pytest

import mapcases
import mapref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "map_unit.npz")


@pytest.fixture(scope="module")
def cases():
    return mapcases.all_pass_cases()


def _same_indices(ob, corner_map, surf_map, corner_q, surf_q, T, ctx):
    m = ob.MapOracle()
    m.set_map(corner_map, surf_map)
    o = m.associate(corner_q, surf_q, T)
    r = mapref.associate_knn(corner_map, surf_map, corner_q, surf_q, T, prune=False)
    for k in ("corner_knn", "surf_knn"):
        assert np.array_equal(o[k], r[k]), f"{ctx} {k}: {np.argwhere(o[k] != r[k])[:5].tolist()}"
    return r


def test_mapref_equals_oracle_on_the_golden_unit(ob):
    g = np.load(GOLD)
    for T in (g["guess"], g["T_out"]):
        _same_indices(ob, g["corner_map"], g["surf_map"], g["corner_last"], g["surf_last"], T, "golden")


@pytest.mark.parametrize("seed,kf", [(5, 12), (11, 25)])
def test_mapref_equals_oracle_on_synthetic_units(ob, synth, seed, kf):
    u = synth.generate_map_unit("config3", seed=seed, n_keyframes=kf, sigma_t=0.1, sigma_r=0.01)
    _same_indices(ob, u.corner_map, u.surf_map, u.corner_last, u.surf_last, u.guess, f"seed {seed}")


def test_mapref_equals_oracle_on_every_case(ob, cases):
    for c in cases:
        _same_indices(ob, *c.clouds(), c.T, c.name)


def test_pruned_search_is_exact_wherever_the_fifth_distance_is_below_one(cases):
    for c in cases:
        for mp, q in ((c.corner_map, c.corner_q), (c.surf_map, c.surf_q)):
            qm = mapref.associate_to_map(q, c.T)
            bi, bd = mapref.knn5_brute(mp, qm)
            pi, pd = mapref.knn5_pruned(mp, qm)
            acc = bd[:, 4] < 1
            assert np.array_equal(bi[acc], pi[acc]) and np.array_equal(bd[acc], pd[acc]), c.name
            assert np.array_equal(acc, pd[:, 4] < 1), c.name


def test_the_cases_contain_their_edges(cases):
    by = {c.name: c for c in cases}
    straddles = sum(c.facts.get("straddling_pairs", 0) for c in cases)
    assert straddles >= 150 and by["straddle-scene"].facts["straddling_pairs"] >= 50
    assert len([n for n in by if n.startswith("straddle-") and n != "straddle-scene"]) == 3 * 2 * 2 * 8
    for n in ("collisions-0", "collisions-1"):
        assert by[n].facts["colliding_points"] >= 1000 and by[n].facts["blocks_with_shared_buckets"] > 0
    assert by["slice-ties"].facts["cross_slice_ties"] >= 100
    assert len(mapcases.FAR_OFFSETS) == 18 and sum(n.startswith("planes-1+") for n in by) == 18
    # the fixed rule keeps every straddler within one cell; the former rule put each two cells away (the builders check
    # that the missed cell's bucket is outside the former block, so the former grid really misses it)
    c = by["straddle-scene"]
    for mp, q in ((c.corner_map, c.corner_q), (c.surf_map, c.surf_q)):
        idx, dist = mapref.knn5(mp, q)
        o = mapref.grid_origin(mp)
        m5 = mapref.xyz(mp)[idx[:, 4]]
        assert (dist[:, 4] < 1).all()
        assert (np.abs(mapref.cell_exact(m5, o) - mapref.cell_exact(q, o)) <= 1).all()
        assert (np.abs(mapref.cell_f32(m5, o) - mapref.cell_f32(q, o)) == 2).any(1).all()


def test_the_oracle_accepts_the_straddlers_and_scan2map_stops_after_one_step(ob):
    c = mapcases.straddle_scene()
    m = ob.MapOracle()
    m.set_map(c.corner_map, c.surf_map)
    a = m.associate(c.corner_q, c.surf_q, c.T)
    assert a["corner_mask"].all() and a["surf_mask"].all()
    T, rep = m.scan2map(c.corner_q, c.surf_q, c.T)
    assert rep.iters == 1 and rep.converged == 1 and rep.n_sel[0] == c.facts["straddling_pairs"] >= 50


def test_the_corridor_is_degenerate_and_the_ground_only_qr_fails(ob):
    c = mapcases.corridor_scene()
    m = ob.MapOracle()
    m.set_map(c.corner_map, c.surf_map)
    T, rep = m.scan2map(c.corner_q, c.surf_q, c.T)
    assert rep.degenerate == 1 and rep.n_sel[0] >= 50 and rep.iters >= 2
    c = mapcases.ground_only_scene()
    m = ob.MapOracle()
    m.set_map(c.corner_map, c.surf_map)
    T, rep = m.scan2map(c.corner_q, c.surf_q, c.T)
    # X = 0: the transform does not move although the scan sits 0.2 m above the ground
    assert rep.n_sel[0] >= 50 and rep.iters == 1 and rep.converged == 1 and rep.delta_r[0] == 0 and rep.delta_t[0] == 0
    assert np.array_equal(T, c.T)
