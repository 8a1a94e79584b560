"""GPU suite for close_loops on mapping nodes built to order (tests/loopnodes.py): each scene's blob is loaded into a
fresh slot and one close_loops report is compared against loopref on the same node (its exact brute-force 1-NN).

Exact: the candidate and latest ids, n_source, n_history_ds, n_corr0, icp_iters, converged and accepted (every scene
has margins, tests/test_loopnodes_cpu.py).  Final transform: rotation entries within 4e-7, translation within
4e-7 (1 + max |coordinate|) m.  Fitness: within 1e-6 relative of getFitnessScore of the device's own final transform
(loopref.fitness_of; with the transform within tolerance this pins it without an absolute floor, which a noiseless
scene's rounding-level fitness would otherwise need).  Degenerate scenes: a proper rotation, no NaN, and
sum |R s + t - q|^2 over the device's final correspondences within 1e-6 relative of the oracle's optimum on them.  The
factor-only scene (10 km out): ids, counts and decisions exact.  The loop factor of accepted scenes, read back from a
save: keys exact, variances six copies of
float32(fitness), R within 1e-6, t within 4e-7 (1 + max |pose coordinate|).  Across slots: a lockstep mixture (and
its permutation) byte-equal to each node alone; LINS_E_TOOBIG from one slot's history leaves every masked slot's saved
blob unchanged; a repeated close adds the same factor twice; a small scene after a large one on the same context
equals the small scene on a fresh context."""
import math
import struct

import numpy as np
import pytest

import loopnodes as ln
import loopref
import mapperref

pytestmark = pytest.mark.gpu
F = np.float32
SCENES = ln.scenes()
BY_NAME = {s.name: s for s in SCENES}
DBL_MAX = np.finfo(np.float64).max


@pytest.fixture(scope="module")
def g(capi):
    return capi.LinsGpu()


@pytest.fixture(scope="module")
def tmpl(g):
    g.mapper_reset()
    g.mapper_loops()
    t = ln.template(g.mapper_save())
    g.mapper_reset()
    return t


def close_alone(g, tmpl, sc):
    g.mapper_reset()
    g.mapper_load(ln.blob(sc.node, tmpl))
    return g.mapper_close_loop()


def factors(blob):
    """(n_loop, FactorRec tuples) of a mapper blob"""
    sec = [struct.unpack_from("<2Q", blob, 48 + 16 * k) for k in range(ln.N_SEC)]
    n_loop = struct.unpack_from("<7i", blob, sec[ln.K_SCALARS][0])[5]
    off, nb = sec[ln.K_FACTORS]
    return n_loop, [struct.unpack_from("<2i18d", blob, off + ln.FACTOR * i) for i in range(nb // ln.FACTOR)]


def wrap(a):
    return (np.asarray(a) + math.pi) % (2 * math.pi) - math.pi


def objective_gap(fin, src, tgt):
    """(device objective, oracle optimum) of sum |R s + t - q|^2 over the device's own final correspondences: q the
    exact 1-NN of each kept source point under the final transform, R s + t in f64 from the f32 entries"""
    s = np.asarray(src, F)[loopref.keep_mask(np.asarray(src, F)[:, 3])]
    idx, _, _ = loopref.nn1_exact(tgt, loopref.xf(fin[:3].astype(F), s))
    s, q = s[idx >= 0, :3].astype(np.float64), np.asarray(tgt, F)[idx[idx >= 0], :3].astype(np.float64)
    R, t = loopref.umeyama(s, q)
    obj = lambda R, t: float(np.sum((s @ R.T + t - q) ** 2))  # noqa: E731
    return obj(fin[:3, :3], fin[:3, 3]), obj(R, t), len(s)


def check(rep, sc, ref):
    assert (rep.closest_history_frame_id, rep.latest_frame_id) == (ref["closest"], ref["latest"])
    if ref["closest"] < 0:
        assert rep.accepted == 0
        return
    i = ref["icp"]
    assert (rep.n_source, rep.n_history_ds, rep.n_corr0) == (i["n_source"], ref["n_history"], i["n_corr0"])
    fin = np.array(rep.final_transform, np.float64).reshape(4, 4)
    scale = ref["scale"]
    # the fitness pass: the device's fitness is getFitnessScore of its own final transform (the transform itself is
    # compared with the oracle's below; a noiseless scene's fitness is f32 rounding, not a quantity of the oracle's)
    own = loopref.fitness_of(fin, ref["src"], ref["tgt"])
    assert rep.fitness == own if own == DBL_MAX else abs(rep.fitness - own) <= 1e-6 * own, (rep.fitness, own)
    assert rep.accepted == int(rep.converged == 1 and not rep.fitness > float(loopref.FITNESS))
    if sc.kind == "degenerate":
        R = fin[:3, :3]
        assert np.isfinite(fin).all() and abs(np.linalg.det(R) - 1) <= 1e-6 and np.abs(R @ R.T - np.eye(3)).max() <= 1e-6
        dev, opt, n = objective_gap(fin, ref["src"], ref["tgt"])
        # (1e-6 relative of the optimum; where the optimum is 0, the f32 entries' rounding at the transform tolerance)
        assert dev <= opt * (1 + 1e-6) + n * (4e-7 * (1 + scale)) ** 2, (dev, opt)
        return
    assert (rep.converged, rep.accepted) == (i["converged"], int(i["converged"] == 1 and not i["fitness"] > float(loopref.FITNESS)))
    if sc.kind == "factor_only":
        return
    assert rep.icp_iters == i["iters"]
    ref_fin = i["final"].astype(np.float64)
    assert np.abs(fin[:3, :3] - ref_fin[:3, :3]).max() <= 4e-7, (fin, ref_fin)
    assert np.abs(fin[:3, 3] - ref_fin[:3, 3]).max() <= 4e-7 * (1 + scale), (fin, ref_fin)


def check_factor(g, rep, sc):
    """the loop factor close_loops added, from a save, against loopref.loop_factor on the device's final transform"""
    P = sc.node.poses
    n_loop, fac = factors(g.mapper_save())
    assert n_loop == 1 and len(fac) == len(P) + 1
    a, b, *v = fac[-1]
    R, t, var = np.array(v[:9]).reshape(3, 3), np.array(v[9:12]), v[12:]
    assert (a, b) == (rep.latest_frame_id, rep.closest_history_frame_id)
    assert var == [float(F(rep.fitness))] * 6 and rep.noise == float(F(rep.fitness))
    fin = np.array(rep.final_transform, np.float64).reshape(4, 4).astype(F)
    z = loopref.loop_factor(fin, P[a], P[b])
    pscale = float(np.abs(P[[a, b], :3]).max())
    assert np.abs(R - z[:3, :3]).max() <= 1e-6 and np.abs(t - z[:3, 3]).max() <= 4e-7 * (1 + pscale)
    assert np.abs(np.array(rep.factor[:3]) - z[:3, 3]).max() <= 4e-7 * (1 + pscale)
    assert np.abs(wrap(np.array(rep.factor[3:]) - mapperref.rot3_xyz(z[:3, :3].tolist()))).max() <= 1e-6


@pytest.mark.parametrize("sc", SCENES, ids=[s.name for s in SCENES])
def test_scene_matches_restatement(g, tmpl, sc):
    rep = close_alone(g, tmpl, sc)
    check(rep, sc, ln.reference(sc.node))
    if sc.expect.get("factor"):
        assert rep.accepted
    if rep.accepted:
        check_factor(g, rep, sc)


MIX = ["cand_at_edges", "cand_d2_below", "cand_nan_pose", "cand_no_poses", "src_empty", "src_intensity", "src_2", "src_129",
       "hist_beyond_100m", "hist_corr_at_1e4", "hist_0", "hist_1025", "hist_tie_tiles", "hist_over_51_keyframes", "fit_accept",
       "far_20km", "factor_yaw_minus_pi"]


def lockstep(capi, tmpl, names, idle=2):
    """names in slots 0.., then `idle` enabled but unmasked slots: one close_loops over the named slots"""
    gl = capi.LinsGpu()
    n = len(names)
    gl.mappers_open(n + idle)
    gl.mappers_load([1] * n + [0] * idle, [ln.blob(BY_NAME[k].node, tmpl) for k in names] + [None] * idle)
    gl.mappers_loops([0] * n + [1] * idle)
    return gl, gl.mappers_close_loops([1] * n + [0] * idle)


def test_lockstep_mixture_equals_each_node_alone(capi, g, tmpl):
    alone = {k: bytes(close_alone(g, tmpl, BY_NAME[k])) for k in MIX}
    _, reps = lockstep(capi, tmpl, MIX)
    assert all(bytes(reps[s]) == alone[k] for s, k in enumerate(MIX))
    assert reps[-1] is None
    perm = list(np.random.default_rng(5).permutation(MIX))
    _, reps = lockstep(capi, tmpl, perm, idle=1)
    assert all(bytes(reps[s]) == alone[k] for s, k in enumerate(perm))


def test_toobig_history_changes_no_slot(capi, g, tmpl):
    names = ["fit_accept", "stop_transform", "hist_1025"]
    gl = capi.LinsGpu()
    gl.mappers_open(4)
    gl.mappers_load([1, 1, 1, 1], [ln.blob(ln.toobig_scene().node, tmpl)] + [ln.blob(BY_NAME[k].node, tmpl) for k in names])
    before = gl.mappers_save([1, 1, 1, 1])
    with pytest.raises(Exception, match="error -4"):
        gl.mappers_close_loops([1, 1, 1, 1])
    assert gl.mappers_save([1, 1, 1, 1]) == before
    reps = gl.mappers_close_loops([0, 1, 1, 1])
    assert all(bytes(reps[s + 1]) == bytes(close_alone(g, tmpl, BY_NAME[k])) for s, k in enumerate(names))


def test_repeated_close_adds_the_same_factor_twice(g, tmpl):
    sc = BY_NAME["stop_transform"]
    a = close_alone(g, tmpl, sc)
    b = g.mapper_close_loop()
    assert a.accepted and bytes(a) == bytes(b)
    n_loop, fac = factors(g.mapper_save())
    assert n_loop == 2 and len(fac) == len(sc.node.poses) + 2 and fac[-1] == fac[-2]


def test_small_scene_after_a_large_one_equals_a_fresh_context(capi, g, tmpl):
    close_alone(g, tmpl, BY_NAME["src_3000"])
    after = bytes(close_alone(g, tmpl, BY_NAME["src_3"]))
    fresh = capi.LinsGpu()
    assert after == bytes(close_alone(fresh, ln.template(_fresh_blob(fresh)), BY_NAME["src_3"]))


def _fresh_blob(gf):
    gf.mapper_reset()
    gf.mapper_loops()
    b = gf.mapper_save()
    gf.mapper_reset()
    return b
