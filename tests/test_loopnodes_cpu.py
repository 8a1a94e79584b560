"""CPU checks of the loop-closure scenes tests/test_gpu_loop_nodes.py runs (tests/loopnodes.py), before any GPU run:
- each scene's mapper blob passes the validator (lins_mapper_blob.hpp's parse, compiled with g++ as
  test_mapper_checkpoint_cpu.py does) with the counts it was built with;
- the restatement (loopref.icp with the exact brute-force 1-NN) reaches the scene's intended branch with a built-in
  margin: a converged fitness at least 10 % away from 0.3; at the stopping iteration the deciding criterion inside its
  threshold by 2x; at every earlier iteration every criterion outside its threshold by 2x; in parity scenes no 1-NN
  gap (second-best minus best distance of a used correspondence) below 1e-6 (1 + max |coordinate|) m, at any
  iteration (tie scenes are exact ties by construction);
- the outcome is stable: a perturbed run (Horn's quaternion in place of the SVD, sums in reverse order) gives the same
  iterations, convergence, first correspondence count and decision, and a final transform within the GPU suite's
  tolerance (4e-7 per rotation entry, 4e-7 (1 + scale) per translation entry), the fitness within 1e-6 relative.
Degenerate scenes (Horn and the SVD may pick different optima) check that both runs give proper rotations and the same
fitness instead; the factor-only scene (10 km out, where the ICP's iterations are not determined) that both runs make
the same decisions.  Every scene also keeps its 1-NN distances at least 1 m^2 from the 1e4 m^2 correspondence limit,
except the distances a scene places there exactly."""
import ctypes as C
import shutil
import subprocess

import numpy as np
import pytest

import loopnodes as ln
import loopref
import mapperref
import test_mapper_checkpoint_cpu as tm

SCENES = ln.scenes()
IDS = [s.name for s in SCENES]


@pytest.fixture(scope="module")
def parse_lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ is not available")
    d = tmp_path_factory.mktemp("loopnodes")
    src, so = d / "mblob_driver.cpp", d / "mblob_driver.so"
    src.write_text(tm.DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC", "-I", tm.CUDA_DIR, "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.blob_check.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    return L


def check_blob(L, node):
    b = np.frombuffer(ln.blob(node, ln.cpu_template()), np.uint8).copy()
    sp, err = np.zeros(64 + 8 * len(node.poses), np.int32), C.create_string_buffer(128)
    assert L.blob_check(b.ctypes.data, len(b), sp.ctypes.data, err, 128) == 0, err.value.decode()
    n = len(node.poses)
    assert list(sp[:8]) == [ln.F_LOOPS, n, 0, n, n, n, 0, 0]
    if n:
        kf = sp[8:8 + 4 * n].reshape(n, 4)
        assert np.array_equal(kf[:, 0], np.arange(n)) and np.array_equal(kf[:, 1:], [[len(c) for c in k] for k in node.clouds])
        assert np.array_equal(sp[8 + 4 * n:8 + 6 * n].reshape(n, 2), [(0, -1)] + [(i - 1, i) for i in range(1, n)])


@pytest.mark.parametrize("sc", SCENES + [ln.toobig_scene()], ids=IDS + ["toobig"])
def test_blob_parses(parse_lib, sc):
    check_blob(parse_lib, sc.node)


def transform_close(a, b, scale):
    a, b = np.asarray(a, np.float64)[:3], np.asarray(b, np.float64)[:3]
    return np.abs(a[:, :3] - b[:, :3]).max() <= 4e-7 and np.abs(a[:, 3] - b[:, 3]).max() <= 4e-7 * (1 + scale)


def transform_outside(x):
    return (1 - x["cos"]) >= 2e-5 or x["tsq"] >= 2e-6


def mse_outside(x):
    d = abs(x["mse"] - x["prev_mse"])
    return d >= 2e-12 and d / x["prev_mse"] >= 2e-6


def accepted(icp):
    return int(icp["converged"] == 1 and not icp["fitness"] > float(loopref.FITNESS))


@pytest.mark.parametrize("sc", SCENES, ids=IDS)
def test_scene_reaches_its_branch_with_margin(sc):
    r = ln.reference(sc.node)
    e = sc.expect
    assert r["closest"] == e["closest"]
    if r["closest"] < 0:
        return
    i = r["icp"]
    for k in ("stop", "n_source", "n_corr0", "n_history", "accepted"):
        if k in e:
            got = {"n_history": r["n_history"], "accepted": accepted(i)}.get(k, i.get(k))
            assert got == e[k], (k, got, e[k])
    if e.get("last_target_used"):
        assert r["n_history"] - 1 in i["corr0"]
    # a 1-NN distance within 1 m^2 of the 1e4 m^2 limit only where the scene puts one exactly, at every iteration
    for x in i["trace"]:
        assert set(x["near_limit"].tolist()) <= set(e.get("at_limit", ())), x["near_limit"]
    if i["converged"]:
        assert abs(i["fitness"] - 0.3) >= 0.03, i["fitness"]
    if sc.kind in ("degenerate", "factor_only"):
        return
    steps = [x for x in i["trace"] if "mse" in x]
    for x in steps[:-1]:
        assert transform_outside(x) and mse_outside(x), x
    if i["stop"] == "transform":
        assert (1 - steps[-1]["cos"]) <= 5e-6 and steps[-1]["tsq"] <= 5e-7, steps[-1]
    elif i["stop"] == "mse":
        x = steps[-1]
        d = abs(x["mse"] - x["prev_mse"])
        assert transform_outside(x) and (d <= 5e-13 or d / x["prev_mse"] <= 5e-7), x
    if sc.kind == "parity":
        tol = 1e-6 * (1 + r["scale"])
        for x in i["trace"]:
            assert x["gap"] is None or not len(x["gap"]) or x["gap"].min() >= tol, (x["gap"].min(), tol)


@pytest.mark.parametrize("sc", SCENES, ids=IDS)
def test_scene_outcome_is_stable(sc):
    a = ln.reference(sc.node)
    if a["closest"] < 0:
        return
    b = ln.reference(sc.node, solver="horn", reverse=True)
    ia, ib = a["icp"], b["icp"]
    assert (ia["n_corr0"], ia["n_source"]) == (ib["n_corr0"], ib["n_source"])
    if sc.kind == "degenerate":
        for i in (ia, ib):
            R = i["final"][:3, :3].astype(np.float64)
            assert np.isfinite(i["final"]).all() and abs(np.linalg.det(R) - 1) <= 1e-6 and np.abs(R @ R.T - np.eye(3)).max() <= 1e-6
        assert abs(ia["fitness"] - ib["fitness"]) <= 1e-6 * ia["fitness"] + 1e-12
        return
    if sc.kind == "factor_only":
        assert (ia["converged"], accepted(ia)) == (ib["converged"], accepted(ib))
        return
    assert (ia["iters"], ia["converged"], accepted(ia)) == (ib["iters"], ib["converged"], accepted(ib))
    assert transform_close(ia["final"], ib["final"], a["scale"]), (ia["final"], ib["final"])
    assert abs(ia["fitness"] - ib["fitness"]) <= 1e-6 * ia["fitness"] + 1e-300


def test_toobig_scene_overflows_the_history_voxel_grid():
    sc = ln.toobig_scene()
    with pytest.raises(mapperref.TooBig):
        ln.reference(sc.node)


def test_exact_nn_against_brute_force_f64_ranking():
    """nn1_exact: the f32 distance's minimum, ties to the lower index, against a per-point loop"""
    rng = np.random.default_rng(3)
    tgt = np.round(rng.uniform(-3, 3, (300, 4)) * 4).astype(np.float32) / 4
    src = np.round(rng.uniform(-3, 3, (200, 4)) * 8).astype(np.float32) / 8
    idx, d, gap = loopref.nn1_exact(tgt, src, chunk=1000)
    for k, p in enumerate(src):
        q = tgt[:, :3] - p[:3]
        dd = (q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]
        j = int(np.flatnonzero(dd == dd.min())[0])
        assert (idx[k], d[k]) == (j, dd[j])
        assert gap[k] == np.sqrt(np.partition(dd.astype(np.float64), 1)[1]) - np.sqrt(float(dd[j]))
    assert (gap == 0).any()  # (the dyadic grid has exact ties)


def test_horn_matches_umeyama():
    rng = np.random.default_rng(4)
    s = rng.uniform(-5, 5, (50, 3))
    R = loopref.Rotation.from_rotvec([0.3, -0.2, 0.5]).as_matrix()
    t = s @ R.T + [1, 2, 3] + rng.normal(0, 0.01, (50, 3))
    (Ra, ta), (Rb, tb) = loopref.umeyama(s, t), loopref.horn(s, t, reverse=True)
    assert np.abs(Ra - Rb).max() < 1e-12 and np.abs(ta - tb).max() < 1e-11
