"""CPU pins of tests/loopref.py, the restatement the loop-closure GPU tests compare against: pcl's Euler helpers and
gtsam's RzRyRx against scipy's Rotation, ICP on noiseless data, the Gauss-Newton back-end against
scipy.optimize.least_squares, and the candidate rule."""
import math

import numpy as np
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

import loopref
import mapperref

F = np.float32


def test_euler_helpers_match_scipy():
    rng = np.random.default_rng(0)
    for _ in range(50):
        r, p, y = rng.uniform(-1.2, 1.2, 3)
        x, yy, z = rng.uniform(-50, 50, 3)
        t = loopref.pcl_transformation(F(x), F(yy), F(z), F(r), F(p), F(y))
        R = Rotation.from_euler("xyz", [float(F(r)), float(F(p)), float(F(y))]).as_matrix()
        assert np.abs(t[:, :3] - R).max() < 1e-6
        e = loopref.pcl_euler(t)
        assert np.allclose([float(v) for v in e], [float(F(x)), float(F(yy)), float(F(z)), float(F(r)), float(F(p)), float(F(y))], atol=2e-6)
        assert np.abs(np.array(mapperref.rot3_rzryrx(r, p, y)) - Rotation.from_euler("xyz", [r, p, y]).as_matrix()).max() < 1e-15
        assert np.allclose(loopref.pose3(r, p, y, x, yy, z)[:3, :3], mapperref.rot3_rzryrx(r, p, y), atol=1e-15)


def test_pose3_exp_log_round_trip():
    rng = np.random.default_rng(1)
    for _ in range(30):
        xi = np.concatenate([rng.uniform(-1, 1, 3), rng.uniform(-5, 5, 3)])
        assert np.allclose(loopref.logmap(loopref.expmap(xi)), xi, atol=1e-12)
    a, b = loopref.pose3(0.1, 0.2, 0.3, 1, 2, 3), loopref.pose3(-0.3, 0.1, 1.2, -4, 0, 2)
    assert np.allclose(a @ loopref.between(a, b), b, atol=1e-12)


def test_icp_recovers_a_rigid_transform():
    rng = np.random.default_rng(2)
    tgt = np.concatenate([rng.uniform(-20, 20, (600, 3)), rng.uniform(0, 100, (600, 1))], 1).astype(F)
    R = Rotation.from_euler("xyz", [0.01, -0.02, 0.03]).as_matrix()
    t = np.array([0.2, -0.1, 0.05])
    src = tgt.copy()
    src[:, :3] = ((tgt[:, :3] - t) @ R).astype(F)  # tgt = R src + t
    src[0, 3] = np.nan  # dropped by the intensity filter
    src[1, 3] = -1.5
    out = loopref.icp(src, tgt)
    assert out["converged"] == 1 and out["n_source"] == len(src) - 2
    T = out["final"].astype(np.float64)
    assert np.abs(T[:3, :3] - R).max() < 1e-5 and np.abs(T[:3, 3] - t).max() < 1e-4
    assert out["fitness"] < 1e-8


def test_icp_without_enough_correspondences():
    tgt = np.array([[0, 0, 0, 1], [1, 0, 0, 1]], F)
    src = np.array([[500, 0, 0, 1], [0, 0, 0.1, 1], [1, 0, 0.1, 1]], F)  # one point beyond 100 m
    out = loopref.icp(src, tgt)
    assert out["converged"] == 0 and out["iters"] == 0 and out["n_corr0"] == 2


def _graph(rng, n=12):
    """A chain with odometry noise and a drift, its prior, and a loop from the last key back to key 0."""
    truth = [loopref.pose3(0, 0, 2 * math.pi * i / n, 10 * math.cos(2 * math.pi * i / n), 10 * math.sin(2 * math.pi * i / n), 0) for i in range(n)]
    fs = [(0, -1, truth[0], loopref.ODOM_VAR)]
    x0 = [truth[0]]
    for i in range(1, n):
        z = loopref.between(truth[i - 1], truth[i]) @ loopref.expmap(np.concatenate([rng.normal(0, 2e-3, 3), rng.normal(0, 2e-2, 3)]))
        fs.append((i - 1, i, z, loopref.ODOM_VAR))
        x0.append(x0[-1] @ z)
    fs.append((n - 1, 0, loopref.between(truth[n - 1], truth[0]), np.full(6, 0.05)))
    return fs, x0, truth


def test_gauss_newton_matches_least_squares():
    fs, x0, truth = _graph(np.random.default_rng(3))
    x = loopref.gn_solve(fs, x0)
    n = len(x0)

    def resid(v):
        xs = [x0[i] @ loopref.expmap(v[6 * i:6 * i + 6]) for i in range(n)]
        return np.concatenate([loopref.factor_error(f, xs) / np.sqrt(np.asarray(f[3])) for f in fs])

    sol = least_squares(resid, np.zeros(6 * n), jac="3-point", method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    xl = [x0[i] @ loopref.expmap(sol.x[6 * i:6 * i + 6]) for i in range(n)]
    assert max(np.abs(a - b).max() for a, b in zip(x, xl)) < 1e-9
    assert loopref.graph_cost(fs, x) <= loopref.graph_cost(fs, xl) * (1 + 1e-12)
    # the loop pulls the drifted chain's end back towards the truth
    assert np.linalg.norm(x[-1][:3, 3] - truth[-1][:3, 3]) < np.linalg.norm(x0[-1][:3, 3] - truth[-1][:3, 3])


def test_candidate_rule():
    poses = np.array([[0, 0, 0, 0, 0, 0, 0.0], [3, 0, 0, 0, 0, 0, 10.0], [1, 0, 0, 0, 0, 0, 50.0], [4.9, 0, 0, 0, 0, 0, 0.0]])
    assert loopref.candidate(poses, (0.5, 0, 0), 60.0) == 0  # nearest first; key 2 is within 30 s
    assert loopref.candidate(poses, (0.5, 0, 0), 25.0) == -1  # every key within 5 m is within 30 s
    assert loopref.candidate(poses, (9.5, 0, 0), 90.0) == 3  # only key 3 is within 5 m
