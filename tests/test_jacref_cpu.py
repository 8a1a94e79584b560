"""CPU: pin tests/jacref.py (the reference of the split Jacobian pass) to the CPU oracle.

The oracle's association at a search iteration >= 1 (brute-force 1-NN, so its IDs are the reference's) gives the IDs,
pointSel, coefficients and accept masks; lins_oracle_measurement_rows gives the reference's rows h = [c ; Rinv^T g_att].
jacref, fed the oracle's IDs, must reproduce pointSel and the masks bit for bit and the coefficients to 1 f32 ulp, its
row formula must give the oracle's rows after the per-unit attitude map, and its exact sums must match the oracle's rows
summed.  Cases: the golden units and fresh config-3 units at their prior and at a perturbed state, the unweighted pass,
lidar_scale = 2.5, a unit with zero rotation, and points with a negative fractional intensity de-skewed by large
angles (the exact sin / cos of axis2Quat, for either sign of the half angle).
"""
import ctypes as C

import numpy as np
import pytest

import jacref

EPS = 2.0 ** -52


def _perturbed(state):
    st = np.array(state, np.float64)
    st[0:3] += [0.05, -0.03, 0.02]
    a = np.array([0.01, -0.02, 0.015])
    th = np.linalg.norm(a)
    dq = np.concatenate([a / th * np.sin(th / 2), [np.cos(th / 2)]])  # (x, y, z, w)
    x1, y1, z1, w1 = dq
    x2, y2, z2, w2 = st[6:10]
    st[6:10] = [w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2]
    return st


def _oracle_assoc(ob, prm, u, state, search=None):
    """The oracle's association of search iteration 1 at `state`.  For icp_freq = 2 that iteration is unweighted and
    reuses the IDs iteration 0 found at the same state for the queries `search` (default: the unit's own)."""
    o = ob.Oracle(prm, use_kdtree=False)
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    if prm.icp_freq > 1:
        qs, qc = search or (u["surf_flat"], u["corner_sharp"])
        o.associate(qs, qc, state, 0)
    return o.associate(u["surf_flat"], u["corner_sharp"], state, 1)


def _ulps_f32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    sp = np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32)).astype(np.float64)
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / sp


def check_unit(ob, prm, sub, state, search=None):
    """jacref of the one-unit batch `sub` at `state` against the oracle; returns jacref's output."""
    u = sub.unit(0)
    a = _oracle_assoc(ob, prm, u, state, search)
    jr = jacref.reference(sub, a["surf_ind"], a["corner_ind"], state[None], prm)
    L = ob.lib()
    h_rows, n_acc = [], 0
    for kind, q in (("surf", "surf_flat"), ("corner", "corner_sharp")):
        rows = getattr(jr, kind)
        assert np.array_equal(rows["sel"], a[kind + "_sel"]), f"{kind} pointSel differs from the oracle's"
        assert np.array_equal(rows["mask"].astype(np.uint8), a[kind + "_mask"]), f"{kind} accept masks differ"
        assert _ulps_f32(rows["coeff"], a[kind + "_coeff"]).max(initial=0) <= 1.0, f"{kind} coeff beyond 1 f32 ulp"
        m = a[kind + "_mask"] == 1
        kp, cf = np.ascontiguousarray(u[q][m]), np.ascontiguousarray(a[kind + "_coeff"][m])
        h6, r = np.zeros((len(kp), 6)), np.zeros(len(kp))
        L.lins_oracle_measurement_rows(C.byref(prm), ob.ptr(np.ascontiguousarray(state)), ob.ptr(kp), ob.ptr(cf), len(kp), ob.ptr(h6), ob.ptr(r))
        p = np.stack([kp["x"], kp["y"], kp["z"]], 1)
        G = jacref.jacobian_rows(p, cf, state, prm.lidar_scale)
        # c and r are computed alike; the attitude columns through the per-unit map ATT (jacref.att_map)
        assert np.array_equal(G[:, :3], h6[:, :3]) and np.array_equal(G[:, 6], r)
        ATT = jacref.att_map(state)
        scale = (np.linalg.norm(p, axis=1) * np.linalg.norm(cf[:, :3], axis=1))[:, None]
        assert (np.abs(G[:, 3:6] @ ATT - h6[:, 3:]) <= 8 * EPS * scale).all(), "g_att does not map onto the oracle's h_att"
        # the oracle's rows in the kernel's basis, for the sums below
        g_att = np.linalg.solve(ATT.T, h6[:, 3:].T).T
        assert (np.abs(g_att - G[:, 3:6]) <= 16 * EPS * scale).all()
        h_rows.append(np.concatenate([h6[:, :3], g_att, r[:, None]], 1))
        n_acc += len(kp)
    H = np.concatenate(h_rows)
    assert (jr.counts[0] == [a["surf_mask"].sum(), a["corner_mask"].sum()]).all()
    want = np.array([float(np.sum(H[:, i].astype(np.longdouble) * H[:, j].astype(np.longdouble))) for i, j in jacref.PAIRS])
    bound = (jr.n_rows[0] + 16) * EPS * jr.scale[0]
    assert (np.abs(jr.sums[0] - want) <= bound).all(), np.abs(jr.sums[0] - want) / np.maximum(bound, 1e-300)
    assert n_acc > 0 or not jr.scale.any()
    return jr


@pytest.fixture(scope="module")
def synth3(synth):
    return synth.generate("config3", n=3, seed0=5150)


@pytest.mark.parametrize("which", ["prior", "perturbed"])
def test_golden_units(ob, golden_batch, which):
    prm = ob.LinsParams.shipped()
    for i in range(golden_batch.n):
        sub = golden_batch.subset([i])
        st = sub.state[0] if which == "prior" else _perturbed(sub.state[0])
        jr = check_unit(ob, prm, sub, st)
        assert jr.counts.sum() > 100


@pytest.mark.parametrize("which", ["prior", "perturbed"])
def test_config3_units(ob, synth3, which):
    prm = ob.LinsParams.shipped()
    for i in range(synth3.n):
        sub = synth3.subset([i])
        check_unit(ob, prm, sub, sub.state[0] if which == "prior" else _perturbed(sub.state[0]))


@pytest.mark.parametrize("kw", [dict(icp_freq=2), dict(lidar_scale=2.5)], ids=["unweighted", "lidar_scale"])
def test_pass_parameters(ob, golden_batch, synth3, kw):
    prm = ob.LinsParams.shipped(**kw)
    for sub in (golden_batch.subset([1]), synth3.subset([0])):
        jr = check_unit(ob, prm, sub, _perturbed(sub.state[0]))
        if "icp_freq" in kw:  # every row with valid IDs and a nonzero residual is accepted
            for kind in ("surf", "corner"):
                rows = getattr(jr, kind)
                assert np.array_equal(rows["mask"], rows["valid"] & (rows["cand"][:, 3] != 0))


def test_zero_rotation(ob, golden_batch):
    sub = golden_batch.subset([2])
    st = sub.state[0].copy()
    st[6:10] = [0.0, 0.0, 0.0, 1.0]
    sub.state[0] = st
    jr = check_unit(ob, ob.LinsParams.shipped(icp_freq=2), sub, st)
    assert (jr.surf["half"] == 0).all() and jr.counts.sum() > 0
    assert np.array_equal(jacref.att_map(st), np.eye(3))


def test_negative_time_points(ob, synth3, defs):
    """Queries whose intensity has a negative fractional part (s < 0) and a scan period that makes |half angle| >= 1/8:
    jacref de-skews them like axis2Quat, whatever the sign and size of the angle.  (The IDs are those of the same
    queries at time 0, so that rows de-skewed this far still have correspondences.)"""
    b = synth3.subset([1])
    clouds = {k: b.clouds[k].copy() for k in b.FIELDS}
    for k in ("surf_flat", "corner_sharp"):
        clouds[k]["intensity"][::2] *= -1.0
    sub = defs.Batch(clouds, b.offsets, b.state, b.cov)
    at0 = []
    for k in ("surf_flat", "corner_sharp"):
        c = clouds[k].copy()
        c["intensity"] = np.trunc(c["intensity"])
        at0.append(c)
    prm = ob.LinsParams.shipped(icp_freq=2, scan_period=0.001)
    jr = check_unit(ob, prm, sub, sub.state[0], search=tuple(at0))
    half = np.concatenate([jr.surf["half"], jr.corner["half"]])
    ok = np.concatenate([jr.surf["mask"], jr.corner["mask"]])
    assert (ok & (half <= -0.125)).sum() > 20 and (ok & (half >= 0.125)).sum() > 20 and half.min() < -1.0


def test_near_midpoint():
    f = np.float32(1.5)
    ulp = float(np.spacing(f))
    mid = float(f) + ulp / 2
    x = np.array([mid, mid * (1 + 2.0 ** -45), mid * (1 + 2.0 ** -40), float(f)])
    assert jacref.near_midpoint(x, np.abs(x)).tolist() == [True, True, False, False]
    # a value formed with cancellation: 2^-49 of its terms' magnitude widens the window
    assert jacref.near_midpoint(x[2:3], 1000 * np.abs(x[2:3])).tolist() == [True]
    assert jacref.near_midpoint(x[2:3], 100 * np.abs(x[2:3])).tolist() == [False]
    # an exact midpoint is excused only where ties are
    assert jacref.near_midpoint(x[:1], np.abs(x[:1]), ties=False).tolist() == [False]
