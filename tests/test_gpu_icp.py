"""The estimateTransform fallback (lins_gpu_estimate_transform: icp_loop + lins_icp_step_kernel) against the oracle on
the scenes where it branches: a corridor whose J^T J has an eigenvalue below 10 at the start pose (the matP projection of
StateEstimator.hpp:1266-1302), too few matched surfs or corners (the early returns of :1175-1184), among them a unit
whose surfs match unweighted but fall below 10 once the robust weight switches on at iter >= icp_freq, and far starts,
one of which stops at num_iter without converging.  Every scene runs with icp_freq 1 and 2; iterations, convergence and
the last search's correspondence IDs must equal the oracle's, the pose within POSE_TOL."""
import numpy as np
import pytest

import filterref as fr

pytestmark = pytest.mark.gpu
POSE_TOL = 1.2e-14  # 10x the worst |pose - oracle| of these scenes on an H100 SXM 80 GB (1.2e-15, the same at 400 W and 700 W)
RINGS = 16
n_ids = [0]  # scenes whose last correspondence IDs were compared


def ray_cast(az, el, world):
    d = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], -1)
    return d * world(d)[:, None]


def corridor(d):
    """Walls at y = +-2, a floor 1.5 m below the sensor, no end within 40 m (those rays return nothing)."""
    with np.errstate(divide="ignore"):
        t = 2.0 / np.abs(d[:, 1])
        t = np.where(d[:, 2] < 0, np.minimum(t, 1.5 / -d[:, 2]), t)
    return np.where(t < 40, t, np.nan)


def yard(d):
    """A 30 m x 18 m walled yard with its floor 1.5 m below the sensor."""
    with np.errstate(divide="ignore"):
        t = np.minimum(15.0 / np.abs(d[:, 0]), 9.0 / np.abs(d[:, 1]))
        t = np.where(d[:, 2] < 0, np.minimum(t, 1.5 / -d[:, 2]), t)
    return t


def scan(rng, defs, world, n_az, frac, noise):
    """A 16-ring sweep: ring r at elevation -15 + 2 r degrees; intensity = ring + frac (frac / 0.1 = the point's s)."""
    pts, ring = [], []
    for r in range(RINGS):
        az = np.sort(rng.uniform(-np.pi, np.pi, n_az))
        p = ray_cast(az, np.full(n_az, np.deg2rad(-15 + 2 * r)), world)
        ok = np.isfinite(p).all(1)
        pts.append(p[ok] + rng.normal(0, noise, (ok.sum(), 3)))
        ring.append(np.full(ok.sum(), r))
    ring = np.concatenate(ring)
    return defs.make_points(np.concatenate(pts), ring + frac)


def unit(rng, defs, world, n_s=300, n_c=60):
    """Targets (the last scan's less-sharp / less-flat clouds) and queries of a second sweep of the same world, with
    s = 0.999 so that the whole pose moves them.  Corner targets / queries are the points on the two lowest rings next
    to a wall-floor edge."""
    noise = 0.0 if world is corridor else 0.005  # (noise on the corridor's planes would observe the along-wall shift)
    tgt = scan(rng, defs, world, 300, 0.05, noise)
    qry = scan(rng, defs, world, 300, 0.0999, noise)

    def edge(c):
        xyz = np.stack([c["x"], c["y"], c["z"]], 1)
        return (np.abs(np.abs(xyz[:, 1]) - 2.0) < 0.3) & (xyz[:, 2] < -1.2) if world is corridor else \
            (np.abs(xyz[:, 2] + 1.5) < 0.3) & ((np.abs(np.abs(xyz[:, 0]) - 15) < 0.5) | (np.abs(np.abs(xyz[:, 1]) - 9) < 0.5))

    sel = lambda c, m, n: c[np.sort(rng.choice(np.flatnonzero(m), min(n, int(m.sum())), replace=False))]
    return dict(surf_less_flat=tgt, corner_less_sharp=tgt[edge(tgt)], surf_flat=sel(qry, ~edge(qry), n_s),
                corner_sharp=sel(qry, edge(qry), n_c))


def start(t, rpy_deg):
    q = fr.rpy2Quat(fr.F64, np.deg2rad(np.asarray(rpy_deg, float)))
    return np.asarray(t, float), q / np.linalg.norm(q)


def jtj_eigenvalues(ob, prm, u, t0, q0):
    """J^T J of the oracle's iteration-0 association (StateEstimator.hpp:1228-1262), rebuilt here."""
    o = ob.Oracle(prm)
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    st = np.zeros(19)
    st[0:3], st[6:10] = t0, q0
    a = o.associate(u["surf_flat"], u["corner_sharp"], st, 0)
    o.close()
    rows = []
    phi = np.zeros(3)
    n = np.linalg.norm(q0[:3])
    if n >= 1e-10:
        phi = q0[:3] / n * (2 * np.arctan2(n, q0[3]))
    for cloud, coeff, mask in ((u["surf_flat"], a["surf_coeff"], a["surf_mask"]), (u["corner_sharp"], a["corner_coeff"], a["corner_mask"])):
        for p, c in zip(cloud[mask.astype(bool)], coeff[mask.astype(bool)]):
            s = (1.0 / 0.1) * (float(p["intensity"]) - int(p["intensity"]))
            R = fr.qtoR(fr.axis2Quat(fr.F64, s * phi))
            P2 = np.array([p["x"], p["y"], p["z"]], float)
            cf = np.array(c[:3], float)
            rows.append(np.concatenate([cf @ (-R @ fr.skew(fr.F64, P2)), cf]))
    J = np.array(rows)
    return np.linalg.eigvalsh(J.T @ J), int(a["surf_mask"].sum()), int(a["corner_mask"].sum())


def oracle_last_ids(ob, defs, prm, u, t0, q0, iters):
    """The oracle's correspondence IDs of the last iteration of an `iters`-iteration run: its pose after iters - 1
    iterations (a shorter run of the same loop), then that iteration's association.  Only used where that iteration
    searched: a second oracle cannot stand for IDs the reference carries over from an earlier search (icp_freq 2, odd
    iterations); test_gpu_fuzz.py pins that carry-over through lins_gpu_associate."""
    o = ob.Oracle(defs.LinsParams.shipped(icp_freq=prm.icp_freq, num_iter=max(iters - 1, 1)))
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    t, q = t0, q0
    if iters > 1:
        t, q, _, _ = o.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
    st = np.zeros(19)
    st[0:3], st[6:10] = t, q
    a = o.associate(u["surf_flat"], u["corner_sharp"], st, iters - 1)
    o.close()
    return a["surf_ind"], a["corner_ind"]


def run_both(gpu, ob, defs, prm, u, t0, q0):
    gpu.set_params(prm)
    gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    o = ob.Oracle(prm)
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    to, qo, ito, cvo = o.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
    o.close()
    tg, qg, itg, cvg = gpu.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
    assert (itg, cvg) == (ito, cvo), (itg, cvg, ito, cvo)
    diff = max(np.abs(tg - to).max(), np.abs(qg - qo).max())
    assert diff <= POSE_TOL, diff
    if (ito - 1) % prm.icp_freq == 0:  # the last iteration searched (see oracle_last_ids)
        si, ci = gpu.download_indices(len(u["surf_flat"]), len(u["corner_sharp"]))
        osi, oci = oracle_last_ids(ob, defs, prm, u, t0, q0, ito)
        assert np.array_equal(si, osi) and np.array_equal(ci, oci), (ito, (si != osi).sum(), (ci != oci).sum())
        n_ids[0] += 1
    return diff, ito, cvo


@pytest.fixture(scope="module")
def scenes(defs):
    rng = np.random.default_rng(41)
    out = dict(corridor=unit(rng, defs, corridor), yard=unit(rng, defs, yard))
    few_s = unit(rng, defs, yard)
    few_s["surf_flat"] = few_s["surf_flat"][:8]
    few_c = unit(rng, defs, yard)
    few_c["corner_sharp"] = few_c["corner_sharp"][:3]
    # 12 floor queries (rings >= 2: the tripod needs a ring below), 4 of them lifted 2 m: all 12 match while the weight is
    # 1, only 8 once s = 1 - 1.8 |res| / sqrt(range) applies (iter >= icp_freq)
    wt = unit(rng, defs, yard)
    q = wt["surf_flat"]
    floor = q[(q["z"] < -1.4) & (q["intensity"] >= 2)][:12].copy()
    floor["z"][::3] += 2.0
    wt["surf_flat"] = floor
    out.update(few_surfs=few_s, few_corners=few_c, weight_drop=wt)
    return out


@pytest.fixture
def ctx(capi):
    """A context of this test's own: the parameters it sets do not outlive it."""
    g = capi.LinsGpu()
    yield g
    g.close()


@pytest.mark.parametrize("icp_freq", [1, 2])
def test_estimate_transform_scenes_match_the_oracle(ctx, ob, defs, scenes, icp_freq):
    gpu = ctx
    prm = defs.LinsParams.shipped(icp_freq=icp_freq)
    worst, seen = 0.0, {}
    # the corridor: one J^T J eigenvalue (translation along the walls) below 10, the rest far above
    u = scenes["corridor"]
    t0, q0 = start((0.3, 0.05, 0.02), (0.5, -0.3, 1.0))
    ev, ns, nc = jtj_eigenvalues(ob, prm, u, t0, q0)
    low = ev[ev < 10]
    assert 1 <= len(low) <= 2 and ns >= 10 and nc >= 5, (ev, ns, nc)
    assert all(abs(e - 10) > 1e-3 * 10 for e in ev) and np.all(np.diff(ev) > 1e-3 * np.maximum(np.abs(ev[1:]), 1e-300)), ev
    d, it, cv = run_both(gpu, ob, defs, prm, u, t0, q0)
    worst, seen["degenerate"] = max(worst, d), (it, cv)
    # too few matched surfs / corners: every iteration returns early, the pose stays where it started
    for name in ("few_surfs", "few_corners"):
        d, it, cv = run_both(gpu, ob, defs, prm, scenes[name], t0, q0)
        assert (it, cv) == (prm.num_iter, False), (name, it, cv)
        worst, seen[name] = max(worst, d), (it, cv)
    # >= 10 matched surfs unweighted, < 10 once the weight switches on: iteration 0 updates, the later ones return early
    u = scenes["weight_drop"]
    t1, q1 = start((0.02, -0.01, 0.0), (0.1, 0.0, 0.0))
    counts = []
    for it in (0, icp_freq):
        o = ob.Oracle(prm)
        o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        st = np.zeros(19)
        st[0:3], st[6:10] = t1, q1
        counts.append(int(o.associate(u["surf_flat"], u["corner_sharp"], st, it)["surf_mask"].sum()))
        o.close()
    assert counts[0] >= 10 > counts[1], counts
    d, it, cv = run_both(gpu, ob, defs, prm, u, t1, q1)
    worst, seen["weight_drop"] = max(worst, d), (it, cv)
    # far starts in the yard: 0.5-2 m and 5-10 degrees away; with num_iter = 3 the farthest cannot converge
    u = scenes["yard"]
    for k, (t, rpy) in enumerate((((0.5, 0.2, 0.0), (0, 0, 5)), ((1.2, -0.8, 0.1), (2, -3, 7)), ((1.5, 1.2, -0.1), (-4, 3, 10)))):
        d, it, cv = run_both(gpu, ob, defs, prm, u, *start(t, rpy))
        worst, seen[f"far{k}"] = max(worst, d), (it, cv)
    short = defs.LinsParams.shipped(icp_freq=icp_freq, num_iter=3)
    d, it, cv = run_both(gpu, ob, defs, short, u, *start((1.5, 1.2, -0.1), (-4, 3, 10)))
    assert (it, cv) == (3, False), (it, cv)
    worst, seen["no_convergence"] = max(worst, d), (it, cv)
    assert n_ids[0] > 0
    print("IDs compared", n_ids[0], "icp_freq", icp_freq, "iters / converged", seen, "worst |pose - oracle|", worst)
