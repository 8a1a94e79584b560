"""GPU suite: the CUDA path (through the C-ABI, ctypes) against the CPU oracle on the same inputs.

Parity bar (BASELINE.json north_star): correspondence indices / accept masks bit-exact, pointSel bit-exact
(f32), pose within 1e-4 m / 1e-4 rad per scan.  Tolerances for the f64 quantities are written in each test.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-4  # m and rad, north_star
STATE_TOL = 1e-7  # the f64 path differs from the oracle only by summation order / libm ulps


def _rot_err(q1, q2):
    d = abs(float(np.dot(q1, q2)))
    return 2 * np.arccos(min(1.0, d))


def _check_assoc(g, o, ctx=""):
    assert np.array_equal(g["surf_sel"], o["surf_sel"]), f"{ctx} surf pointSel not bit-exact"
    assert np.array_equal(g["corner_sel"], o["corner_sel"]), f"{ctx} corner pointSel not bit-exact"
    assert np.array_equal(g["surf_ind"], o["surf_ind"]), f"{ctx} surf indices differ"
    assert np.array_equal(g["corner_ind"], o["corner_ind"]), f"{ctx} corner indices differ"
    assert np.array_equal(g["surf_mask"], o["surf_mask"]) and np.array_equal(g["corner_mask"], o["corner_mask"]), f"{ctx} masks differ"
    for k in ("surf_coeff", "corner_coeff"):
        assert np.allclose(g[k], o[k], rtol=2e-6, atol=1e-9), f"{ctx} {k}"
        # f32 stores of f64 values: all but a handful bit-identical
        assert (g[k] != o[k]).mean() < 1e-3


def test_associate_matches_oracle(gpu, ob, golden_batch, golden_out):
    """Every iteration's association of the forced-10-iteration golden run, at the oracle's own linearisation
    points: pointSel, indices and masks bit-exact."""
    prm = ob.LinsParams.shipped(num_iter=10, force_all_iters=1)
    gpu.set_params(prm)
    for i in range(golden_batch.n):
        u = golden_batch.unit(i)
        o = ob.Oracle(prm, use_kdtree=False)
        o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        lin = golden_out[f"forced10_{i}_lin_state"]
        for it in range(len(lin)):
            go = gpu.associate(u["surf_flat"], u["corner_sharp"], lin[it], it)
            oo = o.associate(u["surf_flat"], u["corner_sharp"], lin[it], it)
            _check_assoc(go, oo, f"unit {i} iter {it}")
            assert np.array_equal(go["surf_ind"], golden_out[f"forced10_{i}_surf_ind"][it])
            assert np.array_equal(go["corner_ind"], golden_out[f"forced10_{i}_corner_ind"][it])
            assert np.array_equal(go["surf_mask"], golden_out[f"forced10_{i}_surf_mask"][it])


@pytest.mark.parametrize("tag,kw", [("shipped", {}), ("forced10", dict(num_iter=10, force_all_iters=1))])
def test_ieskf_matches_oracle_and_golden(gpu, ob, golden_batch, golden_out, tag, kw):
    prm = ob.LinsParams.shipped(**kw)
    gpu.set_params(prm)
    for i in range(golden_batch.n):
        u = golden_batch.unit(i)
        gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        so, co, rep = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
        g = lambda k: golden_out[f"{tag}_{i}_{k}"]  # noqa: E731
        assert [rep.iters, rep.converged, rep.diverged, rep.has_nan] == list(g("iters"))
        assert [list(rep.m_surf[: rep.iters]), list(rep.m_corner[: rep.iters])] == g("m").tolist()
        assert np.allclose(np.array(rep.residual_norm[: rep.iters]), g("rnorm"), rtol=1e-9)
        assert np.allclose(np.array(rep.update_norm[: rep.iters]), g("unorm"), rtol=1e-6, atol=1e-12)
        assert np.abs(so[:3] - g("state")[:3]).max() <= POSE_TOL and _rot_err(so[6:10], g("state")[6:10]) <= POSE_TOL
        assert np.abs(so - g("state")).max() <= STATE_TOL
        assert np.allclose(co, g("cov"), rtol=1e-6, atol=1e-13)
        C = co.reshape(18, 18)
        assert np.array_equal(C, C.T)  # enforceSymmetry


def test_batch_equals_single_and_oracle(gpu, ob, golden_batch):
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    sb, cb, rb = gpu.ieskf_batch(golden_batch)
    so, co, ro, _, _ = ob.ieskf_batch(prm, golden_batch, threads=2)
    assert np.array_equal(rb["iters"], ro["iters"]) and np.array_equal(rb["flags"], ro["flags"])
    assert np.array_equal(rb["scan_id"], np.arange(golden_batch.n))
    assert np.abs(sb - so).max() <= STATE_TOL
    assert np.allclose(cb, co, rtol=1e-6, atol=1e-13)
    assert np.allclose(rb["pose"][:, :3], sb[:, :3]) and np.allclose(rb["pose"][:, 3:], sb[:, 6:10])
    for i in range(golden_batch.n):
        u = golden_batch.unit(i)
        gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        s1, c1, _ = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
        assert np.array_equal(s1, sb[i]) and np.array_equal(c1, cb[i])  # same kernel, deterministic reductions


def test_batch_config3_vs_oracle(gpu, ob, synth):
    """A fresh seeded batch (not a committed fixture): whole-run parity on 48 units."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    b = synth.generate("config3", n=48, seed0=4242)
    sg, cg, rg = gpu.ieskf_batch(b)
    so, co, ro, _, _ = ob.ieskf_batch(prm, b, threads=4)
    assert np.array_equal(rg["iters"], ro["iters"]) and np.array_equal(rg["flags"], ro["flags"])
    assert np.abs(sg[:, :3] - so[:, :3]).max() <= POSE_TOL
    assert max(_rot_err(a, c) for a, c in zip(sg[:, 6:10], so[:, 6:10])) <= POSE_TOL
    assert np.abs(sg - so).max() <= STATE_TOL
    # determinism: a second run is bit-identical
    sg2, cg2, rg2 = gpu.ieskf_batch(b)
    assert np.array_equal(sg, sg2) and np.array_equal(cg, cg2)


def test_dense64_and_stress_queries(gpu, ob, synth):
    """BASELINE.json configs[3] (64x1024) and the literal '2k surf + 500 edge' query counts of configs[0]:
    more queries than one shared-memory tile, more targets than the VLP-16 shape."""
    prm = ob.LinsParams.shipped(num_iter=4, force_all_iters=1)
    gpu.set_params(prm)
    for cfg, n in (("config4", 2), ("config1b", 2)):
        b = synth.generate(cfg, n=n, seed0=77)
        sg, cg, rg = gpu.ieskf_batch(b)
        so, co, ro, _, _ = ob.ieskf_batch(prm, b, threads=2)
        assert np.array_equal(rg["iters"], ro["iters"]) and np.array_equal(rg["flags"], ro["flags"])
        assert np.abs(sg - so).max() <= STATE_TOL
        u = b.unit(0)
        o = ob.Oracle(prm, use_kdtree=True)
        o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        _check_assoc(gpu.associate(u["surf_flat"], u["corner_sharp"], u["state"], 1),
                     o.associate(u["surf_flat"], u["corner_sharp"], u["state"], 1), cfg)


def test_unsorted_rings_take_the_sequential_walk(gpu, ob, golden_batch, defs):
    """Targets in arbitrary ring order: the ring-start table is invalid, the literal sequential walk must give
    the reference's answer (early `break` on the first out-of-window ring)."""
    rng = np.random.default_rng(0)
    u = golden_batch.unit(1)
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    ts = u["surf_less_flat"][rng.permutation(len(u["surf_less_flat"]))[:3000]].copy()
    tc = u["corner_less_sharp"][rng.permutation(len(u["corner_less_sharp"]))].copy()
    o = ob.Oracle(prm, use_kdtree=False)
    o.set_map(ts, tc)
    gpu.set_map(ts, tc)
    _check_assoc(gpu.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0), o.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0))
    # weird ring values (negative / huge) also force the sequential walk
    ts2 = u["surf_less_flat"][:2000].copy()
    ts2["intensity"][::7] += 300.0
    ts2["intensity"][::11] -= 20.0
    o.set_map(ts2, tc)
    gpu.set_map(ts2, tc)
    _check_assoc(gpu.associate(u["surf_flat"], u["corner_sharp"], u["state"], 1), o.associate(u["surf_flat"], u["corner_sharp"], u["state"], 1))


def test_far_and_unmatched_queries(gpu, ob, golden_batch):
    """The device 1-NN index must stay exact when the nearest target is far away: queries displaced by 0.6 m,
    1.3 m, 3 m (outer search rings / brute-force fallback) and 40 m (no target within the 5 m gate)."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    u = golden_batch.unit(2)
    o = ob.Oracle(prm, use_kdtree=False)
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    for shift in (0.6, 1.3, 3.0, 40.0):
        st = u["state"].copy()
        st[0] += shift * 10.0  # s = 10 * frac(intensity) in [0, 1): displaces each query by up to `shift` * 10 * 0.1
        st[2] += 0.3 * shift
        go, oo = gpu.associate(u["surf_flat"], u["corner_sharp"], st, 0), o.associate(u["surf_flat"], u["corner_sharp"], st, 0)
        _check_assoc(go, oo, f"shift {shift}")
    nan_state = u["state"].copy()
    nan_state[0] = np.nan
    go, oo = gpu.associate(u["surf_flat"], u["corner_sharp"], nan_state, 0), o.associate(u["surf_flat"], u["corner_sharp"], nan_state, 0)
    assert np.array_equal(go["surf_ind"], oo["surf_ind"]) and np.array_equal(go["corner_ind"], oo["corner_ind"])
    assert not go["surf_mask"].any() and not oo["surf_mask"].any()


def test_icp_freq_reuses_indices(gpu, ob, golden_batch):
    """ICP_FREQ = 2: odd iterations reuse pointSearch*Ind of the previous one (StateEstimator.hpp:844, :970) and
    the robust weight starts at iter >= ICP_FREQ."""
    prm = ob.LinsParams.shipped(icp_freq=2, num_iter=6, force_all_iters=1)
    gpu.set_params(prm)
    u = golden_batch.unit(0)
    o = ob.Oracle(prm)
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    so, co, ro = o.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
    sg, cg, rg = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
    assert rg.iters == ro.iters == 6
    assert list(rg.m_surf[:6]) == list(ro.m_surf[:6]) and list(rg.m_corner[:6]) == list(ro.m_corner[:6])
    assert np.abs(sg - so).max() <= STATE_TOL


def test_edge_cases_empty_and_ragged(gpu, ob, golden_batch, defs):
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    e = defs.make_points(np.zeros((0, 3)), [])
    u = golden_batch.unit(0)
    # empty queries / empty map / both: one iteration, update == prior difference == 0, converged
    for ms, mc, qs, qc in ((e, e, e, e), (u["surf_less_flat"], u["corner_less_sharp"], e, e), (e, e, u["surf_flat"], u["corner_sharp"])):
        gpu.set_map(ms, mc)
        sg, cg, rg = gpu.ieskf(qs, qc, u["state"], u["cov"])
        o = ob.Oracle(prm)
        o.set_map(ms, mc)
        so, co, ro = o.ieskf(qs, qc, u["state"], u["cov"])
        assert (rg.iters, rg.converged, rg.diverged) == (ro.iters, ro.converged, ro.diverged) == (1, 1, 0)
        assert np.allclose(sg, so, atol=1e-12) and np.allclose(cg, co, rtol=1e-9, atol=1e-15)
    # ragged batch: units with zero queries / zero targets mixed with normal ones
    b = golden_batch
    clouds = {k: b.clouds[k] for k in b.FIELDS}
    offsets = {k: b.offsets[k].copy() for k in b.FIELDS}
    offsets["surf_flat"][2:] = offsets["surf_flat"][2]          # units 2.. have no surf queries
    clouds["surf_flat"] = clouds["surf_flat"][: offsets["surf_flat"][-1]]
    offsets["corner_less_sharp"][1:] = offsets["corner_less_sharp"][1]  # units 1.. have no corner targets
    clouds["corner_less_sharp"] = clouds["corner_less_sharp"][: offsets["corner_less_sharp"][-1]]
    rag = defs.Batch(clouds, offsets, b.state, b.cov)
    sg, cg, rg = gpu.ieskf_batch(rag)
    so, co, ro, _, _ = ob.ieskf_batch(prm, rag, threads=1)
    assert np.array_equal(rg["iters"], ro["iters"]) and np.array_equal(rg["flags"], ro["flags"])
    assert np.abs(sg - so).max() <= STATE_TOL


def test_divergence_is_reported(gpu, ob, golden_batch):
    """NaN prior -> the NaN branch (StateEstimator.hpp:552-563); state_out = prior, cov_out = cov_in."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    u = golden_batch.unit(0)
    gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    o = ob.Oracle(prm)
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    st = u["state"].copy()
    st[3] = np.nan  # velocity does not enter the association, only the update vector
    sg, cg, rg = gpu.ieskf(u["surf_flat"], u["corner_sharp"], st, u["cov"])
    so, co, ro = o.ieskf(u["surf_flat"], u["corner_sharp"], st, u["cov"])
    assert (rg.iters, rg.diverged, rg.has_nan, rg.converged) == (ro.iters, ro.diverged, ro.has_nan, ro.converged) == (1, 1, 1, 0)
    assert np.array_equal(np.isnan(sg), np.isnan(st)) and np.array_equal(cg, u["cov"])
    # residual blow-up branch (:566-570): a second call whose first residual is > 10 x 1e6 cannot happen with
    # finite data; exercise it through lidar_scale instead
    prm2 = ob.LinsParams.shipped(lidar_scale=1e9)
    gpu.set_params(prm2)
    o2 = ob.Oracle(prm2)
    o2.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    sg, cg, rg = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
    so, co, ro = o2.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
    assert (rg.iters, rg.diverged, rg.has_nan) == (ro.iters, ro.diverged, ro.has_nan) == (1, 1, 0)
    assert np.array_equal(sg, u["state"])


def test_update_map_and_stale_index_quirk(gpu, ob, synth):
    """Row F1: transformToEnd + map refresh, including the `>= 5 && >= 20` guard that leaves the 1-NN index on
    the older cloud while the walk cloud advances (StateEstimator.hpp:1156-1160)."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    b = synth.generate("config3", n=1, seed0=9)
    u = b.unit(0)
    ns, nc = b.extra["new_surf_less_flat"], b.extra["new_corner_less_sharp"]
    o = ob.Oracle(prm, use_kdtree=False)
    for o_ in (o, gpu):
        o_.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    sg, cg, rg = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
    s1, c1, rep1 = o.update_map(ns, nc, sg)
    s2, c2, rep2 = gpu.update_map(ns, nc, sg)
    assert rep1 and rep2
    for a, c in ((s1, s2), (c1, c2)):
        A = np.stack([a["x"], a["y"], a["z"]], 1)
        Cc = np.stack([c["x"], c["y"], c["z"]], 1)
        assert np.allclose(A, Cc, rtol=0, atol=2e-6) and (A != Cc).mean() < 1e-3
        assert np.array_equal(a["intensity"], c["intensity"])
    # guard fails (4 corner points): map advances, index does not
    s1, c1, rep1 = o.update_map(ns[:60], nc[:4], sg)
    s2, c2, rep2 = gpu.update_map(ns[:60], nc[:4], sg)
    assert not rep1 and not rep2
    go, oo = gpu.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0), o.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0)
    assert np.array_equal(go["surf_ind"], oo["surf_ind"]) and np.array_equal(go["corner_ind"], oo["corner_ind"])
    assert np.array_equal(go["surf_mask"], oo["surf_mask"])


def test_estimate_transform_fallback(gpu, ob, golden_batch):
    """Row A12: the 6-DoF Gauss-Newton ICP used on divergence and for scan-2 initialisation."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    for i in (0, 1):
        u = golden_batch.unit(i)
        o = ob.Oracle(prm)
        o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        t0, q0 = u["state"][:3], u["state"][6:10]
        to, qo, ito, cvo = o.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
        tg, qg, itg, cvg = gpu.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
        assert (itg, cvg) == (ito, cvo)
        assert np.abs(tg - to).max() <= POSE_TOL and _rot_err(qg, qo) <= POSE_TOL


def test_full_size_properties(gpu, ob, synth):
    """BASELINE.json configs[2] at bench size through size-independent properties: determinism, scan-order
    independence (units are independent), symmetric PSD covariances, unit quaternions, iteration accounting."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    b = synth.generate("config3", n=256, seed0=1000)
    s1, c1, r1 = gpu.ieskf_batch(b)
    perm = np.random.default_rng(1).permutation(b.n)
    s2, c2, r2 = gpu.ieskf_batch(b.subset(perm))
    assert np.array_equal(s1[perm], s2) and np.array_equal(c1[perm], c2) and np.array_equal(r1["iters"][perm], r2["iters"])
    assert np.abs(np.linalg.norm(s1[:, 6:10], axis=1) - 1).max() < 1e-12
    ok = (r1["flags"] & 2) == 0
    C = c1[ok].reshape(-1, 18, 18)
    assert np.array_equal(C, C.transpose(0, 2, 1))
    assert min(np.linalg.eigvalsh(c).min() for c in C) > -1e-9
    assert ((r1["iters"] >= 1) & (r1["iters"] <= prm.num_iter)).all()
    conv = (r1["flags"] & 1) == 1
    assert (r1["iters"][~conv & ok] == prm.num_iter).all()
    # a sample of the batch against the oracle
    idx = list(range(0, 256, 16))
    so, co, ro, _, _ = ob.ieskf_batch(prm, b.subset(idx), threads=4)
    assert np.array_equal(r1["iters"][idx], ro["iters"]) and np.abs(s1[idx] - so).max() <= STATE_TOL


def test_state_estimator_shim_sequence(gpu, ob, synth):
    """Rows B / F3: the C++ mirror of fusion::StateEstimator (csrc/host/state_estimator.hpp) driven like LinsFusion
    drives the reference (Estimator.cpp:204-252) over a synthetic drive.  Scan 1 initialises, scan 2 runs the ICP
    initialiser, every later scan runs performIESKF on the device; each recorded update is replayed through the
    oracle, and the relative motion must track the truth."""
    out = synth.run_sequence("config3", seed=3, n_scans=12)
    assert list(out["status"][:2]) == [1, 3] and (out["status"][2:] == 3).all()  # FIRST_SCAN, then RUNNING
    units = out["units"]
    assert units is not None and units.n == 10
    prm = ob.LinsParams.shipped()
    so, co, ro, _, _ = ob.ieskf_batch(prm, units, threads=2)
    assert np.array_equal(out["iters"], ro["iters"]) and np.array_equal(out["flags"], ro["flags"].astype(np.int32))
    ok = (out["flags"] & 2) == 0
    assert ok.all()
    assert np.abs(out["state_out"][ok] - so[ok]).max() <= STATE_TOL
    # the estimate tracks the true per-scan motion once the filter has settled: the first updates after the ICP
    # initialiser still carry its velocity error in the prior (measured: 0.24, 0.11, 0.03 m, then 1-2 cm)
    terr = np.abs(out["state_out"][:, :3] - units.truth[:, :3])
    assert terr[3:].max() < 0.06 and terr.max() < 0.5, terr
    assert max(_rot_err(a, b) for a, b in zip(out["state_out"][3:, 6:10], units.truth[3:, 3:])) < 5e-3
