"""GPU suite: fuzz parity of the fused kernel's search (VERDICT r1 "next" item 3).

>= 2000 units through lins_gpu_ieskf_batch with the shipped parameters (num_iter 30) against the BRUTE-FORCE oracle:
iteration counts, flags, accepted-measurement counts and residual norms of EVERY iteration, and the correspondence IDs of
the last iteration bit-equal; posterior state within 1e-7.  The units stress exactly what the certificate / azimuth-window
pruning (lins_assoc_az.cuh) could get wrong and the synthetic benchmark data never does:
  * exact duplicate targets (true f32 ties at the 1-NN and in the walks -> lowest index / first visited must win),
  * queries next to the sensor's z axis (rho < 0.1 m: the whole-ring branch of az_halfwidth),
  * priors far from the truth (per-iteration displacement > 1 m: certificates must fail and re-search),
  * random small scenes: any ring count, tiny / empty clouds, queries far outside the map.
Reference: lins/include/StateEstimator.hpp:844-915, :970-1029 (search + walks), :465-600 (loop).
"""
import os

import numpy as np
import pytest

from scenes import STATE_TOL, batch_from_units, compare_units, gpu_batch_run, mutate, oracle_runs, random_scene

pytestmark = pytest.mark.gpu


def test_fuzz_2000_units_against_bruteforce_oracle(gpu, ob, synth, defs):
    rng = np.random.default_rng(20260923)
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    base = synth.generate("config3", n=384, seed0=31000)
    units = []
    for i in range(base.n):
        u = base.unit(i)
        units.append(mutate(rng, u, "none"))
        units.append(mutate(rng, u, "dup"))
        units.append(mutate(rng, u, "axis"))
        units.append(mutate(rng, u, "jump"))
    for _ in range(600):
        units.append(random_scene(rng, defs))
    assert len(units) >= 2000
    batch = batch_from_units(defs, units)

    g = gpu_batch_run(gpu, batch)
    outs = oracle_runs(ob, prm, units, use_kdtree=False)  # brute-force exact 1-NN, lowest index among ties

    def tag_of(i):
        return f"unit {i} (kind {['none', 'dup', 'axis', 'jump'][i % 4] if i < 4 * base.n else 'random'})"

    bad, st = compare_units(units, outs, g, batch, tag_of, STATE_TOL)
    print(f"fuzz: {len(units)} units, {st['n_div']} diverged, {st['n_jump']} with a > 1 m / rad update, worst state diff {st['worst']:.3g} (converged) {st['worst_nc']:.3g} (30 iterations, not converged)")
    assert not bad, (len(bad), bad[:10])
    assert st["n_jump"] >= 100, st["n_jump"]  # the stress really happened


def test_associate_reuses_indices_across_calls_icp_freq2(gpu, ob, golden_batch):
    """ADVICE r1 (medium): with ICP_FREQ > 1 a FRESH launch at iter % ICP_FREQ != 0 must take pointSearch*Ind from the
    context (they persist between calls like the reference's member arrays, StateEstimator.hpp:844, :970) — both through
    lins_gpu_associate(iter odd) and through the odd Gauss-Newton steps of lins_gpu_estimate_transform."""
    prm = ob.LinsParams.shipped(icp_freq=2)
    gpu.set_params(prm)
    for i in (0, 1):
        u = golden_batch.unit(i)
        o = ob.Oracle(prm, use_kdtree=False)
        o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        st0 = u["state"].copy()
        st1 = st0.copy()
        st1[0:3] += [0.05, -0.02, 0.01]
        for it, st in ((0, st0), (1, st1), (2, st1), (3, st0)):
            go, oo = gpu.associate(u["surf_flat"], u["corner_sharp"], st, it), o.associate(u["surf_flat"], u["corner_sharp"], st, it)
            assert np.array_equal(go["surf_ind"], oo["surf_ind"]) and np.array_equal(go["corner_ind"], oo["corner_ind"]), (i, it)
            assert np.array_equal(go["surf_mask"], oo["surf_mask"]) and np.array_equal(go["corner_mask"], oo["corner_mask"]), (i, it)
            assert np.allclose(go["surf_coeff"], oo["surf_coeff"], rtol=2e-6, atol=1e-9)
        t0, q0 = u["state"][:3], u["state"][6:10]
        to, qo, ito, cvo = o.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
        tg, qg, itg, cvg = gpu.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
        assert (itg, cvg) == (ito, cvo)
        assert np.abs(tg - to).max() <= 1e-4 and 2 * np.arccos(min(1.0, abs(float(np.dot(qg, qo))))) <= 1e-4


def test_update_map_stays_on_device(gpu, ob, synth):
    """Row F1 without the round trip: lins_gpu_update_map_ex with lin_state = NULL (the posterior lins_gpu_ieskf left on
    the device) and no read-back must install exactly the map the host-visible call installs — checked through the next
    scan's association against the oracle's updatePointCloud (StateEstimator.hpp:1116-1161)."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    for seed in (9, 10):
        b = synth.generate("config3", n=1, seed0=seed)
        u = b.unit(0)
        ns, nc = b.extra["new_surf_less_flat"], b.extra["new_corner_less_sharp"]
        o = ob.Oracle(prm, use_kdtree=False)
        for o_ in (o, gpu):
            o_.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        sg, cg, rg = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
        assert not rg.diverged
        s1, c1, rep1 = o.update_map(ns, nc, sg)
        assert gpu.update_map_device(ns, nc) == rep1 is True      # device posterior, nothing copied back
        go, oo = gpu.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0), o.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0)
        assert np.array_equal(go["surf_ind"], oo["surf_ind"]) and np.array_equal(go["corner_ind"], oo["corner_ind"])
        assert np.array_equal(go["surf_mask"], oo["surf_mask"]) and np.array_equal(go["corner_mask"], oo["corner_mask"])
        # explicit state + guard failure (map advances, index does not), still without read-back
        s1, c1, rep1 = o.update_map(ns[:60], nc[:4], sg)
        assert gpu.update_map_device(ns[:60], nc[:4], sg) == rep1 is False
        go, oo = gpu.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0), o.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0)
        assert np.array_equal(go["surf_ind"], oo["surf_ind"]) and np.array_equal(go["corner_ind"], oo["corner_ind"])


def test_bag_replay_equals_direct_drive(gpu, ob, synth, tmp_path):
    """Rows F3 + F4 end to end (the BASELINE.json configs[1] code path): the synthetic drive written as a ROS1 bag and
    replayed through the bag reader, image projection, feature extraction and the GPU IESKF must reproduce the run that
    was fed directly — and every recorded update must match the oracle."""
    bag = str(tmp_path / "drive.bag")
    synth.write_sequence_bag(bag, "config3", seed=3, n_scans=8)
    direct = synth.run_sequence("config3", seed=3, n_scans=8)
    replay = synth.run_bag(bag)
    assert list(replay["status"]) == list(direct["status"])
    assert np.array_equal(replay["iters"], direct["iters"]) and np.array_equal(replay["flags"], direct["flags"])
    # (IMU time steps come back from nanosecond stamps: dt differs from the simulator's by ~1e-10 s)
    assert np.abs(replay["state_out"] - direct["state_out"]).max() < 1e-6
    assert np.abs(replay["global_est"] - direct["global_est"]).max() < 1e-5
    units = replay["units"]
    so, co, ro, _, _ = ob.ieskf_batch(ob.LinsParams.shipped(), units, threads=2)
    assert np.array_equal(replay["iters"], ro["iters"]) and np.abs(replay["state_out"] - so).max() <= 1e-7


def test_pinned_direct_upload_equals_host_pack(gpu, capi, synth):
    """lins_gpu_batch_upload with caller-pinned clouds (lins_gpu_host_register) and the raw-DMA + device-pack path
    (LINS_UPLOAD=direct; the default policy picks it when few host threads per context are available, i.e. many ranks on
    one host) must give bit-identical results to the host-pack path, also for ragged / empty clouds."""
    b = synth.generate("config3", n=24, seed0=777)
    s0, c0, r0 = gpu.ieskf_batch(b)
    old = os.environ.get("LINS_UPLOAD")
    try:
        capi.pin_batch(b)
        os.environ["LINS_UPLOAD"] = "pinned"  # fails the call if a cloud is not pinned
        s1, c1, r1 = gpu.ieskf_batch(b)
        os.environ["LINS_UPLOAD"] = "pack"
        s2, c2, r2 = gpu.ieskf_batch(b)
        os.environ["LINS_UPLOAD"] = "hybrid"  # pack threads and the copy engine share the slices
        os.environ["LINS_PACK_THREADS"] = "1"
        big = synth.generate("config3", n=64, seed0=800)  # several 64 K-point slices per cloud
        sb0, cb0, _ = gpu.ieskf_batch(big)
        capi.pin_batch(big)
        p0 = gpu.batch_upload_stats()
        sb1, cb1, _ = gpu.ieskf_batch(big)
        p1 = gpu.batch_upload_stats()
        capi.unpin_batch(big)
        assert np.array_equal(sb0, sb1) and np.array_equal(cb0, cb1)
        assert (p1[0] - p0[0]) + (p1[1] - p0[1]) == sum(int(big.offsets[k][-1]) for k in big.FIELDS) and p1[1] > p0[1]
    finally:
        os.environ.pop("LINS_PACK_THREADS", None)
        capi.unpin_batch(b)
        if old is None:
            os.environ.pop("LINS_UPLOAD", None)
        else:
            os.environ["LINS_UPLOAD"] = old
    assert np.array_equal(s0, s1) and np.array_equal(c0, c1) and np.array_equal(r0["iters"], r1["iters"])
    assert np.array_equal(s0, s2) and np.array_equal(c0, c2)
    # an unpinned cloud under LINS_UPLOAD=pinned is an error, not a silent fallback
    os.environ["LINS_UPLOAD"] = "pinned"
    try:
        with pytest.raises(capi.LinsError):
            gpu.ieskf_batch(synth.generate("config3", n=2, seed0=778))
    finally:
        os.environ.pop("LINS_UPLOAD", None)


def test_packed16_batch_equals_xyzi32(gpu, capi, synth):
    """lins_batch_desc.point_format = LINS_POINTS_PACKED16: clouds handed over as 16-byte (x, y, z, intensity) records
    (pageable -> staged by memcpy; pinned -> one DMA per slice, no pack kernel) give bit-identical results."""
    b = synth.generate("config3", n=40, seed0=901)
    s0, c0, r0 = gpu.ieskf_batch(b)
    p = b.packed16()
    s1, c1, r1 = gpu.ieskf_batch(p)
    capi.pin_batch(p)
    try:
        s2, c2, r2 = gpu.ieskf_batch(p)
    finally:
        capi.unpin_batch(p)
    for s_, c_, r_ in ((s1, c1, r1), (s2, c2, r2)):
        assert np.array_equal(s0, s_) and np.array_equal(c0, c_) and np.array_equal(r0["iters"], r_["iters"])
