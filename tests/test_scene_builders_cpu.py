"""CPU checks of the scene builders behind test_gpu_paths.py: each builder must produce what its GPU test claims to
exercise (ring range, ring order, target counts, bucket occupancy, duplicates), so that an edit to a builder cannot
quietly stop reaching a limit while the GPU test stays green.  The path predicates mirror unit_prologue (lins_gpu.cu)."""
import numpy as np
import pytest

import scenes


@pytest.fixture(scope="module")
def legacy_units(synth, defs):
    base = synth.generate("config3", n=60, seed0=52000)
    return scenes.legacy_batch_units(np.random.default_rng(20261015), defs, base, n_random=40)


def test_legacy_batch_kinds(legacy_units):
    units, tags = legacy_units
    assert len(units) >= 600
    kinds = [t.split()[1] for t in tags]
    # interleaved by kind: every window of len(LEGACY_KINDS) units holds one of each
    assert kinds[: 2 * len(scenes.LEGACY_KINDS)] == list(scenes.LEGACY_KINDS) * 2
    for u, kind in zip(units, kinds):
        ts, tc = u["surf_less_flat"], u["corner_less_sharp"]
        rs, rc = scenes.rings_of(ts), scenes.rings_of(tc)
        assert scenes.unit_indexed(u) == (kind in ("none", "ring_neg_half")), kind
        if kind == "perm":
            assert (np.diff(rs) < 0).any() and (np.diff(rc) < 0).any()
        elif kind in ("ring128", "ring300"):
            assert rs[-1] == int(kind[4:]) and (np.diff(rs) >= 0).all() and (rs[:-1] < scenes.K_MAX_RING).all()
        elif kind == "ring_neg":
            assert tc["intensity"][0] == np.float32(-3.2) and rc[0] == -3 and (np.diff(rc) >= 0).all()
        elif kind == "ring_neg_half":
            assert tc["intensity"][0] == np.float32(-0.5) and rc[0] == 0
    dup = np.array(["dup" in t for t in tags])
    assert 0.3 <= dup.mean() <= 0.37
    for u, d in zip(units, dup):
        assert scenes.has_exact_duplicates(u["surf_less_flat"]) or scenes.has_exact_duplicates(u["corner_less_sharp"]) or not d
    # legacy units with duplicates whose copies sit next to each other: the sequential walks meet exact ties
    adjacent = 0
    for u, kind, d in zip(units, kinds, dup):
        if d and kind in ("ring128", "ring300", "ring_neg"):
            ts = u["surf_less_flat"]
            same = (ts["x"][1:] == ts["x"][:-1]) & (ts["y"][1:] == ts["y"][:-1]) & (ts["z"][1:] == ts["z"][:-1])
            adjacent += int(same.any())
    assert adjacent >= 50
    # config3 and random sources, both with unmodified (indexed) units to share CTAs with the legacy ones
    assert any(t.startswith("random") for t in tags) and sum(t.startswith("config3") for t in tags) >= 300


def test_capacity_units(defs):
    rng = np.random.default_rng(65535)
    for Ts in (65535, 65536):
        for Tc in (65535, 65536):
            u = scenes.capacity_unit(rng, defs, Ts, Tc)
            ts, tc = u["surf_less_flat"], u["corner_less_sharp"]
            assert (len(ts), len(tc)) == (Ts, Tc)
            for t in (ts, tc):
                r = scenes.rings_of(t)
                assert (np.diff(r) >= 0).all() and r.min() == 0 and r.max() == scenes.CAP_RINGS - 1
            assert scenes.cloud_indexable(ts) == (Ts == 65535) and scenes.cloud_indexable(tc) == (Tc == 65535)
            assert scenes.unit_indexed(u) == (Ts == 65535 and Tc == 65535)


@pytest.mark.parametrize("which", ["surf", "corner"])
@pytest.mark.parametrize("parity", [0, 1])
def test_big_bucket_units(defs, which, parity):
    rng = np.random.default_rng(40000)
    u, b = scenes.big_bucket_unit(rng, defs, which, parity)
    tgt, q = (u["surf_less_flat"], u["surf_flat"]) if which == "surf" else (u["corner_less_sharp"], u["corner_sharp"])
    tab = scenes.K_AZ_TAB_S if which == "surf" else scenes.K_AZ_TAB_C
    assert scenes.unit_indexed(u)
    cnt, nb = scenes.bucket_counts(tgt, tab)
    assert b % 2 == parity and cnt[b] >= 40000 and cnt[b ^ 1] >= 1000
    assert cnt.sum() == len(tgt) < scenes.K_MAX_T
    # the big bucket holds exact duplicates, and some queries are exact copies of them (distance-0 ties at the 1-NN)
    r = scenes.rings_of(tgt)
    bb = r.astype(np.int64) * nb + scenes.az_bin(tgt["x"], tgt["y"], nb)
    in_big = tgt[bb == b]
    assert scenes.has_exact_duplicates(in_big)
    key = lambda c: set(zip(c["x"].tolist(), c["y"].tolist(), c["z"].tolist()))  # noqa: E731
    xyz, counts = np.unique(np.stack([in_big["x"], in_big["y"], in_big["z"]], 1), axis=0, return_counts=True)
    dup_pts = set(map(tuple, xyz[counts > 1].tolist()))
    assert len(key(q) & dup_pts) >= 30
    # queries in both buckets
    qb = scenes.rings_of(q).astype(np.int64) * nb + scenes.az_bin(q["x"], q["y"], nb)
    assert (qb == b).sum() >= 100 and (qb == (b ^ 1)).sum() >= 30
    # bucket-interior points only (the edge queries excepted): numpy's atan2 cannot disagree with CUDA's on their bin
    a = np.arctan2(in_big["y"].astype(np.float64), in_big["x"].astype(np.float64))
    frac = (a + np.pi) / (2 * np.pi / nb) % 1.0
    assert frac.min() > 0.05 and frac.max() < 0.95


def test_ring_sweep_units_are_well_posed(ob, defs):
    """The sweep's units must not amplify rounding: the oracle's two equivalent gain forms agree on every residual norm
    far inside the GPU test's 1e-6 bar (an ill-posed unit that keeps jumping for 30 iterations does not)."""
    units, _ = scenes.ring_sweep_units(np.random.default_rng(128), defs)
    prm = ob.LinsParams.shipped()
    for i, u in enumerate(units):
        reps = []
        for form in (ob.FORM_A, ob.FORM_B):
            o = ob.Oracle(prm, use_kdtree=True)
            o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
            reps.append(o.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"], form=form)[2])
            o.close()
        a, b = reps
        assert a.iters == b.iters, i
        ra, rb = np.array(a.residual_norm[: a.iters]), np.array(b.residual_norm[: b.iters])
        assert np.allclose(ra, rb, rtol=1e-8, atol=1e-300), (i, float(np.max(np.abs(ra - rb) / np.maximum(rb, 1e-300))))


def test_ring_sweep_units(defs):
    rng = np.random.default_rng(128)
    units, tags = scenes.ring_sweep_units(rng, defs)
    cases = scenes.ring_sweep_cases()
    names = [c[0] for c in cases]
    assert {f"nrings {n}" for n in scenes.SWEEP_NRINGS} <= set(names)
    by_name = {c[0]: c for c in cases}
    for u, t in zip(units, tags):
        name = t.rsplit(" ", 1)[0]
        _, rs, rc = by_name[name]
        for cloud, want in ((u["surf_less_flat"], rs), (u["corner_less_sharp"], rc)):
            r = scenes.rings_of(cloud)
            assert (np.diff(r) >= 0).all(), t
            assert r.max() == max(want) and set(r.tolist()) <= set(want), t
            if t.endswith("beams"):
                assert set(r.tolist()) == set(want), t
        assert scenes.unit_indexed(u) == (max(max(rs), max(rc)) < scenes.K_MAX_RING), t
    # what the sweep reaches: every bins-per-ring value of both tables, ring 127 indexed, ring 128 legacy
    nbs = {scenes.az_bins_for(int(scenes.rings_of(u["surf_less_flat"]).max()) + 1, scenes.K_AZ_TAB_S) for u in units if scenes.unit_indexed(u)}
    assert nbs == {scenes.K_AZ_TAB_S >> k for k in range(8)}
    tops = {int(scenes.rings_of(u["surf_less_flat"]).max()) for u in units}
    assert {0, 1, 7, 8, 15, 16, 32, 63, 64, 99, 126, 127, 128} <= tops
    assert any(sorted(set(scenes.rings_of(u["surf_less_flat"]).tolist())) == [0, 127] for u in units)
    assert any(int(scenes.rings_of(u["surf_less_flat"]).max()) != int(scenes.rings_of(u["corner_less_sharp"]).max()) for u in units)


def test_global_scratch_units_exceed_shared_memory(synth):
    """config1b units carry thousands of queries: one unit's per-query arrays (140 B per query) exceed the 227 KB of
    shared memory a CTA can have on an H100."""
    b = synth.generate("config1b", n=2, seed0=56000)
    q = np.diff(b.offsets["surf_flat"]) + np.diff(b.offsets["corner_sharp"])
    assert q.min() >= 2500 and q.min() * 140 > 227 * 1024
