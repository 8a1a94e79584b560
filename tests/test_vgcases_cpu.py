"""CPU suite for tests/vgcases.py: every case, episode and step of the plan does what its name claims, checked against
the VoxelGrid of tests/mapperref.py, the independent one of tests/pyfront.py and the mapping oracle, so that the GPU
suite tests/test_gpu_mappers_scale.py cannot silently stop reaching an edge."""
import numpy as np
import pytest

import mapperref
import pyfront
import vgcases as V

F = np.float32


@pytest.fixture(scope="module")
def cat():
    return V.catalogue()


@pytest.fixture(scope="module")
def plan(cat):
    return V.schedule(cat)


def _vg(points, leaf):
    try:
        return mapperref.voxel_grid(mapperref.xyzi(points), leaf)
    except mapperref.TooBig:
        return None


def _bits_nan(a, b):
    """Bit-equal, except that NaN intensities compare by NaN-ness."""
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a[:, 3]), np.isnan(b[:, 3])
    a, b = a.copy(), b.copy()
    a[na, 3] = b[nb, 3] = 0
    return np.array_equal(na, nb) and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_case_outcomes_and_counts_match_both_voxel_grids(cat):
    names = set(cat)
    assert {"empty_corner", "empty_surf", "empty_outlier", "empty_all", "one_point", "n31", "n32", "n33", "all_nonfinite",
            "nonfinite_ends", "voxel_faces", "dense_voxel", "far_coordinate", "nan_intensity"} <= names
    for c in cat.values():
        outs = [_vg(p, leaf) for p, leaf in zip(c.clouds, V.LEAVES)]
        if all(o is not None for o in outs):
            outs.append(_vg(mapperref.to_points(np.concatenate(outs[1:]), V.POINT_DTYPE), 0.4))  # surf DS + outlier DS
        assert any(o is None for o in outs) == (c.expect == "toobig"), c.name
        for p, leaf, o in zip(c.clouds, V.LEAVES, outs):
            if o is not None:
                assert _bits_nan(o, pyfront.voxel_grid(mapperref.xyzi(p), leaf)), c.name
        finite = [np.isfinite(p["intensity"]).all() for p in c.clouds]
        assert all(finite) == (c.name != "nan_intensity"), c.name


def test_edges_are_present(cat):
    for n in (31, 32, 33):
        assert all(len(p) == n for p in cat[f"n{n}"].clouds)
    for p in cat["all_nonfinite"].clouds:
        assert not np.isfinite(np.stack([p["x"], p["y"], p["z"]], 1)).all(1).any()
    for p in cat["nonfinite_ends"].clouds:
        xyz = np.stack([p["x"], p["y"], p["z"]], 1)
        assert not np.isfinite(xyz[0]).all() and not np.isfinite(xyz[-1]).all() and np.isfinite(xyz[1:-1]).all()
    x = cat["voxel_faces"].clouds[0]["x"]
    assert np.signbit(x[x == 0]).any() and (~np.signbit(x[x == 0])).any()
    inv = F(1.0) / F(0.2)
    assert (x * inv == np.floor(x * inv)).sum() >= 10  # points whose product lands on a face
    dv = mapperref.voxel_grid(mapperref.xyzi(cat["dense_voxel"].clouds[0]), 0.2)
    assert len(dv) <= 10 and len(cat["dense_voxel"].clouds[0]) == 900
    p = cat["offset_4e+06"].clouds[1]
    assert np.spacing(F(np.abs(p["x"]).min())) > 0.2  # the f32 ulp exceeds the leaf


def _box(points, leaf):
    q = mapperref.xyzi(points)[:, :3]
    q = q[np.isfinite(q).all(1)]
    inv = F(1.0) / F(leaf)
    lo, hi = np.floor(q.min(0) * inv).astype(np.int64), np.floor(q.max(0) * inv).astype(np.int64)
    return hi - lo + 1


def test_extent_products_at_the_int32_limit(cat):
    assert np.prod(_box(cat["extent_1290"].clouds[0], 0.2)) == 1290 ** 3 < V.INT32_MAX < 1291 ** 3
    assert np.prod(_box(cat["extent_1291"].clouds[0], 0.2)) == 1291 ** 3
    assert _box(cat["int32_extent"].clouds[0], 0.2).tolist() == [V.INT32_MAX, 1, 1]
    assert _box(cat["int32_extent_plus1"].clouds[0], 0.2).tolist() == [V.INT32_MAX + 1, 1, 1]
    # keys next to 2^31 - 1: the f32 differences to the box's floor round up to 2^31
    x = cat["int32_extent"].clouds[0]["x"]
    inv = F(1.0) / F(0.2)
    keys = (np.floor(x * inv) - np.floor(x.min() * inv)).astype(np.int64)
    assert keys.max() == 1 << 31 and ((keys >= V.INT32_MAX - 256) & (keys <= 1 << 31)).sum() >= 2
    assert len(mapperref.voxel_grid(mapperref.xyzi(cat["int32_extent"].clouds[0]), 0.2)) == 5


def test_far_coordinate_has_two_voxels_but_one_int32_clamped_key(cat):
    """The case the device's int cast of the box bounds merged: both bounds clamp to INT32_MAX on x, so div_x = 1."""
    p = mapperref.xyzi(cat["far_coordinate"].clouds[0])
    assert len(mapperref.voxel_grid(p, 0.2)) == len(pyfront.voxel_grid(p, 0.2)) == 2
    inv = F(1.0) / F(0.2)
    b = np.floor(p[:, :3] * inv)
    clamp = lambda v: np.clip(v, -2.0 ** 31, V.INT32_MAX).astype(np.int64)  # noqa: E731  (cvt.rzi.s32.f32)
    min_b, max_b = clamp(b.min(0)), clamp(b.max(0))
    div = max_b - min_b + 1
    assert div[0] == 1
    ijk = clamp(b - min_b.astype(F))
    keys = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    assert keys[0] == keys[1] == 352516608


def test_inf_and_2p62_bounds_are_toobig():
    with pytest.raises(mapperref.TooBig):
        mapperref.voxel_grid(np.array([[3e38, 0, 0, 0]], F), 0.2)  # 3e38 * 5 = inf
    with pytest.raises(mapperref.TooBig):
        mapperref.voxel_grid(np.array([[1e18, 0, 0, 0], [1e18, 0, 0, 0]], F), 0.2)
    assert len(mapperref.voxel_grid(np.array([[9e17, 0, 0, 0]], F), 0.2)) == 1  # 4.5e18 < 2^62


def test_gate_episodes_hit_the_exact_counts(cat, ob, defs):
    for nc, ns in ((10, 100), (11, 100), (10, 101), (11, 101)):
        c = cat[f"gate_{nc}_{ns}"]
        orc = mapperref.MappingOracle(ob.MapOracle(), defs.POINT_DTYPE)
        q, pos = V.GATE_POSE
        r1 = orc.step(100.0, q, pos, *c.clouds)
        assert r1["processed"] and r1["keyframe_saved"] and r1["map_skipped"]
        assert np.abs(orc.poses[0][0]).max() > 0.1  # the key frame's transform is not the identity
        r2 = orc.step(101.0, q, pos, *c.clouds)
        assert (len(orc.clouds["map_corner_ds"]), len(orc.clouds["map_surf_ds"])) == (nc, ns)
        assert r2["map_skipped"] == (not (nc > 10 and ns > 100))
        if not r2["map_skipped"]:
            assert list(r2["map"].n_sel) and max(r2["map"].n_sel) == 0  # nothing within the 1 m searches


def test_every_episode_has_its_outcome_on_the_oracle(cat, plan, ob, defs):
    """Each distinct episode of the plan through the mapping oracle: a toobig case fails in its one cycle; the others
    run all their cycles."""
    seen = {}
    for st in plan:
        for s, ev in (st.fail or {}).items():
            seen.setdefault(("fail", id(ev[3])), ev)
    for ev in seen.values():
        orc = mapperref.MappingOracle(ob.MapOracle(), defs.POINT_DTYPE)
        with pytest.raises(mapperref.TooBig):
            orc.step(*ev)
    eps = {}
    queues = [V.episode_queue(cat, s) for s in range(V.M_SLOTS)]
    for q in queues:
        for _ in range(8):
            ep = next(q)
            eps.setdefault((ep.cases, ep.pose), ep)
    for ep in eps.values():
        if cat[ep.cases[0]].expect == "toobig":
            continue
        orc = mapperref.MappingOracle(ob.MapOracle(), defs.POINT_DTYPE)
        for k, name in enumerate(ep.cases):
            r = orc.step(100.0 + k, ep.pose[0], ep.pose[1], *cat[name].clouds)
            assert r["processed"], ep.cases


def test_plan_reaches_every_P_and_the_big_round(cat, plan):
    Ps = [st.P for st in plan]
    assert set(V.P_TARGETS) <= set(Ps)
    # the boundaries of 5P (round 1) and P (round 2): 5 * 25 = 125 < 128 < 130 = 5 * 26, ...; P = 1 is the 32-bit round 2
    for lo, hi in ((25, 26), (51, 52), (102, 103), (128, 129), (8, 9)):
        assert (5 * lo - 1).bit_length() < (5 * hi - 1).bit_length() or (lo - 1).bit_length() < (hi - 1).bit_length()
    big = [st for st in plan if st.big]
    assert len(big) == 1
    b = big[0]
    n1 = b.round1_points()
    assert n1 > V.BIG_ROUND and n1 > 8 * 132 * 256  # (the GPU suite checks against the device's own SM count)
    sizes = [len(c) for s in sorted(b.events) for c in b.events[s][1][3:]]
    assert 0 in sizes and any(0 < n < 32 for n in sizes) and max(sizes) > 50_000
    # an empty or tiny segment between two large ones
    assert any(sizes[i - 1] > 10_000 and sizes[i] < 32 for i in range(1, len(sizes)))
    # running slots next to non-running ones, at the first and the last index
    assert any(0 in st.events and st.events[0][0] == "run" and st.events.get(1, ("absent",))[0] != "run" for st in plan)
    last = V.M_SLOTS - 1
    assert any(last in st.events and st.events[last][0] == "run" and st.events.get(last - 1, ("absent",))[0] != "run" for st in plan)
    assert sum(1 for st in plan if st.fail) >= 2
    kinds = {k for st in plan for k, _ in st.events.values()}
    assert kinds == {"run", "skip"}
    # every gate case reaches its second cycle (the one whose map is the first cycle's clouds)
    name = {id(c.clouds[0]): n for n, c in cat.items()}
    last, gates = {}, set()
    for st in plan:
        for s, (k, ev) in st.events.items():
            if k == "run":
                n = name.get(id(ev[3]))
                if s not in st.reset and n is not None and n.startswith("gate_") and last.get(s) == n:
                    gates.add(n)
                if s not in st.reset and n is not None and n.endswith("_after_gate") and last.get(s) == "gate_11_101":
                    gates.add(n)
                last[s] = n
    assert gates == {n for n in cat if n.startswith("gate_") or n.endswith("_after_gate")}
    fails = {cat_name for st in plan for ev in (st.fail or {}).values() for cat_name, c in cat.items() if c.clouds[0] is ev[3]}
    assert fails == {n for n, c in cat.items() if c.expect == "toobig"}
