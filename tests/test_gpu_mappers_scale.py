"""GPU suite for the mapping node's VoxelGrid and the lockstep mappers at scale, against the CPU oracle
(tests/mapperref.py with the C++ scan-to-map oracle) on the adversarial clouds of tests/vgcases.py.

* Every catalogue cloud through lins_gpu_voxel_grid at 0.2 and 0.4 m: bit-equal to mapperref.voxel_grid, or
  LINS_E_TOOBIG where it raises TooBig.
* 160 slots stepping queues of short episodes (mappers_reset at every boundary) through a plan whose processed-slot
  counts P cross the bit boundaries of the segmented sorts' keys (5P segments in round 1, P in round 2), with a round of
  more than 600 k points that makes the bounds kernel's lanes walk across segment ends, and steps that fail with
  LINS_E_TOOBIG and are repeated without the failing cloud.  Each slot has its own oracle, compared at every step as
  tests/test_gpu_mapper.py compares the single mapper, and each finished episode is replayed on one spare single
  mapper whose reports must be memcmp-equal.
* The eight drives of tests/test_gpu_mappers.py in 132 slots at full windows, each slot against a single-mapper record
  of its (drive, first event)."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import mapper_drive
import mapperref
import test_gpu_mapper as single
import vgcases as V
from test_gpu_mappers import _split

pytestmark = pytest.mark.gpu
T_TOL = 1e-5
CLOUDS = ("map_corner_ds", "map_surf_ds", "corner_ds", "surf_ds", "outlier_ds", "surf_total_ds")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_cloud(got, want, nan_intensity=False):
    """Bit-equal (n, 4) clouds; with nan_intensity, NaN intensities compare by NaN-ness (their payloads may differ)."""
    if got.shape != want.shape:
        return False
    if nan_intensity:
        ng, nw = np.isnan(got[:, 3]), np.isnan(want[:, 3])
        if not np.array_equal(ng, nw):
            return False
        got, want = got.copy(), want.copy()
        got[ng, 3] = want[nw, 3] = 0
    return np.array_equal(_bits(got), _bits(want))


def _sm_count():
    """The device's multiprocessor count (CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT), read through the driver API."""
    cu = C.CDLL("libcuda.so.1")
    assert cu.cuInit(0) == 0
    dev, n = C.c_int(0), C.c_int(0)
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(n), 16, dev) == 0
    return n.value


@pytest.fixture(scope="module")
def cat():
    return V.catalogue()


def test_single_segment_matches_the_oracle(capi, gpu, cat):
    n = 0
    for c in cat.values():
        for p in c.clouds:
            for leaf in (0.2, 0.4):
                try:
                    want = mapperref.voxel_grid(mapperref.xyzi(p), leaf)
                except mapperref.TooBig:
                    with pytest.raises(capi.LinsError, match="error -4"):
                        gpu.voxel_grid(p, leaf)
                    n += 1
                    continue
                assert _same_cloud(gpu.voxel_grid(p, leaf), want, c.name == "nan_intensity"), (c.name, leaf)
    assert n >= 4


def test_far_coordinate_keeps_its_voxels(gpu, cat):
    """Two points 2^31 voxels out along x at 0.2 m lie in two voxels (int64 box bounds); an int32 cast of the bounds
    clamps both to INT32_MAX, gives div_x = 1 and one key."""
    p = cat["far_coordinate"].clouds[0]
    want = mapperref.voxel_grid(mapperref.xyzi(p), 0.2)
    got = gpu.voxel_grid(p, 0.2)
    assert len(want) == 2 and len(got) == 2 and _same_cloud(got, want)


def _check_processed(ctx, g, s, rep, ro, orc, nan_intensity):
    """One processed slot against its oracle (as test_gpu_mapper._run); the oracle then adopts the device's pose."""
    assert np.array_equal(_bits(rep.transform_guess), _bits(ro["transform_guess"])), ctx
    poses, window, clouds = g.mappers_download(s, rep)
    for k, v in orc.clouds.items():
        assert _same_cloud(clouds[k], v, nan_intensity), f"{ctx} {k}"
    assert rep.map.skipped == ro["map_skipped"], ctx
    assert (rep.keyframe_saved, rep.n_keyframes, rep.loop_candidate) == (ro["keyframe_saved"], ro["n_keyframes"], ro["loop_candidate"]), ctx
    assert list(window) == ro["window"] and rep.window_len == len(ro["window"]), ctx
    counts = (rep.n_map_corner_ds, rep.n_map_surf_ds)
    assert counts == (len(orc.clouds["map_corner_ds"]), len(orc.clouds["map_surf_ds"])), ctx
    if not rep.map.skipped:
        assert rep.map.iters == ro["map"].iters and list(rep.map.n_sel) == list(ro["map"].n_sel), ctx
    assert np.abs(np.array(rep.transform_aft_mapped) - ro["transform_aft_mapped"]).max() <= T_TOL, ctx
    assert len(poses) == len(orc.poses)
    assert np.abs(poses[:, :6] - np.array([p for p, _ in orc.poses])).max() <= T_TOL, ctx
    assert np.array_equal(poses[:, 6], [t for _, t in orc.poses]), ctx
    orc.adopt(np.array(rep.transform_aft_mapped, np.float32), poses[-1] if rep.keyframe_saved else None)
    return counts


def test_lockstep_episodes_match_the_oracle(capi, ob, defs, cat):
    plan = V.schedule(cat)
    M = V.M_SLOTS
    g, spare = capi.LinsGpu(), capi.LinsGpu()
    g.mappers_open(M)
    orc = [None] * M
    hist = [[] for _ in range(M)]  # the current episode's (event, report bytes)
    nan_i = [False] * M
    replays = 0

    def replay(s):
        nonlocal replays
        if not hist[s]:
            return
        spare.mapper_reset()
        for k, (ev, rb) in enumerate(hist[s]):
            assert bytes(spare.mapper_step(*ev)) == rb, f"slot {s} replay event {k}"
        hist[s] = []
        replays += 1

    seen_P, gates, fails, big_n, no_corner = [], set(), 0, 0, 0
    for j, st in enumerate(plan):
        for s in st.reset:
            replay(s)
            orc[s] = mapperref.MappingOracle(ob.MapOracle(), defs.POINT_DTYPE, scan_period=g.params.scan_period)
            nan_i[s] = False
        if st.reset:
            mask = np.zeros(M, np.uint8)
            mask[sorted(st.reset)] = 1
            g.mappers_reset(mask)
        steps = [None] * M
        for s, (_, ev) in st.events.items():
            steps[s] = ev
        if st.fail:
            bad = list(steps)
            for s, ev in st.fail.items():
                bad[s] = ev
            with pytest.raises(capi.LinsError, match="error -4"):
                g.mappers_step(bad)
            fails += 1
        reps = g.mappers_step(steps)
        P = 0
        for s in range(M):
            if steps[s] is None:
                assert reps[s] is None
                continue
            rep, ev = reps[s], steps[s]
            ro = orc[s].step(*ev)
            ctx = f"step {j} slot {s} ({st.events[s][0]})"
            assert (rep.processed, rep.skipped_interval) == (ro["processed"], ro["skipped_interval"]), ctx
            assert rep.processed == (st.events[s][0] == "run"), ctx
            hist[s].append((ev, bytes(rep)))
            nan_i[s] |= any(not np.isfinite(c["intensity"]).all() for c in ev[3:])
            if rep.processed:
                P += 1
                counts = _check_processed(ctx, g, s, rep, ro, orc[s], nan_i[s])
                if counts in ((10, 100), (11, 100), (10, 101), (11, 101)):
                    gates.add(counts + (rep.map.skipped,))
                no_corner += not rep.map.skipped and rep.n_corner_ds == 0  # a map, and no corner query
        assert P == st.P, j
        seen_P.append(P)
        if st.big:
            big_n = st.round1_points()
    for s in range(M):
        replay(s)
    g.close(); spare.close()
    sms = _sm_count()
    print(f"\nlockstep plan: P per step {seen_P}, largest P {max(seen_P)}; big round {big_n} points "
          f"(bounds-kernel stride threshold 8 * {sms} SMs * 256 = {8 * sms * 256}); {fails} failing steps; {replays} replays")
    assert set(V.P_TARGETS) <= set(seen_P) and max(seen_P) == V.M_SLOTS
    assert big_n > V.BIG_ROUND and big_n > 8 * sms * 256
    assert gates == {(10, 100, 1), (11, 100, 1), (10, 101, 1), (11, 101, 0)}
    assert fails >= 2 and replays >= V.M_SLOTS and no_corner >= 2


# ---- full windows at M = 132 -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def drives(synth):
    """The drives of tests/test_gpu_mappers.py."""
    mk = lambda **kw: _split(mapper_drive.make_drive(synth, **kw))  # noqa: E731
    return [
        mk(n_out=36, seed=4, stall_at=50),
        mk(n_out=30, seed=5, stall_at=51),
        mk(n_out=34, seed=6, stall_at=60),
        _split([e for e in mapper_drive.make_drive(synth, n_out=6, stall_at=-1, sparse_first=1) if e[0] == "odom"]),
        _split(single.shim_events(synth, 30, seed=3)),
        _split(single.shim_events(synth, 24, seed=7)),
        mk(n_out=5, seed=8, stall_at=-1),
        mk(n_out=8, seed=9, stall_at=-1),
    ]


def _digest(download):
    poses, window, clouds = download
    h = hashlib.blake2b(digest_size=16)
    for a in (poses, window) + tuple(clouds[k] for k in CLOUDS):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.digest()


def _imu_rows(imu):
    return tuple(np.array(a) for a in zip(*imu)) if imu else None


def test_full_windows_at_132_slots(capi, drives):
    """Slot s runs drive s % 8 from its event (s // 8) % 3 on, starting at step s % 7: every (drive, first event) runs
    once on a single mapper, and each slot that replays it gives memcmp-equal reports and bit-equal downloads."""
    M = 132
    plan = [(s % 8, (s // 8) % 3, s % 7) for s in range(M)]
    ref = capi.LinsGpu()
    rec = {}
    for d, e0, _ in plan:
        if (d, e0) in rec:
            continue
        ref.mapper_reset()
        r = []
        for imu, odom in drives[d][e0:]:
            if imu:
                ref.mapper_imu(*_imu_rows(imu))
            rep = ref.mapper_step(*odom)
            r.append((bytes(rep), _digest(ref.mapper_download(rep)) if rep.processed else None))
        rec[(d, e0)] = r
    ref.close()
    g = capi.LinsGpu()
    g.mappers_open(M)
    n_steps = max(st + len(drives[d]) - e0 for d, e0, st in plan)
    full, compared = 0, 0
    for step in range(n_steps):
        rows, steps = [None] * M, [None] * M
        for s, (d, e0, st) in enumerate(plan):
            k = step - st
            if 0 <= k < len(drives[d]) - e0:
                imu, odom = drives[d][e0 + k]
                rows[s], steps[s] = _imu_rows(imu), odom
        g.mappers_imu(rows)
        reps = g.mappers_step(steps)
        n_full = 0
        for s, (d, e0, st) in enumerate(plan):
            if steps[s] is None:
                assert reps[s] is None
                continue
            rb, dg = rec[(d, e0)][step - st]
            assert bytes(reps[s]) == rb, f"step {step} slot {s} drive {d} from {e0}"
            if reps[s].processed:
                assert _digest(g.mappers_download(s, reps[s])) == dg, f"step {step} slot {s} drive {d} from {e0}"
                n_full += reps[s].window_len == 50
            compared += 1
        full = max(full, n_full)
    g.close()
    assert len(rec) == 24 and full >= 30 and compared > 5000
