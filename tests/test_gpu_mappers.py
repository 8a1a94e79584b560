"""GPU suite for the lockstep mappers (lins_gpu_mappers_*): every slot against a single mapper (lins_gpu_mapper_step) on a
context of its own, fed the same events.  At every event the reports are memcmp-equal (all fields, the scan-to-map
report included), and the key poses, the window and the six downloaded clouds are bit-equal.  The single mapper is
pinned against the CPU oracle in tests/test_gpu_mapper.py, so each slot inherits that oracle through exact equality."""
import ctypes as C

import numpy as np
import pytest

import mapper_drive
import mapperref
import test_gpu_mapper as single

pytestmark = pytest.mark.gpu

CLOUDS = ("map_corner_ds", "map_surf_ds", "corner_ds", "surf_ds", "outlier_ds", "surf_total_ds")


def _split(events):
    """A drive's events -> [(imu rows before the odometry message, odometry message)]."""
    out, imu = [], []
    for e in events:
        if e[0] == "imu":
            imu.append(e[1:4])
        else:
            out.append((imu, e[1:7]))
            imu = []
    return out


class Ref:
    """One drive on a single mapper of its own."""

    def __init__(self, capi):
        self.g = capi.LinsGpu()
        self.g.mapper_reset()

    def feed(self, imu, odom):
        if imu:
            self.g.mapper_imu(*(np.array(a) for a in zip(*imu)))
        return self.g.mapper_step(*odom)


def _same(ctx, got, ref):
    """memcmp-equal reports; bit-equal key poses, window and clouds (sizes from the report)."""
    assert bytes(got) == bytes(ref), ctx


def _same_download(ctx, a, b):
    (pa, wa, ca), (pb, wb, cb) = a, b
    assert pa.shape == pb.shape and np.array_equal(pa.view(np.uint64), pb.view(np.uint64)), ctx
    assert np.array_equal(wa, wb), ctx
    for k in CLOUDS:
        assert ca[k].shape == cb[k].shape and np.array_equal(ca[k].view(np.uint32), cb[k].view(np.uint32)), f"{ctx} {k}"


def run_lockstep(capi, drives, n_slots=None, start=None, queue=False, check=None):
    """Steps the drives in lockstep and compares every slot with its drive's single mapper at every event.
    drives: lists of (imu, odom).  Without `queue`, drive i sits in slot i from step start[i] on and is absent before
    and after its run.  With `queue`, n_slots slots take the drives in order: a slot whose drive ended is reset
    (lins_gpu_mappers_reset) and takes the next one in the same step.  check(step, g, slots, reps) runs after every
    step.  Returns per step the list of (drive index or None, report or None)."""
    M = n_slots or len(drives)
    start = start or [0] * len(drives)
    g = capi.LinsGpu()
    g.mappers_open(M)
    refs = [Ref(capi) for _ in drives]
    pos = [0] * len(drives)
    slot_drive = [None] * M
    pending = list(range(len(drives)))
    log, step = [], 0
    while True:
        reset = np.zeros(M, np.uint8)
        if queue:
            for s in range(M):
                d = slot_drive[s]
                if (d is None or pos[d] >= len(drives[d])) and pending:
                    if d is not None:
                        reset[s] = 1
                    slot_drive[s] = pending.pop(0)
                elif d is not None and pos[d] >= len(drives[d]):
                    slot_drive[s] = None
        else:
            slot_drive = [i if start[i] <= step and pos[i] < len(drives[i]) else None for i in range(M)]
        if all(d is None for d in slot_drive):
            break
        if reset.any():
            g.mappers_reset(reset)
        rows, steps = [], []
        for s in range(M):
            d = slot_drive[s]
            if d is None:
                rows.append(None); steps.append(None)
                continue
            imu, odom = drives[d][pos[d]]
            rows.append(tuple(np.array(a) for a in zip(*imu)) if imu else None)
            steps.append(odom)
        g.mappers_imu(rows)
        reps = g.mappers_step(steps)
        entry = []
        for s in range(M):
            d = slot_drive[s]
            if d is None:
                assert reps[s] is None
                entry.append((None, None))
                continue
            imu, odom = drives[d][pos[d]]
            ref = refs[d].feed(imu, odom)
            ctx = f"step {step} slot {s} drive {d} event {pos[d]}"
            _same(ctx, reps[s], ref)
            if reps[s].processed:
                _same_download(ctx, g.mappers_download(s, reps[s]), refs[d].g.mapper_download(ref))
            pos[d] += 1
            entry.append((d, reps[s]))
        if check:
            check(step, g, slot_drive, reps)
        log.append(entry)
        step += 1
    for r in refs:
        r.g.close()
    g.close()
    return log


@pytest.fixture(scope="module")
def drives(synth):
    mk = lambda **kw: _split(mapper_drive.make_drive(synth, **kw))  # noqa: E731
    return [
        mk(n_out=36, seed=4, stall_at=50),                      # the window fills in a cycle that saves nothing
        mk(n_out=30, seed=5, stall_at=51),
        mk(n_out=34, seed=6, stall_at=60),
        _split([e for e in mapper_drive.make_drive(synth, n_out=6, stall_at=-1, sparse_first=1) if e[0] == "odom"]),  # gate failure
        _split(single.shim_events(synth, 30, seed=3)),          # the shim's own odometry: most cycles interval-skipped
        _split(single.shim_events(synth, 24, seed=7)),
        mk(n_out=5, seed=8, stall_at=-1),
        mk(n_out=8, seed=9, stall_at=-1),
    ]


def test_lockstep_drives_match_single_mappers(capi, drives):
    """Eight drives of different lengths and start steps in lockstep, each bit-identical to its own single mapper."""
    start = [0, 3, 1, 0, 60, 0, 58, 62]
    log = run_lockstep(capi, drives, start=start)
    seen = set()
    for entry in log:
        kinds = set()
        for d, r in entry:
            if d is None:
                kinds.add("absent")
            elif r.skipped_interval:
                kinds.add("skipped")
            elif r.processed and r.window_len == 0:
                kinds.add("no_keyframes")
            elif r.processed and r.window_len == 50:
                kinds.add("full_window")
        if kinds >= {"absent", "skipped", "no_keyframes", "full_window"}:
            seen.add("all_in_one_step")
    assert "all_in_one_step" in seen
    reps = [r for entry in log for d, r in entry if d == 0 and r.processed]
    assert any(r.window_len == 50 for r in reps) and reps[-1].loop_candidate >= 0
    sparse = [r for entry in log for d, r in entry if d == 3 and r.processed]
    assert all(r.map.skipped for r in sparse) and sparse[-1].n_keyframes == 1
    assert any(r.keyframe_saved and not r.map.skipped for entry in log for d, r in entry if d in (4, 5) and r.processed)


def test_slot_hand_over(capi, drives):
    """Six drives queued through two slots: a finished drive's slot is reset and takes the next drive in the same step;
    each drive matches a fresh single mapper."""
    log = run_lockstep(capi, [drives[i] for i in (6, 3, 7, 5, 6, 3)], n_slots=2, queue=True)
    assert len(log) < sum(len(drives[i]) for i in (6, 3, 7, 5, 6, 3))


def test_one_slot_and_a_permutation(capi, drives):
    run_lockstep(capi, [drives[7]])
    run_lockstep(capi, [drives[i] for i in (5, 7, 3, 6)], start=[0, 2, 1, 0])


def _raw_step(capi, g, M, steps, present=None, **override):
    """lins_gpu_mappers_step on a hand-built descriptor; returns the library's return code."""
    time = np.array([s[0] for s in steps], np.float64)
    quat = np.array([s[1] for s in steps], np.float64)
    pos = np.array([s[2] for s in steps], np.float64)
    cl = [capi.pack_csr([s[3 + k] for s in steps]) for k in range(3)]
    arrs = dict(present=present, time=time, quat=quat, pos=pos, corner=cl[0][0], corner_off=cl[0][1], surf=cl[1][0],
                surf_off=cl[1][1], outlier=cl[2][0], outlier_off=cl[2][1])
    arrs.update(override)
    d = capi.LinsMappersDesc(n_slots=override.pop("n_slots", M), **{k: (v if v is None or isinstance(v, int) else v.ctypes.data_as(C.c_void_p))
                                                                     for k, v in arrs.items() if k != "n_slots"})
    return g.L.lins_gpu_mappers_step(g.h, C.byref(d), None)


def test_overflow_and_bad_descriptors_change_no_slot(capi, drives):
    """A slot whose VoxelGrid overflows fails the whole step with LINS_E_TOOBIG, bad descriptors fail with
    LINS_E_INVALID, and afterwards every slot continues bit-identical to single mappers that never saw those calls."""
    ds = [drives[6], drives[7], drives[3]]
    bad_step = 4
    p = np.zeros((3, 8), np.float32)
    p[0, :3], p[1, :3] = -1e5, 1e5  # test_voxel_grid_key_overflow's geometry

    def check(step, g, slots, reps):
        if step != bad_step:
            return
        steps = [ds[d][step + 1][1] for d in range(3)]  # (the next step's IMU rows go in when it runs for real)
        M = len(slots)
        invalid = [dict(n_slots=M + 1)]
        off = capi.pack_csr([s[3] for s in steps])[1].copy(); off[0] = 1
        invalid.append(dict(corner_off=off))
        off = capi.pack_csr([s[4] for s in steps])[1].copy(); off[2] = off[1] - 1
        invalid.append(dict(surf_off=off))
        invalid.append(dict(corner=None))
        for bad in invalid:
            assert _raw_step(capi, g, M, steps, **bad) == -1, bad  # LINS_E_INVALID
        over = list(steps)
        t, q, ps, c, s, o = over[1]
        over[1] = (t + 1.0, q, ps, p, s, o)  # (processed whatever the interval gate would say)
        with pytest.raises(capi.LinsError, match="error -4"):
            g.mappers_step(over)

    run_lockstep(capi, ds, check=check)


def test_independent_of_the_single_mapper_scan2map_and_voxel_grid(capi, drives, defs):
    """lins_gpu_mapper_step, lins_gpu_map_set / scan2map and lins_gpu_voxel_grid interleaved on the context of the
    lockstep mappers give what they give on a context of their own, and so do the mappers."""
    a, b = drives[6], drives[7]
    shared, alone_m, alone_s = capi.LinsGpu(), capi.LinsGpu(), capi.LinsGpu()
    shared.mappers_open(2); alone_m.mappers_open(2)
    shared.mapper_reset(); alone_s.mapper_reset()
    rng = np.random.default_rng(1)
    P = lambda x: mapperref.to_points(x, defs.POINT_DTYPE)  # noqa: E731
    n_s2m = 0
    for k in range(min(len(a), len(b))):
        steps = [a[k][1], b[k][1]]
        r1, r2 = shared.mappers_step(steps), alone_m.mappers_step(steps)
        o1, o2 = shared.mapper_step(*b[k][1]), alone_s.mapper_step(*b[k][1])
        assert bytes(o1) == bytes(o2)
        cloud = rng.uniform(-5, 5, (500, 8)).astype(np.float32)
        assert np.array_equal(shared.voxel_grid(cloud, 0.4).view(np.uint32), alone_s.voxel_grid(cloud, 0.4).view(np.uint32))
        if o1.processed and o1.n_map_surf_ds > 100:
            _same_download(f"step {k} single", shared.mapper_download(o1), alone_s.mapper_download(o2))
            _, _, cl = alone_s.mapper_download(o2)
            mc, ms, qc, qs = (P(cl[n]) for n in ("map_corner_ds", "map_surf_ds", "corner_ds", "surf_total_ds"))
            for g in (shared, alone_s):
                g.map_set(mc, ms)
            t1, m1 = shared.scan2map(qc, qs, o1.transform_guess)
            t2, m2 = alone_s.scan2map(qc, qs, o1.transform_guess)
            assert np.array_equal(t1.view(np.uint32), t2.view(np.uint32)) and bytes(m1) == bytes(m2)
            n_s2m += 1
        for s in range(2):
            assert bytes(r1[s]) == bytes(r2[s])
            if r1[s].processed:
                _same_download(f"step {k} slot {s}", shared.mappers_download(s, r1[s]), alone_m.mappers_download(s, r2[s]))
    assert n_s2m >= 3
    for g in (shared, alone_m, alone_s):
        g.close()
