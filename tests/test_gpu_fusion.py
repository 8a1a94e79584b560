"""GPU suite for transform fusion (lins_gpu_mapper_fuse, lins_gpu_mappers_fuse, lins_gpu_seq_map_fused): the pose
transform_fusion_node publishes for every scan, against the restatement of tests/fusionref.py byte for byte.

The restatement is fed an independent route to the pair the mapping node published: transformAftMapped from the last
processed cycle's report, and transformBefMapped rebuilt from the odometry of the last cycle that ran transformUpdate
(the 10 / 100 gate passed), both zero before the first processed cycle.  A single mapper is fused before each of its
steps on the drives of tests/mapper_drive.py and the shim-published drive of tests/test_gpu_mapper.py; the lockstep
mappers at M = 132 equal single mappers; a bound sequence run's fused poses follow the published poses through absent
and INIT slots, a restart and a save / load at a permutation; bag_replay.replay(map=True) returns what it read at every
step, also when stopped and resumed; tools/run_bags.py --map and tools/run_bag.py --map write integrated.txt."""
import os
import subprocess
import sys

import numpy as np
import pytest

import fusionref as fr
import mapper_drive
import rawcases as rc
import test_gpu_mapper as single
from conftest import ROOT, pkg
from test_gpu_mappers import _split
from test_gpu_seq_checkpoint import _open, _step, logs  # noqa: F401  (logs: the module fixture of eight raw drives)

pytestmark = pytest.mark.gpu
br = pkg("bag_replay")
F = np.float32


class Pair:
    """The fusion node's pair, tracked from the mapper's reports and the odometry it was fed."""

    def __init__(self):
        self.published, self.aft, self.bef = False, np.zeros(6, F), np.zeros(6, F)

    def update(self, rep, quat, pos):
        if rep is None or not rep.processed:
            return
        self.published = True
        self.aft = np.array(rep.transform_aft_mapped, F)
        if not rep.map.skipped:  # transformUpdate: transformBefMapped = transformSum of this cycle
            self.bef = fr.odometry_transform(quat, pos)

    def expect(self, time, quat, pos):
        T, p, q = fr.fuse(quat, pos, self.published, self.aft, self.bef)
        return time, T, p, q


def _same(ctx, got, want):
    time, T, p, q = want
    assert got.valid == 1, ctx
    assert np.float64(got.time).tobytes() == np.float64(time).tobytes(), ctx
    assert np.array(got.transform_mapped, F).tobytes() == T.tobytes(), (ctx, list(got.transform_mapped), T)
    assert np.array(got.pos).tobytes() == p.tobytes() and np.array(got.quat).tobytes() == q.tobytes(), (ctx, got.row(), p, q)


def _none(ctx, got):
    assert got.valid == 0 and bytes(got) == bytes(len(bytes(got))), ctx


def fused_drive(capi, events):
    """A drive on a single mapper with mapper_fuse before every step, checked against the restatement; returns the
    fused poses (bytes) in event order and the reports."""
    g = capi.LinsGpu()
    g.mapper_reset()
    pair, out, reps = Pair(), [], []
    for e in events:
        if e[0] == "imu":
            g.mapper_imu(e[1], e[2], e[3])
            continue
        t, quat, pos = e[1], e[2], e[3]
        got = g.mapper_fuse(t, quat, pos)
        _same(f"event {e[-1]} t {t}", got, pair.expect(t, quat, pos))
        rep = g.mapper_step(*e[1:7])
        pair.update(rep, quat, pos)
        out.append(bytes(got)); reps.append(rep)
    g.close()
    return out, reps


def test_single_mapper_drives(capi, synth):
    """The out-and-back drive (interval skips, a first key frame whose cycle fails the gate), the gate-failure drive (the
    pair stays stale), and the shim's own odometry (most cycles interval-skipped)."""
    _, reps = fused_drive(capi, mapper_drive.make_drive(synth))
    assert reps[0].processed and reps[0].map.skipped and any(r.skipped_interval for r in reps)
    assert sum(1 for r in reps if r.processed and not r.map.skipped) >= 40
    _, reps = fused_drive(capi, [e for e in mapper_drive.make_drive(synth, n_out=6, stall_at=-1, sparse_first=1) if e[0] == "odom"])
    assert all(r.map.skipped for r in reps if r.processed) and sum(r.processed for r in reps) >= 3
    _, reps = fused_drive(capi, single.shim_events(synth, 48, seed=3))
    assert sum(r.skipped_interval for r in reps) >= 20 and sum(1 for r in reps if r.processed and not r.map.skipped) >= 5


def test_fuse_is_read_only_and_checks_its_arguments(capi, synth):
    """mapper_fuse changes nothing (a twin that never fuses steps to the same reports); the lockstep entry's errors."""
    ev = [e for e in mapper_drive.make_drive(synth, n_out=8, seed=9, stall_at=-1) if e[0] == "odom"]
    a, b = capi.LinsGpu(), capi.LinsGpu()
    for e in ev:
        a.mapper_fuse(*e[1:4]); a.mapper_fuse(*e[1:4])
        assert bytes(a.mapper_step(*e[1:7])) == bytes(b.mapper_step(*e[1:7]))
    L = a.L
    assert L.lins_gpu_mapper_fuse(a.h, None, None) == -1
    assert L.lins_gpu_mappers_fuse(a.h, None, None) == -1
    d = capi.LinsMappersDesc(n_slots=1)
    assert L.lins_gpu_mappers_fuse(a.h, d, None) == -3  # no lockstep run
    a.mappers_open(2)
    assert L.lins_gpu_mappers_fuse(a.h, d, None) == -1  # n_slots
    t, q, p = np.zeros(2), np.tile([0.0, 0.0, 0.0, 1.0], 2), np.zeros(6)
    out = (capi.LinsFusedPose * 2)()
    d = capi.LinsMappersDesc(n_slots=2, time=capi.ptr(t), quat=capi.ptr(q), pos=None)
    assert L.lins_gpu_mappers_fuse(a.h, d, out) == -1  # null pos
    d.pos = capi.ptr(p)
    assert L.lins_gpu_mappers_fuse(a.h, d, None) == -1  # null out
    assert L.lins_gpu_mappers_fuse(a.h, d, out) == 0 and out[0].valid == out[1].valid == 1
    a.close(); b.close()


def test_lockstep_132_slots_equal_single_mappers(capi, synth):
    """132 slots tile the eight drives of tests/test_gpu_mappers.py at four start steps; before every step each present
    slot's mappers_fuse equals its drive's single mapper's mapper_fuse at the same event, and absent slots read valid 0."""
    mk = lambda **kw: mapper_drive.make_drive(synth, **kw)  # noqa: E731
    evs = [mk(n_out=36, seed=4, stall_at=50), mk(n_out=30, seed=5, stall_at=51), mk(n_out=34, seed=6, stall_at=60),
           [e for e in mk(n_out=6, stall_at=-1, sparse_first=1) if e[0] == "odom"], single.shim_events(synth, 30, seed=3),
           single.shim_events(synth, 24, seed=7), mk(n_out=5, seed=8, stall_at=-1), mk(n_out=8, seed=9, stall_at=-1)]
    ref = [fused_drive(capi, e)[0] for e in evs]
    drives = [_split(e) for e in evs]
    M = 132
    slot_drive, start = [s % 8 for s in range(M)], [(s // 8) % 4 * 3 for s in range(M)]
    g = capi.LinsGpu()
    g.mappers_open(M)
    step, n_fused = 0, 0
    while True:
        k = [step - start[s] for s in range(M)]
        live = [0 <= k[s] < len(drives[slot_drive[s]]) for s in range(M)]
        if not any(live) and step > max(start):
            break
        g.mappers_imu([tuple(np.array(a) for a in zip(*drives[slot_drive[s]][k[s]][0])) if live[s] and drives[slot_drive[s]][k[s]][0] else None
                       for s in range(M)])
        steps = [drives[slot_drive[s]][k[s]][1] if live[s] else None for s in range(M)]
        fused = g.mappers_fuse(steps)
        out = (capi.LinsFusedPose * M)()  # (the raw entry: an absent slot's record is zeroed)
        present, zt, zq, zp = np.array(live, np.uint8), np.zeros(M), np.tile([0.0, 0.0, 0.0, 1.0], M), np.zeros(3 * M)
        d = capi.LinsMappersDesc(n_slots=M, present=capi.ptr(present), time=capi.ptr(zt), quat=capi.ptr(zq), pos=capi.ptr(zp))
        assert g.L.lins_gpu_mappers_fuse(g.h, d, capi.C.cast(out, capi.C.c_void_p)) == 0
        for s in range(M):
            if live[s]:
                assert bytes(fused[s]) == ref[slot_drive[s]][k[s]], (step, s)
                n_fused += 1
            else:
                assert fused[s] is None
                _none((step, s), out[s])
        g.mappers_step(steps)
        step += 1
    assert n_fused == sum(len(ref[slot_drive[s]]) for s in range(M))
    g.close()


def _shifted(log, t0):
    """log as seen from step t0 on: its scan k at step t0 + k (the entries before t0 are never read)."""
    out = dict(log)
    out["time"] = np.concatenate([np.zeros(t0), log["time"]])
    out["sweeps"] = [np.zeros((0, 4), np.float32)] * t0 + list(log["sweeps"])
    out["imu_last"] = np.concatenate([np.zeros((t0, 6)), log["imu_last"]])
    out["imu_off"] = np.concatenate([np.zeros(t0, log["imu_off"].dtype), log["imu_off"]])
    return out


def test_bound_run(capi, defs, logs):  # noqa: F811
    """Eight drives in a bound run (one absent for a step, every one INIT at first); slot 5 restarted at step 6 with
    another drive; at step 7 every slot is saved and loaded into a run of S + 3 slots at a permutation.  At every step
    each published slot's fused pose equals the restatement fed its published pose and the pair its reports give, the
    others read valid 0, and the loaded run equals the source from each slot's next publish."""
    n = len(logs)
    model = rc.model_of(defs, logs[0])
    T = max(len(l["time"]) for l in logs)
    slot_log = {j: j for j in range(n)}
    lg = list(logs) + [_shifted(logs[1], 6)]
    a = _open(capi, defs, n, True)
    pairs = [Pair() for _ in range(n)]
    rng = np.random.default_rng(2)
    b = perm = None
    kinds = set()
    for t in range(T):
        if t == 6:
            m = np.eye(n, dtype=np.uint8)[5]
            a.seq_restart(m)
            slot_log[5] = n
            pairs[5] = Pair()
            _none("restarted", a.seq_map_fused()[5])
        reps, pub = _step(a, lg, t, slot_log, n, model, True)
        pose, _ = a.seq_map_published()
        fused = a.seq_map_fused()
        for j in range(n):
            li = slot_log[j]
            ctx = f"step {t} slot {j}"
            if not pub[j]:
                _none(ctx, fused[j])
                kinds.add("absent" if t >= len(lg[li]["time"]) or (t == 3 and li == 2) else "unpublished")
                continue
            _same(ctx, fused[j], pairs[j].expect(lg[li]["time"][t], pose[j][3:], pose[j][:3]))
            pairs[j].update(reps[j], pose[j][3:], pose[j][:3])
            if reps[j].processed:
                kinds.add("processed" if not reps[j].map.skipped else "gate")
            elif reps[j].skipped_interval:
                kinds.add("interval")
        if b is not None:
            rb, pbb = _step(b, lg, t, {int(perm[j]): slot_log[j] for j in range(n)}, n + 3, model, True)
            fb = b.seq_map_fused()
            for j in range(n):
                assert bytes(fb[perm[j]]) == bytes(fused[j]), (t, j)
        if t == 7:
            blobs = a.seq_save(np.ones(n, np.uint8))
            perm = rng.permutation(n + 3)[:n]
            b = _open(capi, defs, n + 3, True)
            mask = np.zeros(n + 3, np.uint8); mask[perm] = 1
            bl = [None] * (n + 3)
            for j in range(n):
                bl[perm[j]] = blobs[j]
            b.seq_load(mask, bl)
            assert all(f.valid == 0 for f in b.seq_map_fused())
    assert {"absent", "unpublished", "processed", "interval"} <= kinds, kinds
    with pytest.raises(capi.LinsError, match="error -3"):
        u = _open(capi, defs, 2, False)
        u.seq_map_fused()


def _per_step_reads(capi):
    """A context that records what seq_map_fused returned at every step."""
    class Recorder(capi.LinsGpu):
        def seq_map_fused(self):
            out = super().seq_map_fused()
            self.reads.append([bytes(f) for f in out])
            return out
    g = Recorder()
    g.reads = []
    return g


def test_replay_map_fused(capi, defs, synth, tmp_path):
    """bag_replay.replay(map=True)'s map_fused rows are the per-step reads of the published slots, recording by recording,
    for three simulated bags through two slots; a replay stopped with a checkpoint and resumed returns the same rows;
    tools/run_bags.py --map writes them as the third file (and writes it for tests/golden/tiny.bag)."""
    paths = []
    for seed, n_scans in ((2, 24), (5, 14), (7, 18)):
        paths.append(str(tmp_path / f"b{seed}.bag"))
        synth.write_sequence_bag(paths[-1], config="config3", seed=seed, n_scans=n_scans)
    recs = [br.Recording(p) for p in paths]
    g = _per_step_reads(capi)
    full = br.replay(recs, 2, map=True, gpu=g)
    lengths = [len(r) for r in recs]
    rows = [[] for _ in recs]
    for t, (_, who) in enumerate(br.slot_queue(lengths, 2)):
        for j, w in enumerate(who):
            f = defs.LinsFusedPose.from_buffer_copy(g.reads[t][j])
            if w is not None and f.valid:
                assert f.time == recs[w[0]].stamps[w[1]]
                rows[w[0]].append(f.row())
    for o, r in zip(full, rows):
        assert o["map_fused"].shape == (len(o["map_time"]), 7) and len(r) == len(o["map_time"])
        assert np.array(r, np.float64).reshape(-1, 7).tobytes() == o["map_fused"].tobytes()
    assert all(len(o["map_time"]) >= 8 for o in full) and sum(o["map_processed"].sum() for o in full) >= 6
    ck = str(tmp_path / "ck")
    assert br.replay(recs, 2, map=True, checkpoint=ck, stop_after=9) is None
    got = br.replay(recs, 2, map=True, resume=ck)
    for a, b in zip(full, got):
        assert a["map_fused"].tobytes() == b["map_fused"].tobytes()
    out = tmp_path / "bags"
    tiny = os.path.join(ROOT, "tests", "golden", "tiny.bag")
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "run_bags.py"), paths[0], tiny, "--slots", "1", "--map", "--out", str(out)],
                          stdout=subprocess.DEVNULL)
    integ = np.loadtxt(out / "b2.integrated.txt", ndmin=2)
    assert integ.shape == (len(full[0]["map_time"]), 8) and np.allclose(integ[:, 0], full[0]["map_time"], rtol=0, atol=1e-8)
    assert np.allclose(integ[:, 1:], full[0]["map_fused"], rtol=1e-8, atol=1e-12)
    assert len(open(out / "tiny.integrated.txt").readlines()) == len(open(out / "tiny.mapped.txt").readlines())


def test_run_bag_map_writes_integrated(synth, tmp_path):
    """tools/run_bag.py --map: integrated.txt next to odometry.txt and mapped.txt, one line per published scan."""
    bag = str(tmp_path / "drive.bag")
    synth.write_sequence_bag(bag, n_scans=30, seed=2)
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "run_bag.py"), bag, "--map", "--out", str(tmp_path)], stdout=subprocess.DEVNULL)
    odo = np.loadtxt(tmp_path / "odometry.txt", ndmin=2)
    mapped = np.loadtxt(tmp_path / "mapped.txt", ndmin=2)
    integ = np.loadtxt(tmp_path / "integrated.txt", ndmin=2)
    assert integ.shape == odo.shape and np.array_equal(integ[:, 0], odo[:, 0]) and np.isfinite(integ).all()
    # before the first processed cycle the pair is zero: the fused position is the odometry's (up to f32 rounding)
    assert np.allclose(integ[0, 1:4], odo[0, 1:4], rtol=1e-5, atol=1e-5)
    # once a processed cycle has moved the mapped pose, the fused pose differs from the odometry
    assert mapped[:, 1].sum() >= 6 and np.abs(integ[:, 1:4] - odo[:, 1:4]).max() > 0
