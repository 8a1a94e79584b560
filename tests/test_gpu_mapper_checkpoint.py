"""GPU suite for saving and loading mapping nodes (lins_gpu_mapper(s)_save / _load): a loaded slot continues
bit-identically to the slot it was saved from.

Byte for byte: every later report, download, fused pose, close_loops report and global map of the loaded slot against
the source's continuation; a run that saves at every step against a twin that never saves; a loaded slot saved again
against the blob it was loaded from; the loaded slot's global map right after the load (which reads the rebuilt
map-frame store) against the source's.  Plain lockstep slots at a permutation of a wider run, slots with loop closure on
the drifted, out-and-back and parked drives at the points where the graph and the store change, moves between the
single mapper, the lockstep mappers and a second context, 132 mixed slots under random masks, the refusals (which change
nothing) and the launch counts."""
import ctypes as C

import numpy as np
import pytest

import mapper_drive
import test_gpu_loops as tl

pytestmark = pytest.mark.gpu


class Target:
    """One mapping node: the single mapper of a context (slot None) or slot `slot` of its lockstep run of M slots."""

    def __init__(self, gpu, slot=None, M=1):
        self.g, self.s, self.M = gpu, slot, M
        self.rep = None  # the last processed report

    def _one(self, x):
        v = [None] * self.M
        v[self.s] = x
        return v

    def mask(self):
        m = np.zeros(self.M, np.uint8)
        m[self.s] = 1
        return m

    def imu(self, e):
        if self.s is None:
            self.g.mapper_imu(e[1], e[2], e[3])
        else:
            self.g.mappers_imu(self._one((e[1], e[2], e[3])))

    def fuse(self, e):
        f = self.g.mapper_fuse(*e[1:4]) if self.s is None else self.g.mappers_fuse(self._one(e[1:7]))[self.s]
        return bytes(f)

    def step(self, e):
        rep = self.g.mapper_step(*e[1:7]) if self.s is None else self.g.mappers_step(self._one(e[1:7]))[self.s]
        if rep.processed:
            self.rep = rep
        return rep

    def download(self):
        if self.rep is None:
            return None
        poses, window, clouds = self.g.mapper_download(self.rep) if self.s is None else self.g.mappers_download(self.s, self.rep)
        return poses.tobytes(), window.tobytes(), b"".join(clouds[k].tobytes() for k in sorted(clouds))

    def close(self):
        return self.g.mapper_close_loop() if self.s is None else self.g.mappers_close_loops(self.mask())[self.s]

    def global_map(self):
        if self.s is None:
            rep = self.g.mapper_global_map()
            keys, cloud = self.g.mapper_global_map_download(rep)
        else:
            rep = self.g.mappers_global_map(self.mask())[self.s]
            keys, cloud = self.g.mappers_global_map_download(self.s, rep)
        return bytes(rep), keys.tobytes(), cloud.tobytes()

    def save(self):
        return self.g.mapper_save() if self.s is None else self.g.mappers_save(self.mask())[self.s]

    def load(self, blob):
        if self.s is None:
            self.g.mapper_load(blob)
        else:
            self.g.mappers_load(self.mask(), self._one(blob))


def new_target(capi, kind, loops=False):
    """a fresh node in a new context: the single mapper, or slot 2 of a lockstep run of 4"""
    g = capi.LinsGpu()
    if kind == "single":
        g.mapper_reset()
        if loops:
            g.mapper_loops()
        return Target(g)
    g.mappers_open(4)
    if loops:
        g.mappers_loops([0, 0, 1, 0])
    return Target(g, 2, 4)


# ---- plain lockstep slots --------------------------------------------------------------------------------------------

def plain_drives(synth):
    # the same event layout (IMU and odometry messages at the same indices), three clouds and schedules
    return [mapper_drive.make_drive(synth, seed=4), mapper_drive.make_drive(synth, seed=5, sparse_first=3),
            mapper_drive.make_drive(synth, seed=8, stall_at=30)]


def run_plain(capi, drives, save_every):
    """The drives in lockstep, one per slot, with each slot's fused pose, report and download per event, and with
    save_every every slot's blob after every event (index -1: before the first)."""
    M, n = len(drives), len(drives[0])
    g = capi.LinsGpu()
    g.mappers_open(M)
    nodes = [Target(g, s, M) for s in range(M)]
    log, blobs = [[] for _ in range(M)], []
    if save_every:
        blobs.append(g.mappers_save([1] * M))
    for i in range(n):
        evs = [d[i] for d in drives]
        if evs[0][0] == "imu":
            g.mappers_imu([(e[1], e[2], e[3]) for e in evs])
            for s in range(M):
                log[s].append(None)
        else:
            fused = g.mappers_fuse([e[1:7] for e in evs])
            reps = g.mappers_step([e[1:7] for e in evs])
            for s in range(M):
                if reps[s].processed:
                    nodes[s].rep = reps[s]
                log[s].append((bytes(fused[s]), bytes(reps[s]), nodes[s].download(), reps[s]))
        if save_every:
            blobs.append(g.mappers_save([1] * M))
    return log, blobs


def continue_plain(drive, log, start, target):
    """events start.. of a drive on a loaded node against the source's log"""
    since = False  # a processed cycle since the load (the download's clouds exist again)
    for i in range(start, len(drive)):
        e = drive[i]
        if e[0] == "imu":
            target.imu(e)
            continue
        f = target.fuse(e)
        rep = target.step(e)
        sf, sr, sd, _ = log[i]
        assert f == sf and bytes(rep) == sr, i
        since |= bool(rep.processed)
        if since:
            assert target.download() == sd, i


def test_plain_slots_save_at_every_step_and_continue(capi, synth):
    drives = plain_drives(synth)
    M = len(drives)
    log, blobs = run_plain(capi, drives, save_every=True)
    twin, _ = run_plain(capi, drives, save_every=False)
    for s in range(M):
        assert [x[:3] if x else None for x in log[s]] == [x[:3] if x else None for x in twin[s]], s
    # the checkpoints: before the first key frame, a short window, a full window holding the duplicate id, a first
    # key frame whose map failed the 10 / 100 gate (blob k is the state after event k - 1)
    picks = {"before": 0}
    for s in range(M):
        cycles = 0
        for i, x in enumerate(log[s]):
            if x is None:
                continue
            rep = x[3]
            cycles += rep.processed
            w = np.frombuffer(x[2][1], np.int32) if x[2] else np.zeros(0, np.int32)
            if 0 < rep.window_len < 50 and rep.n_keyframes > 3:
                picks.setdefault("short", i + 1)
            if len(w) == 50 and len(set(w.tolist())) < 50:
                picks.setdefault("duplicate", i + 1)
            if rep.processed and rep.map.skipped and cycles >= 2:  # (a cycle with key frames before it)
                picks.setdefault("gate", i + 1)
    assert set(picks) == {"before", "short", "duplicate", "gate"}, picks
    rng = np.random.default_rng(1)
    for name, k in sorted(picks.items(), key=lambda kv: kv[1]):
        g = capi.LinsGpu()
        g.mappers_open(M + 3)
        perm = rng.permutation(M + 3)[:M]
        blob_list = [None] * (M + 3)
        mask = np.zeros(M + 3, np.uint8)
        for s in range(M):
            blob_list[perm[s]] = blobs[k][s]
            mask[perm[s]] = 1
        g.mappers_load(mask, blob_list)
        again = g.mappers_save(mask)
        for s in range(M):
            assert again[perm[s]] == blobs[k][s], (name, s)
        # the M loaded slots in one run, each against its source (the other 3 slots absent)
        nodes = [Target(g, int(perm[s]), M + 3) for s in range(M)]
        since = [False] * M
        for i in range(k, len(drives[0])):
            evs = [d[i] for d in drives]
            full = [None] * (M + 3)
            if evs[0][0] == "imu":
                for s in range(M):
                    full[perm[s]] = (evs[s][1], evs[s][2], evs[s][3])
                g.mappers_imu(full)
                continue
            for s in range(M):
                full[perm[s]] = evs[s][1:7]
            fused = g.mappers_fuse(full)
            reps = g.mappers_step(full)
            for s in range(M):
                p = int(perm[s])
                sf, sr, sd, _ = log[s][i]
                assert bytes(fused[p]) == sf and bytes(reps[p]) == sr, (name, s, i)
                if reps[p].processed:
                    nodes[s].rep = reps[p]
                    since[s] = True
                if since[s]:
                    assert nodes[s].download() == sd, (name, s, i)
    # a lockstep slot moved into the single mapper of another context
    k = picks["duplicate"]
    t = new_target(capi, "single")
    t.load(blobs[k][1])
    assert t.save() == blobs[k][1]
    continue_plain(drives[1], log[1], k, t)


# ---- slots with loop closure -----------------------------------------------------------------------------------------

def run_loops(capi, events, force_close=()):
    """A drive on the single mapper with loop closure, the loop thread ticked as test_gpu_loops ticks it: the log per
    event (fused pose, report, download, close report, global map at a tick), the tick events, and per checkpoint kind
    (event, whether that event's tick is still to run, blob, global map at the save)."""
    src = new_target(capi, "single", loops=True)
    last_close, log, ticks, points = None, [], set(), {}
    accepted = pending = False
    for i, e in enumerate(events):
        if e[0] == "imu":
            src.imu(e)
            log.append(None)
            continue
        f = src.fuse(e)
        rep = src.step(e)
        d = src.download()
        kind = None
        if rep.processed and pending:  # correctPoses ran in this cycle: after a solve, or on the stale estimate
            kind, pending = ("corrected" if rep.keyframe_saved else "stale"), False
        elif rep.processed and not accepted and rep.n_keyframes >= 3:
            kind = "before"
        if kind and kind not in points:  # (before this event's tick: its closure would change the state)
            points[kind] = (i, True, src.save(), src.global_map())
        kind = None
        lr = gm = None
        if src.rep is not None:
            due = last_close is None or e[1] - last_close >= 1.0  # (a forced tick leaves the 1 s clock alone)
            if due:
                last_close = e[1]
            if due or e[-1] in force_close:
                ticks.add(i)
                lr = src.close()
                gm = src.global_map()
                if lr.accepted:
                    accepted = pending = True
                    kind = "closed"
                lr = bytes(lr)
        log.append((f, bytes(rep), d, lr, gm))
        if kind and kind not in points:
            points[kind] = (i, False, src.save(), src.global_map())
    return log, ticks, points


def continue_loops(events, log, ticks, start, tick_left, target):
    """events start + 1.. on a loaded node against the source's log, after the tick of event start when tick_left"""
    if tick_left and start in ticks:
        assert bytes(target.close()) == log[start][3] and target.global_map() == log[start][4], start
    for i in range(start + 1, len(events)):
        e = events[i]
        if e[0] == "imu":
            target.imu(e)
            continue
        f = target.fuse(e)
        rep = target.step(e)
        sf, sr, sd, slr, sgm = log[i]
        assert f == sf and bytes(rep) == sr, i
        if target.rep is not None:  # (a processed cycle since the load)
            assert target.download() == sd, i
        if i in ticks:
            assert bytes(target.close()) == slr, i
            assert target.global_map() == sgm, i


@pytest.mark.parametrize("drive", ["drifted", "out_and_back", "parked"])
def test_loop_slots_continue_from_every_checkpoint(capi, synth, drive):
    if drive == "drifted":
        events, force = tl.drifted_drive(synth, stall_at=62)[0], {61}
    elif drive == "out_and_back":
        events, force = mapper_drive.make_drive(synth), ()
    else:
        events, force = tl.parked_drive(synth), ()
    log, ticks, points = run_loops(capi, events, force)
    assert "before" in points
    if drive == "drifted":
        assert {"closed", "corrected", "stale"} <= set(points), sorted(points)
    for j, (kind, (i, tick_left, blob, gm)) in enumerate(sorted(points.items())):
        t = new_target(capi, ["single", "lockstep"][j % 2], loops=j % 4 < 2)  # (the fresh slot's own setting is replaced)
        t.load(blob)
        assert t.save() == blob, kind
        assert t.global_map() == gm, kind  # the rebuilt map-frame store
        continue_loops(events, log, ticks, i, tick_left, t)


def test_loaded_slot_refuses_loop_enable_and_has_no_outputs_of_the_last_cycle(capi, synth):
    events, _ = tl.drifted_drive(synth)
    plain = new_target(capi, "lockstep")
    for e in events[:20]:
        plain.step(e)
    t = new_target(capi, "lockstep", loops=True)
    t.load(plain.save())  # (the blob's plain state replaces the fresh slot's loop closure)
    with pytest.raises(capi.LinsError):
        t.g.mappers_loops(t.mask())  # a loaded slot is not fresh
    with pytest.raises(capi.LinsError):
        t.g.mappers_close_loops(t.mask())  # not enabled
    src = new_target(capi, "lockstep", loops=True)
    for e in events[:20]:
        src.step(e)
    blob = src.save()
    t = new_target(capi, "lockstep")
    t.load(blob)
    t.g.mappers_loops(t.mask())  # (enabling an enabled slot is a no-op)
    assert t.save() == blob
    with pytest.raises(capi.LinsError):
        t.g.mappers_global_map_download(t.s, src.g.mappers_global_map(src.mask())[src.s])
    poses, window, clouds = t.g.mappers_download(t.s, src.rep)  # key poses and window, no clouds
    sp, sw, _ = src.g.mappers_download(src.s, src.rep)
    assert np.array_equal(poses, sp) and np.array_equal(window, sw)


# ---- 132 mixed slots ---------------------------------------------------------------------------------------------------

def test_132_mixed_slots_under_random_masks(capi, synth):
    events, _ = tl.drifted_drive(synth)
    M, cut = 132, 60
    loops = np.array([s % 3 != 0 for s in range(M)], np.uint8)
    g = capi.LinsGpu()
    g.mappers_open(M)
    g.mappers_loops(loops)

    def step(gpu, e, slots, perm=None):
        n = gpu._mappers_n
        full = [None] * n
        for s in slots:
            full[s if perm is None else perm[s]] = e[1:7]
        return gpu.mappers_step(full)

    for i, e in enumerate(events[:cut]):
        step(g, e, range(M))
        if i % 2:
            g.mappers_close_loops(loops)
    rng = np.random.default_rng(7)
    masks = [rng.integers(0, 2, M).astype(np.uint8) for _ in range(3)]
    masks.append(1 - np.maximum.reduce(masks))
    blobs = [None] * M
    for m in masks:
        for s, b in enumerate(g.mappers_save(m)):
            if b is not None:
                blobs[s] = b
    assert all(b is not None for b in blobs)
    perm = rng.permutation(M)
    h = capi.LinsGpu()
    h.mappers_open(M)
    n0 = h.launch_count()
    h.mappers_load(np.ones(M, np.uint8), [blobs[int(np.argwhere(perm == p)[0, 0])] for p in range(M)])
    assert h.launch_count() - n0 <= 2
    again = h.mappers_save(np.ones(M, np.uint8))
    for s in range(M):
        assert again[perm[s]] == blobs[s], s
    for i, e in enumerate(events[cut:], cut):
        ra, rb = step(g, e, range(M)), step(h, e, range(M), perm)
        for s in range(M):
            assert bytes(ra[s]) == bytes(rb[perm[s]]), (s, i)
        if i % 2:
            la, lb = g.mappers_close_loops(loops), h.mappers_close_loops(loops[np.argsort(perm)])
            for s in range(M):
                if loops[s]:
                    assert bytes(la[s]) == bytes(lb[perm[s]]), (s, i)


# ---- refusals and launch counts ----------------------------------------------------------------------------------------

def test_refusals_change_nothing(capi, defs, synth):
    events, _ = tl.drifted_drive(synth)
    g = capi.LinsGpu()
    g.mappers_open(3)
    g.mappers_loops([1, 0, 0])
    for e in events[:12]:
        g.mappers_step([e[1:7], e[1:7], None])
    blobs = g.mappers_save([1, 1, 0])
    L, h = g.L, g.h
    # a non-fresh destination (slot 0 stepped), with a fresh one in the same call: nothing loads
    with pytest.raises(capi.LinsError):
        g.mappers_load([1, 0, 1], [blobs[0], None, blobs[1]])
    assert g.mappers_save([1, 1, 0]) == blobs
    g.mappers_load([0, 0, 1], [None, None, blobs[1]])
    assert g.mappers_save([0, 0, 1])[2] == blobs[1]
    # truncated blobs, a flipped byte, wrong offsets, NULL arguments
    t = capi.LinsGpu()
    t.mappers_open(2)
    for bad in (blobs[0][:-16], blobs[0][:100], blobs[0] + b"\0" * 16, b""):
        with pytest.raises(capi.LinsError):
            t.mappers_load([1, 1], [blobs[1], bad])
    flipped = bytearray(blobs[0])
    flipped[60] ^= 4
    with pytest.raises(capi.LinsError):
        t.mappers_load([1, 0], [bytes(flipped), None])
    m = np.ones(2, np.uint8)
    off = np.zeros(3, np.uint64)
    assert L.lins_gpu_mappers_save_size(t.h, None, off.ctypes.data) == -1
    assert L.lins_gpu_mappers_save_size(t.h, m.ctypes.data, None) == -1
    assert L.lins_gpu_mappers_save_size(t.h, m.ctypes.data, off.ctypes.data) == 0
    buf = np.zeros(int(off[-1]), np.uint8)
    wrong = off.copy()
    wrong[1] += 16
    assert L.lins_gpu_mappers_save(t.h, m.ctypes.data, buf.ctypes.data, wrong.ctypes.data) == -1
    assert L.lins_gpu_mappers_save(t.h, m.ctypes.data, None, off.ctypes.data) == -1
    assert L.lins_gpu_mappers_load(t.h, m.ctypes.data, None, off.ctypes.data) == -1
    assert L.lins_gpu_mappers_load(t.h, None, buf.ctypes.data, off.ctypes.data) == -1
    assert L.lins_gpu_mapper_save_size(t.h, None) == -1
    n = C.c_uint64(0)
    assert L.lins_gpu_mapper_save_size(t.h, C.byref(n)) == 0
    assert L.lins_gpu_mapper_save(t.h, buf.ctypes.data, n.value + 16) == -1
    # every refusal above left t's slots fresh: both still load
    t.mappers_load([1, 1], [blobs[1], blobs[0]])
    assert t.mappers_save([1, 1]) == [blobs[1], blobs[0]]
    # a run bound to sequence mode refuses all three lockstep entries
    br = pytest.importorskip("lins---lidar-inertial-slam_b200.bag_replay")
    b = capi.LinsGpu()
    b.seq_open(defs.LinsSeqParams.shipped(), br.shim_init_params(), 2)
    b.seq_map_open()
    seq_blob = b.seq_save([1, 0])[0]
    for call in (lambda: b.mappers_save([1, 0]), lambda: b.mappers_load([1, 0], [blobs[1], None])):
        with pytest.raises(capi.LinsError):
            call()
    mm = np.ones(2, np.uint8)
    assert L.lins_gpu_mappers_save_size(b.h, mm.ctypes.data, np.zeros(3, np.uint64).ctypes.data) == -1
    assert b.seq_save([1, 0])[0] == seq_blob
    # a sequence blob into the mappers, a mapper blob into sequence mode
    with pytest.raises(capi.LinsError, match="magic"):
        t2 = capi.LinsGpu()
        t2.mappers_open(1)
        t2.mappers_load([1], [seq_blob])
    with pytest.raises(capi.LinsError, match="magic"):
        b.seq_load([0, 1], [None, blobs[1]])
    b.seq_load([0, 1], [None, seq_blob])  # (slot 1 is still fresh)


def test_launch_counts(capi, synth):
    events, _ = tl.drifted_drive(synth)
    g = capi.LinsGpu()
    g.mappers_open(4)
    g.mappers_loops([1, 0, 1, 0])
    for e in events[:15]:
        g.mappers_step([e[1:7]] * 4)
    for mask in ([1, 1, 1, 1], [0, 1, 0, 0], [1, 0, 0, 0]):
        n0 = g.launch_count()
        blobs = g.mappers_save(mask)
        assert g.launch_count() - n0 == 1
        h = capi.LinsGpu()
        h.mappers_open(4)
        n0 = h.launch_count()
        h.mappers_load(mask, blobs)
        assert 1 <= h.launch_count() - n0 <= 2
        assert h.mappers_load_phase_ms().shape == (5,)
    s = capi.LinsGpu()
    n0 = s.launch_count()
    s.mapper_load(blobs[0])
    assert s.launch_count() - n0 <= 2
    n0 = s.launch_count()
    assert s.mapper_save() == blobs[0]
    assert s.launch_count() - n0 == 1
