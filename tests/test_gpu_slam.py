"""GPU suite: sequence mode feeding its mapping nodes (lins_gpu_seq_map_open / lins_gpu_seq_map_step).

A bound run (seq_step_raw + seq_map_step) against an unbound twin that does the hand-off on the host (seq_step_raw, then
seq_download / seq_download_init / seq_download_maps, project_scans of the NaN-filtered sweeps for the outlier clouds,
publishTopics' rule restated in tests/slamref.py, and mappers_step from host buffers): at every step the published
flags equal the rule, the mapper reports are byte-equal, every published slot's key poses, window and six clouds are
bit-equal, and the sequence side is bit-equal to the twin's (binding changes no odometry).  Then variations (host
outliers through _pcl / _ex steps, S = 1, a permutation, a queue through fewer slots, a _mixed run), invalid calls that
change nothing, and LINS_E_TOOBIG.  Against the shim: synthetic bags (one with its second scan emptied and a later
scan truncated) replayed with bag_replay.replay(map=True) through fewer slots than bags, each compared with the stream
the C++ shim publishes (synth.run_bag(bag)["map_inputs"]) fed to a single mapper, and tools/run_bags.py --map's files."""
import ctypes as C
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

import rawcases as rc
import slamref as sr
from conftest import ROOT, pkg
from test_gpu_seq_init import init_params
from test_gpu_seq_pcl import _snapshot

pytestmark = pytest.mark.gpu
br = pkg("bag_replay")
ABSENT_JOB = 7


@pytest.fixture(scope="module")
def cases(capi, defs):
    logs, edits = rc.case_logs(defs, 0, gpu=capi.LinsGpu())
    print("drives replaced because a tie decides a pick:", edits.pop("tie_skipped"))
    # one more drive whose second sweep is empty: its estimator falls back from FIRST_SCAN to INIT (a publish of the
    # fresh scan's empty clouds at the identity pose)
    e = {k: (list(v) if k == "sweeps" else v) for k, v in logs[1].items()}
    e["sweeps"][1] = np.zeros((0, 4), np.float32)
    logs.append(e)
    return logs, [rc.pcl_of(defs, l) for l in logs]


def _jobs(logs):
    jobs = []
    for i, l in enumerate(logs):
        ev = list(range(len(l["time"])))
        if i == ABSENT_JOB:
            ev = ev[:3] + [None] + ev[3:]
        jobs.append((i, ev))
    return jobs


def _points(xyzi, defs):
    a = np.asarray(xyzi, np.float32).reshape(-1, 4)
    return defs.make_points(a[:, :3], a[:, 3])


def _xyzi(p):
    return np.stack([p["x"], p["y"], p["z"], p["intensity"]], 1).astype(np.float32) if len(p) else np.zeros((0, 4), np.float32)


def _empty_scan(L):
    return dict(seg=np.zeros((0, 4), np.float32), ground=np.zeros(0, np.uint8), col=np.zeros(0, np.uint32), range=np.zeros(0, np.float32),
                start_ring=np.zeros(L, np.int32), end_ring=np.zeros(L, np.int32), ori=np.zeros(3, np.float32))


def _node(g, s, rep):
    """A mapper slot's key poses, window and clouds as bytes."""
    poses, window, clouds = g.mappers_download(s, rep)
    return [poses.tobytes(), window.tobytes()] + [clouds[k].tobytes() for k in sorted(clouds)]


def run(capi, defs, cases, n_slots, jobs, modes=("raw",), twin=True, mixed=False, params=None):
    """Jobs through a bound run (g) and, with twin, the host composition on an unbound context (h).  modes: the bound
    run's step entry per step, in turn ("raw", "pcl": host outliers, "ex": host features and outliers).  Returns the
    per-job published streams [(stamp, report bytes, node bytes)], and the (fusion before, code) rows reached."""
    logs, pcls = cases
    model = rc.model_of(defs, logs[0])
    L = model.line_num
    g = capi.LinsGpu(params=params)
    g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
    g.seq_map_open()
    h = capi.LinsGpu(params=params)
    h.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
    h.mappers_open(n_slots)
    pub = sr.Publisher(n_slots)
    streams, rows, t = [[] for _ in jobs], set(), 0
    for restart, slots in br.slot_queue([len(ev) for _, ev in jobs], n_slots):
        if restart.any():
            g.seq_restart(restart)
            h.seq_restart(restart)
            h.mappers_reset(restart)
            for s in np.flatnonzero(restart):
                pub.restart(s)
        sweeps, scans, who, imus, scan_imu, time = [], [], [], [], np.zeros((n_slots, 6)), np.zeros(n_slots)
        for j, w in enumerate(slots):
            k = jobs[w[0]][1][w[1]] if w is not None else None
            if k is None:
                sweeps.append(np.zeros((0, 4), np.float32)); scans.append(_empty_scan(L)); who.append(None); imus.append(np.zeros((0, 7)))
                continue
            li = jobs[w[0]][0]
            o = logs[li]["imu_off"]
            sweeps.append(logs[li]["sweeps"][k]); scans.append(pcls[li]["scans"][k]); who.append((w[0], k))
            imus.append(logs[li]["imu"][o[k]:o[k + 1]])
            scan_imu[j] = logs[li]["imu_last"][k]
            time[j] = logs[li]["time"][k]
        step = dict(imu=np.concatenate(imus).reshape(-1, 7), imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32),
                    present=np.array([w is not None for w in who], np.uint8))
        before = h.seq_download_init()["fusion_status"] if twin else None
        h.seq_step_raw(dict(step, sweeps=sweeps), model=model, scan_imu=scan_imu)
        proj = h.project_scans([rc.finite(s) for s in sweeps], model=model)  # (also overwrites the projection state)
        outl = [p["outlier"] if w is not None else np.zeros((0, 4), np.float32) for p, w in zip(proj, who)]
        mode = modes[t % len(modes)]
        if mode == "raw":
            if mixed:
                g.seq_step_raw_mixed(dict(step, sweeps=sweeps), [defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()],
                                     np.zeros(n_slots, np.int32), scan_imu=scan_imu)
            else:
                g.seq_step_raw(dict(step, sweeps=sweeps), model=model, scan_imu=scan_imu)
            g.project_scans([np.zeros((0, 4), np.float32)] * 2, model=model)  # the stash must not read the projection's state
            reps_g, pub_g = g.seq_map_step(time)
        else:
            if mode == "pcl":
                g.seq_step_pcl(dict(step, scans=scans), scan_imu=scan_imu, line_num=L)
            else:
                from test_gpu_seq_raw import _via_ex
                _via_ex(g, capi, dict(step, scans=scans), L, scan_imu)
            reps_g, pub_g = g.seq_map_step(time, outlier=[_points(o, defs) for o in outl])
        d = h.seq_download()
        sa, sb = _snapshot(g), _snapshot(h)
        for k in sa:
            assert (sa[k].tobytes() if isinstance(sa[k], np.ndarray) else sa[k]) == (sb[k].tobytes() if isinstance(sb[k], np.ndarray) else sb[k]), (t, k)
        if twin:
            maps = h.seq_download_maps()
            steps = [None] * n_slots
            for j, w in enumerate(who):
                if w is None:
                    if slots[j] is not None:  # a drive's slot absent for this step
                        rows.add((int(before[j]), sr.IDLE))
                    continue
                code = int(d["status"][j])
                rows.add((int(before[j]), code))
                out = pub.step(j, before[j], code, d["global_state"][j], _xyzi(maps["corner_map"][j]), _xyzi(maps["surf_map"][j]), outl[j])
                if out is not None:
                    steps[j] = (time[j], out[0][3:], out[0][:3], _points(out[1], defs), _points(out[2], defs), _points(out[3], defs))
            reps_h = h.mappers_step(steps)
            assert pub_g.tolist() == [int(x is not None) for x in steps], t
        for j, w in enumerate(who):
            if not pub_g[j]:
                continue
            # (a download is sized by the last processed cycle's report)
            node = _node(g, j, reps_g[j]) if reps_g[j].processed else None
            if twin:
                assert bytes(reps_g[j]) == bytes(reps_h[j]), (t, j)
                assert node is None or node == _node(h, j, reps_h[j]), (t, j)
            streams[w[0]].append((time[j], bytes(reps_g[j]), node))
        t += 1
    return streams, rows


@pytest.fixture(scope="module")
def base(capi, defs, cases):
    return run(capi, defs, cases, len(cases[0]), _jobs(cases[0]))


def test_twin_parity_at_every_step(defs, cases, base):
    streams, rows = base
    I, F, R = sr.FUSION_INIT, sr.FUSION_FIRST_SCAN, sr.FUSION_RUNNING
    print("table rows reached:", sorted(rows))
    assert {(I, sr.INIT_WAIT), (I, sr.FIRST), (F, sr.SECOND), (F, sr.INIT_WAIT), (R, sr.RAN), (R, sr.SKIPPED), (R, sr.IDLE)} <= rows, rows
    print("(RUNNING, ICP) reached by these drives:", (R, sr.ICP) in rows, "(test_icp_fallback forces it)")
    # the empty-second-sweep drive: its first publish carries empty clouds at the identity pose and saves a key frame
    first = streams[len(cases[0]) - 1][0]
    rep = defs.LinsMapperReport.from_buffer_copy(first[1])
    assert rep.processed == 1 and rep.keyframe_saved == 1 and rep.n_corner_ds == rep.n_surf_ds == rep.n_outlier_ds == 0
    assert list(rep.transform_aft_mapped) == [0.0] * 6
    assert all(len(s) > 3 for s in streams)


def test_icp_fallback(capi, defs, cases):
    """lidar_scale = 1e9 makes every running scan's IESKF diverge: each accepted scan is an ICP fallback, whose maps and
    stashed outliers the slot publishes; bit-identical to the host composition at every step."""
    logs = cases[0]
    jobs = [j for j in _jobs(logs) if j[0] in (0, 2, 3, 5, len(logs) - 1)]
    streams, rows = run(capi, defs, cases, len(jobs), jobs, params=defs.LinsParams.shipped(lidar_scale=1e9))
    R = sr.FUSION_RUNNING
    assert (R, sr.ICP) in rows and (R, sr.RAN) not in rows, rows
    assert sum(defs.LinsMapperReport.from_buffer_copy(x[1]).processed for st in streams for x in st) > 5


def _same_streams(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x == y


def test_host_outliers_alternating(capi, defs, cases, base):
    """_raw, _pcl (host outliers) and _ex steps in turn in one bound run: the same streams."""
    streams, _ = run(capi, defs, cases, len(cases[0]), _jobs(cases[0]), modes=("raw", "pcl", "ex"))
    for a, b in zip(streams, base[0]):
        _same_streams(a, b)


def test_single_slot_permutation_queue_and_mixed(capi, defs, cases, base):
    logs = cases[0]
    jobs = _jobs(logs)
    s1, _ = run(capi, defs, cases, 1, [jobs[2]], twin=False)
    _same_streams(s1[0], base[0][2])
    perm = list(np.random.default_rng(5).permutation(len(logs)))
    sp, _ = run(capi, defs, cases, len(logs), [jobs[i] for i in perm], twin=False)
    for j, i in enumerate(perm):
        _same_streams(sp[j], base[0][i])
    # twice the drives through a third of the slots: seq_restart resets the slots' mappers with them
    jq = [(i % len(logs), list(range(len(logs[i % len(logs)]["time"])))) for i in range(2 * len(logs))]
    sq, _ = run(capi, defs, cases, len(logs) // 3, jq)
    for j, (i, _) in enumerate(jq):
        if i != ABSENT_JOB:
            _same_streams(sq[j], base[0][i])
    sm, _ = run(capi, defs, cases, len(logs), jobs, twin=False, mixed=True)
    for a, b in zip(sm, base[0]):
        _same_streams(a, b)


def _raw_map_step(g, defs, n, time=True, outlier=None, off=None):
    t = np.zeros(n)
    d = defs.LinsSeqMapDesc(n_seq=n, time=t.ctypes.data if time else None)
    if off is not None:
        d.outlier_off = off.ctypes.data
        d.outlier = outlier.ctypes.data if outlier is not None else None
    return g.L.lins_gpu_seq_map_step(g.h, C.byref(d), None, None)


def test_invalid_calls_change_nothing(capi, defs, cases):
    """Every rejected call leaves the sequence state, the mappers and the publish state as they were: the snapshot and
    every slot's mapper download are equal around each one, and the run then publishes exactly what a twin that never
    saw the rejected calls publishes."""
    logs, pcls = cases
    model = rc.model_of(defs, logs[0])
    n = 3
    fresh = capi.LinsGpu()
    fresh.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n)
    assert _raw_map_step(fresh, defs, n) == -3  # unbound
    ho = dict(filter_state=np.zeros((1, 19)), filter_cov=np.eye(18).reshape(1, 324), global_state=np.zeros((1, 19)), imu_last=np.zeros((1, 6)),
              surf_map=np.zeros(0, defs.POINT_DTYPE), surf_map_off=np.zeros(2, np.int32), corner_map=np.zeros(0, defs.POINT_DTYPE),
              corner_map_off=np.zeros(2, np.int32))
    ho["filter_state"][0, 9] = ho["global_state"][0, 9] = 1.0
    b = capi.LinsGpu()
    b.seq_begin(defs.LinsSeqParams.shipped(), ho)
    assert b.L.lins_gpu_seq_map_open(b.h) == -1  # a seq_begin run

    ctxs = []
    for _ in range(2):  # g takes the rejected calls, t is its twin
        c = capi.LinsGpu()
        c.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n)
        c.seq_map_open()
        ctxs.append(c)
    g, t = ctxs
    last = [None] * n  # each slot's last processed report

    def step(c, k, raw=True):
        imus = [logs[s]["imu"][logs[s]["imu_off"][k]:logs[s]["imu_off"][k + 1]] for s in range(n)]
        st = dict(imu=np.concatenate(imus), imu_off=np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32))
        si = np.array([logs[s]["imu_last"][k] for s in range(n)])
        if raw:
            c.seq_step_raw(dict(st, sweeps=[logs[s]["sweeps"][k] for s in range(n)]), model=model, scan_imu=si)
        else:
            c.seq_step_pcl(dict(st, scans=[pcls[s]["scans"][k] for s in range(n)]), scan_imu=si, line_num=model.line_num)

    def outl(k):
        return [defs.make_points(p["outlier"][:, :3], p["outlier"][:, 3])
                for p in g.project_scans([rc.finite(logs[s]["sweeps"][k]) for s in range(n)], model=model)]

    def map_step(k, raw=True):
        res = []
        for c in ctxs:
            res.append(c.seq_map_step([logs[s]["time"][k] for s in range(n)], outlier=None if raw else outl(k)))
        (ra, pa), (rb, pb) = res
        assert pa.tolist() == pb.tolist() and all(bytes(x) == bytes(y) for x, y in zip(ra, rb) if x is not None), k
        for s in range(n):
            if ra[s] is not None and ra[s].processed:
                last[s] = ra[s]

    def state():
        snap = _snapshot(g)
        out = [v.tobytes() if isinstance(v, np.ndarray) else v for v in snap.values()]
        for s in range(n):
            out.append(None if last[s] is None else _node(g, s, last[s]))
        return out

    for k in range(8):  # the mappers hold key frames before the rejected calls
        for c in ctxs:
            step(c, k)
        if k == 0:
            assert g.L.lins_gpu_seq_map_open(g.h) == -1  # after a step
        map_step(k)
    assert any(r is not None and r.n_keyframes > 0 for r in last)
    k = 8
    for c in ctxs:
        step(c, k)
    before = state()
    with pytest.raises(capi.LinsError, match="error -1"):  # a step while a publish is pending
        step(g, k + 1)
    pts = np.zeros(1, defs.POINT_DTYPE)
    for rc_, why in ((_raw_map_step(g, defs, n + 1), "n_seq"), (_raw_map_step(g, defs, n, time=False), "NULL time"),
                     (_raw_map_step(g, defs, n, outlier=pts, off=np.array([0, 1, 1, 1], np.int32)), "outliers after a _raw step")):
        assert rc_ == -1, why
        assert state() == before, why
    map_step(k)
    assert _raw_map_step(g, defs, n) == -1  # two map steps for one step
    k = 9
    for c in ctxs:
        step(c, k, raw=False)
    before = state()
    for rc_, why in ((_raw_map_step(g, defs, n), "missing outliers after a _pcl step"),
                     (_raw_map_step(g, defs, n, outlier=pts, off=np.array([0, 1, 0, 1], np.int32)), "bad CSR"),
                     (_raw_map_step(g, defs, n, outlier=None, off=np.array([0, 1, 1, 1], np.int32)), "NULL cloud with points")):
        assert rc_ == -1, why
        assert state() == before, why
    map_step(k, raw=False)
    for k in (10, 11):  # both keep publishing alike
        for c in ctxs:
            step(c, k)
        map_step(k)
    # mappers_open ends the binding
    g.mappers_open(n)
    step(g, 12)
    assert _raw_map_step(g, defs, n) == -3


def test_toobig_changes_no_mapper(capi, defs, cases):
    """A far outlier through a _pcl step: the cycle that reads it returns LINS_E_TOOBIG, no mapper slot changes, the
    publish is committed and the run continues."""
    logs, pcls = cases
    model = rc.model_of(defs, logs[0])
    g = capi.LinsGpu()
    g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), 1)
    g.seq_map_open()
    far = defs.make_points(np.array([[1e30, 0, 0], [-1e30, 0, 0]], np.float32), np.zeros(2, np.float32))
    last, hit = None, None
    for k in range(len(logs[0]["time"])):
        o = logs[0]["imu_off"]
        st = dict(imu=logs[0]["imu"][o[k]:o[k + 1]], imu_off=np.array([0, o[k + 1] - o[k]], np.int32),
                  scans=[pcls[0]["scans"][k]])
        g.seq_step_pcl(st, scan_imu=logs[0]["imu_last"][k][None], line_num=model.line_num)
        if last is None or last.n_keyframes < 2:
            reps, pub = g.seq_map_step([logs[0]["time"][k]], outlier=[np.zeros(0, defs.POINT_DTYPE)])
            last = reps[0] or last
            continue
        kp = np.zeros((last.n_keyframes, 7))
        g._ck(g.L.lins_gpu_mappers_download(g.h, 0, kp.ctypes.data, *[None] * 7))
        try:
            reps, pub = g.seq_map_step([logs[0]["time"][k]], outlier=[far])
            last = reps[0] or last
        except capi.LinsError as e:
            assert "error -4" in str(e)
            kp2 = np.zeros_like(kp)
            g._ck(g.L.lins_gpu_mappers_download(g.h, 0, kp2.ctypes.data, *[None] * 7))
            assert kp2.tobytes() == kp.tobytes()
            assert _raw_map_step(g, defs, 1) == -1  # the publish was committed: nothing pending
            hit = k
            break
    assert hit is not None and hit + 1 < len(logs[0]["time"])
    k = hit + 1
    o = logs[0]["imu_off"]
    g.seq_step_pcl(dict(imu=logs[0]["imu"][o[k]:o[k + 1]], imu_off=np.array([0, o[k + 1] - o[k]], np.int32), scans=[pcls[0]["scans"][k]]),
                   scan_imu=logs[0]["imu_last"][k][None], line_num=model.line_num)


# ---- against the shim ----------------------------------------------------------------------------------------------------
def _bag_tool():
    spec = importlib.util.spec_from_file_location("bag_tool", os.path.join(ROOT, "tools", "bag_tool.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _sweeps(bt, path):
    _, msgs = bt.read_bag(path)
    return [bt.decode_pointcloud2(b) for _, _, b in msgs if bt.index_pointcloud2(b) is not None]


def _ends_finite(bt, path):
    """The shim projects without the NaN removal: a bag replays alike only where every sweep's ends are finite."""
    for m in _sweeps(bt, path):
        xyz = np.stack([m["x"], m["y"], m["z"]], 1)
        if len(xyz) and not np.isfinite(xyz[[0, -1]]).all():
            return False
    return True


def _edited_bag(bt, src, dst):
    """src with its second PointCloud2 emptied and its sixth truncated to (about) its first half, ends finite."""
    conns, msgs = bt.read_bag(src)
    ids = sorted(conns)
    out, k = [], 0
    for cid, t, b in msgs:
        if bt.index_pointcloud2(b) is not None:
            if k in (1, 5):
                m = bt.decode_pointcloud2(b)
                xyz = np.stack([m["x"], m["y"], m["z"]], 1)
                n = 0
                if k == 5:
                    n = len(xyz) // 2
                    while n > 1 and not np.isfinite(xyz[n - 1]).all():
                        n -= 1
                ring = m["ring"][:n] if "ring" in m else None
                b = bt.encode_pointcloud2(m["header"]["seq"], m["header"]["stamp"], xyz[:n], m["intensity"][:n], ring=ring,
                                          frame=m["header"]["frame_id"], fields=m["fields"], point_step=bt.index_pointcloud2(b)["point_step"])
            k += 1
        out.append((ids.index(cid), t, b))
    bt.write_bag(dst, [(conns[c]["topic"], conns[c]["type"], conns[c]["md5sum"], conns[c]["message_definition"]) for c in ids], out)


def test_replayed_bags_against_the_shim(capi, defs, synth, tmp_path):
    """Bags through fewer slots than bags with replay(map=True), each against the shim's published stream fed to a
    single mapper: stamps exact, odometry within 1e-7, cloud sizes, processed / key-frame decisions and n_keyframes
    equal, transformAftMapped and key poses within 1e-5; then tools/run_bags.py --map's two files per bag."""
    bt = _bag_tool()
    paths, seed, replaced = [], 40, 0
    for n_scans in (16, 12, 20, 14, 15):
        while True:
            p = str(tmp_path / f"b{seed}.bag")
            synth.write_sequence_bag(p, config="config3", seed=seed, n_scans=n_scans)
            seed += 1
            if _ends_finite(bt, p):
                break
            replaced += 1
        paths.append(p)
    edited = str(tmp_path / "edited.bag")
    _edited_bag(bt, paths[2], edited)
    paths.append(edited)
    print("bags replaced because a sweep's end is not finite:", replaced)
    recs = [br.Recording(p) for p in paths]
    outs = br.replay(recs, 2, map=True)
    worst_odo = worst_map = 0.0
    for p, o in zip(paths, outs):
        ref = synth.run_bag(p)["map_inputs"]
        assert o["map_time"].tolist() == [m["time"] for m in ref], p
        g = capi.LinsGpu()
        g.mapper_reset()
        last = None
        for k, m in enumerate(ref):
            rep = g.mapper_step(m["time"], m["quat"], m["pos"], m["corner"], m["surf"], m["outlier"])
            worst_odo = max(worst_odo, float(np.abs(o["map_odom"][k] - np.concatenate([m["pos"], m["quat"]])).max()))
            assert (o["map_processed"][k], o["map_keyframes"][k]) == (rep.processed, rep.n_keyframes), (p, k)
            worst_map = max(worst_map, float(np.abs(o["map_aft_mapped"][k] - np.array(rep.transform_aft_mapped)).max()))
            last = rep
        assert o["map_sizes"].tolist() == [[len(m["corner"]), len(m["surf"]), len(m["outlier"])] for m in ref], p
        # (key poses only: a download's window and clouds are sized by the last processed cycle's report)
        poses = np.zeros((last.n_keyframes if last is not None else 0, 7))
        g._ck(g.L.lins_gpu_mapper_download(g.h, poses.ctypes.data, *[None] * 7))
        assert poses.shape == o["key_poses"].shape, p
        if len(poses):
            worst_map = max(worst_map, float(np.abs(poses[:, :6] - o["key_poses"][:, :6]).max()))
            assert np.abs(poses[:, 6] - o["key_poses"][:, 6]).max() == 0.0
    # the edited bag: its estimator falls back to INIT after the emptied second scan
    assert len(outs[-1]["map_time"]) >= 1 and outs[-1]["map_time"][0] == recs[-1].stamps[1]
    print("worst |replay - shim|: odometry", worst_odo, "transform_aft_mapped / key poses", worst_map)
    assert worst_odo < 1e-7 and worst_map < 1e-5
    out = tmp_path / "out"
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "run_bags.py")] + paths[:2] + ["--slots", "1", "--map", "--out", str(out)],
                          stdout=subprocess.DEVNULL)
    for p, o in zip(paths[:2], outs):
        name = os.path.splitext(os.path.basename(p))[0]
        od = [l.split() for l in open(out / f"{name}.odometry.txt")]
        mp = [l.split() for l in open(out / f"{name}.mapped.txt")]
        assert len(od) == len(mp) == len(o["map_time"]) and all(len(r) == 8 for r in od) and all(len(r) == 8 for r in mp)
        assert [float(r[0]) for r in od] == [float("%.9f" % t) for t in o["map_time"]]
        assert np.abs(np.array([[float(v) for v in r[1:]] for r in od]) - o["map_odom"]).max() < 1e-6
        assert [int(r[1]) for r in mp] == o["map_processed"].tolist()
