"""GPU suite: sensor_msgs/PointCloud2 decoded on the device (lins_gpu_decode_cloud2) and sequence mode from the messages
(lins_gpu_seq_step_cloud2, DESIGN.md §4.8).

- decode_cloud2 equals the host decode_pointcloud2 (tools/synth/lins_bag.cpp) on every layout of cloud2cases, mixed in one
  call, with the data fields at every alignment mod 4 and the blob pageable or page-locked; NaN no-returns by NaN-ness,
  everything else bit for bit.
- Invalid descriptors return LINS_E_INVALID and change neither the outputs nor a running sequence.
- seq_step_cloud2 is bit-identical at every step to a twin context fed the host-decoded sweeps through seq_step_raw
  (test_gpu_seq_pcl._snapshot: states, covariances, results, scan_status, maps, correspondence IDs), for VLP-16 and
  64 x 1024 drives in the 32-B and 22-B layouts; S = 1, a permutation, a queue through fewer slots, alternation with
  seq_step_raw.
- bag_replay on bags from synth.write_sequence_bag through fewer slots than bags: bit-identical to the twin path, and
  per bag against synth.run_bag (status_, iterations and flags equal, states within 1e-7).
"""
import ctypes as C

import numpy as np
import pytest

import cloud2cases as cc
from conftest import pkg
from test_gpu_seq_init import init_params
from test_gpu_seq_pcl import _snapshot

pytestmark = pytest.mark.gpu
synth = pkg("synth")


@pytest.fixture(scope="module")
def baglib():
    return cc.baglib()


def _same_points(got, want, who):
    """lins_point records (POINT_DTYPE) against (n, 8) float32 host records: NaN by NaN-ness, the rest bit for bit."""
    g = got.view(np.float32).reshape(-1, 8)
    assert g.shape == want.shape, who
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(g), nan), who
    assert np.array_equal(g.view(np.uint32)[~nan], want.view(np.uint32)[~nan]), who


def _all_layout_msgs(seed=21):
    rng = np.random.default_rng(seed)
    msgs = []
    for name in cc.LAYOUTS:
        for n in (0, 37, 1000):
            if name == "organised" and n % 4:
                n += 4 - n % 4
            msgs.append(cc.message(name, cc.sweep(rng, n), seq=len(msgs))[0])
    return msgs


@pytest.mark.parametrize("gap", [0, 1, 2, 3])
def test_decode_matches_host_on_every_layout_and_alignment(capi, defs, baglib, gap):
    msgs = _all_layout_msgs()
    want = np.concatenate([cc.decode_cpp(baglib, m) for m in msgs])
    assert np.isnan(want[:, 0]).any() and len(want) > 5000
    g = capi.LinsGpu()
    inputs = [cc.as_input(defs, m) for m in msgs]
    for base in range(4):
        out, counts = g.decode_cloud2(inputs, gap=gap, base=base)
        _same_points(out, want, (gap, base))
        assert counts.tolist() == [len(cc.decode_cpp(baglib, m)) for m in msgs]
    assert g.decode_ms() > 0
    # the same blob page-locked: one DMA straight from it
    keep = {}
    d = g.cloud2_desc(inputs, keep, gap=gap, base=1)
    b = keep["blob"]
    assert capi.lib().lins_gpu_host_register(b.ctypes.data, b.nbytes) == 0
    try:
        out, _ = g.decode_cloud2(desc=d)
    finally:
        capi.lib().lins_gpu_host_unregister(b.ctypes.data)
    _same_points(out, want, "pinned")


def test_decode_conversion_edges(capi, defs, baglib):
    """The conversion edges the CPU suite checks on the host (integer extremes, uint32 above 2^24, halfway and overflowing
    doubles, subnormal results, +-0, NaN and signalling NaN, inf) through the device decode, every field misaligned."""
    msgs = cc.edge_messages()
    assert len(msgs) == 8
    want = np.concatenate([cc.decode_cpp(baglib, m) for m in msgs])
    g = capi.LinsGpu()
    for gap in (0, 3):
        out, _ = g.decode_cloud2([cc.as_input(defs, m) for m in msgs], gap=gap)
        _same_points(out, want, gap)
    x = want[:, [0, 1, 2, 4]]
    assert np.isinf(x).any() and np.isnan(x).any() and ((x != 0) & (np.abs(x) < 1.1754942e-38)).any()
    assert (x.view(np.uint32) == 0x80000000).any()


def _bad_descs(defs, capi, good):
    """(what, LinsCloud2Desc, keep) of descriptors that must be rejected."""
    out = []

    def mk(edit_layout=None, edit=None):
        keep = {}
        d = capi.LinsGpu.cloud2_desc(good, keep)
        lays = C.cast(d.layouts, C.POINTER(defs.LinsCloud2Layout))
        if edit_layout:
            edit_layout(lays[1])
        if edit:
            edit(d, keep)
        return d, keep

    def setf(k, v):
        def f(lay):
            setattr(lay, k, v)
        return f

    out.append(("bigendian", *mk(setf("is_bigendian", 1))))
    out.append(("no_x", *mk(lambda l: l.datatype.__setitem__(0, 0))))
    out.append(("datatype_9", *mk(lambda l: l.datatype.__setitem__(2, 9))))
    out.append(("field_past_step", *mk(lambda l: l.offset.__setitem__(3, l.point_step - 3))))
    out.append(("offset_near_2^32", *mk(lambda l: l.offset.__setitem__(1, 2 ** 32 - 2))))
    out.append(("point_past_data", *mk(setf("width", 10 ** 6))))
    out.append(("row_past_data", *mk(lambda l: (setattr(l, "height", 2), setattr(l, "row_step", 2 ** 32 - 1)))))
    out.append(("over_int32_points", *mk(lambda l: (setattr(l, "height", 2 ** 31), setattr(l, "width", 1), setattr(l, "row_step", 0)))))

    def dec(d, keep):
        keep["data_off"][2] = keep["data_off"][1] - 1
    out.append(("decreasing_data_off", *mk(edit=dec)))

    def neg(d, keep):
        keep["data_off"][0] = -1
    out.append(("negative_data_off", *mk(edit=neg)))
    out.append(("null_data", *mk(edit=lambda d, k: setattr(d, "data", None))))
    out.append(("null_layouts", *mk(edit=lambda d, k: setattr(d, "layouts", None))))
    out.append(("null_data_off", *mk(edit=lambda d, k: setattr(d, "data_off", None))))
    return out


def test_invalid_descriptors_change_nothing(capi, defs):
    rng = np.random.default_rng(4)
    good = [cc.as_input(defs, cc.message(n, cc.sweep(rng, 64))[0]) for n in ("velodyne32", "ring_time22", "f64_48")]
    g = capi.LinsGpu()
    log = synth.raw_log("config3", seed=5, n_scans=3)
    g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), 3)
    msgs = [cc.as_input(defs, cc.message("velodyne32", log["sweeps"][0])[0]) for _ in range(3)]
    o = log["imu_off"]
    step = dict(imu=np.concatenate([log["imu"][o[0]:o[1]]] * 3), imu_off=np.array([0, 1, 2, 3]) * (o[1] - o[0]), msgs=msgs)
    g.seq_step_cloud2(step, scan_imu=np.tile(log["imu_last"][0], (3, 1)))
    before = _snapshot(g)
    for what, d, keep in _bad_descs(defs, capi, good):
        out = np.full(200, 7, capi.POINT_DTYPE)
        cnt = np.full(3, -5, np.int32)
        assert g.L.lins_gpu_decode_cloud2(g.h, C.byref(d), out.ctypes.data, cnt.ctypes.data) == -1, what
        assert (out.view(np.uint8) == np.full(200, 7, capi.POINT_DTYPE).view(np.uint8)).all() and (cnt == -5).all(), what
        sd = defs.LinsSeqCloud2Desc()
        sd.n_seq, sd.cloud2 = 3, d
        imu = np.ascontiguousarray(step["imu"], np.float64)
        ioff = np.ascontiguousarray(step["imu_off"], np.int32)
        sd.imu, sd.imu_off = imu.ctypes.data, ioff.ctypes.data
        si = np.ascontiguousarray(np.tile(log["imu_last"][1], (3, 1)))
        assert g.L.lins_gpu_seq_step_cloud2(g.h, C.byref(sd), C.byref(defs.LinsLidarModel.vlp16()), C.byref(defs.LinsFeatureParams.shipped()),
                                            si.ctypes.data) == -1, what
        after = _snapshot(g)
        for k in before:
            assert (before[k].tobytes() == after[k].tobytes()) if isinstance(before[k], np.ndarray) else before[k] == after[k], (what, k)
    # a NULL output with points to write is rejected as well; with no points it is not needed
    keep = {}
    d = g.cloud2_desc(good, keep)
    assert g.L.lins_gpu_decode_cloud2(g.h, C.byref(d), None, None) == -1
    d0 = g.cloud2_desc([cc.as_input(defs, cc.message("velodyne32", np.zeros((0, 4)))[0])], keep)
    assert g.L.lins_gpu_decode_cloud2(g.h, C.byref(d0), None, None) == 0


def _drives(lidar, n, n_scans):
    config = "config4" if lidar == 1 else "config3"
    return [synth.raw_log(config, seed=700 + 13 * s + lidar, n_scans=n_scans - (s % 3)) for s in range(n)]


@pytest.fixture(scope="module")
def vlp_logs():
    return _drives(0, 6, 9)


@pytest.fixture(scope="module")
def dense_logs():
    return _drives(1, 3, 7)


def drive(capi, defs, baglib, logs, n_slots, jobs, layout, alt=False, gap=3):
    """Run jobs (log indices, each from scan 0) through n_slots slots with seq_step_cloud2 (alt: every other step
    seq_step_raw of the host-decoded sweeps instead), a twin context with seq_step_raw of the host-decoded sweeps; the
    snapshots must be bit-identical after every step.  Returns rows[i] = [(scan, snapshot row)]."""
    model = defs.LinsLidarModel.dense64() if int(logs[0]["lidar"]) == 1 else defs.LinsLidarModel.vlp16()
    msgs = [[cc.message(layout, s, seq=k)[0] for k, s in enumerate(l["sweeps"])] for l in logs]
    host = [[cc.decode_cpp(baglib, m)[:, [0, 1, 2, 4]].copy() for m in ms] for ms in msgs]
    for l, hs in zip(logs, host):  # the message holds the sweep exactly
        assert all(np.array_equal(h, s, equal_nan=True) for h, s in zip(hs, l["sweeps"]))
    ctxs = []
    for _ in range(2):
        g = capi.LinsGpu()
        g.seq_open(defs.LinsSeqParams.shipped(), init_params(defs), n_slots)
        ctxs.append(g)
    g, tw = ctxs
    t = 0
    rows = [[] for _ in jobs]
    for restart, who in pkg("bag_replay").slot_queue([len(logs[i]["time"]) for i in jobs], n_slots):
        if restart.any():
            for c in ctxs:
                c.seq_restart(restart)
        imus, si, ins, sweeps = [], np.zeros((n_slots, 6)), [], []
        for j, w in enumerate(who):
            if w is None:
                imus.append(np.zeros((0, 7))); ins.append((defs.LinsCloud2Layout(), b"")); sweeps.append(np.zeros((0, 4), np.float32))
                continue
            l, k = logs[jobs[w[0]]], w[1]
            o = l["imu_off"]
            imus.append(l["imu"][o[k]:o[k + 1]]); si[j] = l["imu_last"][k]
            ins.append(cc.as_input(defs, msgs[jobs[w[0]]][k])); sweeps.append(host[jobs[w[0]]][k])
        imu = np.concatenate(imus).reshape(-1, 7)
        imu_off = np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32)
        pres = np.array([w is not None for w in who], np.uint8)
        if alt and t % 2:
            g.seq_step_raw(dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=pres), model=model, scan_imu=si)
        else:
            g.seq_step_cloud2(dict(imu=imu, imu_off=imu_off, msgs=ins, present=pres), model=model, scan_imu=si, gap=gap)
            assert g.decode_ms() > 0 and g.project_ms() > 0 and g.extract_ms() > 0
        tw.seq_step_raw(dict(imu=imu, imu_off=imu_off, sweeps=sweeps, present=pres), model=model, scan_imu=si)
        a, b = _snapshot(g), _snapshot(tw)
        for key in a:
            same = a[key].tobytes() == b[key].tobytes() if isinstance(a[key], np.ndarray) else a[key] == b[key]
            assert same, f"step {t}: {key}"
        d = g.seq_download()
        for j, w in enumerate(who):
            if w is not None:
                rows[w[0]].append((w[1], (d["global_state"][j].tobytes(), int(d["status"][j]))))
        t += 1
    return rows


@pytest.mark.parametrize("layout", ["velodyne32", "ring_time22"])
def test_seq_step_cloud2_vlp16_equals_raw_twin(capi, defs, baglib, vlp_logs, layout):
    rows = drive(capi, defs, baglib, vlp_logs, len(vlp_logs), list(range(len(vlp_logs))), layout)
    codes = {c for r in rows for _, (_, c) in r}
    assert {defs.SEQ_FIRST, defs.SEQ_SECOND, defs.SEQ_RAN} <= codes, codes


@pytest.mark.parametrize("layout", ["velodyne32", "ring_time22"])
def test_seq_step_cloud2_dense64_equals_raw_twin(capi, defs, baglib, dense_logs, layout):
    drive(capi, defs, baglib, dense_logs, len(dense_logs), list(range(len(dense_logs))), layout)


def test_single_slot_permutation_queue_and_alternation(capi, defs, baglib, vlp_logs):
    n = len(vlp_logs)
    full = drive(capi, defs, baglib, vlp_logs, n, list(range(n)), "velodyne32")
    assert drive(capi, defs, baglib, vlp_logs, 1, [2], "ring_time22")[0] == full[2]
    perm = list(np.random.default_rng(9).permutation(n))
    rows = drive(capi, defs, baglib, vlp_logs, n, perm, "velodyne32")
    assert all(rows[j] == full[i] for j, i in enumerate(perm))
    rows = drive(capi, defs, baglib, vlp_logs, 2, list(range(n)) + [0, 1], "ring_time22")  # fewer slots, restart
    assert rows[:n] == full and rows[n:] == full[:2]
    rows = drive(capi, defs, baglib, vlp_logs, n, list(range(n)), "velodyne32", alt=True)
    assert rows == full


@pytest.fixture(scope="module")
def bags(tmp_path_factory, baglib):
    d = tmp_path_factory.mktemp("bags")
    paths = []
    for s in range(3):
        p = str(d / f"drive{s}.bag")
        synth.write_sequence_bag(p, seed=40 + s, n_scans=10 - 2 * s)
        paths.append(p)
    for p in paths:  # the shim projects without the NaN removal: its sweeps' ends must be finite for the two to agree
        _, msgs = cc.bag_tool.read_bag(p)
        for _, _, b in msgs:
            pts = cc.decode_cpp(baglib, b) if cc.bag_tool.index_pointcloud2(b) else None
            if pts is not None and len(pts):
                assert np.isfinite(pts[[0, -1], :3]).all()
    return paths


class _HostTwin:
    """A LinsGpu whose seq_step_cloud2 decodes the messages on the host (numpy: each field read, then (float), as
    read_scalar does) and runs seq_step_raw."""

    def __init__(self, capi):
        self.g = capi.LinsGpu()

    def __getattr__(self, k):
        return getattr(self.g, k)

    def seq_step_cloud2(self, step, model=None, fp=None, scan_imu=None, desc=None):
        n = desc.n_scans
        off = np.ctypeslib.as_array(C.cast(desc.data_off, C.POINTER(C.c_int64)), (n + 1,))
        lays = C.cast(desc.layouts, C.POINTER(pkg("ctypes_defs").LinsCloud2Layout))
        sweeps = []
        for i in range(n):
            data = np.frombuffer(C.string_at(desc.data + int(off[i]), int(off[i + 1] - off[i])), np.uint8)
            sweeps.append(cc.host_decode(lays[i], data) if step["present"][i] else np.zeros((0, 4), np.float32))
        self.g.seq_step_raw(dict(imu=step["imu"], imu_off=step["imu_off"], sweeps=sweeps, present=step["present"]), model=model,
                            scan_imu=scan_imu)


def test_bag_replay_through_fewer_slots(capi, defs, bags):
    br = pkg("bag_replay")
    recs = [br.Recording(p) for p in bags]
    dev = br.replay(recs, 2)
    twin = br.replay(recs, 2, gpu=_HostTwin(capi))
    for a, b in zip(dev, twin):
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
    worst = 0.0
    for p, o in zip(bags, dev):
        ref = synth.run_bag(p)
        assert np.array_equal(o["status"], ref["status"])
        ran = np.flatnonzero(o["iters"] >= 0)
        assert np.array_equal(ran, np.asarray(ref["scan_index"])), (ran, ref["scan_index"])
        assert np.array_equal(o["iters"][ran], ref["iters"]) and np.array_equal(o["flags"][ran], ref["flags"])
        diff = np.abs(o["global_est"] - ref["global_est"]).max()
        worst = max(worst, diff)
        assert diff <= 1e-7, (p, diff)
        assert len(ran) > 0
    print("worst |replay - run_bag|", worst)
