"""Replay many ROS1 bags (sensor_msgs/PointCloud2 + sensor_msgs/Imu) through sequence mode in lockstep.

Each bag is one recording, scheduled exactly as tools/synth/lins_sequence.cpp lins_seq_run_bag (synth.run_bag) feeds
one StateEstimator, so that run_bag is each bag's contract (LinsFusion, Estimator.cpp:204-252):
  - IMU samples and scans are stably sorted by header stamp;
  - the estimator clock starts one scan_period before the first scan;
  - before each scan, samples are taken from the upper_bound of the estimator time, each with
    dt = min(t_imu, t_scan) - t_est (a sample past the scan is used up to the scan and kept for the next);
  - processPCL's IMU sample is the last propagated one, or (0, 0, G0) / 0 when there is none.
The bags are queued through S slots (lins_gpu_seq_open, lins_gpu_seq_restart when a slot's bag has ended), and every
step hands each present slot's PointCloud2 data field to lins_gpu_seq_step_cloud2 as it is: the decode runs on the
device.  Bags of different sensors run together: each bag names its lidar model, and a step whose slots hold bags of more
than one model goes through lins_gpu_seq_step_cloud2_mixed, each slot projected with its bag's model.  A step's data fields are gathered into one host buffer that is page-locked once (re-registered only when it
grows), so each step's bytes go to the device in one DMA.
With map=True the run is bound to the context's lockstep mappers (lins_gpu_seq_map_open): after every step
lins_gpu_seq_map_step publishes what each slot's LinsFusion::publishTopics would and runs the mapping cycles of the slots
that published, on the device clouds.
A recording may carry its rig (a LinsSlotConfig: scan period, feature thresholds, extrinsic, IMU noise and biases, as a
LINS exp_port.yaml gives them): its slot is configured with it (lins_gpu_seq_configure) when it takes the recording, and
its IMU schedule uses that scan period.  Recordings without one use the run's values.  A recording may also carry its
tuning (a LinsSlotTuning: NUM_ITER, ICP_FREQ, the 1-NN gate, LIDAR_STD, LIDAR_SCALE and imu_misalign_angle): its slot is
tuned with it (lins_gpu_seq_tune) where it is configured, and the device rotates its IMU rows, which stay raw here.
A replay can stop and continue: replay(..., checkpoint=dir, stop_after=k) ends after k steps and writes a checkpoint
directory (every occupied slot saved by lins_gpu_seq_save, and the driver's state), and replay(..., resume=dir) opens a
new context with the same slot count, loads the slots into it (lins_gpu_seq_load) and continues from step k.  The
outputs equal those of a replay that never stopped, byte for byte.
"""
import ctypes as C
import glob
import importlib.util
import itertools
import os

import numpy as np

from . import capi as _capi
from .ctypes_defs import LinsCloud2Desc, LinsCloud2Layout, LinsLidarModel, LinsSeqInitParams, LinsSeqParams, SEQ_ICP, SEQ_RAN

G0 = 9.81  # filter::G0 (parameters.h:62)
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bag_tool():
    spec = importlib.util.spec_from_file_location("bag_tool", os.path.join(_ROOT, "tools", "bag_tool.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def layout(ix):
    """LinsCloud2Layout of a bag_tool.index_pointcloud2 dict."""
    lay = LinsCloud2Layout()
    lay.height, lay.width, lay.point_step, lay.row_step, lay.is_bigendian = ix["height"], ix["width"], ix["point_step"], ix["row_step"], ix["is_bigendian"]
    for k in range(4):
        lay.offset[k], lay.datatype[k] = ix["offset"][k], ix["datatype"][k]
    return lay


class Recording:
    """One bag: its scans (stamp, layout, data field) and, per scan, the processImu rows (dt, acc, gyr) and processPCL's
    IMU sample.  config: the bag's rig (LinsSlotConfig; None = the run's values); its scan_period is the schedule's, and a
    scan_period given as well must equal it.  tuning: the bag's estimator tuning and IMU misalignment (LinsSlotTuning;
    None = the context's lins_params and no rotation)."""

    def __init__(self, path, lidar_topic="/velodyne_points", imu_topic="/imu/data", max_scans=0, scan_period=None, config=None,
                 tuning=None):
        if config is not None and scan_period is not None and scan_period != config.scan_period:
            raise ValueError(f"scan_period {scan_period} differs from the config's {config.scan_period}")
        scan_period = config.scan_period if config is not None else (0.1 if scan_period is None else scan_period)
        self.config = config
        self.tuning = tuning
        bt = _bag_tool()
        conns, msgs = bt.read_bag(path)
        topic = {cid: c["topic"] for cid, c in conns.items()}
        imus, scans = [], []
        for cid, _, b in msgs:
            if topic.get(cid) == imu_topic:
                m = bt.decode_imu(b)
                imus.append((m["header"]["stamp"], m["linear_acceleration"], m["angular_velocity"]))
            elif topic.get(cid) == lidar_topic and (max_scans <= 0 or len(scans) < max_scans):
                ix = bt.index_pointcloud2(b)
                if ix is None:
                    raise ValueError(f"{path}: a PointCloud2 message the decoder rejects")
                scans.append((ix["stamp"], layout(ix), np.frombuffer(b, np.uint8, ix["data_len"], ix["data_start"])))
        imus = [imus[i] for i in np.argsort([t for t, _, _ in imus], kind="stable")]
        scans = [scans[i] for i in np.argsort([t for t, _, _ in scans], kind="stable")]
        self.path = path
        self.stamps = np.array([s[0] for s in scans])
        self.layouts = [s[1] for s in scans]
        self.data = [s[2] for s in scans]
        self.imu, self.imu_last = [], np.zeros((len(scans), 6))
        nxt, t_est = 0, (self.stamps[0] - scan_period) if len(scans) else 0.0
        for k, ts in enumerate(self.stamps):
            rows = []
            while t_est < ts and nxt < len(imus):
                ti, a, g = imus[nxt]
                if ti <= t_est:
                    nxt += 1
                    continue
                dt = min(ti, ts) - t_est
                rows.append((dt, *a, *g))
                t_est += dt
                if ti <= ts:
                    nxt += 1
            t_est = ts
            self.imu.append(np.array(rows, np.float64).reshape(-1, 7))
            self.imu_last[k] = rows[-1][1:] if rows else (0.0, 0.0, G0, 0.0, 0.0, 0.0)

    def __len__(self):
        return len(self.stamps)


class _PinnedBlob:
    """A host byte buffer page-locked once with lins_gpu_host_register (grown, and registered again, when a step needs
    more)."""

    def __init__(self):
        self.a = None

    def get(self, n):
        if self.a is None or len(self.a) < n:
            size = max(n, 1 << 20, 0 if self.a is None else 2 * len(self.a))
            self.release()
            self.a = np.empty(size, np.uint8)
            if _capi.lib().lins_gpu_host_register(self.a.ctypes.data, self.a.nbytes) != 0:
                raise _capi.LinsError("lins_gpu_host_register failed")
        return self.a

    def release(self):
        if self.a is not None:
            _capi.lib().lins_gpu_host_unregister(self.a.ctypes.data)
            self.a = None


def shim_init_params():
    """The filter constants run_bag's StateEstimator uses (lins_sequence.cpp seq_params: zero INIT_BA / INIT_BW)."""
    return LinsSeqInitParams.shipped(init_ba=(0.0, 0.0, 0.0), init_bw=(0.0, 0.0, 0.0))


def slot_queue(lengths, n_slots):
    """Schedule jobs of the given lengths (steps) through n_slots slots, as sequence mode queues recordings: a free slot takes
    the next job on the same step, and a job of length 0 is skipped.  Yields one (restart, who) per step until every job
    has run: restart (n_slots, uint8) flags the slots that take a new job after an earlier one (lins_gpu_seq_restart's
    mask), who[j] is (job, index of the step within the job) or None for a slot without a job."""
    cur, used, nxt = [None] * n_slots, [False] * n_slots, 0
    while True:
        restart = np.zeros(n_slots, np.uint8)
        for j in range(n_slots):
            if cur[j] is not None and cur[j][1] >= lengths[cur[j][0]]:
                cur[j] = None
            while cur[j] is None and nxt < len(lengths):
                if lengths[nxt]:
                    restart[j] = used[j]
                    cur[j], used[j] = [nxt, 0], True
                nxt += 1
        if all(c is None for c in cur):
            return
        yield restart, [(c[0], c[1]) if c is not None else None for c in cur]
        for c in cur:
            if c is not None:
                c[1] += 1


def model_table(recordings, model):
    """(models, model_of): the distinct lidar models of the recordings (a list, in first-use order) and each recording's
    index in it.  model: one LinsLidarModel for every recording, a list with one per recording, or None (VLP-16)."""
    if model is None or isinstance(model, LinsLidarModel):
        return [model or LinsLidarModel.vlp16()], [0] * len(recordings)
    model = list(model)
    if len(model) != len(recordings):
        raise ValueError(f"{len(model)} lidar models for {len(recordings)} recordings")
    models, keys, of = [], [], []
    for m in model:
        k = bytes(m)
        if k not in keys:
            keys.append(k)
            models.append(m)
        of.append(keys.index(k))
    return models, of


# the per-scan lists of a map=True replay and the arrays they become: (dtype, row shape)
_MAP_LISTS = dict(map_time=(np.float64, ()), map_odom=(np.float64, (7,)), map_processed=(np.int32, ()),
                  map_aft_mapped=(np.float32, (6,)), map_keyframes=(np.int32, ()), map_sizes=(np.int32, (3,)),
                  map_fused=(np.float64, (7,)))


def _map_arrays(o):
    """o with its per-published-scan lists as the arrays a finished replay returns."""
    o = dict(o)
    for k, (dt, row) in _MAP_LISTS.items():
        if k in o:
            o[k] = np.array(o[k], dt).reshape((-1,) + row)
    return o


def save_driver_state(path, step, slots, lengths, map, held, out, blob_files):
    """Write a replay's driver state to the file path (an .npz): the number of steps run, the slot count, the recording
    lengths, map, each slot's held recording (-1: none) and its last report's key-frame count (-1: none yet), the output
    dicts so far, and the file of each slot's blob ('' for an unsaved slot).  Written to a temporary file first, then
    renamed over path, so that a reader sees the old state or the new one."""
    a = dict(step=np.int64(step), slots=np.int64(slots), lengths=np.asarray(lengths, np.int64), map=np.int64(bool(map)),
             held_rec=np.array([h[0] if h is not None else -1 for h in held], np.int64),
             held_kf=np.array([h[1] if h is not None and h[1] is not None else -1 for h in held], np.int64),
             blob_files=np.array(blob_files, dtype=np.str_), n_out=np.int64(len(out)))
    for i, o in enumerate(out):
        for k, v in _map_arrays(o).items():
            a[f"out{i}.{k}"] = np.asarray(v)
    tmp = path + ".tmp.npz"
    np.savez(tmp, **a)
    os.replace(tmp, path)


def load_driver_state(path):
    """The driver state save_driver_state wrote: a dict of step, slots, lengths, map, held, out and blob_files, with out
    and held as replay() keeps them while it runs."""
    with np.load(path, allow_pickle=False) as z:
        out = [dict() for _ in range(int(z["n_out"]))]
        for name in z.files:
            if name.startswith("out"):
                i, k = name[3:].split(".", 1)
                v = z[name]
                out[int(i)][k] = list(v) if k in _MAP_LISTS else v
        held = [None if r < 0 else (int(r), None if kf < 0 else int(kf)) for r, kf in zip(z["held_rec"], z["held_kf"])]
        return dict(step=int(z["step"]), slots=int(z["slots"]), lengths=[int(x) for x in z["lengths"]], map=bool(z["map"]),
                    held=held, out=out, blob_files=[str(f) for f in z["blob_files"]])


def write_checkpoint(g, directory, step, who, lengths, map, held, out):
    """Save every slot that holds a recording after `step` steps (lins_gpu_seq_save) and the driver state into directory.
    Each checkpoint's blobs have files of their own, named by step; the driver state names them and is written last, and
    the older blobs go after it."""
    os.makedirs(directory, exist_ok=True)
    blobs = g.seq_save(np.array([w is not None for w in who], np.uint8))
    files = []
    for j, b in enumerate(blobs):
        if b is None:
            files.append("")
            continue
        files.append(f"slot{j}_step{step}.bin")
        with open(os.path.join(directory, files[-1]), "wb") as f:
            f.write(b)
    save_driver_state(os.path.join(directory, "driver.npz"), step, len(who), lengths, map, held, out, files)
    for f in glob.glob(os.path.join(directory, "slot*_step*.bin")):
        if os.path.basename(f) not in files:
            os.remove(f)


def read_checkpoint(directory):
    """The driver state of a checkpoint directory and its slot blobs (bytes, or None for a slot without one)."""
    st = load_driver_state(os.path.join(directory, "driver.npz"))
    blobs = []
    for f in st["blob_files"]:
        if not f:
            blobs.append(None)
            continue
        with open(os.path.join(directory, f), "rb") as fh:
            blobs.append(fh.read())
    return st, blobs


def replay(recordings, slots, model=None, device=0, gpu=None, map=False, checkpoint=None, checkpoint_every=None, stop_after=None,
           resume=None, loops=False, global_map=False):
    """Run the recordings through `slots` slots of one context.  model: one LinsLidarModel for every recording (None =
    VLP-16) or a list with one per recording; a slot is projected with the model of the recording it holds.  Returns per
    recording a dict of per-scan arrays: stamps, status (StateEstimator::status_ after the scan), scan_status (LINS_SEQ_*),
    global_est (n x 7: rn, qbn x y z w), global_state (n x 19), iters and flags (-1 where the scan ran no IESKF).
    map=True also runs each recording's mapping node on what its estimator publishes (the IMU orientation is not fed to
    the mappers, as tools/run_bag.py --map does not), and adds per published scan: map_time, map_odom (m x 7: the
    odometry, YZX position + quaternion x y z w of globalStateYZX_, as fed to the mapper), map_sizes (m x 3: the
    less-sharp, less-flat and outlier cloud sizes), map_processed, map_aft_mapped (m x 6: transformAftMapped) and
    map_keyframes (n_keyframes after the cycle), map_fused (m x 7: transform_fusion_node's pose of the scan, x y z qx qy
    qz qw in /camera_init, lins_gpu_seq_map_fused); and key_poses (the mapper's cloudKeyPoses6D, k x 7, downloaded when
    the recording ends).
    checkpoint: a directory.  With stop_after=k the replay ends after its first k steps, writes a checkpoint there and
    returns None (it returns the outputs as usual when it has fewer steps); with checkpoint_every=N it writes one after
    every N-th step and runs on.  resume: a checkpoint directory written for the same recordings, slot count and map:
    the replay continues from its step in a new context (gpu: one to open it on) and returns what a replay that never
    stopped returns.
    loops=True (with map=True) enables each recording's loop closure (lins_gpu_mappers_loops when a slot takes the
    recording) and ticks its loop thread after a published scan whenever the recording's stamp has advanced >= 1.0 s
    since its last tick (one lins_gpu_mappers_close_loops for all slots due): key_poses are then the corrected ones, and
    loops_accepted counts the recording's closures.  A slot with loop closure cannot be saved, so loops=True takes no
    checkpoint, stop_after or resume.
    global_map=True (with loops=True) builds each recording's global map (lins_gpu_mappers_global_map) when it ends,
    before its slot is handed on, in one call for every slot that finishes at the same step: global_map ((n, 4) float32
    x y z intensity in /camera_init) and global_map_keys (the key frames it concatenates)."""
    models, rec_model = model_table(recordings, model)
    lengths = [len(r) for r in recordings]
    if (stop_after is not None or checkpoint_every) and checkpoint is None:
        raise ValueError("stop_after / checkpoint_every need a checkpoint directory")
    if loops and not map:
        raise ValueError("loops=True needs map=True")
    if global_map and not loops:
        raise ValueError("global_map=True needs loops=True: the global map reads the key frames loop closure keeps")
    if loops and (checkpoint is not None or stop_after is not None or checkpoint_every or resume is not None):
        raise ValueError("loops=True cannot checkpoint or resume: a slot with loop closure is not saved")
    start, blobs = 0, None
    if resume is not None:
        st, blobs = read_checkpoint(resume)
        if st["lengths"] != lengths or st["slots"] != slots or st["map"] != bool(map):
            raise ValueError(f"{resume}: a checkpoint of other recordings, slot count or map setting")
        start = st["step"]
    g = gpu or _capi.LinsGpu(device=device)
    g.seq_open(LinsSeqParams.shipped(), shim_init_params(), slots)
    out = [dict(stamps=r.stamps.copy(), status=np.zeros(len(r), np.int32), scan_status=np.zeros(len(r), np.int32),
                global_est=np.zeros((len(r), 7)), global_state=np.zeros((len(r), 19)), iters=np.full(len(r), -1, np.int32),
                flags=np.full(len(r), -1, np.int32)) for r in recordings]
    held = [None] * slots  # (recording, n_keyframes of its last published report or None) of each slot (map=True)
    if map:
        g.seq_map_open()
        for o in out:
            o.update(map_time=[], map_odom=[], map_processed=[], map_aft_mapped=[], map_keyframes=[], map_sizes=[], map_fused=[],
                     key_poses=np.zeros((0, 7)))
            if loops:
                o["loops_accepted"] = 0
            if global_map:
                o.update(global_map=np.zeros((0, 4), np.float32), global_map_keys=np.zeros(0, np.int32))
    last_tick = [None] * slots  # (loops) the stamp of each slot's last loop-thread tick
    if resume is not None:
        out, held = st["out"], st["held"]
        g.seq_load(np.array([b is not None for b in blobs], np.uint8), blobs)
    blob = _PinnedBlob()

    def finish(js):  # the key poses (and global maps) of the recordings the slots js held, before the slots are handed on
        js = [j for j in js if held[j] is not None]
        if global_map and js:
            mask = np.zeros(slots, np.uint8)
            mask[js] = 1
            for j, rep in enumerate(g.mappers_global_map(mask)):
                if rep is not None:
                    o = out[held[j][0]]
                    o["global_map_keys"], o["global_map"] = g.mappers_global_map_download(j, rep)
        for j in js:
            if held[j][1] is not None:
                kp = np.zeros((held[j][1], 7))
                g._ck(g.L.lins_gpu_mappers_download(g.h, j, _capi.ptr(kp), *[None] * 7))
                out[held[j][0]]["key_poses"] = kp
            held[j] = None

    try:
        for t, (restart, who) in enumerate(itertools.islice(slot_queue(lengths, slots), start, None), start):
            if map:
                finish([j for j in range(slots) if held[j] is not None and (who[j] is None or who[j][0] != held[j][0])])
            if restart.any():
                g.seq_restart(restart)
            if loops:  # a slot taking a recording (after open or its restart) is fresh
                first = np.array([w is not None and w[1] == 0 for w in who], np.uint8)
                if first.any():
                    g.mappers_loops(first)
                    for j in np.flatnonzero(first):
                        last_tick[j] = None
            fresh = [w is not None and w[1] == 0 and getattr(recordings[w[0]], "config", None) is not None for w in who]
            if any(fresh):  # a slot taking a recording with a rig of its own (after open or its restart)
                g.seq_configure(np.array(fresh, np.uint8), [recordings[w[0]].config if f else None for w, f in zip(who, fresh)])
            tuned = [w is not None and w[1] == 0 and getattr(recordings[w[0]], "tuning", None) is not None for w in who]
            if any(tuned):  # ... and one with a tuning of its own
                g.seq_tune(np.array(tuned, np.uint8), [recordings[w[0]].tuning if f else None for w, f in zip(who, tuned)])
            present = np.array([w is not None for w in who], np.uint8)
            imus = [recordings[w[0]].imu[w[1]] if w else np.zeros((0, 7)) for w in who]
            imu_off = np.concatenate([[0], np.cumsum([len(r) for r in imus])]).astype(np.int32)
            scan_imu = np.array([recordings[w[0]].imu_last[w[1]] if w else np.zeros(6) for w in who])
            datas = [recordings[w[0]].data[w[1]] if w else np.zeros(0, np.uint8) for w in who]
            data_off = np.concatenate([[0], np.cumsum([len(d) for d in datas])]).astype(np.int64)
            buf = blob.get(int(data_off[-1]))
            for d, o in zip(datas, data_off):
                buf[o: o + len(d)] = d
            lays = (LinsCloud2Layout * slots)(*[recordings[w[0]].layouts[w[1]] if w else LinsCloud2Layout() for w in who])
            desc = LinsCloud2Desc()
            desc.n_scans, desc.data, desc.data_off, desc.layouts = slots, buf.ctypes.data, data_off.ctypes.data, C.cast(lays, C.c_void_p)
            step = dict(imu=np.concatenate(imus), imu_off=imu_off, present=present)
            if len(models) == 1:
                g.seq_step_cloud2(step, model=models[0], scan_imu=scan_imu, desc=desc)
            else:  # (an absent slot is projected as an empty sweep: any entry in range will do)
                model_of = np.array([rec_model[w[0]] if w else 0 for w in who], np.int32)
                g.seq_step_cloud2_mixed(step, models, model_of, scan_imu=scan_imu, desc=desc)
            d, di = g.seq_download(), g.seq_download_init()
            for j, w in enumerate(who):
                if w is None:
                    continue
                o, k = out[w[0]], w[1]
                o["status"][k], o["scan_status"][k] = di["fusion_status"][j], d["status"][j]
                gs = d["global_state"][j]
                o["global_state"][k] = gs
                o["global_est"][k] = np.concatenate([gs[0:3], gs[6:10]])
                if d["status"][j] in (SEQ_RAN, SEQ_ICP):
                    o["iters"][k], o["flags"][k] = d["results"]["iters"][j], d["results"]["flags"][j]
            if map:
                time = np.array([recordings[w[0]].stamps[w[1]] if w else 0.0 for w in who])
                reps, pub = g.seq_map_step(time)
                pose, sizes = g.seq_map_published()  # (the odometry and cloud sizes each slot's mapper was fed)
                fused = g.seq_map_fused()
                for j, w in enumerate(who):
                    if w is None:
                        continue
                    if held[j] is None:
                        held[j] = (w[0], None)
                    if not pub[j]:
                        continue
                    o, r = out[w[0]], reps[j]
                    held[j] = (w[0], r.n_keyframes)
                    o["map_time"].append(time[j]); o["map_odom"].append(pose[j].copy()); o["map_processed"].append(r.processed)
                    o["map_aft_mapped"].append(list(r.transform_aft_mapped)); o["map_keyframes"].append(r.n_keyframes)
                    o["map_sizes"].append(sizes[j].copy())
                    o["map_fused"].append(fused[j].row())
                if loops:  # the loop thread's 1 Hz tick, on each recording's own stamps
                    due = np.zeros(slots, np.uint8)
                    for j, w in enumerate(who):
                        if w is not None and pub[j] and (last_tick[j] is None or time[j] - last_tick[j] >= 1.0):
                            due[j], last_tick[j] = 1, time[j]
                    if due.any():
                        for j, lr in enumerate(g.mappers_close_loops(due)):
                            if lr is not None and lr.accepted:
                                out[who[j][0]]["loops_accepted"] += 1
            done = t + 1
            if stop_after is not None and done == stop_after:
                write_checkpoint(g, checkpoint, done, who, lengths, map, held, out)
                return None
            if checkpoint_every and done % checkpoint_every == 0:
                write_checkpoint(g, checkpoint, done, who, lengths, map, held, out)
        if map:
            finish(range(slots))
            out = [_map_arrays(o) for o in out]
    finally:
        blob.release()
    return out


def summary(o):
    """A line like tools/run_bag.py's."""
    it = o["iters"][o["iters"] >= 0]
    return "scans %d IESKF updates %d mean iterations %.2f diverged %d" % (
        len(o["stamps"]), len(it), it.mean() if len(it) else 0.0, int(((o["flags"][o["flags"] >= 0] & 2) != 0).sum()))
