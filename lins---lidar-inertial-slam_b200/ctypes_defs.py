"""ctypes mirrors of the C structs in include/lins_gpu.h (the drop-in boundary).

Plain data only: no compute lives here.  numpy structured dtype POINT_DTYPE is layout-identical to
``lins_point`` / ``pcl::PointXYZI`` (32 B; reference lins/include/parameters.h:52).
"""
import ctypes as C

import numpy as np

LINS_MAX_ITER = 64
STATE_DIM = 19
COV_SIZE = 324

POINT_DTYPE = np.dtype(
    {
        "names": ["x", "y", "z", "pad0", "intensity", "pad1", "pad2", "pad3"],
        "formats": [np.float32] * 8,
        "itemsize": 32,
    }
)


class LinsParams(C.Structure):
    _fields_ = [
        ("num_iter", C.c_int32),
        ("icp_freq", C.c_int32),
        ("nearest_feature_search_sq_dist", C.c_double),
        ("lidar_std", C.c_double),
        ("lidar_scale", C.c_double),
        ("scan_period", C.c_double),
        ("verbose", C.c_int32),
        ("force_all_iters", C.c_int32),
    ]

    @classmethod
    def shipped(cls, **kw):
        """lins/config/exp_config/exp_port.yaml:9-20 values."""
        p = cls(30, 1, 25.0, 0.01, 1.0, 0.1, 0, 0)
        for k, v in kw.items():
            setattr(p, k, v)
        return p


class LinsReport(C.Structure):
    _fields_ = [
        ("iters", C.c_int32),
        ("converged", C.c_int32),
        ("diverged", C.c_int32),
        ("has_nan", C.c_int32),
        ("m_surf", C.c_int32 * LINS_MAX_ITER),
        ("m_corner", C.c_int32 * LINS_MAX_ITER),
        ("residual_norm", C.c_double * LINS_MAX_ITER),
        ("update_norm", C.c_double * LINS_MAX_ITER),
    ]


class LinsMapReport(C.Structure):
    """lins_map_report (include/lins_gpu.h, row F2)."""
    _fields_ = [("iters", C.c_int32), ("converged", C.c_int32), ("degenerate", C.c_int32), ("skipped", C.c_int32),
                ("n_sel", C.c_int32 * 10), ("delta_r", C.c_float * 10), ("delta_t", C.c_float * 10)]


class LinsMapperDesc(C.Structure):
    """lins_mapper_desc (include/lins_gpu.h): one mapping cycle's odometry and clouds."""
    _fields_ = [("time", C.c_double), ("quat", C.c_double * 4), ("pos", C.c_double * 3), ("corner", C.c_void_p),
                ("surf", C.c_void_p), ("outlier", C.c_void_p), ("n_corner", C.c_int32), ("n_surf", C.c_int32),
                ("n_outlier", C.c_int32), ("pad", C.c_int32)]


class LinsMappersDesc(C.Structure):
    """lins_mappers_desc (include/lins_gpu.h): one lockstep step of M mapper slots (CSR clouds as lins_batch_desc)."""
    _fields_ = [("n_slots", C.c_int32), ("pad", C.c_int32), ("present", C.c_void_p), ("time", C.c_void_p), ("quat", C.c_void_p),
                ("pos", C.c_void_p), ("corner", C.c_void_p), ("corner_off", C.c_void_p), ("surf", C.c_void_p), ("surf_off", C.c_void_p),
                ("outlier", C.c_void_p), ("outlier_off", C.c_void_p)]


class LinsSeqMapDesc(C.Structure):
    """lins_seq_map_desc (include/lins_gpu.h): the publish step after a sequence step: the scans' stamps and, after a step
    whose scans did not come through the device projection, their outlier clouds (CSR)."""
    _fields_ = [("n_seq", C.c_int32), ("pad", C.c_int32), ("time", C.c_void_p), ("outlier", C.c_void_p), ("outlier_off", C.c_void_p)]


class LinsMapperReport(C.Structure):
    """lins_mapper_report (include/lins_gpu.h)."""
    _fields_ = [("processed", C.c_int32), ("skipped_interval", C.c_int32), ("n_map_corner_ds", C.c_int32),
                ("n_map_surf_ds", C.c_int32), ("n_corner_ds", C.c_int32), ("n_surf_ds", C.c_int32), ("n_outlier_ds", C.c_int32),
                ("n_surf_total_ds", C.c_int32), ("keyframe_saved", C.c_int32), ("n_keyframes", C.c_int32),
                ("window_len", C.c_int32), ("loop_candidate", C.c_int32), ("transform_guess", C.c_float * 6),
                ("transform_aft_mapped", C.c_float * 6), ("map", LinsMapReport)]


class LinsLoopReport(C.Structure):
    """lins_loop_report (include/lins_gpu.h): one performLoopClosure of a mapper slot."""
    _fields_ = [("closest_history_frame_id", C.c_int32), ("latest_frame_id", C.c_int32), ("n_source", C.c_int32),
                ("n_history_ds", C.c_int32), ("icp_iters", C.c_int32), ("n_corr0", C.c_int32), ("converged", C.c_int32),
                ("accepted", C.c_int32), ("fitness", C.c_double), ("final_transform", C.c_float * 16), ("factor", C.c_double * 6),
                ("noise", C.c_double)]


GLOBAL_MAP_PASS_POINTS = 1 << 24  # LINS_GLOBAL_MAP_PASS_POINTS: gathered points per device pass of the global map


class LinsGlobalMapReport(C.Structure):
    """lins_global_map_report (include/lins_gpu.h): one publishGlobalMap of a mapper slot."""
    _fields_ = [("n_key_poses", C.c_int32), ("n_key_frames", C.c_int32), ("n_points", C.c_int64), ("n_map", C.c_int32),
                ("unfiltered", C.c_int32)]


class LinsFusedPose(C.Structure):
    """lins_fused_pose (include/lins_gpu.h): transform_fusion_node's pose of one odometry message."""
    _fields_ = [("time", C.c_double), ("pos", C.c_double * 3), ("quat", C.c_double * 4), ("transform_mapped", C.c_float * 6),
                ("valid", C.c_int32), ("pad", C.c_int32)]

    def row(self):
        """(x, y, z, qx, qy, qz, qw)"""
        return list(self.pos) + list(self.quat)


class LinsScanResult(C.Structure):
    _fields_ = [
        ("scan_id", C.c_int32),
        ("iters", C.c_uint16),
        ("flags", C.c_uint16),
        ("pose", C.c_double * 7),
    ]


SCAN_RESULT_DTYPE = np.dtype(
    [("scan_id", np.int32), ("iters", np.uint16), ("flags", np.uint16), ("pose", np.float64, 7)]
)
assert SCAN_RESULT_DTYPE.itemsize == 64 == C.sizeof(LinsScanResult)


class LinsBatchDesc(C.Structure):
    _fields_ = [
        ("n_scans", C.c_int32),
        ("surf_flat", C.c_void_p),
        ("surf_flat_off", C.c_void_p),
        ("corner_sharp", C.c_void_p),
        ("corner_sharp_off", C.c_void_p),
        ("surf_less_flat", C.c_void_p),
        ("surf_less_flat_off", C.c_void_p),
        ("corner_less_sharp", C.c_void_p),
        ("corner_less_sharp_off", C.c_void_p),
        ("state_in", C.c_void_p),
        ("cov_in", C.c_void_p),
        ("point_format", C.c_int32),  # 0 = 32-B PointXYZI records, 1 = packed 16-B (x, y, z, intensity)
    ]


class LinsSeqParams(C.Structure):
    """lins_seq_params (include/lins_gpu.h, sequence mode)."""
    _fields_ = [("noise", C.c_double * 4), ("init_pos_std", C.c_double * 3), ("init_att_std", C.c_double * 3)]

    @classmethod
    def shipped(cls, acc_n=70000.0, gyr_n=0.1, acc_w=500.0, gyr_w=0.05, init_pos_std=(0.0, 0.0, 0.0), init_att_std=(0.0, 0.0, 0.0)):
        """csrc/host/kalman_filter.hpp FilterParams defaults (exp_port.yaml:29-62); noise as StatePredictor::setNoise."""
        import math
        deg = math.pi / 180.0
        dph, dpsh = deg / 3600.0, deg / math.sqrt(3600.0)
        ug = (9.81 / 1000.0) / 1000.0
        ugpshz = ug / math.sqrt(1.0)
        p = cls()
        for i, v in enumerate((math.pow(acc_n * ug, 2), math.pow(gyr_n * dph, 2), math.pow(acc_w * ugpshz, 2), math.pow(gyr_w * dpsh, 2))):
            p.noise[i] = v
        for i in range(3):
            p.init_pos_std[i], p.init_att_std[i] = init_pos_std[i], init_att_std[i]
        return p


class LinsSeqInitParams(C.Structure):
    """lins_seq_init_params (include/lins_gpu.h): the filter constants sequence initialisation reads."""
    _fields_ = [("init_vel_std", C.c_double * 3), ("init_acc_std", C.c_double * 3), ("init_gyr_std", C.c_double * 3),
                ("init_ba", C.c_double * 3), ("init_bw", C.c_double * 3)]

    @classmethod
    def shipped(cls, init_vel_std=(0.0, 0.0, 0.0), init_acc_std=(0.01, 0.01, 0.02), init_gyr_std=(0.002, 0.002, 0.002),
                init_ba=(-0.015774, 0.143237, -0.0263845), init_bw=(-0.00275058, -0.000165954, 0.00262913)):
        """csrc/host/kalman_filter.hpp FilterParams defaults (exp_port.yaml:29-62)."""
        p = cls()
        for name, v in (("init_vel_std", init_vel_std), ("init_acc_std", init_acc_std), ("init_gyr_std", init_gyr_std),
                        ("init_ba", init_ba), ("init_bw", init_bw)):
            for i in range(3):
                getattr(p, name)[i] = v[i]
        return p


class LinsSeqBeginDesc(C.Structure):
    _fields_ = [
        ("n_seq", C.c_int32),
        ("filter_state", C.c_void_p),
        ("filter_cov", C.c_void_p),
        ("global_state", C.c_void_p),
        ("imu_last", C.c_void_p),
        ("surf_map", C.c_void_p),
        ("surf_map_off", C.c_void_p),
        ("corner_map", C.c_void_p),
        ("corner_map_off", C.c_void_p),
        ("point_format", C.c_int32),
    ]


class LinsFeatureParams(C.Structure):
    """lins_feature_params (include/lins_gpu.h): the feature extraction's constants."""
    _fields_ = [("edge_threshold", C.c_double), ("surf_threshold", C.c_double), ("imu_lidar_extrinsic_angle", C.c_double)]

    @classmethod
    def shipped(cls, edge_threshold=0.5, surf_threshold=0.5, imu_lidar_extrinsic_angle=0.0):
        """exp_port.yaml:7, :12-13 (csrc/host/feature_extraction.hpp FeatureParams defaults)."""
        return cls(edge_threshold, surf_threshold, imu_lidar_extrinsic_angle)


class LinsSlotConfig(C.Structure):
    """lins_slot_config (include/lins_gpu.h): one recording's rig, the exp_port.yaml values that describe its sensors."""
    _fields_ = [("scan_period", C.c_double), ("features", LinsFeatureParams), ("filter", LinsSeqParams), ("init", LinsSeqInitParams)]

    @classmethod
    def shipped(cls, scan_period=0.1, **kw):
        """The shipped rig (LinsFeatureParams / LinsSeqParams / LinsSeqInitParams.shipped) with any of their keyword
        arguments overridden, e.g. shipped(scan_period=0.05, edge_threshold=1.0, acc_n=5e4, init_ba=(0, 0, 0))."""
        import inspect
        parts = []
        for sub in (LinsFeatureParams, LinsSeqParams, LinsSeqInitParams):
            names = inspect.signature(sub.shipped).parameters
            parts.append(sub.shipped(**{k: kw.pop(k) for k in list(kw) if k in names}))
        if kw:
            raise TypeError(f"unknown slot config keys: {sorted(kw)}")
        return cls(scan_period, *parts)


class LinsSlotTuning(C.Structure):
    """lins_slot_tuning (include/lins_gpu.h): one recording's estimator tuning and IMU misalignment."""
    _fields_ = [("num_iter", C.c_int32), ("icp_freq", C.c_int32), ("nearest_feature_search_sq_dist", C.c_double),
                ("lidar_std", C.c_double), ("lidar_scale", C.c_double), ("imu_misalign_angle", C.c_double)]

    @classmethod
    def shipped(cls, **kw):
        """exp_port.yaml's values (NUM_ITER 30, ICP_FREQ 1, the 25 m^2 gate, LIDAR_STD 0.01, LIDAR_SCALE 1, a 3 degree
        imu_misalign_angle) with any field overridden, e.g. shipped(num_iter=12, imu_misalign_angle=0.0)."""
        t = cls(30, 1, 25.0, 0.01, 1.0, 3.0)
        for k, v in kw.items():
            if k not in dict(cls._fields_):
                raise TypeError(f"unknown slot tuning key: {k}")
            setattr(t, k, v)
        return t


class LinsPclDesc(C.Structure):
    """lins_pcl_desc: n segmented scans with their cloud_info, CSR."""
    _fields_ = [("n_scans", C.c_int32), ("line_num", C.c_int32), ("cloud", C.c_void_p), ("cloud_off", C.c_void_p),
                ("ground_flag", C.c_void_p), ("col_ind", C.c_void_p), ("range", C.c_void_p), ("start_ring_index", C.c_void_p),
                ("end_ring_index", C.c_void_p), ("orientation", C.c_void_p), ("point_format", C.c_int32)]


class LinsSeqPclDesc(C.Structure):
    """lins_seq_pcl_desc: one processPCL-shaped scan per sequence."""
    _fields_ = [("n_seq", C.c_int32), ("present", C.c_void_p), ("imu", C.c_void_p), ("imu_off", C.c_void_p), ("pcl", LinsPclDesc)]


FEAT_RING_CAP = 2048  # LINS_FEAT_RING_CAP


class LinsLidarModel(C.Structure):
    """lins_lidar_model: the lidar geometry image projection reads (csrc/host/cloud.hpp LidarModel)."""
    _fields_ = [("line_num", C.c_int32), ("scan_num", C.c_int32), ("ang_res_x", C.c_float), ("ang_res_y", C.c_float),
                ("ang_bottom", C.c_float), ("ground_scan_ind", C.c_int32)]

    # (the C++ LidarModel's constants are float expressions: evaluated in float32 here too)
    @classmethod
    def vlp16(cls):
        """The reference's hard-wired VLP-16 (parameters.h:82-92)."""
        f = np.float32
        return cls(16, 1800, f(0.2), f(2.0), f(15.0) + f(0.1), 5)

    @classmethod
    def dense64(cls):
        """The 64 x 1024 stress shape (LidarModel::dense64)."""
        f = np.float32
        return cls(64, 1024, f(360.0) / f(1024.0), f(45.0) / f(63.0), f(22.5) + f(0.1), 24)


class LinsLidarModels(C.Structure):
    """lins_lidar_models: a table of lidar models and each scan's entry in it (model_of NULL only with one model)."""
    _fields_ = [("n_models", C.c_int32), ("models", C.c_void_p), ("model_of", C.c_void_p)]


class LinsRawDesc(C.Structure):
    """lins_raw_desc: n raw sweeps, CSR."""
    _fields_ = [("n_scans", C.c_int32), ("cloud", C.c_void_p), ("cloud_off", C.c_void_p), ("point_format", C.c_int32)]


class LinsSeqRawDesc(C.Structure):
    """lins_seq_raw_desc: one raw sweep per sequence."""
    _fields_ = [("n_seq", C.c_int32), ("present", C.c_void_p), ("imu", C.c_void_p), ("imu_off", C.c_void_p), ("raw", LinsRawDesc)]


class LinsCloud2Layout(C.Structure):
    """lins_cloud2_layout: what fromROSMsg<PointXYZI> reads of one sensor_msgs/PointCloud2 (x, y, z, intensity in
    offset / datatype order; intensity datatype 0 = absent)."""
    _fields_ = [("height", C.c_uint32), ("width", C.c_uint32), ("point_step", C.c_uint32), ("row_step", C.c_uint32),
                ("offset", C.c_uint32 * 4), ("datatype", C.c_uint8 * 4), ("is_bigendian", C.c_uint8), ("pad_", C.c_uint8 * 3)]


class LinsCloud2Desc(C.Structure):
    """lins_cloud2_desc: n messages' data fields, CSR over one byte blob (int64 offsets), one layout each."""
    _fields_ = [("n_scans", C.c_int32), ("data", C.c_void_p), ("data_off", C.c_void_p), ("layouts", C.c_void_p)]


class LinsSeqCloud2Desc(C.Structure):
    """lins_seq_cloud2_desc: one PointCloud2 message per sequence."""
    _fields_ = [("n_seq", C.c_int32), ("present", C.c_void_p), ("imu", C.c_void_p), ("imu_off", C.c_void_p), ("cloud2", LinsCloud2Desc)]


class LinsSeqStepDesc(C.Structure):
    _fields_ = [
        ("n_seq", C.c_int32),
        ("present", C.c_void_p),
        ("imu", C.c_void_p),
        ("imu_off", C.c_void_p),
        ("surf_flat", C.c_void_p),
        ("surf_flat_off", C.c_void_p),
        ("corner_sharp", C.c_void_p),
        ("corner_sharp_off", C.c_void_p),
        ("surf_less_flat", C.c_void_p),
        ("surf_less_flat_off", C.c_void_p),
        ("corner_less_sharp", C.c_void_p),
        ("corner_less_sharp_off", C.c_void_p),
        ("point_format", C.c_int32),
    ]


SEQ_IDLE, SEQ_SKIPPED, SEQ_RAN, SEQ_ICP = 0, 1, 2, 3  # lins_gpu_seq_download scan_status (LINS_SEQ_*)
SEQ_INIT_WAIT, SEQ_FIRST, SEQ_SECOND = 4, 5, 6        # ... of a slot that initialises (lins_gpu_seq_open runs)
FUSION_INIT, FUSION_FIRST_SCAN, FUSION_RUNNING = 0, 1, 3  # lins_gpu_seq_download_init fusion_status (StateEstimator::status_)


def ptr(a):
    """void* of a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def as_points(a):
    """Return a C-contiguous POINT_DTYPE array view/copy of `a` (n x 8 float32 also accepted)."""
    a = np.asarray(a)
    if a.dtype != POINT_DTYPE:
        a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 8).view(POINT_DTYPE).reshape(-1)
    return np.ascontiguousarray(a)


def make_points(xyz, intensity):
    xyz = np.asarray(xyz, dtype=np.float32).reshape(-1, 3)
    p = np.zeros(len(xyz), dtype=POINT_DTYPE)
    p["x"], p["y"], p["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    p["pad0"] = 1.0
    p["intensity"] = np.asarray(intensity, dtype=np.float32)
    return p


class Batch:
    """Host-side batch of independent (scan pair, prior) units, CSR layout of lins_batch_desc."""

    FIELDS = ("surf_flat", "corner_sharp", "surf_less_flat", "corner_less_sharp")

    def __init__(self, clouds, offsets, state, cov, truth=None, extra=None):
        self.clouds = {k: as_points(clouds[k]) for k in self.FIELDS}
        self.offsets = {k: np.ascontiguousarray(offsets[k], dtype=np.int32) for k in self.FIELDS}
        self.state = np.ascontiguousarray(state, dtype=np.float64).reshape(-1, STATE_DIM)
        self.cov = np.ascontiguousarray(cov, dtype=np.float64).reshape(-1, COV_SIZE)
        self.truth = None if truth is None else np.ascontiguousarray(truth, dtype=np.float64).reshape(-1, 7)
        self.extra = extra or {}
        self.n = len(self.state)
        for k in self.FIELDS:
            assert len(self.offsets[k]) == self.n + 1 and self.offsets[k][-1] == len(self.clouds[k])

    def desc(self):
        d = LinsBatchDesc()
        d.n_scans = self.n
        for k in self.FIELDS:
            setattr(d, k, self.clouds[k].ctypes.data)
            setattr(d, k + "_off", self.offsets[k].ctypes.data)
        d.state_in = self.state.ctypes.data
        d.cov_in = self.cov.ctypes.data
        return d

    def packed16(self):
        """The same batch with its clouds as packed (x, y, z, intensity) float32 records (lins_batch_desc.point_format = 1)."""
        return PackedBatch(self)

    def unit(self, i):
        """The four clouds + prior of unit i."""
        out = {}
        for k in self.FIELDS:
            o = self.offsets[k]
            out[k] = self.clouds[k][o[i] : o[i + 1]]
        out["state"] = self.state[i]
        out["cov"] = self.cov[i]
        return out

    def subset(self, idx):
        idx = list(idx)
        clouds, offsets = {}, {}
        for k in self.FIELDS:
            o = self.offsets[k]
            parts = [self.clouds[k][o[i] : o[i + 1]] for i in idx]
            clouds[k] = np.concatenate(parts) if parts else np.zeros(0, POINT_DTYPE)
            offsets[k] = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
        return Batch(clouds, offsets, self.state[idx], self.cov[idx], None if self.truth is None else self.truth[idx])

    def tile(self, reps):
        """The same units repeated `reps` times (used to push the working set past L2)."""
        clouds, offsets = {}, {}
        for k in self.FIELDS:
            clouds[k] = np.tile(self.clouds[k], reps)
            sizes = np.diff(self.offsets[k])
            offsets[k] = np.concatenate([[0], np.cumsum(np.tile(sizes, reps))]).astype(np.int32)
        return Batch(clouds, offsets, np.tile(self.state, (reps, 1)), np.tile(self.cov, (reps, 1)),
                     None if self.truth is None else np.tile(self.truth, (reps, 1)))

    def save(self, path):
        arrs = {}
        for k in self.FIELDS:
            arrs[k] = self.clouds[k].view(np.float32).reshape(-1, 8)[:, [0, 1, 2, 4]]
            arrs[k + "_off"] = self.offsets[k]
        arrs["state"], arrs["cov"] = self.state, self.cov
        if self.truth is not None:
            arrs["truth"] = self.truth
        np.savez_compressed(path, **arrs)

    @classmethod
    def load(cls, path):
        z = np.load(path)
        clouds = {k: make_points(z[k][:, :3], z[k][:, 3]) for k in cls.FIELDS}
        offsets = {k: z[k + "_off"] for k in cls.FIELDS}
        return cls(clouds, offsets, z["state"], z["cov"], z["truth"] if "truth" in z.files else None)


class PackedBatch:
    """A Batch whose clouds are stored as 16-byte (x, y, z, intensity) records: LINS_POINTS_PACKED16."""

    FIELDS = Batch.FIELDS

    def __init__(self, batch):
        self.n, self.offsets, self.state, self.cov = batch.n, batch.offsets, batch.state, batch.cov
        self.clouds = {}
        for k in self.FIELDS:
            c = batch.clouds[k]
            self.clouds[k] = np.ascontiguousarray(np.stack([c["x"], c["y"], c["z"], c["intensity"]], 1).astype(np.float32)) if len(c) else np.zeros((0, 4), np.float32)

    def desc(self):
        d = LinsBatchDesc()
        d.n_scans = self.n
        for k in self.FIELDS:
            setattr(d, k, self.clouds[k].ctypes.data)
            setattr(d, k + "_off", self.offsets[k].ctypes.data)
        d.state_in = self.state.ctypes.data
        d.cov_in = self.cov.ctypes.data
        d.point_format = 1
        return d
