"""ctypes binding of the C-ABI shared library (include/lins_gpu.h) — the call a Python user makes.

`LinsGpu` mirrors the seam of the reference's ``fusion::StateEstimator`` that the GPU path replaces
(lins/include/StateEstimator.hpp): ``set_map`` ≙ kdtree*->setInputCloud (:363-364, :1156-1160),
``ieskf`` ≙ performIESKF (:465-600), ``associate`` ≙ findCorrespondingSurf/CornerFeatures (:829-1063),
``ieskf_batch`` ≙ performIESKF over many independent (scan pair, prior) units.

There is NO CPU fallback: if the library is missing or no sm_90 device is present this raises.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .ctypes_defs import (Batch, COV_SIZE, LinsBatchDesc, LinsCloud2Desc, LinsCloud2Layout, LinsFeatureParams, LinsLidarModel, LinsLidarModels, LinsFusedPose, LinsGlobalMapReport, LinsLoopReport, LinsMapperDesc, LinsMapperReport, LinsMappersDesc, LinsMapReport, LinsParams, LinsPclDesc,
                          LinsRawDesc, LinsReport, LinsScanResult, LinsSeqBeginDesc, LinsSeqInitParams, LinsSeqParams, LinsSeqPclDesc,
                          LinsSeqCloud2Desc, LinsSeqMapDesc, LinsSeqRawDesc, LinsSeqStepDesc, LinsSlotConfig, LinsSlotTuning, POINT_DTYPE, SCAN_RESULT_DTYPE, STATE_DIM, as_points, make_points, ptr)

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
LIB_PATH = os.path.join(_PKG, "liblins_gpu.so")
CUDA_DIR = os.path.join(_PKG, "csrc", "cuda")

# every symbol include/lins_gpu.h declares
EXPORTS = [
    "lins_gpu_abi_version", "lins_gpu_create", "lins_gpu_destroy", "lins_gpu_last_error", "lins_gpu_set_params",
    "lins_gpu_set_map", "lins_gpu_ieskf", "lins_gpu_associate", "lins_gpu_estimate_transform", "lins_gpu_update_map",
    "lins_gpu_batch_upload", "lins_gpu_batch_run", "lins_gpu_batch_download", "lins_gpu_ieskf_batch",
    "lins_gpu_batch_results_device", "lins_gpu_batch_jacobian_pass", "lins_gpu_launch_count", "lins_gpu_sync",
    "lins_gpu_debug_phase_cycles", "lins_gpu_map_set", "lins_gpu_scan2map", "lins_gpu_map_associate",
    "lins_gpu_host_register", "lins_gpu_host_unregister", "lins_gpu_batch_download_indices", "lins_gpu_update_map_ex",
    "lins_gpu_batch_upload_stats", "lins_gpu_seq_begin", "lins_gpu_seq_step", "lins_gpu_seq_download",
    "lins_gpu_seq_phase_ms", "lins_gpu_seq_download_ieskf", "lins_gpu_seq_download_maps", "lins_gpu_download_indices",
    "lins_gpu_seq_open", "lins_gpu_seq_restart", "lins_gpu_seq_step_ex", "lins_gpu_seq_download_init",
    "lins_gpu_extract_features", "lins_gpu_extract_ms", "lins_gpu_seq_step_pcl", "lins_gpu_project_scans", "lins_gpu_project_ms",
    "lins_gpu_seq_step_raw", "lins_gpu_decode_cloud2", "lins_gpu_decode_ms", "lins_gpu_seq_step_cloud2",
    "lins_gpu_project_scans_mixed", "lins_gpu_seq_step_raw_mixed", "lins_gpu_seq_step_cloud2_mixed",
    "lins_gpu_mapper_reset", "lins_gpu_mapper_imu", "lins_gpu_mapper_step", "lins_gpu_mapper_download", "lins_gpu_voxel_grid",
    "lins_gpu_mappers_open", "lins_gpu_mappers_reset", "lins_gpu_mappers_imu", "lins_gpu_mappers_step", "lins_gpu_mappers_download",
    "lins_gpu_seq_map_open", "lins_gpu_seq_map_step", "lins_gpu_seq_map_published", "lins_gpu_seq_configure", "lins_gpu_seq_tune",
    "lins_gpu_seq_save_size", "lins_gpu_seq_save", "lins_gpu_seq_load", "lins_gpu_mapper_fuse", "lins_gpu_mappers_fuse",
    "lins_gpu_seq_map_fused", "lins_gpu_mappers_loops", "lins_gpu_mappers_close_loops", "lins_gpu_mapper_loops",
    "lins_gpu_mapper_close_loop", "lins_gpu_mappers_global_map", "lins_gpu_mappers_global_map_download",
    "lins_gpu_mapper_global_map", "lins_gpu_mapper_global_map_download", "lins_gpu_mappers_save_size", "lins_gpu_mappers_save",
    "lins_gpu_mappers_load", "lins_gpu_mapper_save_size", "lins_gpu_mapper_save", "lins_gpu_mapper_load", "lins_gpu_mappers_load_phase_ms",
    "lins_gpu_mappers_store_bytes", "lins_gpu_mapper_store_bytes",
]

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper)
NVCC_COMMON = NVCC_ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]
# translation units and their extra flags: lins_gpu.cu (the fused kernel and most of the C-ABI), lins_upload.cu (batch
# upload), lins_map.cu (row F2's host side), lins_seq.cu (sequence mode), lins_features.cu (feature extraction),
# lins_projection.cu (image projection), lins_cloud2.cu (PointCloud2 decoding), lins_mapper.cu (the mapping node's cycle), lins_mappers.cu (many mapping nodes in lockstep), lins_loops.cu (their loop closure), lins_checkpoint.cu (saving and loading sequence-mode slots and mapping nodes) — all bit-exact, so no multiply-add contraction: the association and the map
# fits depend on it — and lins_jacobian.cu (the tolerance-checked split Jacobian kernel: contraction allowed)
UNITS = [("lins_gpu.cu", ["-fmad=false"]), ("lins_upload.cu", ["-fmad=false"]), ("lins_map.cu", ["-fmad=false"]),
         ("lins_seq.cu", ["-fmad=false"]), ("lins_features.cu", ["-fmad=false"]), ("lins_projection.cu", ["-fmad=false"]),
         ("lins_cloud2.cu", ["-fmad=false"]), ("lins_mapper.cu", ["-fmad=false"]), ("lins_mappers.cu", ["-fmad=false"]),
         ("lins_loops.cu", ["-fmad=false"]), ("lins_checkpoint.cu", ["-fmad=false"]), ("lins_jacobian.cu", [])]


def build(force=False, verbose=False):
    """Compile csrc/cuda/*.cu -> liblins_gpu.so for sm_90a (nvcc cross-compiles without a GPU)."""
    # (this file too: a library built with other flags, e.g. for another architecture, is stale)
    deps = [os.path.join(CUDA_DIR, u) for u, _ in UNITS] + [os.path.join(_ROOT, "include", "lins_gpu.h"), os.path.abspath(__file__)]
    for d in (CUDA_DIR, os.path.join(os.path.dirname(CUDA_DIR), "host")):  # every header the translation units include
        deps += [os.path.join(d, f) for f in sorted(os.listdir(d)) if f.endswith((".cuh", ".hpp", ".h"))]
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(s) for s in deps):
        return LIB_PATH
    objdir = os.path.join(_PKG, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    for unit, flags in UNITS:
        obj = os.path.join(objdir, os.path.splitext(unit)[0] + ".o")
        subprocess.check_call(["nvcc"] + NVCC_COMMON + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, os.path.join(CUDA_DIR, unit)])
        objs.append(obj)
    subprocess.check_call(["nvcc"] + NVCC_ARCH + ["-shared", "-o", LIB_PATH] + objs)
    return LIB_PATH


_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: run __graft_entry__.build() (there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        vp, i32p, f32p, u8p, f64p = C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
        L.lins_gpu_create.argtypes = [C.POINTER(LinsParams), C.c_int, vp, C.POINTER(vp)]
        L.lins_gpu_destroy.argtypes = [vp]
        L.lins_gpu_destroy.restype = None
        L.lins_gpu_last_error.argtypes = [vp]
        L.lins_gpu_last_error.restype = C.c_char_p
        L.lins_gpu_set_params.argtypes = [vp, C.POINTER(LinsParams)]
        L.lins_gpu_set_map.argtypes = [vp, vp, C.c_int, vp, C.c_int]
        L.lins_gpu_ieskf.argtypes = [vp, vp, C.c_int, vp, C.c_int, f64p, f64p, f64p, f64p, C.POINTER(LinsReport)]
        L.lins_gpu_associate.argtypes = [vp, vp, C.c_int, vp, C.c_int, f64p, C.c_int, i32p, i32p, f32p, f32p, u8p, u8p, f32p, f32p]
        L.lins_gpu_estimate_transform.argtypes = [vp, vp, C.c_int, vp, C.c_int, f64p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.lins_gpu_update_map.argtypes = [vp, vp, C.c_int, vp, C.c_int, f64p, C.POINTER(C.c_int)]
        L.lins_gpu_update_map_ex.argtypes = [vp, vp, C.c_int, vp, C.c_int, f64p, vp, vp, C.POINTER(C.c_int)]
        L.lins_gpu_batch_upload.argtypes = [vp, C.POINTER(LinsBatchDesc)]
        L.lins_gpu_batch_run.argtypes = [vp]
        L.lins_gpu_batch_download.argtypes = [vp, f64p, f64p, vp, vp]
        L.lins_gpu_ieskf_batch.argtypes = [vp, C.POINTER(LinsBatchDesc), f64p, f64p, vp]
        L.lins_gpu_batch_results_device.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_int)]
        L.lins_gpu_batch_jacobian_pass.argtypes = [vp, f64p]
        L.lins_gpu_launch_count.argtypes = [vp]
        L.lins_gpu_launch_count.restype = C.c_int64
        L.lins_gpu_sync.argtypes = [vp]
        L.lins_gpu_debug_phase_cycles.argtypes = [vp, C.c_int, vp]
        L.lins_gpu_map_set.argtypes = [vp, vp, C.c_int, vp, C.c_int]
        L.lins_gpu_scan2map.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp, C.POINTER(LinsMapReport)]
        L.lins_gpu_map_associate.argtypes = [vp, vp, C.c_int, vp, C.c_int, vp] + [vp] * 6
        L.lins_gpu_host_register.argtypes = [vp, C.c_size_t]
        L.lins_gpu_batch_download_indices.argtypes = [vp, vp, vp]
        L.lins_gpu_batch_upload_stats.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.lins_gpu_host_unregister.argtypes = [vp]
        L.lins_gpu_seq_begin.argtypes = [vp, C.POINTER(LinsSeqParams), C.POINTER(LinsSeqBeginDesc)]
        L.lins_gpu_seq_step.argtypes = [vp, C.POINTER(LinsSeqStepDesc)]
        L.lins_gpu_seq_download.argtypes = [vp, f64p, f64p, f64p, vp, vp, vp]
        L.lins_gpu_seq_phase_ms.argtypes = [vp, vp]
        L.lins_gpu_seq_download_ieskf.argtypes = [vp] + [vp] * 7
        L.lins_gpu_seq_download_maps.argtypes = [vp] + [vp] * 6
        L.lins_gpu_download_indices.argtypes = [vp, vp, vp]
        L.lins_gpu_seq_open.argtypes = [vp, C.POINTER(LinsSeqParams), C.POINTER(LinsSeqInitParams), C.c_int32]
        L.lins_gpu_seq_restart.argtypes = [vp, vp]
        L.lins_gpu_seq_configure.argtypes = [vp, vp, vp]
        L.lins_gpu_seq_tune.argtypes = [vp, vp, vp]
        L.lins_gpu_seq_step_ex.argtypes = [vp, C.POINTER(LinsSeqStepDesc), vp]
        L.lins_gpu_seq_download_init.argtypes = [vp, vp, vp, vp, vp]
        L.lins_gpu_extract_features.argtypes = [vp, C.POINTER(LinsFeatureParams), C.POINTER(LinsPclDesc)] + [vp] * 6
        L.lins_gpu_extract_ms.argtypes = [vp, vp]
        L.lins_gpu_seq_step_pcl.argtypes = [vp, C.POINTER(LinsSeqPclDesc), C.POINTER(LinsFeatureParams), vp]
        L.lins_gpu_project_scans.argtypes = [vp, C.POINTER(LinsLidarModel), C.POINTER(LinsRawDesc)] + [vp] * 9
        L.lins_gpu_project_ms.argtypes = [vp, vp]
        L.lins_gpu_seq_step_raw.argtypes = [vp, C.POINTER(LinsSeqRawDesc), C.POINTER(LinsLidarModel), C.POINTER(LinsFeatureParams), vp]
        L.lins_gpu_decode_cloud2.argtypes = [vp, C.POINTER(LinsCloud2Desc), vp, vp]
        L.lins_gpu_decode_ms.argtypes = [vp, vp]
        L.lins_gpu_seq_step_cloud2.argtypes = [vp, C.POINTER(LinsSeqCloud2Desc), C.POINTER(LinsLidarModel), C.POINTER(LinsFeatureParams), vp]
        L.lins_gpu_project_scans_mixed.argtypes = [vp, C.POINTER(LinsLidarModels), C.POINTER(LinsRawDesc)] + [vp] * 9
        L.lins_gpu_seq_step_raw_mixed.argtypes = [vp, C.POINTER(LinsSeqRawDesc), C.POINTER(LinsLidarModels), C.POINTER(LinsFeatureParams), vp]
        L.lins_gpu_seq_step_cloud2_mixed.argtypes = [vp, C.POINTER(LinsSeqCloud2Desc), C.POINTER(LinsLidarModels), C.POINTER(LinsFeatureParams), vp]
        L.lins_gpu_mapper_reset.argtypes = [vp]
        L.lins_gpu_mapper_imu.argtypes = [vp, vp, vp, vp, C.c_int]
        L.lins_gpu_mapper_step.argtypes = [vp, C.POINTER(LinsMapperDesc), C.POINTER(LinsMapperReport)]
        L.lins_gpu_mapper_download.argtypes = [vp] + [vp] * 8
        L.lins_gpu_voxel_grid.argtypes = [vp, vp, C.c_int, C.c_float, vp, C.POINTER(C.c_int)]
        L.lins_gpu_mappers_open.argtypes = [vp, C.c_int32]
        L.lins_gpu_mappers_reset.argtypes = [vp, vp]
        L.lins_gpu_mappers_imu.argtypes = [vp, vp, vp, vp, vp]
        L.lins_gpu_mappers_step.argtypes = [vp, C.POINTER(LinsMappersDesc), vp]
        L.lins_gpu_mappers_download.argtypes = [vp, C.c_int32] + [vp] * 8
        L.lins_gpu_seq_map_open.argtypes = [vp]
        L.lins_gpu_seq_map_step.argtypes = [vp, C.POINTER(LinsSeqMapDesc), vp, vp]
        L.lins_gpu_seq_map_published.argtypes = [vp, vp, vp]
        L.lins_gpu_seq_save_size.argtypes = [vp, vp, vp]
        L.lins_gpu_seq_save.argtypes = [vp, vp, vp, vp]
        L.lins_gpu_seq_load.argtypes = [vp, vp, vp, vp]
        L.lins_gpu_mapper_fuse.argtypes = [vp, C.POINTER(LinsMapperDesc), C.POINTER(LinsFusedPose)]
        L.lins_gpu_mappers_fuse.argtypes = [vp, C.POINTER(LinsMappersDesc), vp]
        L.lins_gpu_mappers_loops.argtypes = [vp, vp]
        L.lins_gpu_mappers_close_loops.argtypes = [vp, vp, vp]
        L.lins_gpu_mapper_loops.argtypes = [vp]
        L.lins_gpu_mapper_close_loop.argtypes = [vp, C.POINTER(LinsLoopReport)]
        L.lins_gpu_seq_map_fused.argtypes = [vp, vp]
        L.lins_gpu_mappers_global_map.argtypes = [vp, vp, vp]
        L.lins_gpu_mappers_global_map_download.argtypes = [vp, C.c_int32, vp, vp]
        L.lins_gpu_mapper_global_map.argtypes = [vp, C.POINTER(LinsGlobalMapReport)]
        L.lins_gpu_mapper_global_map_download.argtypes = [vp, vp, vp]
        L.lins_gpu_mappers_save_size.argtypes = [vp, vp, vp]
        L.lins_gpu_mappers_save.argtypes = [vp, vp, vp, vp]
        L.lins_gpu_mappers_load.argtypes = [vp, vp, vp, vp]
        L.lins_gpu_mapper_save_size.argtypes = [vp, C.POINTER(C.c_uint64)]
        L.lins_gpu_mapper_save.argtypes = [vp, vp, C.c_uint64]
        L.lins_gpu_mapper_load.argtypes = [vp, vp, C.c_uint64]
        L.lins_gpu_mappers_load_phase_ms.argtypes = [vp, vp]
        L.lins_gpu_mappers_store_bytes.argtypes = [vp, vp, vp, vp, vp]
        L.lins_gpu_mapper_store_bytes.argtypes = [vp, vp, vp, vp]
        _LIB = L
    return _LIB


class LinsError(RuntimeError):
    pass


def _points_from_xyzi(a):
    """POINT_DTYPE records of an (m x 4) float32 (x, y, z, intensity) array (pad0 = 1, as pcl's PointXYZI)."""
    a = np.asarray(a, np.float32).reshape(-1, 4)
    out = np.zeros(len(a), POINT_DTYPE)
    out["x"], out["y"], out["z"], out["intensity"] = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
    out["pad0"] = 1.0
    return out


def pin_batch(batch):
    """Page-lock the four cloud arrays of a host batch in place (lins_gpu_host_register): lins_gpu_batch_upload then DMAs
    the raw records straight from them.  Returns the list of pinned arrays; call unpin_batch before they are freed."""
    L = lib()
    pinned = []
    for k in Batch.FIELDS:
        a = batch.clouds[k]
        if a.nbytes == 0:
            continue
        rc = L.lins_gpu_host_register(a.ctypes.data, a.nbytes)
        if rc != 0:
            unpin_arrays(pinned)
            raise LinsError(f"lins_gpu_host_register failed with {rc}")
        pinned.append(a)
    batch._pinned = pinned
    return pinned


def unpin_arrays(arrays):
    L = lib()
    for a in arrays:
        L.lins_gpu_host_unregister(a.ctypes.data)


def unpin_batch(batch):
    unpin_arrays(getattr(batch, "_pinned", []))
    batch._pinned = []


def pack_csr(clouds):
    """Per-slot clouds (point arrays, or None for none) -> (one POINT_DTYPE array, int32 offsets of len(clouds) + 1):
    slot s's points are [off[s], off[s + 1])."""
    parts = [as_points(c) if c is not None else np.zeros(0, POINT_DTYPE) for c in clouds]
    off = np.zeros(len(parts) + 1, np.int32)
    off[1:] = np.cumsum([len(p) for p in parts])
    # (joined as plain float32 rows: numpy concatenates structured records far more slowly)
    pts = np.concatenate([p.view(np.float32).reshape(-1, 8) for p in parts]).view(POINT_DTYPE).reshape(-1) if parts else np.zeros(0, POINT_DTYPE)
    return pts, off


def _odometry_arrays(steps):
    """The present flags, stamps, quaternions (M x 4) and positions (M x 3) of lockstep steps[s] = (time, quat_xyzw, pos,
    ...) or None (an absent slot: identity odometry)."""
    M = len(steps)
    present = np.array([st is not None for st in steps], np.uint8)
    time = np.array([float(st[0]) if st is not None else 0.0 for st in steps], np.float64)
    quat = np.array([[float(v) for v in st[1]] if st is not None else [0.0, 0.0, 0.0, 1.0] for st in steps], np.float64).reshape(M, 4)
    pos = np.array([[float(v) for v in st[2]] if st is not None else [0.0] * 3 for st in steps], np.float64).reshape(M, 3)
    return present, time, quat, pos


class LinsGpu:
    """One context = one CUDA device + one stream (pass ``stream=torch.cuda.current_stream().cuda_stream`` to
    share torch's stream so torch.cuda.Event timing sees the kernels)."""

    def __init__(self, params=None, device=0, stream=None):
        self.L = lib()
        self.params = params or LinsParams.shipped()
        h = C.c_void_p()
        rc = self.L.lins_gpu_create(C.byref(self.params), device, C.c_void_p(stream or 0), C.byref(h))
        if rc != 0:
            raise LinsError(f"lins_gpu_create failed with {rc} (no sm_90 CUDA device? there is no CPU fallback)")
        self.h = h
        self._batch_n = 0

    def close(self):
        if getattr(self, "h", None):
            self.L.lins_gpu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise LinsError(f"error {rc}: {self.L.lins_gpu_last_error(self.h).decode()}")

    def set_params(self, params):
        self.params = params
        self._ck(self.L.lins_gpu_set_params(self.h, C.byref(params)))

    def launch_count(self):
        return int(self.L.lins_gpu_launch_count(self.h))

    def sync(self):
        self._ck(self.L.lins_gpu_sync(self.h))

    def phase_cycles(self, enable=True, read=False):
        out = np.zeros(64, np.int64) if read else None
        self._ck(self.L.lins_gpu_debug_phase_cycles(self.h, int(enable), ptr(out)))
        return out

    # ---- single-scan seam ---------------------------------------------------------------------------------
    def set_map(self, surf_less_flat, corner_less_sharp):
        s, c = as_points(surf_less_flat), as_points(corner_less_sharp)
        self._ck(self.L.lins_gpu_set_map(self.h, ptr(s), len(s), ptr(c), len(c)))

    def ieskf(self, surf_flat, corner_sharp, state, cov):
        s, c = as_points(surf_flat), as_points(corner_sharp)
        st = np.ascontiguousarray(state, dtype=np.float64).reshape(STATE_DIM)
        cv = np.ascontiguousarray(cov, dtype=np.float64).reshape(COV_SIZE)
        so, co, rep = np.zeros(STATE_DIM), np.zeros(COV_SIZE), LinsReport()
        self._ck(self.L.lins_gpu_ieskf(self.h, ptr(s), len(s), ptr(c), len(c), ptr(st), ptr(cv), ptr(so), ptr(co), C.byref(rep)))
        return so, co, rep

    def associate(self, surf_flat, corner_sharp, lin_state, it):
        s, c = as_points(surf_flat), as_points(corner_sharp)
        ns, nc = len(s), len(c)
        st = np.ascontiguousarray(lin_state, dtype=np.float64).reshape(STATE_DIM)
        out = dict(
            surf_ind=np.full((ns, 3), -2, np.int32), corner_ind=np.full((nc, 2), -2, np.int32),
            surf_coeff=np.zeros((ns, 4), np.float32), corner_coeff=np.zeros((nc, 4), np.float32),
            surf_mask=np.zeros(ns, np.uint8), corner_mask=np.zeros(nc, np.uint8),
            surf_sel=np.zeros((ns, 3), np.float32), corner_sel=np.zeros((nc, 3), np.float32),
        )
        self._ck(self.L.lins_gpu_associate(self.h, ptr(s), ns, ptr(c), nc, ptr(st), int(it), ptr(out["surf_ind"]),
                                           ptr(out["corner_ind"]), ptr(out["surf_coeff"]), ptr(out["corner_coeff"]),
                                           ptr(out["surf_mask"]), ptr(out["corner_mask"]), ptr(out["surf_sel"]),
                                           ptr(out["corner_sel"])))
        return out

    def download_indices(self, n_surf, n_corner):
        """(surf_ind (n_surf, 3), corner_ind (n_corner, 2)) of the last single-scan call's last search iteration."""
        si, ci = np.full((n_surf, 3), -2, np.int32), np.full((n_corner, 2), -2, np.int32)
        self._ck(self.L.lins_gpu_download_indices(self.h, ptr(si), ptr(ci)))
        return si, ci

    def estimate_transform(self, surf_flat, corner_sharp, t, q_xyzw):
        s, c = as_points(surf_flat), as_points(corner_sharp)
        pose = np.ascontiguousarray(np.concatenate([np.asarray(t, float), np.asarray(q_xyzw, float)]))
        it, cv = C.c_int(0), C.c_int(0)
        self._ck(self.L.lins_gpu_estimate_transform(self.h, ptr(s), len(s), ptr(c), len(c), ptr(pose), C.byref(it), C.byref(cv)))
        return pose[:3].copy(), pose[3:].copy(), it.value, bool(cv.value)

    def update_map(self, surf_less_flat, corner_less_sharp, lin_state):
        """In-place transformToEnd of the two clouds (returned) + conditional map refresh."""
        s, c = as_points(surf_less_flat).copy(), as_points(corner_less_sharp).copy()
        st = np.ascontiguousarray(lin_state, dtype=np.float64).reshape(STATE_DIM)
        rep = C.c_int(0)
        self._ck(self.L.lins_gpu_update_map(self.h, ptr(s), len(s), ptr(c), len(c), ptr(st), C.byref(rep)))
        return s, c, bool(rep.value)

    def update_map_device(self, surf_less_flat, corner_less_sharp, lin_state=None):
        """Map refresh that stays on the device: no read-back, no synchronisation; lin_state None = the posterior of the
        last ieskf() call, still resident."""
        s, c = as_points(surf_less_flat), as_points(corner_less_sharp)
        st = None if lin_state is None else np.ascontiguousarray(lin_state, dtype=np.float64).reshape(STATE_DIM)
        rep = C.c_int(0)
        self._ck(self.L.lins_gpu_update_map_ex(self.h, ptr(s), len(s), ptr(c), len(c), ptr(st), None, None, C.byref(rep)))
        return bool(rep.value)

    # ---- row F2: scan-to-map refinement of the mapping node ---------------------------------------------------------
    def map_set(self, corner_from_map, surf_from_map):
        c, s = as_points(corner_from_map), as_points(surf_from_map)
        self._ck(self.L.lins_gpu_map_set(self.h, ptr(c), len(c), ptr(s), len(s)))

    def scan2map(self, corner_last, surf_last, transform):
        """≙ the iteration loop of scan2MapOptimization; returns (transformTobeMapped, LinsMapReport)."""
        c, s = as_points(corner_last), as_points(surf_last)
        t = np.array(transform, np.float32).copy()
        rep = LinsMapReport()
        self._ck(self.L.lins_gpu_scan2map(self.h, ptr(c), len(c), ptr(s), len(s), ptr(t), C.byref(rep)))
        return t, rep

    def map_associate(self, corner_last, surf_last, transform):
        c, s = as_points(corner_last), as_points(surf_last)
        t = np.ascontiguousarray(transform, np.float32)
        out = dict(corner_knn=np.zeros((len(c), 5), np.int32), surf_knn=np.zeros((len(s), 5), np.int32),
                   corner_coeff=np.zeros((len(c), 4), np.float32), surf_coeff=np.zeros((len(s), 4), np.float32),
                   corner_mask=np.zeros(len(c), np.uint8), surf_mask=np.zeros(len(s), np.uint8))
        self._ck(self.L.lins_gpu_map_associate(self.h, ptr(c), len(c), ptr(s), len(s), ptr(t), ptr(out["corner_knn"]), ptr(out["surf_knn"]),
                                               ptr(out["corner_coeff"]), ptr(out["surf_coeff"]), ptr(out["corner_mask"]), ptr(out["surf_mask"])))
        return out

    # ---- the mapping node's cycle (lins_gpu_mapper_*) ---------------------------------------------------------------
    def mapper_reset(self):
        self._ck(self.L.lins_gpu_mapper_reset(self.h))

    def mapper_imu(self, time, roll, pitch):
        """imuHandler for each (stamp, roll, pitch) (the roll / pitch getRPY gave for the message's orientation)."""
        t, r, p = (np.ascontiguousarray(np.atleast_1d(a), np.float64) for a in (time, roll, pitch))
        self._ck(self.L.lins_gpu_mapper_imu(self.h, ptr(t), ptr(r), ptr(p), len(t)))

    def mapper_step(self, time, quat_xyzw, pos, corner, surf, outlier):
        """One mapping cycle from the odometry message (stamp, orientation, position) and the three YZX clouds;
        returns the LinsMapperReport."""
        c, s, o = as_points(corner), as_points(surf), as_points(outlier)
        d = LinsMapperDesc(time=float(time), quat=(C.c_double * 4)(*[float(v) for v in quat_xyzw]),
                           pos=(C.c_double * 3)(*[float(v) for v in pos]), corner=ptr(c), surf=ptr(s), outlier=ptr(o),
                           n_corner=len(c), n_surf=len(s), n_outlier=len(o))
        rep = LinsMapperReport()
        self._ck(self.L.lins_gpu_mapper_step(self.h, C.byref(d), C.byref(rep)))
        return rep

    def mapper_fuse(self, time, quat_xyzw, pos):
        """transform_fusion_node's pose (LinsFusedPose) for this odometry message against the mapper's state now: call it
        before the mapper_step of the same message."""
        d = LinsMapperDesc(time=float(time), quat=(C.c_double * 4)(*[float(v) for v in quat_xyzw]), pos=(C.c_double * 3)(*[float(v) for v in pos]))
        out = LinsFusedPose()
        self._ck(self.L.lins_gpu_mapper_fuse(self.h, C.byref(d), C.byref(out)))
        return out

    def mapper_download(self, rep):
        """Key poses (n x 7: x, y, z, roll, pitch, yaw, time), the window's ids, and the last processed cycle's clouds
        ((n, 4) float32: map_corner_ds, map_surf_ds, corner_ds, surf_ds, outlier_ds, surf_total_ds) whose sizes `rep`,
        that cycle's report, gives."""
        return self._download_node(lambda *out: self.L.lins_gpu_mapper_download(self.h, *out), rep)

    def _download_node(self, call, rep):
        """A mapping node's download through call(key_poses, window, six clouds), sized by its last cycle's report."""
        poses = np.zeros((rep.n_keyframes, 7))
        window = np.zeros(rep.window_len, np.int32)
        names = ("map_corner_ds", "map_surf_ds", "corner_ds", "surf_ds", "outlier_ds", "surf_total_ds")
        sizes = (rep.n_map_corner_ds, rep.n_map_surf_ds, rep.n_corner_ds, rep.n_surf_ds, rep.n_outlier_ds, rep.n_surf_total_ds)
        clouds = {k: np.zeros((n, 4), np.float32) for k, n in zip(names, sizes)}
        self._ck(call(ptr(poses), ptr(window), *[ptr(clouds[k]) for k in names]))
        return poses, window, clouds

    def voxel_grid(self, cloud, leaf):
        """pcl::VoxelGrid<PointXYZI> on the device: (n_voxels, 4) float32 (x, y, z, intensity) centroids."""
        p = as_points(cloud)
        out = np.zeros((max(len(p), 1), 4), np.float32)
        n = C.c_int(0)
        self._ck(self.L.lins_gpu_voxel_grid(self.h, ptr(p), len(p), float(leaf), ptr(out), C.byref(n)))
        return out[:n.value].copy()

    # ---- many mapping nodes in lockstep (lins_gpu_mappers_*) ------------------------------------------------------
    def mappers_open(self, n_slots):
        self._ck(self.L.lins_gpu_mappers_open(self.h, int(n_slots)))
        self._mappers_n = int(n_slots)

    def mappers_reset(self, mask):
        m = np.ascontiguousarray(mask, np.uint8).reshape(-1)
        assert len(m) == self._mappers_n
        self._ck(self.L.lins_gpu_mappers_reset(self.h, ptr(m)))

    def mappers_imu(self, rows):
        """imuHandler per slot: rows[s] = (times, rolls, pitches) of slot s (None or empty: no message)."""
        per = [[np.atleast_1d(np.asarray(a, np.float64)) for a in (r if r is not None else ((), (), ()))] for r in rows]
        off = np.zeros(len(per) + 1, np.int32)
        off[1:] = np.cumsum([len(t) for t, _, _ in per])
        t, r, p = (np.ascontiguousarray(np.concatenate([x[k] for x in per]) if per else np.zeros(0)) for k in range(3))
        self._ck(self.L.lins_gpu_mappers_imu(self.h, ptr(off), ptr(t), ptr(r), ptr(p)))

    def mappers_step(self, steps):
        """One lockstep step: steps[s] = (time, quat_xyzw, pos, corner, surf, outlier) of slot s, or None for an absent
        slot.  Returns the list of LinsMapperReport (None for absent slots)."""
        M = len(steps)
        present, time, quat, pos = _odometry_arrays(steps)
        clouds = [pack_csr([st[3 + k] if st is not None else None for st in steps]) for k in range(3)]
        d = LinsMappersDesc(n_slots=M, present=ptr(present), time=ptr(time), quat=ptr(quat), pos=ptr(pos),
                            corner=ptr(clouds[0][0]), corner_off=ptr(clouds[0][1]), surf=ptr(clouds[1][0]), surf_off=ptr(clouds[1][1]),
                            outlier=ptr(clouds[2][0]), outlier_off=ptr(clouds[2][1]))
        reps = (LinsMapperReport * M)()
        self._ck(self.L.lins_gpu_mappers_step(self.h, C.byref(d), C.cast(reps, C.c_void_p)))
        return [reps[s] if present[s] else None for s in range(M)]

    def mappers_fuse(self, steps):
        """mapper_fuse for every slot of a lockstep step: steps[s] = (time, quat_xyzw, pos, ...) of slot s, or None for an
        absent slot.  Returns the list of LinsFusedPose (None for absent slots)."""
        M = len(steps)
        present, time, quat, pos = _odometry_arrays(steps)
        d = LinsMappersDesc(n_slots=M, present=ptr(present), time=ptr(time), quat=ptr(quat), pos=ptr(pos))
        out = (LinsFusedPose * M)()
        self._ck(self.L.lins_gpu_mappers_fuse(self.h, C.byref(d), C.cast(out, C.c_void_p)))
        return [out[s] if present[s] else None for s in range(M)]

    def mappers_download(self, slot, rep):
        """mapper_download of one slot: (key poses, window, clouds) with the sizes its last processed cycle's report gives."""
        return self._download_node(lambda *out: self.L.lins_gpu_mappers_download(self.h, int(slot), *out), rep)

    # ---- loop closure of the mapping nodes (lins_gpu_mapper(s)_loops / close_loop(s)) ----------------------------
    def mapper_loops(self):
        """Enable loop closure on the single mapper (fresh: before its first step)."""
        self._ck(self.L.lins_gpu_mapper_loops(self.h))

    def mapper_close_loop(self):
        """One performLoopClosure of the single mapper: its LinsLoopReport."""
        rep = LinsLoopReport()
        self._ck(self.L.lins_gpu_mapper_close_loop(self.h, C.byref(rep)))
        return rep

    def mappers_loops(self, mask):
        """Enable loop closure on the masked lockstep slots (each fresh)."""
        m = np.ascontiguousarray(mask, np.uint8).reshape(-1)
        assert len(m) == self._mappers_n
        self._ck(self.L.lins_gpu_mappers_loops(self.h, ptr(m)))

    def mappers_close_loops(self, mask):
        """performLoopClosure of every masked (enabled) slot in one device pass: a LinsLoopReport per masked slot, None
        elsewhere."""
        m = np.ascontiguousarray(mask, np.uint8).reshape(-1)
        assert len(m) == self._mappers_n
        reps = (LinsLoopReport * len(m))()
        self._ck(self.L.lins_gpu_mappers_close_loops(self.h, ptr(m), C.cast(reps, C.c_void_p)))
        return [reps[s] if m[s] else None for s in range(len(m))]

    # ---- the key-frame stores' bytes (lins_gpu_mapper(s)_store_bytes) -------------------------------------------------
    def mappers_store_bytes(self, mask=None):
        """The masked lockstep slots' key-frame store bytes: (device (M,) uint64, host (M,) uint64, host_reserved int).
        device: 16 x the points of a slot's device store; host: 16 x the points of its host store (0 on a plain slot);
        host_reserved: the run's pinned slabs and large blocks.  Unmasked entries are 0.  Host bookkeeping only."""
        m = self._mapper_mask(np.ones(getattr(self, "_mappers_n", 0), np.uint8) if mask is None else mask)
        dev, host, res = np.zeros(len(m), np.uint64), np.zeros(len(m), np.uint64), np.zeros(1, np.uint64)
        self._ck(self.L.lins_gpu_mappers_store_bytes(self.h, ptr(m), ptr(dev), ptr(host), ptr(res)))
        return dev, host, int(res[0])

    def mapper_store_bytes(self):
        """The single mapper's key-frame store bytes: (device, host, host_reserved) as mappers_store_bytes gives them."""
        out = np.zeros(3, np.uint64)
        self._ck(self.L.lins_gpu_mapper_store_bytes(self.h, ptr(out[0:1]), ptr(out[1:2]), ptr(out[2:3])))
        return int(out[0]), int(out[1]), int(out[2])

    # ---- the global map of the mapping nodes (lins_gpu_mapper(s)_global_map(_download)) ---------------------------
    def mapper_global_map(self):
        """publishGlobalMap of the single mapper (loop closure enabled): its LinsGlobalMapReport."""
        rep = LinsGlobalMapReport()
        self._ck(self.L.lins_gpu_mapper_global_map(self.h, C.byref(rep)))
        return rep

    def mapper_global_map_download(self, rep):
        """(key ids (n_key_frames int32), cloud (n_map, 4) float32 x y z intensity) of the single mapper's last global map,
        with the sizes its report `rep` gives."""
        keys, cloud = np.zeros(rep.n_key_frames, np.int32), np.zeros((rep.n_map, 4), np.float32)
        self._ck(self.L.lins_gpu_mapper_global_map_download(self.h, ptr(keys), ptr(cloud)))
        return keys, cloud

    def mappers_global_map(self, mask):
        """publishGlobalMap of every masked (enabled) lockstep slot: a LinsGlobalMapReport per masked slot, None elsewhere."""
        m = np.ascontiguousarray(mask, np.uint8).reshape(-1)
        assert len(m) == self._mappers_n
        reps = (LinsGlobalMapReport * len(m))()
        self._ck(self.L.lins_gpu_mappers_global_map(self.h, ptr(m), C.cast(reps, C.c_void_p)))
        return [reps[s] if m[s] else None for s in range(len(m))]

    def mappers_global_map_download(self, slot, rep):
        """mapper_global_map_download of one lockstep slot."""
        keys, cloud = np.zeros(rep.n_key_frames, np.int32), np.zeros((rep.n_map, 4), np.float32)
        self._ck(self.L.lins_gpu_mappers_global_map_download(self.h, int(slot), ptr(keys), ptr(cloud)))
        return keys, cloud

    # ---- saving and loading mapping nodes (lins_gpu_mapper(s)_save / _load) ------------------------------------------
    def mappers_save(self, mask):
        """Save the lockstep slots with mask[s] != 0: a list of M entries, each slot's blob (bytes, self-contained: it loads
        into a fresh lockstep slot or a fresh single mapper of any context of this library build) or None where the mask
        is 0.  The run is unchanged."""
        return self._save_blobs(self.L.lins_gpu_mappers_save_size, self.L.lins_gpu_mappers_save, self._mapper_mask(mask))

    def mappers_load(self, mask, blobs):
        """Load blobs[s] (bytes, as mappers_save or mapper_save returned it) into every lockstep slot with mask[s] != 0,
        each still fresh (no step since open / its last reset); blobs has M entries (None where the mask is 0).  All or
        nothing."""
        self._load_blobs(self.L.lins_gpu_mappers_load, self._mapper_mask(mask), blobs)

    def mapper_save(self):
        """The single mapper's blob (bytes)."""
        n = C.c_uint64(0)
        self._ck(self.L.lins_gpu_mapper_save_size(self.h, C.byref(n)))
        buf = np.zeros(max(n.value, 1), np.uint8)
        self._ck(self.L.lins_gpu_mapper_save(self.h, ptr(buf), n.value))
        return buf[:n.value].tobytes()

    def mapper_load(self, blob):
        """Load a blob (as mapper_save or mappers_save returned it) into the single mapper, still fresh."""
        buf = np.frombuffer(bytes(blob) or b"\0", np.uint8)
        self._ck(self.L.lins_gpu_mapper_load(self.h, ptr(buf), len(bytes(blob))))

    def mappers_load_phase_ms(self):
        """The last mapper load's host phases in ms: (validation, allocation, staging, device, bookkeeping)."""
        out = np.zeros(5)
        self._ck(self.L.lins_gpu_mappers_load_phase_ms(self.h, ptr(out)))
        return out

    def _mapper_mask(self, mask):
        m = np.ascontiguousarray(mask, dtype=np.uint8).reshape(-1)
        if len(m) != getattr(self, "_mappers_n", -1):
            raise ValueError(f"mask has {len(m)} entries, the run {getattr(self, '_mappers_n', 0)}")
        return m

    # ---- sequence mode feeding its mapping nodes (lins_gpu_seq_map_*) ---------------------------------------------
    def seq_map_open(self):
        """Bind the open sequence run (seq_open, before its first step) to S fresh lockstep mapper slots: slot s feeds
        mapper slot s."""
        self._ck(self.L.lins_gpu_seq_map_open(self.h))
        self._mappers_n = self._seq_n

    def seq_map_step(self, time, outlier=None):
        """publishTopics after the last sequence step and the published slots' mapping cycles.  time: S scan stamps;
        outlier: after a seq_step / seq_step_pcl step, the S outlier clouds its scans came with (None after seq_step_raw /
        seq_step_cloud2).  Returns (reports: a LinsMapperReport per published slot, None elsewhere; published: S uint8)."""
        n = self._seq_n
        t = np.ascontiguousarray(time, np.float64).reshape(-1)
        if len(t) != n:
            raise ValueError(f"time has {len(t)} entries, the run {n}")
        d = LinsSeqMapDesc(n_seq=n, time=ptr(t))
        if outlier is not None:
            pts, off = pack_csr(outlier)
            d.outlier, d.outlier_off = ptr(pts), ptr(off)
        reps = (LinsMapperReport * n)()
        published = np.zeros(n, np.uint8)
        self._ck(self.L.lins_gpu_seq_map_step(self.h, C.byref(d), C.cast(reps, C.c_void_p), ptr(published)))
        return [reps[s] if published[s] else None for s in range(n)], published

    def seq_map_published(self):
        """What each slot publishes, as the last seq_map_step fed a published slot's mapper: (pose (S, 7): globalStateYZX_,
        position + quaternion x y z w; sizes (S, 3): points of the less-sharp, less-flat and outlier YZX clouds)."""
        pose, sizes = np.zeros((self._seq_n, 7)), np.zeros((self._seq_n, 3), np.int32)
        self._ck(self.L.lins_gpu_seq_map_published(self.h, ptr(pose), ptr(sizes)))
        return pose, sizes

    def seq_map_fused(self):
        """Each slot's LinsFusedPose of the last seq_map_step (valid = 0: the slot did not publish)."""
        out = (LinsFusedPose * self._seq_n)()
        self._ck(self.L.lins_gpu_seq_map_fused(self.h, C.cast(out, C.c_void_p)))
        return list(out)

    # ---- batched mode ------------------------------------------------------------------------------------------
    def batch_upload(self, batch):
        d = batch.desc()
        self._keep = batch  # keep the host arrays alive while the async copies are in flight
        self._ck(self.L.lins_gpu_batch_upload(self.h, C.byref(d)))
        self._batch_n = batch.n

    def batch_upload_stats(self):
        """(points uploaded as host-packed 16-B records, points uploaded as raw 32-B records), cumulative."""
        a, b = C.c_int64(0), C.c_int64(0)
        self._ck(self.L.lins_gpu_batch_upload_stats(self.h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def batch_run(self):
        self._ck(self.L.lins_gpu_batch_run(self.h))

    def batch_download(self, states=True, covs=True, reports=False):
        n = self._batch_n
        so = np.zeros((n, STATE_DIM)) if states else None
        co = np.zeros((n, COV_SIZE)) if covs else None
        res = np.zeros(n, dtype=SCAN_RESULT_DTYPE)
        reps = (LinsReport * n)() if reports else None
        self._ck(self.L.lins_gpu_batch_download(self.h, ptr(so), ptr(co), ptr(res), C.cast(reps, C.c_void_p) if reports else None))
        return so, co, res, reps

    def batch_download_indices(self, batch: Batch):
        """(surf_ind (Ns_total, 3), corner_ind (Nc_total, 2)) of the resident batch's last search iteration."""
        si = np.full((int(batch.offsets["surf_flat"][-1]), 3), -2, np.int32)
        ci = np.full((int(batch.offsets["corner_sharp"][-1]), 2), -2, np.int32)
        self._ck(self.L.lins_gpu_batch_download_indices(self.h, ptr(si), ptr(ci)))
        return si, ci

    def ieskf_batch(self, batch, covs=True):
        """upload + run + download through host buffers: the end-to-end entry point."""
        d = batch.desc()
        n = batch.n
        so = np.zeros((n, STATE_DIM))
        co = np.zeros((n, COV_SIZE)) if covs else None
        res = np.zeros(n, dtype=SCAN_RESULT_DTYPE)
        self._ck(self.L.lins_gpu_ieskf_batch(self.h, C.byref(d), ptr(so), ptr(co), ptr(res)))
        self._batch_n = n
        return so, co, res

    def batch_results_device(self):
        p, n = C.c_void_p(), C.c_int(0)
        self._ck(self.L.lins_gpu_batch_results_device(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def batch_jacobian_pass(self, want_accum=False):
        """The split Jacobian pass over the resident batch; with want_accum its (n, 30) sums (include/lins_gpu.h)."""
        acc = np.zeros((self._batch_n, 30)) if want_accum else None
        self._ck(self.L.lins_gpu_batch_jacobian_pass(self.h, ptr(acc)))
        return acc

    # ---- sequence mode ---------------------------------------------------------------------------------------------
    def seq_begin(self, params, handover):
        """Hand over S running sequences (each right after its processSecondScan).  `handover`: dict with filter_state
        (S x 19), filter_cov (S x 324), global_state (S x 19), imu_last (S x 6), surf_map / corner_map (POINT_DTYPE clouds)
        and their (S + 1) offsets surf_map_off / corner_map_off."""
        h = {k: np.ascontiguousarray(handover[k], dtype=np.float64) for k in ("filter_state", "filter_cov", "global_state", "imu_last")}
        for k in ("surf_map", "corner_map"):
            h[k] = as_points(handover[k])
            h[k + "_off"] = np.ascontiguousarray(handover[k + "_off"], dtype=np.int32)
        d = LinsSeqBeginDesc()
        d.n_seq = len(h["surf_map_off"]) - 1
        for k, v in h.items():
            setattr(d, k, v.ctypes.data)
        self._ck(self.L.lins_gpu_seq_begin(self.h, C.byref(params), C.byref(d)))
        self._seq_n = d.n_seq

    def seq_open(self, params, init_params, n_seq):
        """Open n_seq empty slots that start from their first scan (lins_gpu_seq_open).  params: LinsSeqParams,
        init_params: LinsSeqInitParams."""
        self._ck(self.L.lins_gpu_seq_open(self.h, C.byref(params), C.byref(init_params), int(n_seq)))
        self._seq_n = int(n_seq)

    def seq_restart(self, mask):
        """Put the slots with mask[s] != 0 back into the fresh state of seq_open (their next scan is a first scan)."""
        self._ck(self.L.lins_gpu_seq_restart(self.h, ptr(self._slot_mask(mask))))

    def seq_configure(self, mask, configs):
        """Configure the slots with mask[s] != 0, each still fresh (no step since seq_open / its last seq_restart), with
        their own rig: configs is a LinsSlotConfig per slot (S entries; None where the mask is 0).  A restart returns a slot
        to the run's values."""
        m = self._slot_mask(mask)
        if len(configs) != self._seq_n:
            raise ValueError(f"{len(configs)} configs, the run has {self._seq_n} slots")
        arr = (LinsSlotConfig * self._seq_n)(*[c if c is not None else LinsSlotConfig() for c in configs])
        self._ck(self.L.lins_gpu_seq_configure(self.h, ptr(m), C.cast(arr, C.c_void_p)))

    def seq_tune(self, mask, tunings):
        """Tune the slots with mask[s] != 0, each still fresh, with their own estimator tuning and IMU misalignment:
        tunings is a LinsSlotTuning per slot (S entries; None where the mask is 0).  A restart returns a slot to untuned."""
        m = self._slot_mask(mask)
        if len(tunings) != self._seq_n:
            raise ValueError(f"{len(tunings)} tunings, the run has {self._seq_n} slots")
        arr = (LinsSlotTuning * self._seq_n)(*[t if t is not None else LinsSlotTuning() for t in tunings])
        self._ck(self.L.lins_gpu_seq_tune(self.h, ptr(m), C.cast(arr, C.c_void_p)))

    def seq_save(self, mask):
        """Save the slots with mask[s] != 0: a list of S entries, each slot's blob (bytes, self-contained: it can be
        written to a file alone and loaded into a fresh slot of any seq_open run of this library build) or None where the
        mask is 0.  The run is unchanged."""
        return self._save_blobs(self.L.lins_gpu_seq_save_size, self.L.lins_gpu_seq_save, self._slot_mask(mask))

    def seq_load(self, mask, blobs):
        """Load blobs[s] (bytes, as seq_save returned it) into every slot with mask[s] != 0, each still fresh (no step
        since seq_open / its last seq_restart); blobs has S entries (None where the mask is 0).  All or nothing."""
        self._load_blobs(self.L.lins_gpu_seq_load, self._slot_mask(mask), blobs)

    def _save_blobs(self, save_size, save, m):
        """seq_save / mappers_save through their C entries: each slot's blob, None where m is 0"""
        off = np.zeros(len(m) + 1, np.uint64)
        self._ck(save_size(self.h, ptr(m), ptr(off)))
        buf = np.zeros(max(int(off[-1]), 1), np.uint8)
        self._ck(save(self.h, ptr(m), ptr(buf), ptr(off)))
        return [buf[int(off[s]): int(off[s + 1])].tobytes() if m[s] else None for s in range(len(m))]

    def _load_blobs(self, load, m, blobs):
        """seq_load / mappers_load through their C entry"""
        if len(blobs) != len(m):
            raise ValueError(f"{len(blobs)} blobs, the run has {len(m)} slots")
        parts = [bytes(blobs[s]) if m[s] else b"" for s in range(len(m))]
        off = np.zeros(len(m) + 1, np.uint64)
        off[1:] = np.cumsum([len(p) for p in parts])
        buf = np.frombuffer(b"".join(parts) or b"\0", np.uint8)
        self._ck(load(self.h, ptr(m), ptr(buf), ptr(off)))

    def _slot_mask(self, mask):
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        if len(m) != self._seq_n:
            raise ValueError(f"mask has {len(m)} entries, the run {self._seq_n}")
        return m

    def seq_download_init(self):
        """dict: fusion_status (S; StateEstimator::status_ of every slot) and, for the slots whose last scan was a second
        scan (LINS_SEQ_SECOND), its estimateTransform result: icp_pose (S x 7: t, q xyzw), icp_iters, icp_converged (zero
        elsewhere)."""
        n = self._seq_n
        out = dict(fusion_status=np.zeros(n, np.int32), icp_pose=np.zeros((n, 7)), icp_iters=np.zeros(n, np.int32),
                   icp_converged=np.zeros(n, np.int32))
        self._ck(self.L.lins_gpu_seq_download_init(self.h, ptr(out["fusion_status"]), ptr(out["icp_pose"]), ptr(out["icp_iters"]),
                                                   ptr(out["icp_converged"])))
        return out

    def seq_step(self, step, scan_imu=None):
        """Advance every present sequence by one scan.  `step`: dict with imu (k x 7: dt, acc, gyr) + imu_off, the four
        feature clouds (Batch.FIELDS) + their offsets (<name>_off), and optionally present (S, uint8).  scan_imu (S x 6:
        acc, gyr): the IMU sample that comes with each scan, needed while a present slot initialises."""
        keep, d = {}, LinsSeqStepDesc()
        si = self._seq_step_common(d, step, scan_imu, keep)
        for k in Batch.FIELDS:
            keep[k] = as_points(step[k])
            keep[k + "_off"] = np.ascontiguousarray(step[k + "_off"], dtype=np.int32)
            setattr(d, k, keep[k].ctypes.data)
            setattr(d, k + "_off", keep[k + "_off"].ctypes.data)
        d.point_format = int(step.get("point_format", 0))
        if si is None:
            self._ck(self.L.lins_gpu_seq_step(self.h, C.byref(d)))
        else:
            self._ck(self.L.lins_gpu_seq_step_ex(self.h, C.byref(d), ptr(si)))

    @staticmethod
    def _seq_step_common(d, step, scan_imu, keep):
        """Fill what every seq_step* descriptor d shares from `step` (n_seq, imu, imu_off and, when given, present) and check
        scan_imu against n_seq.  The arrays d points at are added to `keep`.  Returns scan_imu as an (S x 6) array, or None."""
        keep["imu"] = np.ascontiguousarray(step["imu"], dtype=np.float64)
        keep["imu_off"] = np.ascontiguousarray(step["imu_off"], dtype=np.int32)
        d.n_seq = len(keep["imu_off"]) - 1
        d.imu, d.imu_off = keep["imu"].ctypes.data, keep["imu_off"].ctypes.data
        if step.get("present") is not None:
            keep["present"] = np.ascontiguousarray(step["present"], dtype=np.uint8)
            d.present = keep["present"].ctypes.data
        if scan_imu is None:
            return None
        si = keep["scan_imu"] = np.ascontiguousarray(scan_imu, dtype=np.float64).reshape(-1, 6)
        if len(si) != d.n_seq:
            raise ValueError(f"scan_imu has {len(si)} rows, the step {d.n_seq}")
        return si

    @staticmethod
    def _pcl_desc(scans, line_num, keep):
        """LinsPclDesc of a list of segmented scans (dicts: seg (m x 4 float32 x, y, z, intensity, or POINT_DTYPE), ground,
        col, range, start_ring, end_ring, ori (3)); the arrays it points at are added to `keep`."""
        n = len(scans)
        segs = [as_points(s["seg"]) if np.asarray(s["seg"]).dtype == POINT_DTYPE else _points_from_xyzi(s["seg"]) for s in scans]
        off = np.zeros(n + 1, np.int32)
        off[1:] = np.cumsum([len(a) for a in segs])
        cat = lambda k, t: np.ascontiguousarray(np.concatenate([np.asarray(s[k], t).reshape(-1) for s in scans]) if n else np.zeros(0, t))  # noqa: E731
        keep.update(cloud=np.ascontiguousarray(np.concatenate(segs)) if n else np.zeros(0, POINT_DTYPE), cloud_off=off,
                    ground_flag=cat("ground", np.uint8), col_ind=cat("col", np.uint32), range=cat("range", np.float32),
                    start_ring_index=cat("start_ring", np.int32), end_ring_index=cat("end_ring", np.int32), orientation=cat("ori", np.float32))
        for k in ("start_ring_index", "end_ring_index"):
            if len(keep[k]) != n * line_num:
                raise ValueError(f"{k}: {len(keep[k])} entries for {n} scans of {line_num} rings")
        d = LinsPclDesc()
        d.n_scans, d.line_num, d.point_format = n, int(line_num), 0
        for k in ("cloud", "cloud_off", "ground_flag", "col_ind", "range", "start_ring_index", "end_ring_index", "orientation"):
            setattr(d, k, keep[k].ctypes.data)
        return d

    def extract_features(self, scans, line_num=16, params=None, undist=False):
        """Feature extraction of segmented scans on the device (lins_gpu_extract_features).  Returns one dict per scan with
        surf_flat, corner_sharp, surf_less_flat, corner_less_sharp (and undist when asked for) as (k x 4) float32
        (x, y, z, intensity) arrays."""
        keep = {}
        d = self._pcl_desc(scans, line_num, keep)
        n, total = d.n_scans, int(keep["cloud_off"][-1])
        outs = [np.zeros(max(total, 1), POINT_DTYPE) for _ in range(5)]
        counts = np.zeros((max(n, 1), 4), np.int32)
        fp = params or LinsFeatureParams.shipped()
        self._ck(self.L.lins_gpu_extract_features(self.h, C.byref(fp), C.byref(d), *[ptr(o) for o in outs[:4]],
                                                  ptr(outs[4]) if undist else None, ptr(counts)))
        x4 = lambda a: np.stack([a["x"], a["y"], a["z"], a["intensity"]], 1).astype(np.float32)  # noqa: E731
        names = ("surf_flat", "corner_sharp", "surf_less_flat", "corner_less_sharp")
        res = []
        off = keep["cloud_off"]
        for i in range(n):
            r = {k: x4(outs[c][off[i]: off[i] + counts[i, c]]) for c, k in enumerate(names)}
            if undist:
                r["undist"] = x4(outs[4][off[i]: off[i + 1]])
            res.append(r)
        return res

    def extract_ms(self):
        """CUDA-event time (ms) of the last extraction kernel."""
        ms = np.zeros(1, np.float32)
        self._ck(self.L.lins_gpu_extract_ms(self.h, ptr(ms)))
        return float(ms[0])

    @staticmethod
    def _raw_desc(sweeps, point_format, keep):
        """LinsRawDesc of a list of raw sweeps (POINT_DTYPE arrays, or (m x 3 / m x 4) float32 x, y, z[, intensity]);
        point_format 1 sends them as packed 16-B records.  The arrays it points at are added to `keep`."""
        n = len(sweeps)

        def points(s):
            a = np.asarray(s)
            if a.dtype == POINT_DTYPE:
                return as_points(a)
            a = np.asarray(a, np.float32)
            a = a.reshape(len(a), -1) if a.size else a.reshape(0, 4)  # (an empty sweep)
            return make_points(a[:, :3], a[:, 3] if a.shape[1] > 3 else np.zeros(len(a), np.float32))

        pts = [points(s) for s in sweeps]
        off = np.zeros(n + 1, np.int32)
        off[1:] = np.cumsum([len(a) for a in pts])
        cloud = np.ascontiguousarray(np.concatenate(pts)) if n else np.zeros(0, POINT_DTYPE)
        if point_format == 1:
            cloud = np.ascontiguousarray(np.stack([cloud["x"], cloud["y"], cloud["z"], cloud["intensity"]], 1).astype(np.float32))
        keep.update(cloud=cloud, cloud_off=off)
        d = LinsRawDesc()
        d.n_scans, d.point_format = n, int(point_format)
        d.cloud, d.cloud_off = cloud.ctypes.data, off.ctypes.data
        return d

    def project_scans(self, sweeps, model=None, point_format=0):
        """Image projection of raw sweeps on the device (lins_gpu_project_scans).  Returns one dict per sweep in the form
        extract_features takes: seg (m x 4 float32 x, y, z, intensity), ground, col, range, start_ring, end_ring, ori (3),
        plus outlier (k x 4)."""
        model = model or LinsLidarModel.vlp16()
        return self._project(sweeps, point_format, model.line_num, self.L.lins_gpu_project_scans, model)

    def project_scans_mixed(self, sweeps, models, model_of, point_format=0):
        """project_scans with sweep i projected by models[model_of[i]] (lins_gpu_project_scans_mixed); model_of may be None
        with one model.  start_ring / end_ring hold max(line_num) entries per sweep, those past its own model's line_num 0."""
        keep = {}
        t = self.models_table(models, model_of, keep)
        return self._project(sweeps, point_format, max(m.line_num for m in models), self.L.lins_gpu_project_scans_mixed, t)

    @staticmethod
    def models_table(models, model_of, keep):
        """LinsLidarModels of a list of LinsLidarModel and one entry per scan (or None); the arrays it points at are added
        to `keep`."""
        keep["models"] = (LinsLidarModel * max(len(models), 1))(*models)
        t = LinsLidarModels()
        t.n_models, t.models = len(models), C.cast(keep["models"], C.c_void_p)
        if model_of is not None:
            keep["model_of"] = np.ascontiguousarray(model_of, dtype=np.int32)
            t.model_of = keep["model_of"].ctypes.data
        return t

    def _project(self, sweeps, point_format, L, entry, model):
        """project_scans / project_scans_mixed: the outputs of the C entry `entry` called with `model` (a LinsLidarModel or
        a LinsLidarModels table), with L ring entries per sweep."""
        keep = {}
        d = self._raw_desc(sweeps, point_format, keep)
        n, total = d.n_scans, int(keep["cloud_off"][-1])
        rec = np.float32 if point_format == 1 else POINT_DTYPE
        shape = (max(total, 1), 4) if point_format == 1 else max(total, 1)
        seg, outl = np.zeros(shape, rec), np.zeros(shape, rec)
        ground, col, rng = np.zeros(max(total, 1), np.uint8), np.zeros(max(total, 1), np.uint32), np.zeros(max(total, 1), np.float32)
        sr, er = np.zeros((max(n, 1), max(L, 1)), np.int32), np.zeros((max(n, 1), max(L, 1)), np.int32)
        ori, counts = np.zeros((max(n, 1), 3), np.float32), np.zeros((max(n, 1), 2), np.int32)
        self._ck(entry(self.h, C.byref(model), C.byref(d), ptr(seg), ptr(ground), ptr(col), ptr(rng), ptr(outl), ptr(sr), ptr(er), ptr(ori), ptr(counts)))
        x4 = (lambda a: a.astype(np.float32)) if point_format == 1 else (  # noqa: E731
            lambda a: np.stack([a["x"], a["y"], a["z"], a["intensity"]], 1).astype(np.float32).reshape(-1, 4))
        off = keep["cloud_off"]
        res = []
        for i in range(n):
            o, m, k = off[i], counts[i, 0], counts[i, 1]
            res.append(dict(seg=x4(seg[o: o + m]), ground=ground[o: o + m].copy(), col=col[o: o + m].copy(), range=rng[o: o + m].copy(),
                            start_ring=sr[i].copy(), end_ring=er[i].copy(), ori=ori[i].copy(), outlier=x4(outl[o: o + k])))
        return res

    def project_ms(self):
        """CUDA-event time (ms) of the last projection kernel."""
        ms = np.zeros(1, np.float32)
        self._ck(self.L.lins_gpu_project_ms(self.h, ptr(ms)))
        return float(ms[0])

    def seq_step_pcl(self, step, fp=None, scan_imu=None, line_num=16):
        """Advance every present sequence by one processPCL-shaped scan (lins_gpu_seq_step_pcl): `step` has imu + imu_off as
        in seq_step, scans (one segmented scan per slot, as extract_features takes them; an absent slot's may be empty) and
        optionally present."""
        keep, d = {}, LinsSeqPclDesc()
        si = self._seq_step_common(d, step, scan_imu, keep)
        d.pcl = self._pcl_desc(step["scans"], line_num, keep)
        fp = fp or LinsFeatureParams.shipped()
        self._ck(self.L.lins_gpu_seq_step_pcl(self.h, C.byref(d), C.byref(fp), ptr(si)))

    def seq_step_raw(self, step, model=None, fp=None, scan_imu=None, point_format=0):
        """Advance every present sequence by one raw sweep (lins_gpu_seq_step_raw: image projection with copyPointCloud's NaN
        removal, feature extraction and the filter step on the device): `step` has imu + imu_off as in seq_step, sweeps (one
        raw sweep per slot, as project_scans takes them; an absent slot's may be empty) and optionally present.  model: the
        LinsLidarModel every slot shares (None = VLP-16)."""
        self._seq_step_sweeps(self.L.lins_gpu_seq_step_raw, model or LinsLidarModel.vlp16(), {}, step, fp, scan_imu, point_format)

    def seq_step_raw_mixed(self, step, models, model_of, fp=None, scan_imu=None, point_format=0):
        """seq_step_raw with slot s's sweep projected by models[model_of[s]] (lins_gpu_seq_step_raw_mixed): models is a list
        of LinsLidarModel, model_of one entry per slot, absent slots included (None with one model)."""
        keep = {}
        t = self.models_table(models, model_of, keep)
        self._seq_step_sweeps(self.L.lins_gpu_seq_step_raw_mixed, t, keep, step, fp, scan_imu, point_format)

    def _seq_step_sweeps(self, entry, model, keep, step, fp, scan_imu, point_format):
        """seq_step_raw / seq_step_raw_mixed: the C entry `entry` called with `model` (a LinsLidarModel or a LinsLidarModels
        table); `keep` holds what model points at."""
        d = LinsSeqRawDesc()
        si = self._seq_step_common(d, step, scan_imu, keep)
        d.raw = self._raw_desc(step["sweeps"], point_format, keep)
        fp = fp or LinsFeatureParams.shipped()
        self._ck(entry(self.h, C.byref(d), C.byref(model), C.byref(fp), ptr(si)))

    @staticmethod
    def cloud2_desc(msgs, keep, gap=0, base=0):
        """LinsCloud2Desc of PointCloud2 messages [(LinsCloud2Layout, data field bytes)], their data fields back to back in
        one blob.  gap: bytes after each data field (inside its range, as the rest of a message record in a bag chunk), so
        the fields start at any alignment; base: bytes before the first.  The arrays it points at are added to `keep`."""
        n = len(msgs)
        parts, off, pos = [np.zeros(base, np.uint8)], np.zeros(n + 1, np.int64), base
        off[0] = base
        for i, (_, data) in enumerate(msgs):
            a = np.frombuffer(bytes(data), np.uint8)
            parts += [a, np.full(gap, 0xA5, np.uint8)]
            pos += len(a) + gap
            off[i + 1] = pos
        blob = np.ascontiguousarray(np.concatenate(parts)) if parts else np.zeros(0, np.uint8)
        lays = (LinsCloud2Layout * max(n, 1))(*[m[0] for m in msgs])
        keep.update(blob=blob, data_off=off, layouts=lays)
        d = LinsCloud2Desc()
        d.n_scans, d.data, d.data_off, d.layouts = n, blob.ctypes.data, off.ctypes.data, C.cast(lays, C.c_void_p)
        return d

    def decode_cloud2(self, msgs=None, desc=None, gap=0, base=0):
        """pcl::fromROSMsg<PointXYZI> of PointCloud2 messages on the device (lins_gpu_decode_cloud2): msgs as cloud2_desc takes
        them, or a prepared LinsCloud2Desc.  Returns (POINT_DTYPE records of every message back to back, counts)."""
        keep = {}
        d = desc if desc is not None else self.cloud2_desc(msgs, keep, gap, base)
        lays = C.cast(d.layouts, C.POINTER(LinsCloud2Layout)) if d.n_scans else None
        total = sum(int(lays[i].width) * int(lays[i].height) for i in range(d.n_scans))
        out, counts = np.zeros(max(total, 1), POINT_DTYPE), np.zeros(max(d.n_scans, 1), np.int32)
        self._ck(self.L.lins_gpu_decode_cloud2(self.h, C.byref(d), ptr(out), ptr(counts)))
        return out[:total], counts[: d.n_scans]

    def decode_ms(self):
        """CUDA-event time (ms) of the last PointCloud2 decode kernel."""
        ms = np.zeros(1, np.float32)
        self._ck(self.L.lins_gpu_decode_ms(self.h, ptr(ms)))
        return float(ms[0])

    def seq_step_cloud2(self, step, model=None, fp=None, scan_imu=None, desc=None, gap=0):
        """Advance every present sequence by one sensor_msgs/PointCloud2 message (lins_gpu_seq_step_cloud2: the decode, then
        what seq_step_raw runs): `step` has imu + imu_off as in seq_step, msgs (one (layout, data) per slot, as cloud2_desc
        takes them; an absent slot's is not read) or desc (a prepared LinsCloud2Desc), and optionally present."""
        self._seq_step_msgs(self.L.lins_gpu_seq_step_cloud2, model or LinsLidarModel.vlp16(), {}, step, fp, scan_imu, desc, gap)

    def seq_step_cloud2_mixed(self, step, models, model_of, fp=None, scan_imu=None, desc=None, gap=0):
        """seq_step_cloud2 with slot s's message projected by models[model_of[s]] (lins_gpu_seq_step_cloud2_mixed): models
        and model_of as seq_step_raw_mixed takes them."""
        keep = {}
        t = self.models_table(models, model_of, keep)
        self._seq_step_msgs(self.L.lins_gpu_seq_step_cloud2_mixed, t, keep, step, fp, scan_imu, desc, gap)

    def _seq_step_msgs(self, entry, model, keep, step, fp, scan_imu, desc, gap):
        """seq_step_cloud2 / seq_step_cloud2_mixed: the C entry `entry` called with `model` (a LinsLidarModel or a
        LinsLidarModels table); `keep` holds what model points at."""
        d = LinsSeqCloud2Desc()
        si = self._seq_step_common(d, step, scan_imu, keep)
        d.cloud2 = desc if desc is not None else self.cloud2_desc(step["msgs"], keep, gap)
        fp = fp or LinsFeatureParams.shipped()
        self._ck(entry(self.h, C.byref(d), C.byref(model), C.byref(fp), ptr(si)))

    def seq_download(self, reports=False):
        """dict: global_state, filter_state (S x 19), filter_cov (S x 324), results (SCAN_RESULT_DTYPE), status (S) and,
        when asked for, reports (LinsReport array)."""
        n = self._seq_n
        out = dict(global_state=np.zeros((n, STATE_DIM)), filter_state=np.zeros((n, STATE_DIM)), filter_cov=np.zeros((n, COV_SIZE)),
                   results=np.zeros(n, dtype=SCAN_RESULT_DTYPE), status=np.zeros(n, np.int32))
        reps = (LinsReport * n)() if reports else None
        self._ck(self.L.lins_gpu_seq_download(self.h, ptr(out["global_state"]), ptr(out["filter_state"]), ptr(out["filter_cov"]),
                                              ptr(out["results"]), C.cast(reps, C.c_void_p) if reports else None, ptr(out["status"])))
        if reports:
            out["reports"] = reps
        return out

    def seq_phase_ms(self):
        """CUDA-event times (ms) of the last seq_step's phases: predict, IESKF, divergence check + ICP fallback, post + map."""
        ms = np.zeros(4, np.float32)
        self._ck(self.L.lins_gpu_seq_phase_ms(self.h, ptr(ms)))
        return ms

    def seq_download_ieskf(self):
        """The last step's IESKF: prior_state / prior_cov (every sequence), state_out / cov_out, and per sequence that ran its
        last-iteration correspondence IDs: surf_ind[s] (ns, 3), corner_ind[s] (nc, 2) (None for a sequence that did not run)."""
        n = self._seq_n
        off = np.zeros(2 * (n + 1), np.int32)
        self._ck(self.L.lins_gpu_seq_download_ieskf(self.h, None, None, None, None, ptr(off), None, None))
        so, co = off[: n + 1], off[n + 1:]
        out = dict(prior_state=np.zeros((n, STATE_DIM)), prior_cov=np.zeros((n, COV_SIZE)), state_out=np.zeros((n, STATE_DIM)),
                   cov_out=np.zeros((n, COV_SIZE)))
        si, ci = np.zeros((so[-1], 3), np.int32), np.zeros((co[-1], 2), np.int32)
        ran = so[-1] + co[-1] > 0
        self._ck(self.L.lins_gpu_seq_download_ieskf(self.h, ptr(out["prior_state"]), ptr(out["prior_cov"]),
                                                    ptr(out["state_out"]) if ran else None, ptr(out["cov_out"]) if ran else None,
                                                    None, ptr(si), ptr(ci)))
        out["surf_ind"] = [si[so[s]:so[s + 1]] for s in range(n)]
        out["corner_ind"] = [ci[co[s]:co[s + 1]] for s in range(n)]
        return out

    def seq_download_maps(self):
        """The maps the next step searches: per sequence surf_map, corner_map, surf_tree, corner_tree (POINT_DTYPE clouds)
        and stale (S,)."""
        n = self._seq_n
        off = np.zeros(4 * (n + 1), np.int32)
        self._ck(self.L.lins_gpu_seq_download_maps(self.h, ptr(off), None, None, None, None, None))
        o = off.reshape(4, n + 1)
        bufs = [np.zeros((o[c, -1], 4), np.float32) for c in range(4)]
        stale = np.zeros(n, np.uint8)
        self._ck(self.L.lins_gpu_seq_download_maps(self.h, None, *[ptr(b) for b in bufs], ptr(stale)))
        out = dict(stale=stale)
        for c, name in enumerate(("surf_map", "corner_map", "surf_tree", "corner_tree")):
            pts = np.zeros(o[c, -1], POINT_DTYPE)
            pts["x"], pts["y"], pts["z"], pts["intensity"] = bufs[c][:, 0], bufs[c][:, 1], bufs[c][:, 2], bufs[c][:, 3]
            out[name] = [pts[o[c, s]:o[c, s + 1]] for s in range(n)]
        return out
