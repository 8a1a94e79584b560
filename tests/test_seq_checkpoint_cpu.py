"""CPU checks of saving and loading sequence-mode slots: the slot-blob validator (csrc/cuda/lins_slot_blob.hpp, compiled
with g++ next to a synthetic blob writer) accepts what the writer makes and rejects every truncation, every bit flip of
the header and section table, counts that run past the end, a window id without a stored key frame, too many key frames
and an out-of-range status; and the replay driver's checkpoint pieces (slot_queue fast-forward, the driver state file)."""
import ctypes as C
import importlib
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_DIR = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")

# A synthetic writer and the validator behind a C ABI.  spec: flags, fusion, stale, n_map[4], n_outlier, n_poses, n_window,
# n_keyframes, then the window ids, then (id, n[3]) per key frame.  Data sections get a byte pattern; a configured /
# tuned blob gets valid values.
DRIVER = r"""
#include "lins_slot_blob.hpp"
#include <vector>
using namespace lins_blob;
static const BuildSizes kSz = {304, 304, LINS_MAPPER_IMU_QUEUE, 10, 24};
extern "C" uint64_t blob_make(const int* sp, uint8_t* out, uint64_t cap) {
  Counts c;
  const uint32_t flags = sp[0];
  c.bound = flags & kBound;
  for (int k = 0; k < 4; ++k) c.n_map[k] = sp[3 + k];
  c.n_outlier = sp[7]; c.n_poses = sp[8]; c.n_window = sp[9]; c.n_keyframes = sp[10];
  const int* win = sp + 11;
  const int* kf = win + c.n_window;
  for (int i = 0; i < c.n_keyframes; ++i) c.n_kf_points += kf[4 * i + 1] + kf[4 * i + 2] + kf[4 * i + 3];
  Header h;
  layout(c, kSz, h);
  if (h.total > cap) return h.total;
  for (uint64_t i = 0; i < h.total; ++i) out[i] = (uint8_t)(i * 131 + 7);
  h.magic = kMagic; h.version = kVersion; h.flags = flags; h.sizes = kSz; h.n_sections = kNumSections;
  std::memcpy(out, &h, sizeof(h));
  Scalars s;
  std::memset(&s, 0, sizeof(s));
  s.fusion = sp[1]; s.stale = sp[2];
  for (int k = 0; k < 4; ++k) s.n_map[k] = sp[3 + k];
  s.n_outlier = sp[7]; s.n_poses = sp[8]; s.n_window = sp[9]; s.n_keyframes = sp[10];
  if (flags & kConfigured) { s.cfg.scan_period = 0.1; }
  if (flags & kTuned) { s.tune.num_iter = 30; s.tune.icp_freq = 1000; }
  std::memcpy(out + h.sec[kScalars].off, &s, sizeof(s));
  if (c.bound) {
    MapperRec m;
    std::memset(&m, 0, sizeof(m));
    m.imuPointerLast = -1;
    std::memcpy(out + h.sec[kMapper].off, &m, sizeof(m));
    std::memcpy(out + h.sec[kWindow].off, win, 4 * c.n_window);
    for (int i = 0; i < c.n_keyframes; ++i) {
      KeyframeRec r = {kf[4 * i], {kf[4 * i + 1], kf[4 * i + 2], kf[4 * i + 3]}};
      std::memcpy(out + h.sec[kKeyframes].off + sizeof(r) * i, &r, sizeof(r));
    }
  }
  return h.total;
}
extern "C" int blob_check(const uint8_t* p, uint64_t len, int* sp, char* err, int errcap) {
  View v;
  const char* bad = parse(p, len, kSz, v);
  if (bad) { std::snprintf(err, errcap, "%s", bad); return 1; }
  const Scalars& s = v.sc;
  int* o = sp;
  *o++ = v.h.flags; *o++ = s.fusion; *o++ = s.stale;
  for (int k = 0; k < 4; ++k) *o++ = s.n_map[k];
  *o++ = s.n_outlier; *o++ = s.n_poses; *o++ = s.n_window; *o++ = s.n_keyframes;
  for (int i = 0; i < s.n_window; ++i) *o++ = v.window(i);
  for (int i = 0; i < s.n_keyframes; ++i) { KeyframeRec r = v.keyframe(i); *o++ = r.id; for (int a = 0; a < 3; ++a) *o++ = r.n[a]; }
  return 0;
}
"""

HEADER_BYTES = 208   # sizeof(Header)
SCALARS = 208        # the scalar section's offset
F_BOUND, F_CONFIGURED, F_TUNED = 1, 2, 4


@pytest.fixture(scope="module")
def blob_lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ is not available")
    d = tmp_path_factory.mktemp("blob")
    src, so = d / "blob_driver.cpp", d / "blob_driver.so"
    src.write_text("#include <cstdio>\n" + DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC", "-I", CUDA_DIR, "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.blob_make.restype = C.c_uint64
    L.blob_make.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.blob_check.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    return L


def spec(flags=F_BOUND, fusion=3, stale=1, n_map=(40, 7, 30, 5), n_outlier=9, n_poses=12, window=None, keyframes=None):
    window = list(range(12)) if window is None else window
    keyframes = [(i, 3 + i % 4, 20 + i, i % 3) for i in range(12)] if keyframes is None else keyframes
    if not flags & F_BOUND:
        n_outlier, n_poses, window, keyframes = 0, 0, [], []
    return [flags, fusion, stale, *n_map, n_outlier, n_poses, len(window), len(keyframes), *window, *[x for k in keyframes for x in k]]


def make(L, sp):
    sp_a = np.array(sp, np.int32)
    n = L.blob_make(sp_a.ctypes.data, None, 0)
    buf = np.zeros(n, np.uint8)
    assert L.blob_make(sp_a.ctypes.data, buf.ctypes.data, n) == n
    return buf


def check(L, buf, n=None):
    """(None, spec) for an accepted blob, else (the validator's message, None)."""
    out = np.zeros(4096, np.int32)
    err = C.create_string_buffer(256)
    b = np.ascontiguousarray(buf, np.uint8)
    rc = L.blob_check(b.ctypes.data if len(b) else None, len(b) if n is None else n, out.ctypes.data, err, 256)
    return (err.value.decode(), None) if rc else (None, out)


@pytest.mark.parametrize("sp", [spec(), spec(flags=0), spec(flags=0, stale=0, n_map=(10, 3, 0, 0)), spec(flags=F_BOUND | F_CONFIGURED | F_TUNED),
                                spec(fusion=0, stale=0, n_map=(0, 0, 0, 0), n_poses=0, window=[], keyframes=[]),
                                spec(fusion=1, n_poses=60, window=list(range(10, 60)) + [], keyframes=[(i, 1, 2, 3) for i in range(9, 60)]),
                                spec(n_poses=51, window=list(range(1, 50)) + [50], keyframes=[(i, 1, 1, 1) for i in range(0, 51)]),
                                spec(n_poses=52, window=list(range(2, 51)) + [50], keyframes=[(i, 0, 4, 1) for i in range(2, 52)])])
def test_synthetic_blobs_accepted_and_round_trip(blob_lib, sp):
    buf = make(blob_lib, sp)
    assert len(buf) % 16 == 0
    err, got = check(blob_lib, buf)
    assert err is None, err
    assert got[:len(sp)].tolist() == sp


def test_every_truncation_rejected(blob_lib):
    buf = make(blob_lib, spec())
    for n in range(len(buf)):
        err, _ = check(blob_lib, buf[:n])
        assert err is not None, n
    # and a blob read with a length other than its own
    assert check(blob_lib, np.concatenate([buf, np.zeros(16, np.uint8)]))[0] is not None


@pytest.mark.parametrize("flags", [0, F_BOUND])
def test_every_header_and_section_table_bit_flip_rejected(blob_lib, flags):
    buf = make(blob_lib, spec(flags=flags))
    for byte in range(HEADER_BYTES):
        for bit in range(8):
            b = buf.copy()
            b[byte] ^= 1 << bit
            err, _ = check(blob_lib, b)
            assert err is not None, (byte, bit)


def _scalar(buf, field, value):
    off = SCALARS + dict(fusion=0, stale=4, yzx=8, pad=12, n_map0=16, n_map1=20, n_map2=24, n_map3=28, n_outlier=32, n_poses=36,
                         n_window=40, n_keyframes=44)[field]
    b = buf.copy()
    b[off: off + 4] = np.frombuffer(np.int32(value).tobytes(), np.uint8)
    return b


@pytest.mark.parametrize("field,value", [("n_map0", 1 << 30), ("n_map3", 2), ("n_outlier", 1 << 20), ("n_poses", -1), ("n_window", 13),
                                         ("n_keyframes", 13), ("n_map1", -1), ("n_outlier", 10)])
def test_counts_past_the_end_rejected(blob_lib, field, value):
    buf = make(blob_lib, spec())
    assert check(blob_lib, _scalar(buf, field, value))[0] is not None


@pytest.mark.parametrize("field,value", [("fusion", 2), ("fusion", -1), ("fusion", 4), ("stale", 2), ("yzx", 3), ("pad", 1)])
def test_out_of_range_status_rejected(blob_lib, field, value):
    buf = make(blob_lib, spec())
    err, _ = check(blob_lib, _scalar(buf, field, value))
    assert err is not None


def test_mapper_state_checks(blob_lib):
    ok = spec(n_poses=5, window=[0, 1, 2, 3], keyframes=[(i, 1, 1, 1) for i in range(5)])
    assert check(blob_lib, make(blob_lib, ok))[0] is None
    # a window id that names no stored key frame
    err, _ = check(blob_lib, make(blob_lib, spec(n_poses=5, window=[0, 1, 7], keyframes=[(i, 1, 1, 1) for i in range(5)])))
    assert err and "window" in err
    # more than 51 stored key frames
    err, _ = check(blob_lib, make(blob_lib, spec(n_poses=60, window=list(range(8, 58)), keyframes=[(i, 1, 1, 1) for i in range(8, 60)])))
    assert err and "51" in err
    # a key frame stored twice, one of no key pose, a negative cloud count
    for kfs in ([(0, 1, 1, 1), (0, 1, 1, 1), (1, 1, 1, 1)], [(0, 1, 1, 1), (1, 1, 1, 1), (5, 1, 1, 1)], [(0, 1, 1, 1), (1, -1, 1, 1)]):
        assert check(blob_lib, make(blob_lib, spec(n_poses=2, window=[0], keyframes=kfs)))[0] is not None
    # the newest key frame, or one the next window takes, missing
    assert check(blob_lib, make(blob_lib, spec(n_poses=3, window=[0, 1], keyframes=[(0, 1, 1, 1), (1, 1, 1, 1)])))[0] is not None
    assert check(blob_lib, make(blob_lib, spec(n_poses=3, window=[2], keyframes=[(0, 1, 1, 1), (2, 1, 1, 1)])))[0] is not None
    # an unbound blob with mapper counts, a 1-NN cloud without the stale flag
    assert check(blob_lib, _scalar(make(blob_lib, spec(flags=0)), "n_poses", 1))[0] is not None
    assert check(blob_lib, make(blob_lib, spec(stale=0)))[0] is not None


def _bag_replay():
    return importlib.import_module("lins---lidar-inertial-slam_b200.bag_replay")


@pytest.mark.parametrize("lengths,slots", [([5, 0, 3, 7, 1, 4], 2), ([9, 2, 2, 6], 3), ([4, 4, 4], 5), ([1] * 7, 1)])
def test_slot_queue_fast_forward(lengths, slots):
    br = _bag_replay()
    full = [(r.tolist(), w) for r, w in br.slot_queue(lengths, slots)]
    for k in range(len(full) + 1):
        tail = [(r.tolist(), w) for r, w in itertools.islice(br.slot_queue(lengths, slots), k, None)]
        assert tail == full[k:]


def test_driver_state_round_trips(tmp_path):
    br = _bag_replay()
    rng = np.random.default_rng(3)
    out = []
    for n, m in ((6, 3), (4, 0)):
        o = dict(stamps=rng.random(n), status=rng.integers(0, 4, n).astype(np.int32), scan_status=rng.integers(0, 6, n).astype(np.int32),
                 global_est=rng.random((n, 7)), global_state=rng.random((n, 19)), iters=rng.integers(-1, 30, n).astype(np.int32),
                 flags=rng.integers(-1, 4, n).astype(np.int32), key_poses=rng.random((2, 7)))
        o.update(map_time=[np.float64(t) for t in rng.random(m)], map_odom=[rng.random(7) for _ in range(m)],
                 map_processed=[int(x) for x in rng.integers(0, 2, m)],
                 map_aft_mapped=[[float(np.float32(x)) for x in rng.random(6)] for _ in range(m)],
                 map_keyframes=[int(x) for x in rng.integers(0, 9, m)], map_sizes=[rng.integers(0, 99, 3).astype(np.int32) for _ in range(m)])
        out.append(o)
    held = [(1, 5), None, (0, None)]
    path = str(tmp_path / "driver.npz")
    br.save_driver_state(path, 7, 3, [6, 4], True, held, out, ["slot0_step7.bin", "", "slot2_step7.bin"])
    st = br.load_driver_state(path)
    assert (st["step"], st["slots"], st["lengths"], st["map"], st["held"]) == (7, 3, [6, 4], True, held)
    assert st["blob_files"] == ["slot0_step7.bin", "", "slot2_step7.bin"]
    for a, b in zip(out, st["out"]):
        fa, fb = br._map_arrays(a), br._map_arrays(b)
        assert fa.keys() == fb.keys()
        for k in fa:
            assert fa[k].dtype == fb[k].dtype and fa[k].shape == fb[k].shape and fa[k].tobytes() == fb[k].tobytes(), k
        # a list keeps growing after a resume: the restored rows, then new ones, give the same array
        assert br._map_arrays(dict(map_odom=b["map_odom"] + [np.ones(7)]))["map_odom"].tobytes() == \
            br._map_arrays(dict(map_odom=a["map_odom"] + [np.ones(7)]))["map_odom"].tobytes()
    # written again, the file's state is the same byte for byte
    path2 = str(tmp_path / "driver2.npz")
    br.save_driver_state(path2, st["step"], st["slots"], st["lengths"], st["map"], st["held"], st["out"], st["blob_files"])
    st2 = br.load_driver_state(path2)
    for a, b in zip(st["out"], st2["out"]):
        for k in a:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes()


def test_replay_checkpoint_arguments():
    br = _bag_replay()
    with pytest.raises(ValueError):
        br.replay([], 2, stop_after=3)
    with pytest.raises(ValueError):
        br.replay([], 2, checkpoint_every=3)
