"""CPU checks of saving and loading mapping nodes: the mapper-blob validator (csrc/cuda/lins_mapper_blob.hpp, compiled with
g++ next to a synthetic blob writer) accepts what the writer makes, plain and with loop closure, and rejects every
truncation, every bit flip of the header and section table, counts that run past the end, the plain-slot mapper rules,
and each loop-closure rule broken: a missing key frame, an estimate count other than the key poses', the prior not
first, a chain factor out of order, a loop end out of range, closed without a loop factor, NaN / inf values and a
variance <= 0."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_DIR = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")

# A synthetic writer and the validator behind a C ABI.  spec: flags, n_poses, n_window, n_keyframes, n_factors, n_est,
# n_loop, closed, then the window ids, then (id, n[3]) per key frame, then (a, b) per factor.  Data sections get a byte
# pattern; factors get R = I, t = 0, variances 1e-6; estimates R = I, t = 0.
DRIVER = r"""
#include "lins_mapper_blob.hpp"
#include <cstdio>
using namespace lins_mblob;
static const BuildSizes kSz = {304, LINS_MAPPER_IMU_QUEUE, LINS_MAPPER_WINDOW, sizeof(FactorRec)};
extern "C" uint64_t blob_make(const int* sp, uint8_t* out, uint64_t cap) {
  Counts c;
  const uint32_t flags = sp[0];
  c.n_poses = sp[1]; c.n_window = sp[2]; c.n_keyframes = sp[3]; c.n_factors = sp[4]; c.n_est = sp[5];
  const int* win = sp + 8;
  const int* kf = win + c.n_window;
  const int* fac = kf + 4 * c.n_keyframes;
  for (int i = 0; i < c.n_keyframes; ++i) c.n_kf_points += kf[4 * i + 1] + kf[4 * i + 2] + kf[4 * i + 3];
  Header h;
  layout(c, kSz, h);
  if (h.total > cap) return h.total;
  for (uint64_t i = 0; i < h.total; ++i) out[i] = (uint8_t)(i * 131 + 7);
  h.magic = kMagic; h.version = kVersion; h.flags = flags; h.sizes = kSz; h.n_sections = kNumSections; h.pad = 0;
  std::memcpy(out, &h, sizeof(h));
  Scalars s;
  std::memset(&s, 0, sizeof(s));
  s.n_poses = sp[1]; s.n_window = sp[2]; s.n_keyframes = sp[3]; s.n_factors = sp[4]; s.n_est = sp[5]; s.n_loop = sp[6]; s.closed = sp[7];
  s.time = 123.5;
  std::memcpy(out + h.sec[kScalars].off, &s, sizeof(s));
  MapperRec m;
  std::memset(&m, 0, sizeof(m));
  m.imuPointerLast = -1;
  std::memcpy(out + h.sec[kMapper].off, &m, sizeof(m));
  std::memcpy(out + h.sec[kWindow].off, win, 4 * c.n_window);
  for (int i = 0; i < c.n_keyframes; ++i) {
    KeyframeRec r = {kf[4 * i], {kf[4 * i + 1], kf[4 * i + 2], kf[4 * i + 3]}};
    std::memcpy(out + h.sec[kKeyframes].off + sizeof(r) * i, &r, sizeof(r));
  }
  for (int i = 0; i < c.n_factors; ++i) {
    FactorRec f;
    std::memset(&f, 0, sizeof(f));
    f.a = fac[2 * i]; f.b = fac[2 * i + 1];
    f.R[0] = f.R[4] = f.R[8] = 1.0;
    for (int k = 0; k < 6; ++k) f.var[k] = 1e-6;
    std::memcpy(out + h.sec[kFactors].off + sizeof(f) * i, &f, sizeof(f));
  }
  for (int i = 0; i < c.n_est; ++i) {
    EstRec e;
    std::memset(&e, 0, sizeof(e));
    e.R[0] = e.R[4] = e.R[8] = 1.0;
    std::memcpy(out + h.sec[kEst].off + sizeof(e) * i, &e, sizeof(e));
  }
  return h.total;
}
extern "C" int blob_check(const uint8_t* p, uint64_t len, int* sp, char* err, int errcap) {
  View v;
  const char* bad = parse(p, len, kSz, v);
  if (bad) { std::snprintf(err, errcap, "%s", bad); return 1; }
  const Scalars& s = v.sc;
  int* o = sp;
  *o++ = v.h.flags; *o++ = s.n_poses; *o++ = s.n_window; *o++ = s.n_keyframes; *o++ = s.n_factors; *o++ = s.n_est;
  *o++ = s.n_loop; *o++ = s.closed;
  for (int i = 0; i < s.n_window; ++i) *o++ = v.window(i);
  for (int i = 0; i < s.n_keyframes; ++i) { KeyframeRec r = v.keyframe(i); *o++ = r.id; for (int a = 0; a < 3; ++a) *o++ = r.n[a]; }
  for (int i = 0; i < s.n_factors; ++i) { FactorRec f = v.factor(i); *o++ = f.a; *o++ = f.b; }
  return 0;
}
"""

HEADER_BYTES = 192  # sizeof(Header)
SEC_TABLE = 48      # the section table's offset in the header
K_SCALARS, K_MAPPER, K_POSES, K_WINDOW, K_KEYFRAMES, K_KFCLOUDS, K_LOOP, K_FACTORS, K_EST = range(9)
FACTOR_BYTES = 152
F_LOOPS = 1


@pytest.fixture(scope="module")
def blob_lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ is not available")
    d = tmp_path_factory.mktemp("mblob")
    src, so = d / "mblob_driver.cpp", d / "mblob_driver.so"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC", "-I", CUDA_DIR, "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.blob_make.restype = C.c_uint64
    L.blob_make.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.blob_check.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    return L


def plain(n_poses=12, window=None, keyframes=None):
    window = list(range(n_poses)) if window is None else window
    keyframes = [(i, 3 + i % 4, 20 + i, i % 3) for i in range(n_poses)] if keyframes is None else keyframes
    return [0, n_poses, len(window), len(keyframes), 0, 0, 0, 0, *window, *[x for k in keyframes for x in k]]


def loop_factors(n_poses, loops=()):
    """the graph mapper_loops_save / close_loops build: prior, chains, and each loop (after chain factor `at`, ends a, b)"""
    f = [(0, -1)] if n_poses else []
    for n in range(1, n_poses):
        f.append((n - 1, n))
        f += [(a, b) for at, a, b in loops if at == n]
    return f


def with_loops(n_poses=60, window=None, factors=None, n_est=None, n_loop=None, closed=0, keyframes=None):
    window = list(range(max(0, n_poses - 50), n_poses)) if window is None else window
    keyframes = [(i, 2 + i % 3, 10 + i % 7, i % 2) for i in range(n_poses)] if keyframes is None else keyframes
    factors = loop_factors(n_poses, [(40, 40, 3), (55, 55, 2)] if n_poses > 55 else []) if factors is None else factors
    n_loop = sum(1 for a, b in factors[1:] if b != a + 1) if n_loop is None else n_loop
    n_est = n_poses if n_est is None else n_est
    return [F_LOOPS, n_poses, len(window), len(keyframes), len(factors), n_est, n_loop, closed, *window,
            *[x for k in keyframes for x in k], *[x for f in factors for x in f]]


def make(L, sp):
    sp_a = np.array(sp, np.int32)
    n = L.blob_make(sp_a.ctypes.data, None, 0)
    buf = np.zeros(n, np.uint8)
    assert L.blob_make(sp_a.ctypes.data, buf.ctypes.data, n) == n
    return buf


def check(L, buf, n=None):
    """(None, spec) for an accepted blob, else (the validator's message, None)."""
    out = np.zeros(1 << 14, np.int32)
    err = C.create_string_buffer(256)
    b = np.ascontiguousarray(buf, np.uint8)
    rc = L.blob_check(b.ctypes.data if len(b) else None, len(b) if n is None else n, out.ctypes.data, err, 256)
    return (err.value.decode(), None) if rc else (None, out)


def section(buf, k):
    return struct.unpack_from("<QQ", bytes(buf[SEC_TABLE + 16 * k: SEC_TABLE + 16 * k + 16]))


ACCEPTED = [plain(), plain(n_poses=0, window=[], keyframes=[]),
            plain(n_poses=60, window=list(range(10, 60)), keyframes=[(i, 1, 2, 3) for i in range(9, 60)]),
            plain(n_poses=52, window=list(range(2, 51)) + [50], keyframes=[(i, 0, 4, 1) for i in range(2, 52)]),
            with_loops(), with_loops(n_poses=0, window=[]), with_loops(n_poses=1, window=[0]), with_loops(closed=1),
            with_loops(n_poses=30, window=[], factors=loop_factors(30, [(29, 29, 29)]), closed=1),
            with_loops(n_poses=1100, window=list(range(1050, 1100)))]


@pytest.mark.parametrize("sp", ACCEPTED)
def test_synthetic_blobs_accepted_and_round_trip(blob_lib, sp):
    buf = make(blob_lib, sp)
    assert len(buf) % 16 == 0
    err, got = check(blob_lib, buf)
    assert err is None, err
    assert got[:len(sp)].tolist() == sp


def test_loop_blob_carries_body_clouds_of_every_key_frame(blob_lib):
    sp = with_loops(n_poses=7, window=list(range(7)), factors=loop_factors(7), keyframes=[(i, 1, 2, 3) for i in range(7)])
    buf = make(blob_lib, sp)
    assert section(buf, K_KFCLOUDS)[1] == 16 * 7 * 6
    assert section(buf, K_FACTORS)[1] == FACTOR_BYTES * 7 and section(buf, K_EST)[1] == 96 * 7


@pytest.mark.parametrize("sp", [plain(), with_loops(n_poses=8, window=list(range(8)))])
def test_every_truncation_rejected(blob_lib, sp):
    buf = make(blob_lib, sp)
    for n in range(len(buf)):
        err, _ = check(blob_lib, buf[:n])
        assert err is not None, n
    assert check(blob_lib, np.concatenate([buf, np.zeros(16, np.uint8)]))[0] is not None


@pytest.mark.parametrize("sp", [plain(), with_loops(n_poses=8, window=list(range(8)))])
def test_every_header_and_section_table_bit_flip_rejected(blob_lib, sp):
    buf = make(blob_lib, sp)
    for byte in range(HEADER_BYTES):
        for bit in range(8):
            b = buf.copy()
            b[byte] ^= 1 << bit
            err, _ = check(blob_lib, b)
            assert err is not None, (byte, bit)


def _scalar(buf, field, value):
    off = section(buf, K_SCALARS)[0] + dict(n_poses=0, n_window=4, n_keyframes=8, n_factors=12, n_est=16, n_loop=20, closed=24)[field]
    b = buf.copy()
    b[off: off + 4] = np.frombuffer(np.int32(value).tobytes(), np.uint8)
    return b


@pytest.mark.parametrize("sp", [plain(), with_loops()])
@pytest.mark.parametrize("field,value", [("n_poses", 1 << 30), ("n_poses", -1), ("n_window", 51), ("n_keyframes", 1 << 20),
                                         ("n_factors", 1 << 24), ("n_est", 1 << 26), ("n_est", -1), ("n_loop", -1), ("n_keyframes", 13)])
def test_counts_past_the_end_rejected(blob_lib, sp, field, value):
    assert check(blob_lib, _scalar(make(blob_lib, sp), field, value))[0] is not None


def test_plain_slot_mapper_checks(blob_lib):
    err, _ = check(blob_lib, make(blob_lib, plain(n_poses=5, window=[0, 1, 7], keyframes=[(i, 1, 1, 1) for i in range(5)])))
    assert err and "window" in err
    err, _ = check(blob_lib, make(blob_lib, plain(n_poses=60, window=list(range(8, 58)), keyframes=[(i, 1, 1, 1) for i in range(8, 60)])))
    assert err and "51" in err
    for kfs in ([(0, 1, 1, 1), (0, 1, 1, 1), (1, 1, 1, 1)], [(0, 1, 1, 1), (1, 1, 1, 1), (5, 1, 1, 1)], [(0, 1, 1, 1), (1, -1, 1, 1)]):
        assert check(blob_lib, make(blob_lib, plain(n_poses=2, window=[0], keyframes=kfs)))[0] is not None
    assert check(blob_lib, make(blob_lib, plain(n_poses=3, window=[0, 1], keyframes=[(0, 1, 1, 1), (1, 1, 1, 1)])))[0] is not None
    assert check(blob_lib, make(blob_lib, plain(n_poses=3, window=[2], keyframes=[(0, 1, 1, 1), (2, 1, 1, 1)])))[0] is not None
    # a plain blob with loop-closure state, a bad IMU pointer
    for field in ("n_loop", "closed"):
        assert check(blob_lib, _scalar(make(blob_lib, plain()), field, 1))[0] is not None, field
    b = make(blob_lib, plain())
    off = section(b, K_MAPPER)[0] + 4 * (36 + 2 * 200) + 8 * 200  # imuPointerFront
    b[off: off + 4] = np.frombuffer(np.int32(200).tobytes(), np.uint8)
    assert check(blob_lib, b)[0] is not None


def test_loop_closure_rules(blob_lib):
    n = 20
    ok = dict(n_poses=n, window=list(range(n)))
    assert check(blob_lib, make(blob_lib, with_loops(**ok, factors=loop_factors(n, [(12, 12, 1)]))))[0] is None
    bad = {
        "missing key frame": with_loops(**ok, keyframes=[(i, 1, 1, 1) for i in range(n) if i != 4]),
        "n_est < n_poses": with_loops(**ok, n_est=n - 1),
        "n_est > n_poses": with_loops(**ok, n_est=n + 1),
        "prior not first": with_loops(**ok, factors=[(0, 1), (0, -1)] + loop_factors(n)[2:]),
        "no prior": with_loops(**ok, factors=loop_factors(n)[1:]),
        "second prior": with_loops(**ok, factors=loop_factors(n) + [(0, -1)], n_loop=0),
        "chain out of order": with_loops(**ok, factors=[(0, -1), (1, 2), (0, 1)] + loop_factors(n)[3:]),
        "chain missing": with_loops(**ok, factors=loop_factors(n)[:-1]),
        "chain past the poses": with_loops(**ok, factors=loop_factors(n) + [(n - 1, n)]),
        "loop end out of range": with_loops(**ok, factors=loop_factors(n) + [(n, 3)], n_loop=1),
        "loop end negative": with_loops(**ok, factors=loop_factors(n) + [(5, -2)], n_loop=1),
        "loop count": with_loops(**ok, factors=loop_factors(n, [(12, 12, 1)]), n_loop=2),
        "closed without a loop factor": with_loops(**ok, factors=loop_factors(n), closed=1),
        "closed flag": with_loops(**ok, factors=loop_factors(n, [(12, 12, 1)]), closed=2),
    }
    for what, sp in bad.items():
        assert check(blob_lib, make(blob_lib, sp))[0] is not None, what


@pytest.mark.parametrize("where", ["R", "t", "var", "est"])
@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf])
def test_non_finite_values_rejected(blob_lib, where, value):
    buf = make(blob_lib, with_loops(n_poses=10, window=list(range(10))))
    assert check(blob_lib, buf)[0] is None
    if where == "est":
        off = section(buf, K_EST)[0] + 96 * 3 + 8 * 10
    else:
        off = section(buf, K_FACTORS)[0] + FACTOR_BYTES * 4 + 8 + 8 * dict(R=4, t=9 + 2, var=12 + 5)[where]
    buf[off: off + 8] = np.frombuffer(np.float64(value).tobytes(), np.uint8)
    assert check(blob_lib, buf)[0] is not None


@pytest.mark.parametrize("value", [0.0, -0.0, -1e-6])
def test_variance_not_positive_rejected(blob_lib, value):
    buf = make(blob_lib, with_loops(n_poses=10, window=list(range(10))))
    off = section(buf, K_FACTORS)[0] + FACTOR_BYTES * 0 + 8 + 8 * (12 + 3)
    buf[off: off + 8] = np.frombuffer(np.float64(value).tobytes(), np.uint8)
    assert check(blob_lib, buf)[0] is not None


def test_odometry_time_must_be_finite(blob_lib):
    buf = make(blob_lib, plain())
    off = section(buf, K_SCALARS)[0] + 40
    buf[off: off + 8] = np.frombuffer(np.float64(np.nan).tobytes(), np.uint8)
    assert check(blob_lib, buf)[0] is not None


def test_sequence_blob_magic_is_not_a_mapper_blob(blob_lib):
    buf = make(blob_lib, plain())
    buf[:8] = np.frombuffer(struct.pack("<Q", 0x544F4C53534E494C), np.uint8)  # "LINSSLOT"
    err, _ = check(blob_lib, buf)
    assert err and "magic" in err
