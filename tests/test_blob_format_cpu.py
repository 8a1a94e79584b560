"""CPU checks that the sequence-mode slot blob and the mapper blob keep their bytes and their validators' words, against
tests/golden/blob_format.json (tests/golden/make_blob_format_golden.py wrote it when each format had a header of its
own): for each format, the section table and total of a grid of counts (bound and unbound, plain and with loop closure,
zero and large counts), the SHA-256 of the synthetic blobs of the validator tests' writers, and the validator's exact
message for every truncation and every single-bit flip of the header and section table of small blobs.  The writers
and validators are those of test_seq_checkpoint_cpu.py and test_mapper_checkpoint_cpu.py, compiled with g++."""
import ctypes as C
import hashlib
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_mapper_checkpoint_cpu as tm
import test_seq_checkpoint_cpu as ts

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blob_format.json")

# the section table of counts c (seq: bound, n_map[4], n_outlier, n_poses, n_window, n_keyframes, n_kf_points; mapper:
# n_poses, n_window, n_keyframes, n_kf_points, n_factors, n_est) into sec as (offset, bytes) pairs; returns the total
LAYOUT = {
    "seq": r"""
extern "C" uint64_t blob_layout(const int64_t* c, uint64_t* sec) {
  Counts k;
  k.bound = c[0] != 0;
  for (int i = 0; i < 4; ++i) k.n_map[i] = c[1 + i];
  k.n_outlier = c[5]; k.n_poses = c[6]; k.n_window = c[7]; k.n_keyframes = c[8]; k.n_kf_points = c[9];
  Header h;
  layout(k, kSz, h);
  std::memcpy(sec, h.sec, sizeof(h.sec));
  return h.total;
}
""",
    "mapper": r"""
extern "C" uint64_t blob_layout(const int64_t* c, uint64_t* sec) {
  Counts k;
  k.n_poses = c[0]; k.n_window = c[1]; k.n_keyframes = c[2]; k.n_kf_points = c[3]; k.n_factors = c[4]; k.n_est = c[5];
  Header h;
  layout(k, kSz, h);
  std::memcpy(sec, h.sec, sizeof(h.sec));
  return h.total;
}
""",
}
SECTIONS = {"seq": 10, "mapper": 9}
BIG = (1 << 31) - 1
COUNTS = {
    "seq": [[0] * 10, [1] + [0] * 9, [0, 40, 7, 30, 5, 0, 0, 0, 0, 0], [1, 40, 7, 30, 5, 9, 12, 12, 12, 400],
            [1, 1, 0, 0, 0, 0, 1, 1, 1, 1], [1, 3, 3, 3, 3, 3, 60, 50, 51, 7], [0, 1 << 20, 1 << 19, 1 << 18, 1 << 17, 0, 0, 0, 0, 0],
            [1, BIG, BIG, BIG, BIG, BIG, BIG, 50, 51, BIG]],
    "mapper": [[0] * 6, [1, 1, 1, 1, 0, 0], [12, 12, 12, 400, 0, 0], [60, 50, 51, 7, 0, 0], [60, 50, 60, 900, 62, 60],
               [1100, 50, 1100, 1 << 20, 1101, 1100], [BIG, 50, BIG, BIG, BIG, BIG]],
}
SEQ_SPECS = [ts.spec(), ts.spec(flags=0), ts.spec(flags=0, stale=0, n_map=(10, 3, 0, 0)), ts.spec(flags=ts.F_BOUND | ts.F_CONFIGURED | ts.F_TUNED),
             ts.spec(fusion=0, stale=0, n_map=(0, 0, 0, 0), n_poses=0, window=[], keyframes=[]),
             ts.spec(n_poses=52, window=list(range(2, 51)) + [50], keyframes=[(i, 0, 4, 1) for i in range(2, 52)])]
SPECS = {"seq": SEQ_SPECS, "mapper": tm.ACCEPTED}
# the blobs whose truncations and header bit flips are recorded
SMALL = {"seq": [ts.spec(flags=0), ts.spec()], "mapper": [tm.plain(), tm.with_loops(n_poses=8, window=list(range(8)))]}
HEADER_BYTES = {"seq": ts.HEADER_BYTES, "mapper": tm.HEADER_BYTES}


def compile_formats(d):
    """the two writers and validators, each with blob_layout, built in directory d"""
    libs = {}
    for name, mod in (("seq", ts), ("mapper", tm)):
        src, so = os.path.join(d, f"{name}_format.cpp"), os.path.join(d, f"{name}_format.so")
        with open(src, "w") as f:
            f.write("#include <cstdio>\n" + mod.DRIVER + LAYOUT[name])
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC", "-I", ts.CUDA_DIR, "-o", so, src])
        L = C.CDLL(so)
        L.blob_make.restype = C.c_uint64
        L.blob_make.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.blob_check.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
        L.blob_layout.restype = C.c_uint64
        L.blob_layout.argtypes = [C.c_void_p, C.c_void_p]
        libs[name] = L
    return libs


def _runs(msgs):
    """messages as [message, run length] runs"""
    out = []
    for m in msgs:
        if out and out[-1][0] == m:
            out[-1][1] += 1
        else:
            out.append([m, 1])
    return out


def record(libs):
    """what the fixture holds, from the compiled formats"""
    out = {}
    for name, L in libs.items():
        mod = ts if name == "seq" else tm
        layouts = []
        for c in COUNTS[name]:
            ca, sec = np.array(c, np.int64), np.zeros(2 * SECTIONS[name], np.uint64)
            total = L.blob_layout(ca.ctypes.data, sec.ctypes.data)
            layouts.append({"counts": c, "total": int(total), "sections": sec.reshape(-1, 2).tolist()})
        sha = [hashlib.sha256(mod.make(L, sp).tobytes()).hexdigest() for sp in SPECS[name]]
        small = []
        for sp in SMALL[name]:
            buf = mod.make(L, sp)
            trunc = [mod.check(L, buf[:n])[0] for n in range(len(buf))]
            flips = []
            for byte in range(HEADER_BYTES[name]):
                for bit in range(8):
                    b = buf.copy()
                    b[byte] ^= 1 << bit
                    flips.append(mod.check(L, b)[0])
            small.append({"spec": sp, "truncations": _runs(trunc), "bit_flips": _runs(flips)})
        out[name] = {"layouts": layouts, "sha256": sha, "messages": small}
    return out


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ is not available")
    return compile_formats(str(tmp_path_factory.mktemp("formats")))


def test_formats_match_the_fixture(libs):
    with open(FIXTURE) as f:
        want = json.load(f)
    got = record(libs)
    for name in ("seq", "mapper"):
        for k in ("layouts", "sha256", "messages"):
            assert got[name][k] == want[name][k], (name, k)
