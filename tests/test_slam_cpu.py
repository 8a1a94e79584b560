"""CPU suite: sequence mode's publish step restated (tests/slamref.py) — globalStateYZX_ bit for bit against the library's
header (csrc/host/global_state_yzx.hpp, compiled here with g++) and against scipy's rotations, and publishTopics' rule
over status sequences that reach every row of its table."""
import os
import subprocess

import numpy as np
import pytest

import slamref as sr
from conftest import ROOT


def _states(n, seed):
    rng = np.random.default_rng(seed)
    rn = rng.normal(scale=rng.choice([1e-3, 1.0, 50.0, 3e3], n)[:, None], size=(n, 3))
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[:4] = [[0, 0, 0, 1], [1, 0, 0, 0], [0, 0.6, 0.8, 0], [0, 0, 0, -1]]  # (identity, half turns, -identity)
    rn[0] = 0.0
    return rn, q


def test_yzx_pose_matches_the_header_bit_for_bit(tmp_path):
    rn, q = _states(4000, 11)
    inp = tmp_path / "in.bin"
    np.concatenate([rn, q], 1).astype(np.float64).tofile(inp)
    src = tmp_path / "t.cpp"
    src.write_text('#include <cstdio>\n#include "global_state_yzx.hpp"\n'
                   'int main(int, char** v) { FILE* f = std::fopen(v[1], "rb"); FILE* o = std::fopen(v[2], "wb"); double r[7], out[7];\n'
                   '  while (std::fread(r, sizeof(double), 7, f) == 7) { lins::global_state_yzx(r, r + 3, out, out + 3); std::fwrite(out, sizeof(double), 7, o); }\n'
                   '  std::fclose(f); std::fclose(o); return 0; }\n')
    exe = tmp_path / "t"
    host = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "host")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", host, "-o", str(exe), str(src)])
    subprocess.check_call([str(exe), str(inp), str(tmp_path / "out.bin")])
    got = np.fromfile(tmp_path / "out.bin", np.float64).reshape(-1, 7)
    want = sr.yzx_pose(rn, q)
    assert got.tobytes() == want.tobytes()


def test_yzx_pose_against_scipy():
    from scipy.spatial.transform import Rotation as R

    rn, q = _states(2000, 12)
    got = sr.yzx_pose(rn, q)
    P = np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0]], float)  # (x, y, z) -> (y, z, x)
    assert np.abs(got[:, :3] - rn @ P.T).max() <= 1e-15 * np.maximum(1.0, np.abs(rn).max())
    Rq = R.from_matrix(P @ R.from_quat(q).as_matrix() @ P.T).as_matrix()
    assert np.abs(R.from_quat(got[:, 3:]).as_matrix() - Rq).max() < 1e-15 * 8
    assert np.abs(np.linalg.norm(got[:, 3:], axis=1) - 1).max() < 1e-15 * 4
    # the identity stays the identity exactly
    assert sr.yzx_pose(np.zeros(3), np.array([0, 0, 0, 1.0])).tolist() == [0, 0, 0, 0, 0, 0, 1]


def _run(seq):
    """Drive one slot through [(code or 'restart')], tracking StateEstimator::status_ as processPCL does; returns the
    (fusion before, code, published?, pose, cloud sizes) rows."""
    p = sr.Publisher(1)
    fusion, rows, k = sr.FUSION_INIT, [], 0
    for code in seq:
        if code == "restart":
            p.restart(0)
            fusion = sr.FUSION_INIT
            continue
        k += 1
        g = np.zeros(19)
        g[0:3] = (k, 2 * k, 3 * k)
        g[9] = 1.0
        c = np.full((k, 4), k, np.float32)
        out = p.step(0, fusion, code, g, c[:1], c[:2], c[:3])
        rows.append((fusion, code, out is not None, None if out is None else out[0], None if out is None else [len(x) for x in out[1:]]))
        if code == sr.INIT_WAIT:
            fusion = sr.FUSION_INIT
        elif code == sr.FIRST:
            fusion = sr.FUSION_FIRST_SCAN
        elif code == sr.SECOND:
            fusion = sr.FUSION_RUNNING
    return rows


def test_publish_rule_reaches_every_row():
    I, F, Rn = sr.FUSION_INIT, sr.FUSION_FIRST_SCAN, sr.FUSION_RUNNING
    ident = [0, 0, 0, 0, 0, 0, 1]
    rows = _run([sr.INIT_WAIT, sr.FIRST, sr.INIT_WAIT, sr.FIRST, sr.SECOND, sr.RAN, sr.SKIPPED, sr.ICP, sr.IDLE, sr.RAN,
                 "restart", sr.IDLE, sr.FIRST, sr.SECOND])
    seen = {(f, c) for f, c, *_ in rows}
    assert {(I, sr.INIT_WAIT), (I, sr.FIRST), (F, sr.SECOND), (F, sr.INIT_WAIT), (Rn, sr.RAN), (Rn, sr.ICP), (Rn, sr.SKIPPED),
            (Rn, sr.IDLE), (I, sr.IDLE)} <= seen
    pub = [r[2] for r in rows]
    assert pub == [False, False, True, False, True, True, True, True, False, True, False, False, True]
    # FIRST_SCAN -> INIT_WAIT: the empty clouds of the fresh scan, the identity pose
    assert rows[2][3].tolist() == ident and rows[2][4] == [0, 0, 0]
    # SECOND: its clouds and pose (scan 5: rn = (5, 10, 15) -> YZX (10, 15, 5))
    assert rows[4][4] == [1, 2, 3] and rows[4][3][:3].tolist() == [10.0, 15.0, 5.0]
    # SKIPPED republishes the previous clouds and pose
    assert rows[6][4] == rows[5][4] and rows[6][3].tolist() == rows[5][3].tolist()
    assert rows[7][4] == [1, 2, 3] and rows[7][3][:3].tolist() == [16.0, 24.0, 8.0]
    # an absent slot publishes nothing; after a restart the next first scan / second scan start again
    assert rows[11][4] is None and rows[12][4] == [1, 2, 3] and rows[12][3][:3].tolist() == [26.0, 39.0, 13.0]


def test_restart_forgets_the_published_state():
    p = sr.Publisher(2)
    c = np.ones((3, 4), np.float32)
    g = np.zeros(19); g[0] = 4.0; g[9] = 1.0
    p.step(0, sr.FUSION_FIRST_SCAN, sr.SECOND, g, c, c, c)
    p.step(1, sr.FUSION_FIRST_SCAN, sr.SECOND, g, c, c, c)
    p.restart(0)
    out0 = p.step(0, sr.FUSION_FIRST_SCAN, sr.INIT_WAIT)
    out1 = p.step(1, sr.FUSION_RUNNING, sr.SKIPPED)
    assert out0[0].tolist() == [0, 0, 0, 0, 0, 0, 1] and [len(x) for x in out0[1:]] == [0, 0, 0]
    assert out1[0][:3].tolist() == [0.0, 0.0, 4.0] and [len(x) for x in out1[1:]] == [3, 3, 3]
    # the clouds are permuted to (y, z, x, intensity)
    a = np.arange(8, dtype=np.float32).reshape(2, 4)
    assert sr.to_yzx(a).tolist() == [[1, 2, 0, 3], [5, 6, 4, 7]]
