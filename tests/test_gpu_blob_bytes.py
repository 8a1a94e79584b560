"""GPU suite: the bytes of saved blobs stay those of the committed fixture (tests/golden/checkpoint_sha256.json).

The length and SHA-256 of every blob saved at fixed steps of drives the checkpoint suites already run: sequence mode,
unbound and bound; a lockstep mapper slot and the single mapper, each plain and with loop closure (the drifted drive of
test_gpu_loops, saved after its loop has closed).  A library build that writes other bytes for the same run fails here,
so a blob saved by one build loads into any other build that passes."""
import hashlib
import json
import os

import numpy as np
import pytest

import mapper_drive
import rawcases as rc
import test_gpu_loops as tl
import test_gpu_mapper_checkpoint as tm
import test_gpu_seq_checkpoint as ts

pytestmark = pytest.mark.gpu
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "checkpoint_sha256.json")
SEQ_SAVES = (0, 3, 6, 13)  # the steps after which every sequence-mode slot is saved
MAPPER_SAVE_EVERY = 8      # a mapper drive saves after every 8th odometry message and after its last event


def _digest(blob):
    return [len(blob), hashlib.sha256(blob).hexdigest()]


def _seq(capi, defs, logs, bound):
    n = len(logs)
    model = rc.model_of(defs, logs[0])
    g = ts._open(capi, defs, n, bound)
    ts._rig(defs, g, [0, 1], [1, 4], n)
    out = {}
    for t in range(max(len(l["time"]) for l in logs)):
        ts._step(g, logs, t, {j: j for j in range(n)}, n, model, bound)
        if t in SEQ_SAVES:
            out[f"step{t}"] = [_digest(b) for b in g.seq_save(np.ones(n, np.uint8))]
    return out


def _mapper(capi, events, kind, loops, force_close=()):
    """the drive on a fresh node (the single mapper, or slot 2 of 4 lockstep slots), its loop thread ticked once a
    second of drive time as test_gpu_loops ticks it; the digests of its saves, and whether a loop closed before the last"""
    t = tm.new_target(capi, kind, loops=loops)
    out, last_close, odom, closed = {}, None, 0, False
    for i, e in enumerate(events):
        if e[0] == "imu":
            t.imu(e)
        else:
            t.fuse(e)
            t.step(e)
            odom += 1
            if loops and t.rep is not None:
                due = last_close is None or e[1] - last_close >= 1.0
                if due:
                    last_close = e[1]
                if due or e[-1] in force_close:
                    closed |= bool(t.close().accepted)
        if (e[0] != "imu" and odom % MAPPER_SAVE_EVERY == 0) or i == len(events) - 1:
            out[f"event{i}"] = _digest(t.save())
    return out, closed


def digests(capi, defs, synth):
    logs = rc.case_logs(defs, 0, gpu=capi.LinsGpu())[0][:8]
    out = {f"seq_{'bound' if b else 'unbound'}": _seq(capi, defs, logs, b) for b in (False, True)}
    plain = mapper_drive.make_drive(synth, seed=5, sparse_first=3)
    drifted = tl.drifted_drive(synth, stall_at=62)[0]
    for kind in ("lockstep", "single"):
        out[f"{kind}_plain"], _ = _mapper(capi, plain, kind, False)
        out[f"{kind}_loops"], closed = _mapper(capi, drifted, kind, True, force_close={61})
        assert closed, kind
    return out


def test_saved_blobs_match_the_fixture(capi, defs, synth):
    with open(FIXTURE) as f:
        want = json.load(f)
    got = digests(capi, defs, synth)
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k], k
