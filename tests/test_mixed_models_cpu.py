"""CPU suite: the host side of one lidar model per scan — the lins_lidar_models layout, tools/run_bags.py's --lidar-model
(one value or one per bag), and the model table and model_of that bag_replay.replay hands a context (through a fake
context that records its calls)."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, pkg


def test_lidar_models_layout_matches_header(defs, tmp_path):
    T = defs.LinsLidarModels
    assert C.sizeof(T) == 24
    assert (T.n_models.offset, T.models.offset, T.model_of.offset) == (0, 8, 16)
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lins_gpu.h"\n'
                   'int main(){printf("%zu %zu %zu %zu\\n", sizeof(lins_lidar_models), offsetof(lins_lidar_models, n_models),'
                   ' offsetof(lins_lidar_models, models), offsetof(lins_lidar_models, model_of));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    assert [int(x) for x in subprocess.check_output([str(exe)]).split()] == [24, 0, 8, 16]


def _run_bags():
    spec = importlib.util.spec_from_file_location("run_bags", os.path.join(ROOT, "tools", "run_bags.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_run_bags_lidar_model_argument(defs):
    rb = _run_bags()
    vlp, dense = bytes(defs.LinsLidarModel.vlp16()), bytes(defs.LinsLidarModel.dense64())
    assert bytes(rb.lidar_models("0", 3)) == vlp and bytes(rb.lidar_models("1", 1)) == dense
    assert [bytes(m) for m in rb.lidar_models("0,1,1", 3)] == [vlp, dense, dense]
    assert [bytes(m) for m in rb.lidar_models("1, 0", 2)] == [dense, vlp]
    for spec, n in (("0,1", 3), ("0,1,1", 2), ("2", 1), ("0,x", 2), ("", 1)):
        with pytest.raises(ValueError):
            rb.lidar_models(spec, n)
    with pytest.raises(SystemExit):  # (argparse's error exit, before any bag is read)
        rb.main(["a.bag", "b.bag", "--lidar-model", "0,1,0"])


class _Rec:
    """A recording as replay reads it: n scans with no IMU rows and empty data fields."""

    def __init__(self, n):
        self.stamps = np.arange(n, dtype=np.float64)
        self.imu = [np.zeros((0, 7)) for _ in range(n)]
        self.imu_last = np.zeros((n, 6))
        self.data = [np.zeros(0, np.uint8) for _ in range(n)]
        self.layouts = [pkg("ctypes_defs").LinsCloud2Layout() for _ in range(n)]

    def __len__(self):
        return len(self.stamps)


class _FakeGpu:
    """Records the step calls replay makes: ("cloud2", model bytes, None) or ("mixed", [model bytes], model_of)."""

    def __init__(self):
        self.calls, self.restarts = [], []

    def seq_open(self, params, init_params, n):
        self.n = n

    def seq_restart(self, mask):
        self.restarts.append((len(self.calls), list(mask)))

    def seq_step_cloud2(self, step, model=None, fp=None, scan_imu=None, desc=None):
        self.calls.append(("cloud2", bytes(model), None, list(step["present"])))

    def seq_step_cloud2_mixed(self, step, models, model_of, fp=None, scan_imu=None, desc=None):
        self.calls.append(("mixed", [bytes(m) for m in models], list(model_of), list(step["present"])))

    def seq_download(self):
        return dict(status=np.zeros(self.n, np.int32), global_state=np.zeros((self.n, 19)),
                    results=np.zeros(self.n, pkg("ctypes_defs").SCAN_RESULT_DTYPE))

    def seq_download_init(self):
        return dict(fusion_status=np.zeros(self.n, np.int32))


class _Blob:
    def __init__(self):
        self.a = np.zeros(1, np.uint8)

    def get(self, n):
        if len(self.a) < n:
            self.a = np.zeros(n, np.uint8)
        return self.a

    def release(self):
        pass


@pytest.fixture
def br(monkeypatch):
    m = pkg("bag_replay")
    monkeypatch.setattr(m, "_PinnedBlob", _Blob)  # (page-locking needs a device)
    return m


def test_replay_builds_the_table_and_model_of(br, defs):
    vlp, dense = defs.LinsLidarModel.vlp16(), defs.LinsLidarModel.dense64()
    V, D = bytes(vlp), bytes(dense)
    g = _FakeGpu()
    # lengths 2, 3, 1 through 2 slots: rec 0 and 1 first; at step 2 rec 0 has ended and its slot takes rec 2
    br.replay([_Rec(2), _Rec(3), _Rec(1)], 2, model=[vlp, dense, vlp], gpu=g)
    assert g.calls == [("mixed", [V, D], [0, 1], [1, 1]), ("mixed", [V, D], [0, 1], [1, 1]), ("mixed", [V, D], [0, 1], [1, 1])]
    assert g.restarts == [(2, [1, 0])]
    # the dense recording first: the table is in first-use order; a slot without a recording gets entry 0
    g = _FakeGpu()
    br.replay([_Rec(1), _Rec(3), _Rec(1)], 2, model=[dense, vlp, dense], gpu=g)
    assert g.calls == [("mixed", [D, V], [0, 1], [1, 1]), ("mixed", [D, V], [0, 1], [1, 1]), ("mixed", [D, V], [0, 1], [0, 1])]
    assert g.restarts == [(1, [1, 0])]


def test_replay_with_one_model_keeps_seq_step_cloud2(br, defs):
    dense = defs.LinsLidarModel.dense64()
    for model in (dense, [dense, defs.LinsLidarModel.dense64(), dense]):
        g = _FakeGpu()
        br.replay([_Rec(2), _Rec(1), _Rec(1)], 2, model=model, gpu=g)
        assert [c[:3] for c in g.calls] == [("cloud2", bytes(dense), None)] * 2
    g = _FakeGpu()
    br.replay([_Rec(1)], 1, gpu=g)
    assert g.calls == [("cloud2", bytes(defs.LinsLidarModel.vlp16()), None, [1])]
    with pytest.raises(ValueError):
        br.replay([_Rec(1), _Rec(1)], 1, model=[dense], gpu=_FakeGpu())
