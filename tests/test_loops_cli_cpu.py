"""Loop closure's replay options that are refused before any device work: loops without the mapper, and loops with a
checkpoint (a slot with loop closure is not saved)."""
import importlib
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
br = importlib.import_module("lins---lidar-inertial-slam_b200.bag_replay")


@pytest.mark.parametrize("kw", [dict(loops=True), dict(map=True, loops=True, checkpoint="d", checkpoint_every=2),
                                dict(map=True, loops=True, checkpoint="d", stop_after=1), dict(map=True, loops=True, resume="d")])
def test_replay_refuses(kw):
    with pytest.raises(ValueError):
        br.replay([], 1, **kw)


@pytest.mark.parametrize("args", [["--loops"], ["--map", "--loops", "--checkpoint-every", "2", "d"], ["--map", "--loops", "--resume", "d"]])
def test_run_bags_refuses(args, tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_bags.py"), str(tmp_path / "none.bag")] + args,
                       capture_output=True, text=True)
    assert r.returncode == 2 and "--loops" in r.stderr
