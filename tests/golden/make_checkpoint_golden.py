"""Generates tests/golden/checkpoint_sha256.json on a machine with an H100 (run from the repo root:
python tests/golden/make_checkpoint_golden.py): the length and SHA-256 of the blobs tests/test_gpu_blob_bytes.py saves,
with the library as the tree builds it."""
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_gpu_blob_bytes as tb  # noqa: E402


def main(path=tb.FIXTURE):
    pkg = "lins---lidar-inertial-slam_b200"
    capi, defs, synth = (importlib.import_module(f"{pkg}.{m}") for m in ("capi", "ctypes_defs", "synth"))
    synth.build()
    out = tb.digests(capi, defs, synth)
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", path, {k: len(v) for k, v in out.items()})


if __name__ == "__main__":
    main(*sys.argv[1:])
