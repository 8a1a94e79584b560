"""Generates tests/golden/blob_format.json (run from the repo root: python tests/golden/make_blob_format_golden.py): the
section tables, synthetic blob digests and validator messages tests/test_blob_format_cpu.py checks, from the blob
format headers as the tree holds them (g++ only)."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_blob_format_cpu as tb  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as d:
        out = tb.record(tb.compile_formats(d))
    with open(tb.FIXTURE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", tb.FIXTURE)


if __name__ == "__main__":
    main()
