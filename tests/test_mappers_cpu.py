"""CPU suite for the lockstep mappers (lins_gpu_mappers_*): the lins_mappers_desc mirror against the header, compiled
with the system C compiler, and the CSR packing of per-slot clouds that capi.LinsGpu.mappers_step hands to the library."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT


def test_mappers_desc_matches_header(defs):
    fields = ("n_slots", "present", "time", "quat", "pos", "corner", "corner_off", "surf", "surf_off", "outlier", "outlier_off")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "lins_gpu.h"\nint main(){printf("%zu' + ' %zu' * len(fields) + '\\n", sizeof(lins_mappers_desc)'
           + "".join(f", offsetof(lins_mappers_desc, {f})" for f in fields) + ");return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "s"), os.path.join(d, "s.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert got == [C.sizeof(defs.LinsMappersDesc)] + [getattr(defs.LinsMappersDesc, f).offset for f in fields]


def test_pack_csr_of_per_slot_clouds(capi, defs):
    rng = np.random.default_rng(2)
    clouds = [rng.standard_normal((n, 8)).astype(np.float32) for n in (3, 0, 5)]
    clouds.insert(1, None)  # an absent slot: no points
    pts, off = capi.pack_csr(clouds)
    assert pts.dtype == defs.POINT_DTYPE and pts.flags["C_CONTIGUOUS"]
    assert off.dtype == np.int32 and off.tolist() == [0, 3, 3, 3, 8]
    for s, c in enumerate(clouds):
        want = np.zeros((0, 8), np.float32) if c is None else c
        assert np.array_equal(pts[off[s]:off[s + 1]].view(np.float32).reshape(-1, 8), want)
    pts, off = capi.pack_csr([None, None])
    assert len(pts) == 0 and off.tolist() == [0, 0, 0]
