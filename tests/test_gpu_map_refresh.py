"""GPU suite: the single-scan seam's map (lins_gpu_set_map, lins_gpu_update_map, lins_gpu_update_map_ex) through drives
of calls on both sides of the `>= 5 && >= 20` guard (StateEstimator.hpp:1156-1160): surf 19 / 20, corner 4 / 5, empty
clouds, stale states, an update_map before any set_map, a set_map after a stale state and rejected calls in between.
After every call, lins_gpu_ieskf and lins_gpu_associate against the brute-force oracle taken through the same calls,
the read-back clouds against the oracle's transformToEnd, and the launch count of every call."""

import numpy as np
import pytest

from scenes import assoc_mismatches, single_mismatches

pytestmark = pytest.mark.gpu

# A drive: (call, surf points, corner points) of the new clouds (None: the whole cloud).  "set": set_map; "upd":
# update_map with read-back and the last posterior as lin_state; "dev": update_map_ex on the posterior the last ieskf
# left on the device, no read-back; "bad": an update_map_ex that is rejected (a negative count, a null cloud).
DRIVES = {
    "guard_boundaries": [("set", None, None), ("upd", 19, 5), ("upd", 20, 4), ("upd", 20, 5), ("upd", 19, 4), ("upd", 19, 4),
                         ("dev", 20, 5), ("upd", 0, 0), ("dev", 20, 0), ("upd", 0, 5), ("upd", None, None)],
    "before_set_map": [("upd", 60, 4), ("upd", 19, 5), ("dev", None, None), ("upd", 20, 4)],
    "before_set_map_passing": [("upd", None, None), ("upd", 60, 4)],
    "set_after_stale": [("set", None, None), ("upd", 60, 4), ("dev", 30, 3), ("set", 200, 40), ("upd", 20, 5), ("upd", 19, 5),
                        ("set", None, None)],
    "rejected_in_between": [("set", None, None), ("upd", 60, 4), ("bad", -1, 5), ("upd", 20, 5), ("bad", 5, -1), ("upd", 0, 4),
                            ("bad", 20, None), ("dev", 20, 5)],
}


def _cut(cloud, k):
    return cloud if k is None else cloud[:k]


def _check_readback(g, o):
    for a, c in zip(g, o):
        assert len(a) == len(c)
        A = np.stack([a["x"], a["y"], a["z"]], 1)
        Cc = np.stack([c["x"], c["y"], c["z"]], 1)
        assert np.allclose(A, Cc, rtol=0, atol=2e-6)
        assert np.array_equal(a["intensity"], c["intensity"])


@pytest.mark.parametrize("drive", sorted(DRIVES))
def test_seam_map_refresh_drive(capi, ob, synth, drive):
    b = synth.generate("config3", n=1, seed0=9)
    u = b.unit(0)
    new = (b.extra["new_surf_less_flat"], b.extra["new_corner_less_sharp"])
    prm = ob.LinsParams.shipped()
    g, o = capi.LinsGpu(prm), ob.Oracle(prm, use_kdtree=False)
    try:
        if DRIVES[drive][0][0] != "set":  # no map yet: the single-scan calls fail, and launch nothing
            for call in (lambda: g.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"]),
                         lambda: g.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0),
                         lambda: g.estimate_transform(u["surf_flat"], u["corner_sharp"], u["state"][:3], u["state"][6:10])):
                with pytest.raises(capi.LinsError, match="error -3"):
                    call()
            assert g.launch_count() == 0
        post = np.ascontiguousarray(u["state"], np.float64)
        for step, (op, ks, kc) in enumerate(DRIVES[drive]):
            ctx = (drive, step, op, ks, kc)
            n0 = g.launch_count()
            if op == "set":
                s, c = _cut(u["surf_less_flat"], ks), _cut(u["corner_less_sharp"], kc)
                g.set_map(s, c)
                o.set_map(s, c)
                assert g.launch_count() == n0, ctx
            elif op == "bad":
                # (kc None: a null corner cloud of 20 points)
                rc = g.L.lins_gpu_update_map_ex(g.h, new[0].ctypes.data, ks, None if kc is None else new[1].ctypes.data,
                                                20 if kc is None else kc, post.ctypes.data, None, None, None)
                assert rc == -1, ctx  # LINS_E_INVALID
                assert g.launch_count() == n0, ctx
            else:
                s, c = _cut(new[0], ks), _cut(new[1], kc)
                so, co, rep_o = o.update_map(s, c, post)
                if op == "upd":
                    sg, cg, rep_g = g.update_map(s, c, post)
                    _check_readback((sg, cg), (so, co))
                else:
                    rep_g = g.update_map_device(s, c)
                assert rep_g == rep_o == (len(c) >= 5 and len(s) >= 20), ctx
                assert g.launch_count() == n0 + (len(s) > 0) + (len(c) > 0), ctx
            # the next scan against the map the calls left: association at iteration 0, then the whole IESKF (whose
            # posterior stays on the device for a "dev" call)
            n0 = g.launch_count()
            bad = assoc_mismatches(g.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0),
                                   o.associate(u["surf_flat"], u["corner_sharp"], u["state"], 0))
            assert not bad, (ctx, bad)
            assert g.launch_count() == n0 + 1, ctx
            so, co, rep, tr = o.ieskf_trace(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
            oo = dict(state=so, iters=rep.iters, flags=(rep.converged | (rep.diverged << 1) | (rep.has_nan << 2)),
                      m_surf=list(rep.m_surf[: rep.iters]), m_corner=list(rep.m_corner[: rep.iters]), rnorm=np.array(rep.residual_norm[: rep.iters]))
            sg, cg, rg = g.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
            bad = single_mismatches(u, sg, rg, oo)
            assert not bad, (ctx, bad)
            assert g.launch_count() == n0 + 2, ctx
            post = np.ascontiguousarray(sg)
    finally:
        g.close()
        o.close()
