"""GPU suite: parity of the fused IESKF kernel on every search path and at every limit the code declares.

unit_prologue (lins_gpu.cu) sends a unit down the indexed path — the (ring, azimuth-bin) index of lins_assoc_az.cuh —
when both target clouds are ring-sorted, every ring is in [0, 128), there is no stale 1-NN index and Ts, Tc < 65536;
everything else takes the legacy path (brute-force 1-NN + the literal sequential walks, lins_assoc.cuh).  The fuzz test
(test_gpu_fuzz.py) covers the indexed path on ring-sorted clouds of 1-40 rings; this module covers the rest:
  1. legacy units through the whole loop, sharing CTAs with indexed units, at ICP_FREQ 1 / 2 / 3 and 1 / 2 / 3 resident
     units per CTA; the stale-index state and lins_gpu_estimate_transform on a legacy map,
  2. the 16-bit index limits: T = 65535 (indexed) / 65536 (legacy), a bucket of >= 40 000 targets next to a populated
     neighbour half of its counter word,
  3. ring counts 1 ... 128 (every change of the bins per ring, ring 127 indexed, ring 128 legacy), sparse ring sets,
  4. per-query arrays in global scratch (units too large for shared memory),
  5. num_iter = LINS_MAX_ITER with every iteration forced: the report arrays exactly full.
Parity bar (scenes.compare_units): iteration counts and flags, per-iteration accepted-measurement counts and residual
norms, the last iteration's correspondence IDs bit-equal, posterior within 1e-7 when converged; associate() outputs
(pointSel, IDs, masks) bit-exact.  Oracle: brute force, or the kd-tree (exact, same lowest-index tie-break, pinned
against brute force in test_oracle_cpu.py) for the 65 k-target units.
Reference: lins/include/StateEstimator.hpp:844-915, :970-1029 (search + walks), :465-600 (loop), :1156-1160 (map refresh).
"""
import os

import numpy as np
import pytest

import scenes
from scenes import (assoc_mismatches, batch_from_units, compare_units, gpu_batch_run, oracle_runs, single_mismatches)

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-4


def _fresh_ctx(capi, **env):
    """A new context created with the given environment (LINS_SLOTS / LINS_VERBOSE are read by lins_gpu_create)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return capi.LinsGpu()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _assert_batch_parity(what, units, tags, outs, g, batch):
    bad, st = compare_units(units, outs, g, batch, lambda i: f"{what}: unit {i} ({tags[i]})")
    assert not bad, (len(bad), bad[:10])
    return st


def _with_ordinary_units(synth, units, tags, seed0, n=8):
    """The given units interleaved with n config3 units (indexed), so that they share CTAs with ordinary work."""
    base = synth.generate("config3", n=n, seed0=seed0)
    out_u, out_t = [], []
    for i in range(max(n, len(units))):
        if i < n:
            out_u.append(base.unit(i)); out_t.append("config3")
        if i < len(units):
            out_u.append(units[i]); out_t.append(tags[i])
    return out_u, out_t


# ---- 1. legacy path ----------------------------------------------------------------------------------------------------
def test_legacy_units_share_ctas_across_icp_freq_and_slots(capi, ob, synth, defs, capfd):
    """>= 600 units interleaved by kind (permuted targets, a ring of 128 / 300 / -3.2, the -0.5 control and unmodified
    units; a third with exact duplicate targets) through the whole loop, at 1, 2 and 3 resident units per CTA: every
    CTA mixes legacy and indexed units, the legacy walks see exact ties, ICP_FREQ > 1 reuses legacy IDs by original
    index.  Bit-identical across slot counts, equal to the brute-force oracle."""
    rng = np.random.default_rng(20261015)
    base = synth.generate("config3", n=60, seed0=52000)
    units, tags = scenes.legacy_batch_units(rng, defs, base, n_random=40)
    assert len(units) >= 600
    batch = batch_from_units(defs, units)
    ctxs = {s: _fresh_ctx(capi, LINS_SLOTS=str(s), LINS_VERBOSE="1") for s in (1, 2, 3)}
    try:
        for kw in ({}, dict(icp_freq=2), dict(icp_freq=3)):
            prm = ob.LinsParams.shipped(**kw)
            outs = oracle_runs(ob, prm, units)
            ref = None
            for s, ctx in ctxs.items():
                ctx.set_params(prm)
                capfd.readouterr()
                g = gpu_batch_run(ctx, batch)
                err = capfd.readouterr().err
                assert f"slots {s} " in err, err  # (the batch's queries fit shared memory at every slot count)
                _assert_batch_parity(f"icp_freq {prm.icp_freq}, {s} slots", units, tags, outs, g, batch)
                if ref is None:
                    ref = g
                    continue
                for k in ("state", "cov", "surf_ind", "corner_ind"):
                    assert np.array_equal(g[k], ref[k]), (prm.icp_freq, s, k)
                assert np.array_equal(g["res"], ref["res"]), (prm.icp_freq, s)
                assert bytes(g["reps"]) == bytes(ref["reps"]), (prm.icp_freq, s)
    finally:
        for c in ctxs.values():
            c.close()


def test_legacy_associate_reload_and_estimate_transform(gpu, ob, synth, defs):
    """ICP_FREQ = 2 on legacy maps: a fresh associate() at an odd iteration reloads the IDs of the previous call from
    global memory (original indices, not slots), and estimate_transform's odd Gauss-Newton steps do the same."""
    rng = np.random.default_rng(7)
    base = synth.generate("config3", n=2, seed0=53000)
    for i in range(base.n):
        for kind in ("perm", "ring128", "ring_neg"):
            u = scenes.legacy_variant(rng, base.unit(i), kind, dup=True)
            assert not scenes.unit_indexed(u)
            for kw in ({}, dict(icp_freq=2)):
                prm = ob.LinsParams.shipped(**kw)
                gpu.set_params(prm)
                o = ob.Oracle(prm, use_kdtree=False)
                o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
                gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
                st0 = u["state"].copy()
                st1 = st0.copy()
                st1[0:3] += [0.05, -0.02, 0.01]
                for it, st in ((0, st0), (1, st1), (2, st1), (3, st0)):
                    bad = assoc_mismatches(gpu.associate(u["surf_flat"], u["corner_sharp"], st, it), o.associate(u["surf_flat"], u["corner_sharp"], st, it))
                    assert not bad, (i, kind, prm.icp_freq, it, bad)
                t0, q0 = u["state"][:3], u["state"][6:10]
                to, qo, ito, cvo = o.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
                tg, qg, itg, cvg = gpu.estimate_transform(u["surf_flat"], u["corner_sharp"], t0, q0)
                assert (itg, cvg) == (ito, cvo), (i, kind, prm.icp_freq)
                assert np.abs(tg - to).max() <= POSE_TOL and 2 * np.arccos(min(1.0, abs(float(np.dot(qg, qo))))) <= POSE_TOL
                o.close()


@pytest.mark.parametrize("walk", ["smaller", "larger"])
def test_stale_index_through_the_loop(gpu, ob, synth, walk):
    """A map refresh that fails the `>= 5 && >= 20` guard (StateEstimator.hpp:1156-1160) advances the walk clouds but
    not the 1-NN index; the next lins_gpu_ieskf runs the legacy path against the older index.  Walk cloud smaller than
    the index cloud (IDs from the index beyond the walk cloud find nothing) and larger."""
    for seed in (9, 10):
        b = synth.generate("config3", n=1, seed0=seed)
        u = b.unit(0)
        ns, nc = b.extra["new_surf_less_flat"], b.extra["new_corner_less_sharp"]
        ts, tc = u["surf_less_flat"], u["corner_less_sharp"]
        if walk == "larger":
            ts, tc = ts[: len(ts) // 3], tc[: len(tc) // 3]
            ws, wc = ns, nc[:4]
            assert len(ws) > len(ts)
        else:
            ws, wc = ns[:60], nc[:4]
            assert len(ws) < len(ts)
        for kw in ({}, dict(icp_freq=2)):
            prm = ob.LinsParams.shipped(**kw)
            gpu.set_params(prm)
            o = ob.Oracle(prm, use_kdtree=False)
            o.set_map(ts, tc)
            gpu.set_map(ts, tc)
            _, _, rep1 = o.update_map(ws, wc, u["state"])
            _, _, rep2 = gpu.update_map(ws, wc, u["state"])
            assert not rep1 and not rep2
            so, co, rep, tr = o.ieskf_trace(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
            oo = dict(state=so, iters=rep.iters, flags=(rep.converged | (rep.diverged << 1) | (rep.has_nan << 2)),
                      m_surf=list(rep.m_surf[: rep.iters]), m_corner=list(rep.m_corner[: rep.iters]), rnorm=np.array(rep.residual_norm[: rep.iters]))
            sg, cg, rg = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
            bad = single_mismatches(u, sg, rg, oo)
            assert not bad, (seed, walk, prm.icp_freq, bad)
            for k in sorted({0, rep.iters - 1}):  # the search at the first and the last linearisation point
                bad = assoc_mismatches(gpu.associate(u["surf_flat"], u["corner_sharp"], tr["lin_state"][k], k),
                                       o.associate(u["surf_flat"], u["corner_sharp"], tr["lin_state"][k], k))
                assert not bad, (seed, walk, prm.icp_freq, k, bad)
            o.close()


# ---- 2. index capacity -------------------------------------------------------------------------------------------------
def _single_and_batch(gpu, ob, synth, defs, units, tags, seed0):
    """Each unit on its own (set_map + associate at iteration 0 and at a later point of the oracle's trace + ieskf), then
    all of them in one batch with ordinary units.  kd-tree oracle (exact, lowest index among ties)."""
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    outs = oracle_runs(ob, prm, units, use_kdtree=True)
    for u, t, o in zip(units, tags, outs):
        orc = ob.Oracle(prm, use_kdtree=True)
        orc.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        gpu.set_map(u["surf_less_flat"], u["corner_less_sharp"])
        later = min(2, o["iters"] - 1)
        for it, st in ((0, u["state"]), (later, o["lin_state"][later])):
            bad = assoc_mismatches(gpu.associate(u["surf_flat"], u["corner_sharp"], st, it), orc.associate(u["surf_flat"], u["corner_sharp"], st, it))
            assert not bad, (t, it, bad)
        orc.close()
        sg, cg, rg = gpu.ieskf(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
        bad = single_mismatches(u, sg, rg, o)
        assert not bad, (t, bad)
    mixed, mtags = _with_ordinary_units(synth, units, tags, seed0)
    batch = batch_from_units(defs, mixed)
    _assert_batch_parity("batch", mixed, mtags, oracle_runs(ob, prm, mixed, use_kdtree=True), gpu_batch_run(gpu, batch), batch)


def test_target_count_65535_indexed_65536_legacy(gpu, ob, synth, defs):
    """Ts, Tc in {65535, 65536}, all four combinations: 65535 fills the 16-bit bucket table (table[TAB] = 65535), 65536
    switches the unit to the legacy path."""
    rng = np.random.default_rng(65535)
    units, tags = [], []
    for Ts in (65535, 65536):
        for Tc in (65535, 65536):
            u = scenes.capacity_unit(rng, defs, Ts, Tc)
            assert (len(u["surf_less_flat"]), len(u["corner_less_sharp"])) == (Ts, Tc)
            assert scenes.unit_indexed(u) == (Ts < 65536 and Tc < 65536)
            units.append(u)
            tags.append(f"Ts {Ts} Tc {Tc}")
    _single_and_batch(gpu, ob, synth, defs, units, tags, seed0=54000)


def test_bucket_of_40000_targets_next_to_its_counter_half(gpu, ob, synth, defs):
    """One (ring, azimuth-bin) bucket b with >= 40 000 targets (past the top bit of its 16-bit counter half) and bucket
    b ^ 1, the other half of the same counter word, populated; b even and b odd, surf and corner targets.  Queries land in
    the big bucket (exact ties there), in b ^ 1 and on their shared edge."""
    rng = np.random.default_rng(40000)
    units, tags = [], []
    for which in ("surf", "corner"):
        for parity in (0, 1):
            u, b = scenes.big_bucket_unit(rng, defs, which, parity)
            tgt = u["surf_less_flat" if which == "surf" else "corner_less_sharp"]
            cnt, _ = scenes.bucket_counts(tgt, scenes.K_AZ_TAB_S if which == "surf" else scenes.K_AZ_TAB_C)
            assert scenes.unit_indexed(u) and b % 2 == parity and cnt[b] >= 40000 and cnt[b ^ 1] >= 1000, (which, parity)
            units.append(u)
            tags.append(f"{which} bucket {b}")
    _single_and_batch(gpu, ob, synth, defs, units, tags, seed0=55000)


# ---- 3. ring counts ----------------------------------------------------------------------------------------------------
def test_ring_count_sweep(gpu, ob, defs):
    """Rings 0 .. n-1 for n in 1, 2, 3, 5, 8, 9, 16, 17, 33, 64, 65, 100, 127, 128 (indexed: every power-of-two change of
    the bins per ring, 8 and 16 rings, top ring 127 — the last one the 7-bit ring field of a slot word holds), a top ring
    of 128 (legacy), the sparse sets {0, 127} and every 7th ring, and surf / corner clouds with different ring counts;
    multi-beam geometry and random scenes."""
    rng = np.random.default_rng(128)
    units, tags = scenes.ring_sweep_units(rng, defs)
    batch = batch_from_units(defs, units)
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    g = gpu_batch_run(gpu, batch)
    _assert_batch_parity("ring sweep", units, tags, oracle_runs(ob, prm, units), g, batch)


# ---- 4. global scratch -------------------------------------------------------------------------------------------------
def test_per_query_arrays_in_global_scratch(capi, ob, synth, defs, capfd):
    """A batch whose largest unit (config1b: thousands of queries) does not fit shared memory: every CTA keeps its
    per-query arrays in global scratch and stages queries without TMA."""
    b1, b3 = synth.generate("config1b", n=24, seed0=56000), synth.generate("config3", n=24, seed0=57000)
    units, tags = [], []
    for i in range(24):
        units += [b1.unit(i), b3.unit(i)]
        tags += ["config1b", "config3"]
    batch = batch_from_units(defs, units)
    ctx = _fresh_ctx(capi, LINS_VERBOSE="1")
    try:
        for kw in ({}, dict(icp_freq=2)):
            prm = ob.LinsParams.shipped(**kw)
            ctx.set_params(prm)
            capfd.readouterr()
            g = gpu_batch_run(ctx, batch)
            err = capfd.readouterr().err
            assert "(per-query arrays in global scratch)" in err, err
            _assert_batch_parity(f"icp_freq {prm.icp_freq}", units, tags, oracle_runs(ob, prm, units), g, batch)
    finally:
        ctx.close()


# ---- 5. num_iter = LINS_MAX_ITER ---------------------------------------------------------------------------------------
def test_num_iter_64_fills_every_report_entry(gpu, ob, synth, defs):
    """num_iter = 64 with every iteration forced: all 64 entries of every unit's report (neighbouring units' reports
    included) equal the oracle's."""
    rng = np.random.default_rng(64)
    base = synth.generate("config3", n=6, seed0=58000)
    units = [base.unit(i) for i in range(4)]
    units += [scenes.legacy_variant(rng, base.unit(4), "perm", True), scenes.legacy_variant(rng, base.unit(5), "ring128", True)]
    tags = ["config3"] * 4 + ["perm dup", "ring128 dup"]
    prm = ob.LinsParams.shipped(num_iter=scenes.LINS_MAX_ITER, force_all_iters=1)
    gpu.set_params(prm)
    batch = batch_from_units(defs, units)
    g = gpu_batch_run(gpu, batch)
    outs = oracle_runs(ob, prm, units)
    _assert_batch_parity("num_iter 64", units, tags, outs, g, batch)
    for i, o in enumerate(outs):
        r, ro = g["reps"][i], o["rep"]
        assert r.iters == ro.iters == 64 and (r.converged, r.diverged, r.has_nan) == (ro.converged, ro.diverged, ro.has_nan), (i, r.iters, ro.iters)
        assert list(r.m_surf) == list(ro.m_surf) and list(r.m_corner) == list(ro.m_corner), i
        assert np.allclose(r.residual_norm, ro.residual_norm, rtol=1e-6, atol=1e-300), i
        # (update norms shrink to ~1e-12 once the iteration has settled: an absolute floor, still far below any entry
        # that was left unwritten or written by a neighbour)
        assert np.allclose(r.update_norm, ro.update_norm, rtol=1e-6, atol=1e-9), i
