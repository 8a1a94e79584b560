"""Certificate counters of the fused kernel's phase timers (lins_assoc.cuh: kCertSlots) on the config3 bench shape: a run
with the timers on computes exactly what a run with them off computes, swaps of the stored front-runners are accepted,
and every checked certificate is either accepted or failed for one reason.  (Parity of the certified answers with the
brute-force oracle is held by test_gpu_fuzz.py and test_gpu_parity.py.)"""
import importlib

import numpy as np
import pytest

capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
synth = importlib.import_module("lins---lidar-inertial-slam_b200.synth")
defs = importlib.import_module("lins---lidar-inertial-slam_b200.ctypes_defs")

CERT_SLOTS = 40


def _run(g, b, timers):
    g.batch_upload(b)
    g.phase_cycles(enable=timers)
    g.batch_run()
    g.sync()
    t = g.phase_cycles(enable=False, read=True) if timers else None
    st, cov, res, _ = g.batch_download(states=True, covs=True)
    si, ci = g.batch_download_indices(b)
    return (st, cov, res, si, ci), t


@pytest.mark.gpu
def test_timers_change_nothing_and_certificate_counters_add_up():
    b = synth.generate("config3", n=200, seed0=1000)
    g = capi.LinsGpu(defs.LinsParams.shipped())
    off, _ = _run(g, b, False)
    on, t = _run(g, b, True)
    for x, y in zip(off, on):
        if isinstance(x, np.ndarray) and x.dtype.names:
            assert x.tobytes() == y.tobytes()
        else:
            assert np.array_equal(x, y)
    for half in (0, 1):  # closest point, walks
        c = [(int(t[CERT_SLOTS + k]) >> (32 * half)) & 0xffffffff for k in range(8)]
        checked, accepted, failed, swaps = c[0], c[1], sum(c[2:6]), c[7]
        assert checked > 0 and checked == accepted + failed, c
        assert 0 < swaps <= accepted, c


@pytest.mark.gpu
def test_swapped_answers_match_the_bruteforce_oracle(gpu, ob, synth, defs):
    # config3 units as the bench runs them and the same units with priors 1-4 m off (certificates must fail, swap and
    # re-search): iteration counts, flags, per-iteration counts and norms and the last iteration's correspondence IDs
    # equal to the brute-force oracle, states within the suite's tolerance
    from scenes import STATE_TOL, batch_from_units, compare_units, gpu_batch_run, mutate, oracle_runs
    rng = np.random.default_rng(20261015)
    prm = ob.LinsParams.shipped()
    gpu.set_params(prm)
    base = synth.generate("config3", n=96, seed0=1000)
    units = [base.unit(i) for i in range(base.n)] + [mutate(rng, base.unit(i), "jump") for i in range(base.n)]
    batch = batch_from_units(defs, units)
    gpu.phase_cycles(enable=True)
    g = gpu_batch_run(gpu, batch)
    t = gpu.phase_cycles(enable=False, read=True)
    outs = oracle_runs(ob, prm, units, use_kdtree=False)
    bad, st = compare_units(units, outs, g, batch, lambda i: f"unit {i} ({'bench' if i < base.n else 'prior off'})", STATE_TOL)
    assert not bad, (len(bad), bad[:10])
    assert st["n_jump"] >= 20, st["n_jump"]
    swaps = [(int(t[CERT_SLOTS + 7]) >> (32 * h)) & 0xffffffff for h in (0, 1)]
    assert min(swaps) > 0, swaps  # the swap path really ran in this batch
