"""GPU: the split Jacobian kernel (lins_jacobian_mma_kernel through lins_gpu_batch_jacobian_pass) against jacref.

Every unit's 30 outputs are compared, with no unit skipped:
  * counts exact, except +-1 per marginal row of that kind (jacref: an f32 rounding a few f64 ulps from a tie);
  * each sum e: |got - ref| <= (n_rows + 16) 2^-52 A_e + sum over marginal rows of |a_i b_i|' (jacref.JacRef.bound);
  * over the module, marginal rows are fewer than 1e-4 of all rows, so the test cannot pass by excusing rows.

How much the bound leaves a wrong kernel, measured by perturbing the reference by hand and comparing it with itself on
the four golden units (IDs of the oracle's association at the prior, 218-273 rows each; the bound on sum r r is about
6e-14 of it): dropping one accepted row misses the worst sum's bound by a factor of 1.5e11 to 3e12, swapping g3 / g4 by
9e11 to 1.4e12, the unweighted rule in a weighted pass by 9e13 to 1.2e15.  A dropped trip, a transposed MMA fragment or
a wrong weight is at least as large.
"""
import ctypes as C
import time

import numpy as np
import pytest

import jacref

pytestmark = pytest.mark.gpu

TALLY = dict(units=0, rows=0, marginal=0, parts=set())


@pytest.fixture(scope="module", autouse=True)
def tally():
    t0 = time.time()
    yield TALLY
    print(f"\njacobian pass vs jacref: P reached {sorted(TALLY['parts'])}, {TALLY['units']} units, {TALLY['rows']} rows, "
          f"{TALLY['marginal']} marginal rows, {time.time() - t0:.1f} s")
    assert TALLY["marginal"] < 1e-4 * TALLY["rows"]


@pytest.fixture(scope="module")
def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def parts(n, sm):
    from conftest import pkg

    L = pkg("capi").lib()
    L.lins_jacobian_parts.argtypes = [C.c_int, C.c_int]
    return int(L.lins_jacobian_parts(n, sm))


def sizes_by_parts(sm):
    """{P: the batch sizes lins_jacobian_parts cuts into P parts}, up to 16 units per resident warp."""
    by_p = {}
    for n in range(1, 16 * sm * 8):
        by_p.setdefault(parts(n, sm), []).append(n)
    return by_p


@pytest.fixture(scope="module")
def pool(synth):
    """1000 config-3 units: the bench's batch."""
    return synth.generate("config3", 1000)


def make_batch(defs, units):
    """A Batch of unit dicts (the four clouds, state, cov)."""
    clouds, offsets = {}, {}
    for k in defs.Batch.FIELDS:
        parts_ = [defs.as_points(u[k]) for u in units]
        clouds[k] = np.concatenate(parts_) if parts_ else np.zeros(0, defs.POINT_DTYPE)
        offsets[k] = np.concatenate([[0], np.cumsum([len(p) for p in parts_])]).astype(np.int32)
    return defs.Batch(clouds, offsets, np.array([u["state"] for u in units]), np.array([u["cov"] for u in units]))


def run_pass(gpu, ob, batch, pass_prm=None, run_prm=None):
    """upload -> run -> download (states, IDs) -> [set_params] -> jacobian pass.  Returns (accum, jacref)."""
    run_prm = run_prm or ob.LinsParams.shipped()
    gpu.set_params(run_prm)
    gpu.batch_upload(batch)
    gpu.batch_run()
    so, _, _, _ = gpu.batch_download(covs=False)
    si, ci = gpu.batch_download_indices(batch)
    pass_prm = pass_prm or run_prm
    gpu.set_params(pass_prm)
    acc = gpu.batch_jacobian_pass(want_accum=True)
    return acc, jacref.reference(batch, si, ci, so, pass_prm)


def check(acc, jr, what, sm=None):
    """Every unit's 30 outputs within the bound; tallies units, rows, marginal rows and the part count."""
    d = np.abs(acc[:, :28] - jr.sums)
    b = jr.bound()
    bad = ~(d <= b)
    if bad.any():
        u, e = np.unravel_index(np.argmax(np.where(bad, d / np.maximum(b, 1e-300), 0)), d.shape)
        raise AssertionError(f"{what}: {bad.sum()} sums of {bad.any(1).sum()} units beyond the bound; worst unit {u} entry {e}: "
                             f"got {acc[u, e]!r} ref {jr.sums[u, e]!r} |diff| {d[u, e]:.3e} bound {b[u, e]:.3e} "
                             f"(rows {jr.n_rows[u]}, accepted {jr.counts[u].tolist()}, marginal {jr.marginal[u].tolist()})")
    dc = np.abs(acc[:, 28:30] - jr.counts)
    assert (dc <= jr.marginal).all(), f"{what}: counts differ in units {np.nonzero((dc > jr.marginal).any(1))[0][:10]}"
    TALLY["units"] += jr.n
    TALLY["rows"] += int(jr.n_rows.sum())
    TALLY["marginal"] += int(jr.marginal.sum())
    if sm is not None:
        TALLY["parts"].add(parts(jr.n, sm))
    print(f"{what}: {jr.n} units, {int(jr.n_rows.sum())} rows, {int(jr.counts.sum())} accepted, {int(jr.marginal.sum())} marginal")


def test_every_part_count(gpu, ob, pool, sm_count):
    """Batch sizes that cut each unit into P = 4, 3, 2 and 1 parts (lins_jacobian_parts: the largest batch of each P > 1,
    the smallest of P = 1), so every merge path through part_acc / part_cnt and the direct write run."""
    by_p = sizes_by_parts(sm_count)
    assert {1, 2, 3, 4} <= set(by_p), sorted(by_p)
    big = pool.tile(2)
    for P, n in ((4, max(by_p[4])), (3, max(by_p[3])), (2, max(by_p[2])), (1, min(by_p[1]))):
        b = big.subset(range(n)) if n <= big.n else big.tile(-(-n // big.n)).subset(range(n))
        acc, jr = run_pass(gpu, ob, b)
        assert parts(b.n, sm_count) == P
        check(acc, jr, f"P = {P} (n = {n})", sm_count)


def test_bench_shape(gpu, ob, pool, sm_count):
    """bench.py's roofline_jacobian batch: the 1000 units tiled five times, every unit, one part each."""
    b = pool.tile(5)
    assert parts(b.n, sm_count) == 1
    acc, jr = run_pass(gpu, ob, b)
    check(acc, jr, "bench shape", sm_count)


def _shaped_units(defs, pool, P):
    """Units whose query count ns + nc hits a trip boundary (0, 1, 31 .. 65, 32 P +- 1), plus ns = 0, nc = 0, an empty
    unit and a unit whose queries all lie 100 m from the map (every ID -1, every row rejected)."""
    out, zero = [], []
    totals = [0, 1, 31, 32, 33, 63, 64, 65, 32 * P - 1, 32 * P, 32 * P + 1]
    for j, t in enumerate(totals):
        u = dict(pool.unit(3 + j))
        ns = min(len(u["surf_flat"]), (t + 1) // 2)
        u["surf_flat"], u["corner_sharp"] = u["surf_flat"][:ns], u["corner_sharp"][: t - ns]
        assert len(u["surf_flat"]) + len(u["corner_sharp"]) == t
        out.append(u)
    u = dict(pool.unit(20)); u["surf_flat"] = u["surf_flat"][:0]; out.append(u)
    u = dict(pool.unit(21)); u["corner_sharp"] = u["corner_sharp"][:0]; out.append(u)
    u = dict(pool.unit(22))
    for k in defs.Batch.FIELDS:
        u[k] = u[k][:0]
    zero.append(len(out)); out.append(u)
    u = dict(pool.unit(23))
    for k in ("surf_flat", "corner_sharp"):
        u[k] = u[k].copy(); u[k]["x"] += 100.0
    zero.append(len(out)); out.append(u)
    return out, zero


@pytest.mark.parametrize("P", [4, 1])
def test_trip_tails_and_empty_units(gpu, ob, defs, pool, sm_count, P):
    """The shaped units mixed with full ones, in a batch cut into 4 parts and in one of single parts."""
    shaped, zero = _shaped_units(defs, pool, P)
    fill = [pool.unit(i) for i in range(100, 110)] if P == 4 else [pool.unit(i % pool.n) for i in range(100, 100 + 2 * sm_count * 8)]
    units = []
    for i, u in enumerate(shaped):  # spread the shaped units over the batch
        units.append(u)
        units.extend(fill[i * len(fill) // len(shaped):(i + 1) * len(fill) // len(shaped)])
    zero = [next(k for k, v in enumerate(units) if v is shaped[z]) for z in zero]
    b = make_batch(defs, units)
    assert parts(b.n, sm_count) == P
    acc, jr = run_pass(gpu, ob, b)
    check(acc, jr, f"trip tails, P = {P}", sm_count)
    si, ci = gpu.batch_download_indices(b)
    assert (si[b.offsets["surf_flat"][zero[1]]:b.offsets["surf_flat"][zero[1] + 1]] == -1).any()
    for z in zero:
        assert (acc[z] == 0).all(), (z, acc[z])


def test_unmatched_and_far_queries(gpu, ob, defs, pool, sm_count):
    """A third of the queries displaced by 40 m: their IDs are -1 and their rows rejected; the rest still count."""
    units, far = [], []
    for i in range(40):
        u = dict(pool.unit(200 + i))
        for k in ("surf_flat", "corner_sharp"):
            u[k] = u[k].copy(); u[k]["x"][::3] += 40.0
        far.append(np.arange(len(u["surf_flat"])) % 3 == 0)
        units.append(u)
    far = np.concatenate(far)
    b = make_batch(defs, units)
    acc, jr = run_pass(gpu, ob, b)
    si, ci = gpu.batch_download_indices(b)
    assert (si[far] == -1).any(axis=1).mean() > 0.9 and (ci == -1).any()
    assert not jr.surf["mask"][(si == -1).any(axis=1)].any() and jr.counts.sum() > 0
    check(acc, jr, "unmatched", sm_count)


@pytest.mark.parametrize("kw", [dict(icp_freq=2), dict(lidar_scale=2.5), dict(scan_period=0.002, icp_freq=2)],
                         ids=["unweighted", "lidar_scale", "exact_sincos"])
def test_pass_parameters(gpu, ob, pool, sm_count, kw):
    """set_params between batch_run and the pass: the unweighted rule, lidar_scale, and a scan period short enough that
    |half angle| >= 1/8, so the kernel takes sincos instead of the Taylor polynomials."""
    b = pool.subset(range(300, 364))
    acc, jr = run_pass(gpu, ob, b, pass_prm=ob.LinsParams.shipped(**kw))
    if "scan_period" in kw:
        half = np.concatenate([jr.surf["half"][jr.surf["mask"]], jr.corner["half"][jr.corner["mask"]]])
        assert (half >= 0.125).sum() > 100, half.max()
    check(acc, jr, f"parameters {kw}", sm_count)


def test_negative_time_points(gpu, ob, defs, pool, sm_count):
    """Half the queries with a negative fractional intensity (-0.1 .. -0.2) and a pass scan period of 1 ms: s down to
    -200, half angles down to about -3 rad.  The kernel must rotate them by sincos, like axis2Quat; its Taylor polynomials
    are only accurate for |half| < 1/8."""
    units = []
    for i in range(64):
        u = dict(pool.unit(400 + i))
        for k in ("surf_flat", "corner_sharp"):
            u[k] = u[k].copy()
            u[k]["intensity"][1::2] = -(u[k]["intensity"][1::2] + np.float32(0.1))
        units.append(u)
    b = make_batch(defs, units)
    acc, jr = run_pass(gpu, ob, b, pass_prm=ob.LinsParams.shipped(scan_period=0.001, icp_freq=2))
    half = np.concatenate([jr.surf["half"][jr.surf["mask"]], jr.corner["half"][jr.corner["mask"]]])
    assert (half <= -0.125).sum() > 1000 and half.min() < -2.0, half.min()
    check(acc, jr, "negative time", sm_count)


def test_determinism_and_part_reset(gpu, ob, defs, pool, sm_count):
    """Two passes are bit-equal; the same units in a 4-part and a 1-part batch agree within the bound; a pass after a
    different pass (other weights, other batch size) is still right, so part_cnt is reset."""
    small = pool.subset(range(500, 524))
    assert parts(small.n, sm_count) == 4
    acc4, jr4 = run_pass(gpu, ob, small)
    again = gpu.batch_jacobian_pass(want_accum=True)
    assert np.array_equal(acc4, again)
    gpu.set_params(ob.LinsParams.shipped(icp_freq=2))
    unw = gpu.batch_jacobian_pass(want_accum=True)
    so, _, _, _ = gpu.batch_download(covs=False)
    si, ci = gpu.batch_download_indices(small)
    check(unw, jacref.reference(small, si, ci, so, ob.LinsParams.shipped(icp_freq=2)), "unweighted after weighted", sm_count)
    gpu.set_params(ob.LinsParams.shipped())
    assert np.array_equal(gpu.batch_jacobian_pass(want_accum=True), acc4)
    # the same 24 units inside a batch of single parts, then the small batch again
    big = pool.subset(list(range(0, 500)) + list(range(500, 524)) + list(range(524, 1000)) + list(range(0, 200)))
    assert parts(big.n, sm_count) == 1
    acc1, jr1 = run_pass(gpu, ob, big)
    check(acc1, jr1, "1-part batch", sm_count)
    assert (np.abs(acc1[500:524] - acc4) <= 2 * np.concatenate([jr4.bound(), jr4.marginal], 1)).all()
    mid = pool.subset(range(max(sizes_by_parts(sm_count)[3])))
    acc_mid, jr_mid = run_pass(gpu, ob, mid)
    check(acc_mid, jr_mid, f"P = {parts(mid.n, sm_count)} batch", sm_count)
    acc4b, _ = run_pass(gpu, ob, small)
    assert np.array_equal(acc4b, acc4)


def test_accum_abi_writes_n_by_30(gpu, ob, pool):
    """lins_gpu_batch_jacobian_pass writes exactly n x 30 doubles (include/lins_gpu.h): a guard band of NaN canaries
    after them survives, and the 30 columns are what the Python wrapper returns."""
    b = pool.subset(range(700, 733))
    gpu.set_params(ob.LinsParams.shipped())
    gpu.batch_upload(b)
    gpu.batch_run()
    n = b.n
    guard = 2 * n + 64  # wide enough that a 32-double row stride would land inside the buffer, on the canaries
    canary = np.uint64(0x7FF8DEADBEEF0001)
    buf = np.zeros(n * 30 + guard, np.float64)
    buf.view(np.uint64)[n * 30:] = canary
    gpu._ck(gpu.L.lins_gpu_batch_jacobian_pass(gpu.h, buf.ctypes.data_as(C.c_void_p)))
    tail = buf.view(np.uint64)[n * 30:]
    assert (tail == canary).all(), f"{int((tail != canary).sum())} of {guard} canaries after the n x 30 buffer overwritten"
    wrapped = gpu.batch_jacobian_pass(want_accum=True)
    assert wrapped.shape == (n, 30)
    assert np.array_equal(buf[: n * 30].reshape(n, 30), wrapped[:, :30])
