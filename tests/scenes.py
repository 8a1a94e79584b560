"""Scene builders and the parity comparison shared by the GPU parity modules (test_gpu_fuzz.py, test_gpu_paths.py).

Every builder returns units as dicts of the four clouds (POINT_DTYPE, intensity = ring + fraction) + prior state and
covariance, the layout of ctypes_defs.Batch.unit().  test_scene_builders_cpu.py checks on the host that each builder
produces what its GPU test claims to exercise (ring range, ring order, target counts, bucket occupancy, duplicates).
Nothing here needs a GPU.
"""
import concurrent.futures as cf
import os

import numpy as np

STATE_TOL = 1e-7
LINS_MAX_ITER = 64

# ---- numpy mirror of the kernel's index limits (lins_kernels.cuh, lins_assoc_az.cuh) ----------------------------------
K_MAX_RING = 128         # kMaxRing: rings outside [0, 128) take the legacy path
K_AZ_TAB_S, K_AZ_TAB_C = 4096, 1024  # kAzTabS / kAzTabC: (ring, azimuth-bin) table entries
K_MAX_T = 65536          # the indexed path needs T < 65536 (16-bit bucket tables and counters)
F = np.float32
PI = F(3.14159265358979)


def az_bin(x, y, nb):
    """lins_assoc_az.cuh az_bin in float32 (numpy's atan2 may differ from CUDA's by an ulp: keep test points off the
    bin edges)."""
    a = np.arctan2(np.asarray(y, F), np.asarray(x, F)).astype(F)
    b = np.floor((a + PI) * (F(nb) * (F(0.5) / PI))).astype(np.int64)
    return np.clip(b, 0, nb - 1)


def az_bins_for(nrings, tab):
    p2 = 1
    while p2 < nrings:
        p2 <<= 1
    return tab // p2


def rings_of(cloud):
    """int(intensity) as the C cast computes it (truncation towards zero)."""
    return cloud["intensity"].astype(np.int32)


def cloud_indexable(cloud):
    """check_ring_sorted + the T bound of unit_prologue for one target cloud."""
    r = rings_of(cloud)
    return len(cloud) < K_MAX_T and bool(((r >= 0) & (r < K_MAX_RING)).all()) and bool((np.diff(r) >= 0).all())


def unit_indexed(u):
    """Does the kernel take the indexed path for this unit (both target clouds indexable)?"""
    return cloud_indexable(u["surf_less_flat"]) and cloud_indexable(u["corner_less_sharp"])


def has_exact_duplicates(cloud):
    xyz = np.stack([cloud["x"], cloud["y"], cloud["z"]], 1)
    return len(xyz) > 0 and len(np.unique(xyz, axis=0)) < len(xyz)


def bucket_counts(cloud, tab):
    """Targets per (ring, azimuth-bin) bucket, b = ring * nb + bin, of an indexable cloud; also returns nb."""
    r = rings_of(cloud)
    nb = az_bins_for(int(r.max()) + 1, tab)
    b = r.astype(np.int64) * nb + az_bin(cloud["x"], cloud["y"], nb)
    return np.bincount(b, minlength=(int(r.max()) + 1) * nb), nb


# ---- batches -----------------------------------------------------------------------------------------------------------
def batch_from_units(defs, units):
    clouds, offsets = {}, {}
    for k in defs.Batch.FIELDS:
        parts = [u[k] for u in units]
        clouds[k] = np.concatenate(parts) if parts else np.zeros(0, defs.POINT_DTYPE)
        offsets[k] = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
    return defs.Batch(clouds, offsets, np.stack([u["state"] for u in units]), np.stack([u["cov"] for u in units]))


def copy_unit(u):
    return {k: (v.copy() if hasattr(v, "copy") else v) for k, v in u.items()}


# ---- the fuzz scenes ---------------------------------------------------------------------------------------------------
def dup_targets(rng, cloud, frac):
    """Insert exact copies of a fraction of the points right after the original (keeps the ring order)."""
    n = len(cloud)
    if n == 0:
        return cloud
    pick = np.sort(rng.choice(n, size=max(1, int(frac * n)), replace=False))
    reps = np.ones(n, int)
    reps[pick] += rng.integers(1, 3, len(pick))
    return np.repeat(cloud, reps)


def mutate(rng, u, kind):
    u = copy_unit(u)
    if kind == "dup":
        u["surf_less_flat"] = dup_targets(rng, u["surf_less_flat"], 0.15)
        u["corner_less_sharp"] = dup_targets(rng, u["corner_less_sharp"], 0.3)
    elif kind == "axis":  # queries at rho < 0.1 m and a few targets near the axis too
        for k in ("surf_flat", "corner_sharp"):
            q = u[k]
            m = rng.random(len(q)) < 0.08
            q["x"][m] = rng.uniform(-0.05, 0.05, m.sum()).astype(np.float32)
            q["y"][m] = rng.uniform(-0.05, 0.05, m.sum()).astype(np.float32)
            q["z"][m] = rng.uniform(-2.0, 2.0, m.sum()).astype(np.float32)
        t = u["surf_less_flat"]
        m = rng.random(len(t)) < 0.01
        t["x"][m] = rng.uniform(-0.08, 0.08, m.sum()).astype(np.float32)
        t["y"][m] = rng.uniform(-0.08, 0.08, m.sum()).astype(np.float32)
    elif kind == "jump":  # prior 1-4 m / up to 0.1 rad off with a covariance that lets the update move that far
        st = u["state"]
        st[0:3] += rng.normal(0, 1.0, 3) * rng.uniform(1.0, 4.0)
        ax = rng.normal(0, 0.03, 3)
        th = np.linalg.norm(ax)
        dq = np.r_[ax / th * np.sin(th / 2), np.cos(th / 2)]
        x1, y1, z1, w1 = st[6:10]
        x2, y2, z2, w2 = dq
        st[6:10] = [w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                    w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2]
        P = u["cov"].reshape(18, 18)
        P[np.arange(3), np.arange(3)] += 4.0
        P[np.arange(6, 9), np.arange(6, 9)] += 0.01
    return u


def random_prior(rng):
    """A prior near the identity pose with a random SPD covariance (column-major, as the ABI takes it)."""
    st = np.zeros(19)
    st[0:3] = rng.normal(0, 0.2, 3)
    ax = rng.normal(0, 0.01, 3)
    th = np.linalg.norm(ax)
    st[6:9] = ax / th * np.sin(th / 2)
    st[9] = np.cos(th / 2)
    st[18] = -9.81
    A = rng.normal(0, 1, (18, 18))
    cov = (A @ A.T) * 1e-4 + np.diag(np.r_[np.full(3, 0.05), np.full(3, 0.01), np.full(3, 1e-3), np.full(9, 1e-4)])
    return st, cov.T.reshape(-1)


def queries_near(rng, tgt, n, sigma=0.3, far_frac=0.1):
    """n queries: targets displaced by N(0, sigma) per axis, a fraction of them 60 m away; ring = the target's ring,
    plus a de-skew fraction in [0, 0.1)."""
    pick = tgt[rng.integers(0, len(tgt), n)].copy()
    for ax in ("x", "y", "z"):
        pick[ax] += rng.normal(0, sigma, n).astype(np.float32)
    far = rng.random(n) < far_frac
    pick["x"][far] += 60.0
    pick["intensity"] = (np.floor(pick["intensity"]) + 0.1 * rng.random(n) * 0.999).astype(np.float32)
    return pick


def random_scene(rng, defs, rings=None, surf_sizes=(0, 3, 25, 300, 1500), corner_sizes=(0, 2, 6, 80, 400)):
    """A small random unit: ring-sorted targets (on 1..40 rings, or on the given ring set), sometimes empty / tiny clouds,
    queries near and far."""
    nr = int(rng.integers(1, 41)) if rings is None else None
    ring_set = None if rings is None else np.asarray(sorted(rings))

    def cloud(n, spread):
        ring = np.sort(rng.integers(0, nr, n)) if ring_set is None else np.sort(rng.choice(ring_set, n))
        az = rng.uniform(-np.pi, np.pi, n)
        rho = rng.uniform(0.5, 30.0, n) * spread
        xyz = np.stack([rho * np.cos(az), rho * np.sin(az), rng.uniform(-2, 2, n)], 1)
        if n and rng.random() < 0.5:  # quantised coordinates: plenty of exact distance ties
            xyz = np.round(xyz * 4) / 4
        return defs.make_points(xyz, ring + 0.1 * rng.random(n) * 0.999)

    ts = cloud(int(rng.choice(surf_sizes)), 1.0)
    tc = cloud(int(rng.choice(corner_sizes)), 1.0)

    def queries(n, tgt):
        if n == 0 or len(tgt) == 0:
            return cloud(n, 1.0)
        return queries_near(rng, tgt, n)

    qs = queries(int(rng.choice([0, 1, 40, 200])), ts)
    qc = queries(int(rng.choice([0, 1, 20, 90])), tc)
    st, cov = random_prior(rng)
    return dict(surf_flat=qs, corner_sharp=qc, surf_less_flat=ts, corner_less_sharp=tc, state=st, cov=cov)


# ---- multi-beam geometry -----------------------------------------------------------------------------------------------
ELEV_LO, ELEV_HI = np.radians(-25.0), np.radians(15.0)


def beam_elevation(ring, nrings):
    return ELEV_LO + (ELEV_HI - ELEV_LO) * np.asarray(ring, float) / max(nrings - 1, 1)


def box_world(az, el):
    """Ray cast from a sensor 1.7 m above the floor of a 40 m x 24 m walled yard: unit directions -> hit points."""
    d = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], -1)
    with np.errstate(divide="ignore"):
        t = np.minimum(20.0 / np.abs(d[:, 0]), 12.0 / np.abs(d[:, 1]))
        t = np.where(d[:, 2] < 0, np.minimum(t, 1.7 / -d[:, 2]), t)
    return d * np.minimum(t, 80.0)[:, None]


def multibeam_cloud(rng, defs, counts, nrings_geom, noise=0.01):
    """Ring-sorted targets: counts[r] points on ring r (beam elevation spread over -25..+15 deg for nrings_geom beams) at
    random azimuths, in random order within the ring."""
    xyz, ring = [], []
    for r in sorted(counts):
        n = int(counts[r])
        if n == 0:
            continue
        az = rng.uniform(-np.pi, np.pi, n)
        p = box_world(az, np.full(n, beam_elevation(r, nrings_geom))) + rng.normal(0, noise, (n, 3))
        xyz.append(p)
        ring.append(np.full(n, r))
    if not xyz:
        return defs.make_points(np.zeros((0, 3)), [])
    ring = np.concatenate(ring)
    return defs.make_points(np.concatenate(xyz), ring + 0.1 * rng.random(len(ring)) * 0.999)


def multibeam_unit(rng, defs, surf_rings, corner_rings, per_ring_s=40, per_ring_c=8, nq_s=200, nq_c=60):
    """Surf and corner targets on the given ring sets (they may differ) of one sensor, queries 2 cm (per axis) from
    them.  (With 10 cm a 3-ring unit moved ~1 m per iteration for all 30 iterations: such a unit amplifies the last-bit
    differences of equivalent f64 algebra until even the oracle's two gain forms differ by 2e-5 in the residual norm,
    past the 1e-6 bar, while its searches stay identical.)"""
    top = max(max(surf_rings), max(corner_rings)) + 1
    ts = multibeam_cloud(rng, defs, {r: per_ring_s for r in surf_rings}, top)
    tc = multibeam_cloud(rng, defs, {r: per_ring_c for r in corner_rings}, top)
    st, cov = random_prior(rng)
    st[0:3] *= 0.25
    return dict(surf_flat=queries_near(rng, ts, nq_s, 0.02), corner_sharp=queries_near(rng, tc, nq_c, 0.02),
                surf_less_flat=ts, corner_less_sharp=tc, state=st, cov=cov)


# ---- legacy-path units (§1 of test_gpu_paths.py) -----------------------------------------------------------------------
# kind -> what is done to the targets; every kind but "none" and "ring_neg_half" makes the unit take the legacy path
LEGACY_KINDS = ("perm", "ring128", "ring300", "ring_neg", "ring_neg_half", "none")


def legacy_variant(rng, u, kind, dup):
    """A copy of unit u whose targets take the legacy path (or, for "none" / "ring_neg_half", stay indexed)."""
    u = copy_unit(u)
    if dup:
        u["surf_less_flat"] = dup_targets(rng, u["surf_less_flat"], 0.15)
        u["corner_less_sharp"] = dup_targets(rng, u["corner_less_sharp"], 0.3)
    ts, tc = u["surf_less_flat"], u["corner_less_sharp"]
    if kind == "perm":  # both clouds in arbitrary ring order
        u["surf_less_flat"], u["corner_less_sharp"] = ts[rng.permutation(len(ts))], tc[rng.permutation(len(tc))]
    elif kind in ("ring128", "ring300"):  # the last surf target (the largest ring) moves to ring 128 / 300: still sorted
        ts["intensity"][-1] = (128.0 if kind == "ring128" else 300.0) + (ts["intensity"][-1] % 1.0)
    elif kind == "ring_neg":  # first corner target on ring -3.2 (int() = -3): still sorted, below range
        tc["intensity"][0] = -3.2
    elif kind == "ring_neg_half":  # control: int(-0.5) = 0, the unit stays indexed
        tc["intensity"][0] = -0.5
    return u


def legacy_batch_units(rng, defs, base, n_random):
    """Every unit of `base` (a synth Batch) and n_random random scenes, each in every LEGACY_KINDS variant, interleaved by
    kind; about a third with exact duplicate targets.  Returns (units, tags)."""
    srcs = [base.unit(i) for i in range(base.n)]
    srcs += [random_scene(rng, defs, rings=range(int(rng.integers(2, 41))), surf_sizes=(25, 300, 1500), corner_sizes=(25, 80, 400))
             for _ in range(n_random)]  # (two rings at least: a permutation must break the ring order)
    units, tags = [], []
    for j, src in enumerate(srcs):
        for k, kind in enumerate(LEGACY_KINDS):
            dup = (j + k) % 3 == 0
            units.append(legacy_variant(rng, src, kind, dup))
            tags.append(f"{'config3' if j < base.n else 'random'} {kind}{' dup' if dup else ''}")
    return units, tags


# ---- index-capacity units (§2) -----------------------------------------------------------------------------------------
CAP_RINGS = 16


def capacity_cloud(rng, defs, T, nrings=CAP_RINGS):
    """Exactly T ring-sorted targets spread evenly over nrings rings."""
    counts = {r: T // nrings + (1 if r < T % nrings else 0) for r in range(nrings)}
    return multibeam_cloud(rng, defs, counts, nrings)


def capacity_unit(rng, defs, Ts, Tc):
    ts, tc = capacity_cloud(rng, defs, Ts), capacity_cloud(rng, defs, Tc)
    st, cov = random_prior(rng)
    st[0:3] *= 0.25
    return dict(surf_flat=queries_near(rng, ts, 300, 0.1), corner_sharp=queries_near(rng, tc, 100, 0.1),
                surf_less_flat=ts, corner_less_sharp=tc, state=st, cov=cov)


BIG_RING = 7


def big_bucket_unit(rng, defs, which, parity, n_big=40000, n_dup=1500, n_nb=2500, n_ring=1000, n_other=800, nrings=CAP_RINGS):
    """One (ring, azimuth-bin) bucket b of the `which` ("surf" / "corner") targets with n_big + n_dup >= 40 000 targets
    (n_dup of them exact copies, adjacent to their original) and bucket b ^ 1 — the other 16-bit half of b's counter
    word — with n_nb targets; b % 2 == parity.  The rest of ring BIG_RING and the other rings hold a few targets each.
    Queries: near the big bucket, exact copies of its duplicated targets, near bucket b ^ 1 and on the edge between the
    two.  Returns (unit, b)."""
    nb = az_bins_for(nrings, K_AZ_TAB_S if which == "surf" else K_AZ_TAB_C)
    k = nb // 2 - 8 + parity
    binw = 2 * np.pi / nb
    el = beam_elevation(BIG_RING, nrings)

    def in_bin(kk, n, lo=0.1, hi=0.9):  # azimuths well inside bin kk, ranges 4..30 m on ring BIG_RING
        az = -np.pi + binw * (kk + rng.uniform(lo, hi, n))
        rho = rng.uniform(4.0, 30.0, n)
        return np.stack([rho * np.cos(az), rho * np.sin(az), rho * np.tan(el) + rng.normal(0, 0.02, n)], 1)

    big = in_bin(k, n_big)
    reps = np.ones(n_big, int)
    reps[rng.choice(n_big, n_dup, replace=False)] += 1
    big = np.repeat(big, reps, axis=0)
    nbr = in_bin(k ^ 1, n_nb)
    az = rng.uniform(-np.pi, np.pi, 4 * n_ring)
    rest = box_world(az, np.full(len(az), el))
    rest = rest[np.abs(az_bin(rest[:, 0], rest[:, 1], nb) - k) > 2][:n_ring]  # the rest of the ring, away from both buckets
    ring_xyz = np.concatenate([big, nbr, rest])
    ring_pts = defs.make_points(ring_xyz, BIG_RING + 0.1 * rng.random(len(ring_xyz)) * 0.999)
    below = multibeam_cloud(rng, defs, {r: n_other for r in range(BIG_RING)}, nrings)
    above = multibeam_cloud(rng, defs, {r: n_other for r in range(BIG_RING + 1, nrings)}, nrings)
    tgt = np.concatenate([below, ring_pts, above])
    other = multibeam_cloud(rng, defs, {r: 40 for r in range(nrings)}, nrings)

    # queries: 200 near the big bucket, 60 exact copies of duplicated targets, 60 near bucket b ^ 1, 60 on the shared edge
    off = len(below)
    starts = np.r_[0, np.cumsum(reps)[:-1]]  # first copy of each big-bucket target
    dup_first = off + starts[reps > 1]
    q_big = tgt[off + rng.integers(0, len(big), 200)].copy()
    for a in ("x", "y", "z"):
        q_big[a] += rng.normal(0, 0.05, 200).astype(np.float32)
    q_tie = tgt[rng.choice(dup_first, 60, replace=False)].copy()
    q_nb = tgt[off + len(big) + rng.integers(0, n_nb, 60)].copy()
    for a in ("x", "y", "z"):
        q_nb[a] += rng.normal(0, 0.05, 60).astype(np.float32)
    edge = -np.pi + binw * max(k, k ^ 1) + rng.uniform(-0.02, 0.02, 60) * binw
    rho = rng.uniform(4.0, 30.0, 60)
    q_edge = defs.make_points(np.stack([rho * np.cos(edge), rho * np.sin(edge), rho * np.tan(el)], 1), np.full(60, float(BIG_RING)))
    q = np.concatenate([q_big, q_tie, q_nb, q_edge])
    q["intensity"] = (np.floor(q["intensity"]) + 0.1 * rng.random(len(q)) * 0.999).astype(np.float32)
    q_other = queries_near(rng, other, 60, 0.1)
    st, cov = random_prior(rng)
    st[0:3] *= 0.1
    st[6:9] *= 0.1
    st[9] = np.sqrt(1.0 - (st[6:9] ** 2).sum())
    u = dict(state=st, cov=cov)
    if which == "surf":
        u.update(surf_flat=q, corner_sharp=q_other, surf_less_flat=tgt, corner_less_sharp=other)
    else:
        u.update(surf_flat=q_other, corner_sharp=q, surf_less_flat=other, corner_less_sharp=tgt)
    return u, BIG_RING * nb + k


# ---- ring-count sweep (§3) ---------------------------------------------------------------------------------------------
# rings 0 .. n-1: every change of the bins per ring (az_bins_for: 4096 / next_pow2(n) surf, 1024 / next_pow2(n) corner),
# 8 and 16 rings, and n = 128 (top ring 127, the last one the 7-bit ring field of a slot word holds)
SWEEP_NRINGS = (1, 2, 3, 5, 8, 9, 16, 17, 33, 64, 65, 100, 127, 128)


def ring_sweep_cases():
    """(name, surf ring set, corner ring set): every ring count of SWEEP_NRINGS on both clouds, a top ring of 128 (legacy),
    sparse sets, and clouds with different ring counts in one unit."""
    cases = [(f"nrings {n}", list(range(n)), list(range(n))) for n in SWEEP_NRINGS]
    cases += [("top ring 128", list(range(129)), list(range(129))), ("rings {0, 127}", [0, 127], [0, 127]),
              ("every 7th ring", list(range(0, 128, 7)), list(range(0, 128, 7))), ("surf 64 / corner 9", list(range(64)), list(range(9))),
              ("surf 17 / corner 100", list(range(17)), list(range(100))), ("surf top ring 128 / corner 8", list(range(129)), list(range(8)))]
    return cases


def ring_sweep_units(rng, defs, per_case_beam=3, per_case_random=2):
    """Per case: multi-beam units and random scenes whose target clouds both reach their case's top ring."""
    units, tags = [], []
    for name, rs, rc in ring_sweep_cases():
        for _ in range(per_case_beam):
            units.append(multibeam_unit(rng, defs, rs, rc, per_ring_s=max(8, 2400 // len(rs)), per_ring_c=max(2, 300 // len(rc))))
            tags.append(f"{name} beams")
        for _ in range(per_case_random):
            u = random_scene(rng, defs, rings=rs, surf_sizes=(300, 1500), corner_sizes=(80, 400))
            tc = random_scene(rng, defs, rings=rc, surf_sizes=(80, 400))["surf_less_flat"]
            u["corner_less_sharp"] = tc
            u["surf_flat"] = queries_near(rng, u["surf_less_flat"], 200, 0.1)
            u["corner_sharp"] = queries_near(rng, tc, 60, 0.1)
            for k, top in (("surf_less_flat", max(rs)), ("corner_less_sharp", max(rc))):  # reach the top ring
                u[k]["intensity"][-1] = top + (u[k]["intensity"][-1] % 1.0)
            units.append(u)
            tags.append(f"{name} random")
    return units, tags


# ---- the oracle and the comparison -------------------------------------------------------------------------------------
def oracle_run(ob, prm, u, use_kdtree=False):
    """The oracle's run of one unit: report, final state and the last iteration's correspondence IDs."""
    o = ob.Oracle(prm, use_kdtree=use_kdtree)  # brute force: exact 1-NN, lowest index among ties (kd-tree: same answers)
    o.set_map(u["surf_less_flat"], u["corner_less_sharp"])
    so, co, rep, tr = o.ieskf_trace(u["surf_flat"], u["corner_sharp"], u["state"], u["cov"])
    out = dict(state=so, cov=co, rep=rep, iters=rep.iters, flags=(rep.converged | (rep.diverged << 1) | (rep.has_nan << 2)),
               m_surf=list(rep.m_surf[: rep.iters]), m_corner=list(rep.m_corner[: rep.iters]),
               rnorm=np.array(rep.residual_norm[: rep.iters]), lin_state=tr["lin_state"],
               surf_ind=tr["surf_ind"][-1] if rep.iters else None, corner_ind=tr["corner_ind"][-1] if rep.iters else None)
    o.close()
    return out


def oracle_runs(ob, prm, units, use_kdtree=False):
    with cf.ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 4)) as ex:
        return list(ex.map(lambda u: oracle_run(ob, prm, u, use_kdtree), units))


def gpu_batch_run(gpu, batch):
    """One lins_gpu_ieskf_batch pass: states, covariances, result records, reports and the last iteration's IDs."""
    gpu.batch_upload(batch)
    gpu.batch_run()
    sg, cg, rg, reps = gpu.batch_download(states=True, covs=True, reports=True)
    si, ci = gpu.batch_download_indices(batch)
    return dict(state=sg, cov=cg, res=rg, reps=reps, surf_ind=si, corner_ind=ci)


def compare_units(units, outs, g, batch, tag_of, state_tol=STATE_TOL):
    """The parity bar of the fuzz test, unit by unit: iteration count and flags, per-iteration accepted-measurement
    counts, residual norms (rtol 1e-9 over the first three iterations, 1e-6 over all), the last iteration's
    correspondence IDs bit-equal, the posterior within state_tol when converged (1e-5 after the last iteration otherwise),
    the prior when diverged.  Returns (mismatches, stats)."""
    rg, reps, sg, si, ci = g["res"], g["reps"], g["state"], g["surf_ind"], g["corner_ind"]
    so_off, co_off = batch.offsets["surf_flat"], batch.offsets["corner_sharp"]
    st = dict(n_div=0, n_jump=0, worst=0.0, worst_nc=0.0)
    bad = []
    for i, o in enumerate(outs):
        tag = tag_of(i)
        r = reps[i]
        n_it = o["iters"]
        if int(rg["iters"][i]) != n_it or int(rg["flags"][i]) != o["flags"]:
            bad.append((tag, "iters / flags", int(rg["iters"][i]), n_it, int(rg["flags"][i]), o["flags"]))
            continue
        if list(r.m_surf[:n_it]) != o["m_surf"] or list(r.m_corner[:n_it]) != o["m_corner"]:
            bad.append((tag, "accepted-measurement counts"))
            continue
        # residual norms: equal to f64 summation order while the iteration is contracting; a unit that never converges
        # (random scenes, 30 iterations) amplifies the 1e-15 differences of the f64 algebra from pass to pass
        rn_g, rn_o = np.array(r.residual_norm[:n_it]), o["rnorm"]
        if not (np.allclose(rn_g[:3], rn_o[:3], rtol=1e-9, atol=1e-300, equal_nan=True) and np.allclose(rn_g, rn_o, rtol=1e-6, atol=1e-300, equal_nan=True)):
            bad.append((tag, "residual norms", float(np.nanmax(np.abs(rn_g - rn_o) / np.maximum(np.abs(rn_o), 1e-300)))))
            continue
        if n_it and not (np.array_equal(si[so_off[i] : so_off[i + 1]], o["surf_ind"]) and np.array_equal(ci[co_off[i] : co_off[i + 1]], o["corner_ind"])):
            bad.append((tag, "correspondence IDs of the last iteration"))
            continue
        if o["flags"] & 2:
            st["n_div"] += 1
            if not np.allclose(sg[i], units[i]["state"], equal_nan=True):
                bad.append((tag, "diverged unit must return the prior"))
        else:
            d = float(np.abs(sg[i] - o["state"]).max())
            conv = bool(o["flags"] & 1)
            if conv:
                st["worst"] = max(st["worst"], d)
            else:
                st["worst_nc"] = max(st["worst_nc"], d)
            if d > (state_tol if conv else 1e-5):  # (north_star: 1e-4)
                bad.append((tag, "state", d, "converged" if conv else "not converged"))
        un = np.array(r.update_norm[:n_it])
        if len(un) and un.max() > 1.0:
            st["n_jump"] += 1
    return bad, st


def single_mismatches(u, sg, rep, o, state_tol=STATE_TOL):
    """compare_units' bar for one lins_gpu_ieskf call (its IDs are checked through lins_gpu_associate instead)."""
    n_it = o["iters"]
    flags = rep.converged | (rep.diverged << 1) | (rep.has_nan << 2)
    if rep.iters != n_it or flags != o["flags"]:
        return [("iters / flags", rep.iters, n_it, flags, o["flags"])]
    bad = []
    if list(rep.m_surf[:n_it]) != o["m_surf"] or list(rep.m_corner[:n_it]) != o["m_corner"]:
        bad.append("accepted-measurement counts")
    rn_g, rn_o = np.array(rep.residual_norm[:n_it]), o["rnorm"]
    if not (np.allclose(rn_g[:3], rn_o[:3], rtol=1e-9, atol=1e-300, equal_nan=True) and np.allclose(rn_g, rn_o, rtol=1e-6, atol=1e-300, equal_nan=True)):
        bad.append("residual norms")
    if o["flags"] & 2:
        if not np.allclose(sg, u["state"], equal_nan=True):
            bad.append("diverged unit must return the prior")
    elif np.abs(sg - o["state"]).max() > (state_tol if o["flags"] & 1 else 1e-5):
        bad.append(("state", float(np.abs(sg - o["state"]).max())))
    return bad


def assoc_mismatches(g, o):
    """Keys on which two association outputs differ: pointSel, IDs and masks bit-exact, coefficients to f32 rounding."""
    bad = [k for k in ("surf_sel", "corner_sel", "surf_ind", "corner_ind", "surf_mask", "corner_mask") if not np.array_equal(g[k], o[k])]
    bad += [k for k in ("surf_coeff", "corner_coeff") if not np.allclose(g[k], o[k], rtol=2e-6, atol=1e-9)]
    return bad
