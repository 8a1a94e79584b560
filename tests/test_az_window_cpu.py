"""Property test (CPU, numpy float32) of the azimuth window the indexed searches scan (lins_assoc_az.cuh: az_bin,
az_halfwidth, az_window; DESIGN.md §4.1 "Exactness of the search"): a target whose (ring, azimuth) bucket lies outside the
window built for the squared radius U must be farther from the query than sqrt(U) — otherwise a search could miss its
minimum.  numpy's float32 arctan2 / arcsin differ from CUDA's by an ulp or two; the window carries 1e-5 rad and a spare
bin on each side for exactly that, so the property has to hold with either library."""
import numpy as np

from scenes import PI, F, az_bin


def az_halfwidth(U, rho):
    r = np.sqrt(U, dtype=F) * F(1.002) + F(1.0e-5)
    with np.errstate(invalid="ignore", divide="ignore"):
        th = (np.arcsin(np.minimum(r / rho, F(1.0)), dtype=F) + F(1.0e-5)).astype(F)
    return np.where(r < rho, th, F(4.0)).astype(F)


def az_window(nb, aq, th):
    inv_binw = F(nb) * (F(0.5) / PI)
    nbins = (F(2.0) * th * inv_binw).astype(np.int64) + 3
    whole = ~(th < PI) | (nbins >= nb)
    b = np.floor((aq - th + PI) * inv_binw).astype(np.int64) - 1
    b = np.mod(b, nb)
    return np.where(whole, 0, b), np.where(whole, nb, nbins)


def test_targets_outside_the_window_are_beyond_the_radius():
    rng = np.random.default_rng(3)
    checked = 0
    for nb in (64, 256, 1024):
        for trial in range(200):
            # a query anywhere (also close to the sensor axis), a radius from millimetres to the 5 m gate
            rho_q = F(10 ** rng.uniform(-2, 2))
            aq_true = rng.uniform(-np.pi, np.pi)
            q = np.array([rho_q * np.cos(aq_true), rho_q * np.sin(aq_true), rng.uniform(-3, 3)], dtype=F)
            U = F(10 ** rng.uniform(-6, np.log10(25.0)))
            aq = np.arctan2(q[1], q[0]).astype(F)
            rho = np.sqrt(q[0] * q[0] + q[1] * q[1], dtype=F)
            blo, nbins = az_window(nb, aq, az_halfwidth(U, rho))
            # targets: a shell around the query at ~the radius (the adversarial distance), plus points all around the sensor
            n = 4000
            dirs = rng.standard_normal((n, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
            shell = q[None, :] + (dirs * np.sqrt(U) * rng.uniform(0.5, 1.2, (n, 1))).astype(F)
            ring = np.stack([rho_q * np.cos(a := rng.uniform(-np.pi, np.pi, n)), rho_q * np.sin(a), np.full(n, q[2])], -1)
            t = np.concatenate([shell, ring]).astype(F)
            tb = az_bin(t[:, 0], t[:, 1], nb)
            inside = np.mod(tb - blo, nb) < nbins
            d2 = ((t.astype(np.float64) - q.astype(np.float64)) ** 2).sum(1)
            bad = ~inside & (d2 <= float(U))
            assert not bad.any(), (nb, q, U, t[bad][:3], d2[bad][:3], int(blo), int(nbins))
            checked += int((~inside).sum())
    assert checked > 100000  # (the windows are not trivially the whole ring)
