"""Property test (CPU, numpy float32) of the block rule of the grid 5-NN (lins_map.cuh grid_cell; DESIGN.md §4.4).  The
grid scans the 3 x 3 x 3 block of 1 m cells around a query's cell and is exact for every point the 1 m gate can accept
only if EVERY map point whose f32 distance is < 1 lies within one cell of the query on every axis.  The GPU suite checks
the consequence on scenes (test_gpu_map_grid.py); this checks the rule itself on a million pairs placed at cell faces,
where f32 rounding decides.

The former rule, floorf of the f32 difference x - ox, breaks near a power of two from a negative origin: the worked
example below is pinned as a pair it put two cells apart.  The device now floors the difference taken in f64."""
import numpy as np

import mapref

F = np.float32


def _nudge(v, steps):
    """v moved by `steps` ulps (per element, |steps| <= 8)."""
    v = v.copy()
    for _ in range(8):
        mv = steps != 0
        v = np.where(mv, np.nextafter(v, np.where(steps > 0, F(np.inf), F(-np.inf)), dtype=F), v)
        steps = steps - np.sign(steps)
    return v


def _pairs(rng, n):
    """Query / neighbour pairs snapped to cell faces: origins of both signs with |o| from 0.1 to 1e5 m, queries within
    a few ulps of o + k, neighbours either anywhere within 1 m or within a few ulps of query +- 1 on one axis."""
    o = (np.where(rng.random((n, 3)) < 0.7, -1.0, 1.0) * 10.0 ** rng.uniform(-1, 5, (n, 3))).astype(F)
    k = np.floor(10.0 ** rng.uniform(0, 5, (n, 3)) * np.where(rng.random((n, 3)) < 0.8, 1.0, -1.0))
    p2 = 2.0 ** rng.integers(0, 17, (n, 3))
    k = np.where(rng.random((n, 3)) < 0.5, p2, k)  # powers of two from the origin
    # a third of the origins near -k, where coordinates resolve finer than the difference and rounding moves cells
    o = np.where((rng.random(n) < 0.33)[:, None] & (k == p2), (-k * rng.uniform(0.5, 1.5, (n, 3))).astype(F), o)
    q = _nudge((o.astype(np.float64) + k).astype(F), rng.integers(-8, 9, (n, 3)))
    near = (q + rng.uniform(-1, 1, (n, 3)) * F(0.577)).astype(F)
    axis = rng.integers(0, 3, n)
    edge = q.copy()
    sgn = np.where(rng.random(n) < 0.5, F(1), F(-1))
    r = np.arange(n)
    edge[r, axis] = _nudge((q[r, axis] + sgn).astype(F), rng.integers(-8, 2, n) * sgn.astype(np.int64))
    small = (rng.normal(0, 1e-4, (n, 3)) * (rng.random((n, 3)) < 0.3)).astype(F)
    small[r, axis] = 0
    edge = (edge + small).astype(F)
    m = np.where((rng.random(n) < 0.4)[:, None], near, edge)
    return o, q, m


def test_exact_cells_put_every_pair_within_one_metre_in_the_block():
    rng = np.random.default_rng(20)
    total = within = former_misses = 0
    for _ in range(10):
        o, q, m = _pairs(rng, 100_000)
        d = mapref.sqdist(q, m)
        sel = d < F(1)
        gap = np.abs(mapref.cell_exact(m, o) - mapref.cell_exact(q, o))
        bad = sel & (gap > 1).any(1)
        assert not bad.any(), (o[bad][:3], q[bad][:3], m[bad][:3])
        former = np.abs(mapref.cell_f32(m, o) - mapref.cell_f32(q, o))
        former_misses += int((sel & (former > 1).any(1)).sum())
        total += len(q)
        within += int(sel.sum())
    assert total >= 1_000_000 and within >= 500_000
    # the sample reaches the faces where rounding decides: the former rule misses many of these pairs
    assert former_misses >= 100, former_misses


def test_the_worked_example_is_outside_the_former_block_and_inside_the_new_one():
    o = np.array([-50, 0, 0], F)
    q = np.array([[14 - 3 * 2.0 ** -20, 0.5, 0.5]], F)
    m = np.array([[15 - 2.0 ** -18, 0.5, 0.5]], F)
    assert q[0, 0] == F(14 - 3 * 2.0 ** -20) and m[0, 0] == F(15 - 2.0 ** -18)  # (both exact in f32)
    d = mapref.sqdist(q, m)[0]
    assert d < F(1) and d == F(1 - 2.0 ** -19)
    assert F(q[0, 0] - o[0]) == F(64 - 2.0 ** -18) and F(m[0, 0] - o[0]) == F(65)
    assert mapref.cell_f32(q, o)[0, 0] == 63 and mapref.cell_f32(m, o)[0, 0] == 65  # two cells apart: missed
    assert mapref.cell_exact(q, o)[0, 0] == 63 and mapref.cell_exact(m, o)[0, 0] == 64


def test_saturated_cells_stay_adjacent():
    """Beyond 2^31 m from the origin the cell saturates; the block arithmetic wraps in uint32, so a saturated query's
    block still holds its saturated neighbours (and NaN -> cell 0)."""
    o = np.zeros(3, F)
    q = np.array([[2.0 ** 31 + 4096, 0, 0], [-(2.0 ** 31) - 4096, 0, 0], [1e30, 0, 0], [np.nan, 0, 0]], F)
    c = mapref.cell_exact(q, o)
    assert c[0, 0] == mapref.INT_MAX and c[1, 0] == mapref.INT_MIN and c[2, 0] == mapref.INT_MAX and c[3, 0] == 0
    nb = 4096
    own = mapref.grid_hash(c) & np.uint64(nb - 1)
    assert all(own[i] in mapref.block_buckets(c[i], nb) for i in range(len(c)))
