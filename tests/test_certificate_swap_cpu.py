"""The certificate rule of the fused kernel with swaps (lins_assoc_az.cuh: cert_check), checked on a numpy model with exact
f32 keys: of the two stored front-runners re-evaluated at the query's new position, the one with the smaller key is the
answer of a search there if its distance + moved + 2e-4 m < bound (bound = the third best distance at the search
position), whether it is the old winner or the runner-up.  Covers both key forms the kernel uses — the closest point's
(distance, index) and the walks' (distance, visiting order) — three-way near-ties, queries sliding along a ring, steps
from 1e-4 m to 0.3 m and winners that leave the gate.  The rule must never certify an answer that differs from brute
force, must certify strictly more than the rule without swaps, and must fail when the displacement or the 2e-4 m slack
is left out."""
import numpy as np

f32 = np.float32
GATE = f32(25.0)
SLACK = f32(2e-4)


def sqd(q, T):
    d = (q[None, :] - T).astype(f32)
    return ((d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def keys(q, T, lo):
    return (sqd(q, T).view(np.uint32).astype(np.uint64) << np.uint64(32)) | lo


def scene(rng, trial):
    """targets, query at the search position and the query after one step"""
    kind = trial % 4
    if kind == 0:  # a ring of 10 m radius, points 3.5 cm apart, query sliding along it
        n = int(rng.integers(5, 40))
        a0 = rng.uniform(-np.pi, np.pi)
        ang = a0 + np.arange(n) * 0.0035
        T = np.stack([10 * np.cos(ang), 10 * np.sin(ang), np.full(n, -1.5)], 1).astype(f32)
        T = T[rng.permutation(n)]
        k = rng.uniform(1, n - 2)
        p0 = np.array([10 * np.cos(a0 + k * 0.0035), 10 * np.sin(a0 + k * 0.0035), -1.5], f32) + rng.standard_normal(3).astype(f32) * f32(0.01)
        t = np.array([-np.sin(a0 + k * 0.0035), np.cos(a0 + k * 0.0035), 0.0])  # along the ring
        step = t * rng.uniform(-1, 1) * 10 ** rng.uniform(-4, np.log10(0.3)) + rng.standard_normal(3) * 1e-4
    else:
        n = int(rng.integers(3, 60))
        T = (rng.standard_normal((n, 3)) * rng.uniform(0.05, 3.0)).astype(f32)
        p0 = (rng.standard_normal(3) * 0.5).astype(f32)
        if kind == 1:  # near-tie between two targets
            p0 = ((T[0] + T[1]) / 2 + rng.standard_normal(3).astype(f32) * f32(1e-3)).astype(f32)
        elif kind == 2:  # three-way near-tie: three targets on a small circle around the query
            c = rng.standard_normal(3).astype(f32)
            r = rng.uniform(0.02, 0.5)
            for j in range(3):
                u = rng.standard_normal(3)
                T[j] = (c + r * u / np.linalg.norm(u) + rng.standard_normal(3) * 1e-5).astype(f32)
            p0 = c
        else:  # far away: the winner can leave the gate
            p0 = (p0 + rng.standard_normal(3) * 4.5).astype(f32)
        step = rng.standard_normal(3) * 10 ** rng.uniform(-4, np.log10(0.3))
    return T, p0, (p0 + step.astype(f32)).astype(f32)


def rule(p0, p1, T, lo, slack=SLACK, swap=True, use_moved=True):
    """-> certified answer (index into T) or None, and the brute-force answer at p1"""
    k0 = keys(p0, T, lo)
    order = np.argsort(k0)
    w, r = int(order[0]), int(order[1])
    bound = np.sqrt(sqd(p0, T)[order[2]])
    moved = np.sqrt(sqd(p1, p0[None, :])[0]) if use_moved else f32(0)
    k1 = keys(p1, T, lo)
    m = r if k1[r] < k1[w] else w
    if m != w and not swap:
        return None
    dm = sqd(p1, T)[m]
    ok = bool(dm < GATE) and bool(np.sqrt(dm) + moved + slack < bound)
    return (m if ok else None), int(np.argmin(k1))


def run(slack=SLACK, swap=True, use_moved=True, seed=11, trials=6000):
    rng = np.random.default_rng(seed)
    certified = swaps = wrong = 0
    for trial in range(trials):
        T, p0, p1 = scene(rng, trial)
        n = len(T)
        # closest point: (distance, index); walks: (distance, visiting order) with a random closest point c
        c = int(rng.integers(0, n))
        j = np.arange(n, dtype=np.int64)
        walk_lo = np.where(j > c, j - c - 1, n + (c - j)).astype(np.uint64)  # forward first, then backward
        for lo in (np.arange(n, dtype=np.uint64), walk_lo):
            out = rule(p0, p1, T, lo, slack, swap, use_moved)
            if out is None:
                continue
            got, truth = out
            if got is None:
                continue
            certified += 1
            swaps += got != int(np.argmin(keys(p0, T, lo)))
            wrong += got != truth
    return certified, swaps, wrong


def test_swap_rule_never_certifies_a_changed_answer_and_certifies_more():
    certified, swaps, wrong = run()
    assert wrong == 0
    base, base_swaps, base_wrong = run(swap=False)
    assert base_wrong == 0 and base_swaps == 0
    assert certified > base and swaps > 200, (certified, base, swaps)


def test_rule_without_the_displacement_is_caught():
    # the displacement since the search is what keeps a certified answer exact once the query moves: without it the
    # model certifies answers brute force does not return
    _, _, wrong = run(use_moved=False)
    assert wrong > 0


def test_rule_without_the_slack_is_caught():
    # f32 rounding of the distances: the query moves by one ulp (2 um) between three targets at almost the same distance.
    # Without the 2e-4 m slack the rule certifies the swapped runner-up although brute force returns another target;
    # with it, the case is searched.  (Found by a seeded random search over such geometries.)
    p0 = np.array([-17.841394424438477, 20.866867065429688, 35.89086151123047], f32)
    p1 = np.array([-17.841392517089844, 20.866867065429688, 35.89086151123047], f32)
    T = np.array([[-16.392593383789062, 21.100555419921875, 35.977596282958984],
                  [-17.55706214904785, 20.94627571105957, 34.450721740722656],
                  [-19.29019546508789, 20.633180618286133, 35.80412673950195]], f32)
    lo = np.arange(3, dtype=np.uint64)
    got, truth = rule(p0, p1, T, lo, slack=f32(0))
    assert got is not None and got != truth
    got, truth = rule(p0, p1, T, lo)
    assert got is None
