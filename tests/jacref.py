"""jacref: an independent numpy restatement of the split Jacobian pass (lins_jacobian_mma_kernel, reached through
lins_gpu_batch_jacobian_pass), with exact sums and the tolerance scales its tests use.

For every query of a resident batch it computes what the kernel is specified to compute, from the correspondence IDs
the batch's last search iteration left (batch_download_indices) and the batch's posterior (batch_download's state_out):

  * the de-skew transformToStart (StateEstimator.hpp:1066-1080): fi = w - (float)(int)w, s = (1.f / scan_period) * fi,
    axis2Quat(s * phi) with phi = Quat2axis(q), rotate, add s * rn, round to f32;
  * the plane / line residual (StateEstimator.hpp:917-951, :1031-1060) with the reference's f32 rounding points, the
    robust weight when the pass is weighted (icp_freq == 1: the weight of a search iteration >= 1) and the accept rule
    s > 0.1 && res != 0;
  * the factored Jacobian row g = [c ; p x (R^T c)], r = lidar_scale * coeff.w, with c = coeff.xyz, p the raw query and R
    the posterior's rotation.  The reference's (and the oracle's) row is h = [c ; Rinv^T g_att] with Rinv =
    Rinvleft(-Quat2axis(q)): the fused solve applies that per-unit linear map once to the folded sums (att_map below);

and per unit the 28 sums of the kernel's layout (0..20 the upper triangle of sum g g^T row-major, 21..26 sum g r,
27 sum r r) plus the accepted surf / corner counts.  Per-row arithmetic is float64 in the kernel's operation order,
without multiply-add contraction; each sum is formed in extended precision (np.longdouble, 64-bit mantissa), so its
error is below n * 2^-64 of its condition scale.

Tolerance scales.  For each sum e = sum_i a_i b_i, scale[e] = sum_i |a_i|' |b_i|' where |.|' is the magnitude the row
entry is computed from: |c_k| and |r| for the exact entries (c and r are f32 values the kernel reproduces bit for
bit), and |p| |c| (2-norms) for g_3..5, whose cross product can cancel: a kernel that evaluates R^T c and the cross product
with contraction differs from this one by a few f64 ulps of |p| |c|, not of |g_k|.

Marginal rows.  A row is marginal when one of the f32 roundings in its chain (sel, the plane residual, the line's |P|
and d12, the weight, the three coeff entries) has a float64 argument x within 2^-44 |x| of an f32 rounding midpoint, or,
for an argument formed with cancellation, within 2^-49 (8 f64 ulps) of the magnitude of its terms: |p| + |s rn_k| for
sel, |P0 - P1| for the plane residual, |s| times the cross products' term scale for coeff.  A kernel that differs by a
few f64 ulps there (contraction, the hoisted de-skew axis, Taylor sin / cos) may round such a value the other way and so
change the row or flip its accept decision.  The one exception
is a robust weight exactly on a midpoint: 1.8 |res| of an f32 res often lies on a coarse lattice (9/5 times a short
mantissa), so 1 - 1.8 |res| is an exact f32 midpoint in about 2 % of the line rows; the weight's inputs are f32 values the
kernel reproduces, and both evaluations open to it (with and without contracting 1 - 1.8 |res| into one fma) give that
exact midpoint, which rounds to even either way.  Nothing else is excused: excuse[e] = sum over marginal rows of |a_i|' |b_i|' of the row as it would be accepted.
"""
import math

import numpy as np

N_SUMS = 28
MARGIN = 2.0 ** -44       # of the value itself
MARGIN_SCALE = 2.0 ** -49  # of the magnitude scale of a value formed with cancellation: 8 f64 ulps of its terms
# (a, b) column pairs of G = [g0..g5, r] for each of the 28 sums, in the kernel's order
PAIRS = [(i, j) for i in range(6) for j in range(i, 6)] + [(i, 6) for i in range(6)] + [(6, 6)]
assert len(PAIRS) == N_SUMS
if np.finfo(np.longdouble).nmant < 63:  # pragma: no cover - x86-64 long double has 63 explicit mantissa bits
    raise ImportError("jacref needs an extended-precision np.longdouble for its exact sums")

_sin, _cos, _atan2 = np.frompyfunc(math.sin, 1, 1), np.frompyfunc(math.cos, 1, 1), math.atan2


def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _dot3(a, b):
    """Eigen's 3-element order x0 + (x1 + x2)."""
    return a[..., 0] * b[..., 0] + (a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2])


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def near_midpoint(x, scale, ties=True):
    """Does float64 x lie within max(MARGIN |x|, MARGIN_SCALE scale) of the midpoint between two adjacent float32 values?
    ties=False: a value exactly on a midpoint does not count (see the robust weights)."""
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = x.astype(np.float32)
        toward = np.where(x >= f.astype(np.float64), np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
        mid = 0.5 * (f.astype(np.float64) + np.nextafter(f, toward).astype(np.float64))
        win = np.maximum(MARGIN * np.abs(x), MARGIN_SCALE * np.asarray(scale, np.float64))
        near = np.isfinite(mid) & (np.abs(x - mid) <= win)
        return near if ties else near & (x != mid)


def quat2axis(q):
    """math_utils.h Quat2axis of one quaternion (x, y, z, w)."""
    x, y, z, w = (float(v) for v in q)
    mag = math.sqrt(x * x + y * y + z * z)
    v = np.array([x, y, z])
    if mag >= 1e-10:
        a = 2.0 * _atan2(mag, w)
        while a >= math.pi:
            a -= 2.0 * math.pi
        while a < -math.pi:
            a += 2.0 * math.pi
        v = v / mag * a
    return v


def rot_matrix(q):
    """QuaternionBase::toRotationMatrix of (x, y, z, w), row-major 3 x 3."""
    x, y, z, w = (float(v) for v in q)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]])


def rinvleft(axis):
    """math_utils.h Rinvleft (3 x 3, row-major)."""
    theta = float(np.sqrt(_dot3(axis, axis)))
    if theta < 1e-10:
        return np.eye(3)
    h = theta / 2.0
    a = axis / theta
    s = h * (math.cos(h) / math.sin(h))
    sk = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return (s * np.eye(3) + np.outer((1.0 - s) * a, a)) - h * sk


def att_map(state):
    """The per-unit linear map from the kernel's g_3..5 to the reference row's attitude columns: h_3..5 = ATT^T g_3..5,
    ATT = Rinvleft(-Quat2axis(q)).  (h_att = (c^T N) Rinv with N = -R skew(p), and c^T N = (p x R^T c)^T = g_att^T.)"""
    return rinvleft(-quat2axis(np.asarray(state)[6:10]))


def _deskew(p, w, unit, states, scan_period):
    """transformToStart of every query: (sel f32 (m, 3), sel marginal (m,), s (m,), half angle (m,))."""
    fi = (w - np.trunc(w).astype(np.float32)).astype(np.float32)
    s = (1.0 / scan_period) * fi.astype(np.float64)
    phi = np.array([quat2axis(st[6:10]) for st in states]).reshape(-1, 3)
    rn = np.asarray(states, np.float64).reshape(-1, 19)[:, 0:3]
    v = s[:, None] * phi[unit]
    theta = np.sqrt(_dot3(v, v))
    small = theta < 1e-10
    th = np.where(small, 1.0, theta)
    t = v / th[:, None]
    half = theta / 2.0
    sn, cs = _sin(half).astype(np.float64), _cos(half).astype(np.float64)
    qw = np.where(small, 1.0, cs)
    qv = np.where(small[:, None], 0.0, t * sn[:, None])
    P = p.astype(np.float64)
    uv = _cross(qv, P)
    uv = uv + uv
    c = _cross(qv, uv)
    rp = (P + qw[:, None] * uv) + c
    T = s[:, None] * rn[unit]
    x = rp + T
    scale = np.sqrt(_dot3(P, P))[:, None] + np.abs(T)
    return _f32(x), near_midpoint(x, scale).any(1), s, 0.5 * (s * np.sqrt(_dot3(phi, phi))[unit])


def _plane(sel, t1, t2, t3, weighted):
    P0, P1, P2, P3 = (a.astype(np.float64) for a in (sel, t1, t2, t3))
    M = _cross(P1 - P2, P1 - P3)
    d = P0 - P1
    r = _dot3(d, M)
    m = np.sqrt(_dot3(M, M))
    with np.errstate(divide="ignore", invalid="ignore"):
        res64 = r / m
        jac = M / m[:, None]
    res = _f32(res64)
    marg = near_midpoint(res64, np.sqrt(_dot3(d, d)))
    if weighted:
        sf = sel.astype(np.float32)
        n2 = (sf[:, 0] * sf[:, 0] + sf[:, 1] * sf[:, 1]) + sf[:, 2] * sf[:, 2]
        rt = np.sqrt(np.sqrt(n2))
        with np.errstate(divide="ignore", invalid="ignore"):
            q = 1.8 * np.abs(res).astype(np.float64) / rt.astype(np.float64)
        s64 = 1.0 - q
        marg |= near_midpoint(s64, 1.0 + np.abs(q), ties=False)
        s = _f32(s64)
    else:
        s = np.ones(len(res), np.float32)
    # |M_k| <= |P1 - P2| |P1 - P3|: the cross product's terms, which a contracted evaluation rounds differently
    with np.errstate(divide="ignore", invalid="ignore"):
        jscale = np.sqrt(_dot3(P1 - P2, P1 - P2) * _dot3(P1 - P3, P1 - P3)) / m
    return res, s, jac, jscale, marg


def _line(sel, t1, t2, weighted):
    P0, P1, P2 = (a.astype(np.float64) for a in (sel, t1, t2))
    P = _cross(P0 - P1, P0 - P2)
    r64, d64 = np.sqrt(_dot3(P, P)), np.sqrt(_dot3(P1 - P2, P1 - P2))
    marg = near_midpoint(r64, r64) | near_midpoint(d64, d64)
    r, d12 = _f32(r64), _f32(d64)
    with np.errstate(divide="ignore", invalid="ignore"):
        res = (r / d12).astype(np.float32)
        a = P2 - P1
        num = np.stack([P[:, 1] * a[:, 2] + P[:, 2] * (-a[:, 1]), P[:, 0] * (-a[:, 2]) + P[:, 2] * a[:, 0],
                        P[:, 0] * a[:, 1] + P[:, 1] * (-a[:, 0])], 1)
        den = (d12 * r).astype(np.float32).astype(np.float64)
        jac = num / den[:, None]
        jscale = r64 * np.sqrt(_dot3(a, a)) / den  # |P| |a| / den >= |jac|
    if weighted:
        s64 = 1.0 - 1.8 * np.abs(res).astype(np.float64)
        marg |= near_midpoint(s64, 1.0 + 1.8 * np.abs(res), ties=False)
        s = _f32(s64)
    else:
        s = np.ones(len(res), np.float32)
    return res, s, jac, jscale, marg


def _rows(kind, pts, ids, targets, toff, unit, states, prm):
    """Every query of one kind (surf: 3 IDs, corner: 2) of every unit: dict of per-row arrays."""
    m = len(pts)
    p = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float32)
    w = np.asarray(pts["intensity"], np.float32)
    sel, marg, s_t, half = _deskew(p, w, unit, states, prm.scan_period)
    T = (toff[unit + 1] - toff[unit]).astype(np.int64)
    k = ids.shape[1]
    valid = np.all((ids >= 0) & (ids < T[:, None]), 1)
    g = np.clip(ids, 0, None).astype(np.int64) + toff[unit][:, None]
    g = np.where(valid[:, None], g, 0)
    tgt = np.stack([targets["x"], targets["y"], targets["z"]], 1).astype(np.float32) if len(targets) else np.zeros((1, 3), np.float32)
    tri = [tgt[g[:, j]] if len(targets) else np.zeros((m, 3), np.float32) for j in range(k)]
    weighted = 1 >= prm.icp_freq
    if kind == "surf":
        res, s, jac, jscale, m2 = _plane(sel, tri[0], tri[1], tri[2], weighted)
    else:
        res, s, jac, jscale, m2 = _line(sel, tri[0], tri[1], weighted)
    s64 = s.astype(np.float64)
    c64 = s64[:, None] * jac
    with np.errstate(invalid="ignore"):
        m2 |= near_midpoint(c64, (np.abs(s64) * jscale)[:, None]).any(1)
        accept = valid & (s64 > 0.1) & (res != 0)
    coeff = np.zeros((m, 4), np.float32)
    cand = np.concatenate([_f32(c64), (s * res).astype(np.float32)[:, None]], 1)  # the coefficients if accepted
    coeff[accept] = cand[accept]
    marg = valid & (marg | m2)
    return dict(unit=unit, p=p, sel=sel, s=s_t, half=half, valid=valid, mask=accept, coeff=coeff, cand=cand, marginal=marg)


def jacobian_rows(p, coeff, state, lidar_scale):
    """G = [g0..g5, r] (m, 7) of queries p (m, 3) with coefficients coeff (m, 4), all linearised at one state."""
    p, coeff = np.asarray(p, np.float32).reshape(-1, 3), np.asarray(coeff, np.float32).reshape(-1, 4)
    return _jacobian_rows(p, coeff, np.broadcast_to(rot_matrix(np.asarray(state)[6:10]), (len(p), 3, 3)), lidar_scale)[0]


def _jacobian_rows(p, coeff, R, lidar_scale):
    """G = [g0..g5, r] (m, 7) and the magnitude scales of its entries, R (m, 3, 3) per row."""
    c = coeff[:, :3].astype(np.float64)
    r = lidar_scale * coeff[:, 3].astype(np.float64)
    cx, cy, cz = c[:, 0], c[:, 1], c[:, 2]
    u = [R[:, 0, j] * cx + R[:, 1, j] * cy + R[:, 2, j] * cz for j in range(3)]
    px, py, pz = (p[:, j].astype(np.float64) for j in range(3))
    G = np.stack([cx, cy, cz, py * u[2] - pz * u[1], pz * u[0] - px * u[2], px * u[1] - py * u[0], r], 1)
    pc = np.sqrt(_dot3(p.astype(np.float64), p.astype(np.float64))) * np.sqrt(_dot3(c, c))
    S = np.abs(G)
    S[:, 3:6] = pc[:, None]
    return G, S


def _unit_sums(vals, unit, n, dtype):
    """Per-unit sums of vals (m, k) over rows grouped by unit (rows of a unit contiguous, units ascending)."""
    out = np.zeros((n,) + vals.shape[1:], dtype)
    if len(vals) == 0:
        return out
    starts = np.searchsorted(unit, np.arange(n))
    ends = np.searchsorted(unit, np.arange(n), side="right")
    has = ends > starts
    if has.any():
        out[has] = np.add.reduceat(vals.astype(dtype), starts[has], axis=0)
    return out


class JacRef:
    """The pass's reference outputs.  Per unit: sums (n, 28), counts (n, 2), scale / excuse (n, 28), n_rows (n,),
    marginal (n, 2) marginal rows of each kind.  Per kind ('surf', 'corner'): the per-row dict of _rows plus
    rows (m, 7) = [g0..g5, r] of the accepted rows (zero elsewhere)."""

    def bound(self):
        """|kernel - reference| allowed for each of the (n, 28) sums."""
        return (self.n_rows + 16)[:, None] * 2.0 ** -52 * self.scale + self.excuse

    def accum(self):
        """The (n, 30) layout lins_gpu_batch_jacobian_pass writes."""
        return np.concatenate([self.sums, self.counts.astype(np.float64)], 1)


def reference(batch, surf_ind, corner_ind, states, prm):
    """jacref of the resident batch `batch` with the IDs of batch_download_indices, the linearisation states (n, 19)
    and the LinsParams of the pass."""
    n = batch.n
    states = np.asarray(states, np.float64).reshape(n, 19)
    Rs = np.array([rot_matrix(st[6:10]) for st in states]).reshape(n, 3, 3)
    out = JacRef()
    out.n = n
    sums = np.zeros((n, N_SUMS), np.longdouble)
    out.scale, out.excuse = np.zeros((n, N_SUMS)), np.zeros((n, N_SUMS))
    out.counts, out.marginal = np.zeros((n, 2), np.int64), np.zeros((n, 2), np.int64)
    out.n_rows = np.zeros(n, np.int64)
    for kk, (kind, q, t, ids) in enumerate((("surf", "surf_flat", "surf_less_flat", surf_ind), ("corner", "corner_sharp", "corner_less_sharp", corner_ind))):
        qoff = batch.offsets[q].astype(np.int64)
        unit = np.repeat(np.arange(n), np.diff(qoff))
        rows = _rows(kind, batch.clouds[q], np.asarray(ids).reshape(len(unit), -1), batch.clouds[t], batch.offsets[t].astype(np.int64), unit, states, prm)
        G, S = _jacobian_rows(rows["p"], rows["cand"], Rs[unit], prm.lidar_scale)
        acc, mg = rows["mask"], rows["marginal"]
        Ga = np.where(acc[:, None], G, 0.0)
        for e, (a, b) in enumerate(PAIRS):
            sums[:, e] += _unit_sums(Ga[:, a].astype(np.longdouble) * Ga[:, b].astype(np.longdouble), unit, n, np.longdouble)
            SS = S[:, a] * S[:, b]
            out.scale[:, e] += _unit_sums(np.where(acc, SS, 0.0), unit, n, np.float64)
            out.excuse[:, e] += _unit_sums(np.where(mg, SS, 0.0), unit, n, np.float64)
        out.counts[:, kk] = _unit_sums(acc.astype(np.int64), unit, n, np.int64)
        out.marginal[:, kk] = _unit_sums(mg.astype(np.int64), unit, n, np.int64)
        out.n_rows += np.diff(qoff)
        rows["rows"] = Ga
        rows["scales"] = S
        setattr(out, kind, rows)
    out.sums = sums.astype(np.float64)
    return out
