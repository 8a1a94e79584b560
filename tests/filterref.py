"""An independent float64 restatement of the reference filter algebra that sequence mode runs on the device: the
StatePredictor of KalmanFilter.hpp, the IMU pre-integration of integrationBase.h and the parts of StateEstimator.hpp
that move the state between scans (processImu, processFirstScan / processSecondScan, integrateTransformation, reset(1),
the roll / pitch correction).  Written from the reference's source the way npref.py is; it does not use this project's
C++ or CUDA code.

The reference is followed literally where it is not the textbook operation:
  * `quaternion * vector` is Eigen's _transformVector, v + 2 w (q_v x v) + q_v x (2 q_v x v), also on quaternions that
    are not unit; toRotationMatrix is Eigen's formula, also unnormalised; `q.inverse()` is the conjugate over the squared
    norm; `Matrix * Quaternion` is M R(q);
  * rpy2Quat discards its `Q.normalized()` (math_utils.h:146), axis2Quat returns the identity for theta < 1e-10,
    sign(x) is +1 for x >= 0 (and -1 for NaN);
  * predict's Ft uses the current gyro sample in its att-att block and the new attitude in its vel blocks;
  * reset(1) builds the covariance with the pre-reset q, then resets the state; gn is rotated by the already-identity q
    and rescaled to 9.81;
  * the pre-integration rotates acc_1 by the unnormalised delta_q * (1, w dt / 2) and normalises afterwards.

States are the C-ABI's 19 numbers: rn[0..2] vn[3..5] q(x, y, z, w)[6..9] ba[10..12] bw[13..15] gn[16..18];
covariances are 18x18 matrices in the error-state order pos vel att acc gyr gra.  Every function takes `m`, the scalar
backend: F64 (numpy float64, NaN where the reference's libm gives NaN) or MP (mpmath at the working precision, for the
self-check).  Inputs are not modified."""
import math
import types

import numpy as np

# ---- constants: parameters.h:63-71 and exp_port.yaml:29-75 ---------------------------------------------------------
G0 = 9.81
DEG = math.pi / 180.0
DPH = DEG / 3600.0
DPSH = DEG / math.sqrt(3600.0)
MG = G0 / 1000.0
UG = MG / 1000.0
UGPSHZ = UG / math.sqrt(1.0)

YAML = dict(acc_n=70000.0, gyr_n=0.1, acc_w=500.0, gyr_w=0.05,
            init_pos_std=(0.0, 0.0, 0.0), init_vel_std=(0.0, 0.0, 0.0), init_att_std=(0.0, 0.0, 0.0),
            init_acc_std=(0.01, 0.01, 0.02), init_gyr_std=(0.002, 0.002, 0.002),
            init_ba=(-0.015774, 0.143237, -0.0263845), init_bw=(-0.00275058, -0.000165954, 0.00262913))

POS, VEL, ATT, ACC, GYR, GRA = 0, 3, 6, 9, 12, 15        # error-state blocks (KalmanFilter.hpp:40-45)
S_RN, S_VN, S_Q, S_BA, S_BW, S_GN = 0, 3, 6, 10, 13, 16  # the 19-number state


def _f64_asin(x):
    with np.errstate(invalid="ignore"):
        return float(np.arcsin(x))


def _f64_div(a, b):
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.float64(a) / np.float64(b)


F64 = types.SimpleNamespace(sin=math.sin, cos=math.cos, sqrt=lambda x: float(np.sqrt(np.float64(x))), asin=_f64_asin,
                            atan2=lambda y, x: float(np.arctan2(y, x)), div=_f64_div, f=float, dtype=np.float64)


def mp_backend():
    import mpmath

    return types.SimpleNamespace(sin=mpmath.sin, cos=mpmath.cos, sqrt=mpmath.sqrt, asin=mpmath.asin, atan2=mpmath.atan2,
                                 div=lambda a, b: a / b, f=mpmath.mpf, dtype=object)


def vec(m, x):
    return np.array([m.f(v) for v in x], dtype=m.dtype)


def zeros(m, *shape):
    a = np.empty(shape, dtype=m.dtype)
    a.fill(m.f(0))
    return a


def eye(m, n):
    a = zeros(m, n, n)
    for i in range(n):
        a[i, i] = m.f(1)
    return a


def cross(a, b):
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]], dtype=a.dtype)


def norm(m, v):
    return m.sqrt(sum(x * x for x in v))


def skew(m, v):
    z = m.f(0)
    return np.array([[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]], dtype=m.dtype)


def sign(x):
    return 1 if x >= 0 else -1


# ---- quaternions (x, y, z, w) with Eigen's semantics ----------------------------------------------------------------
def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], dtype=a.dtype)


def qrot(q, v):
    """Eigen's `q * v` (_transformVector): no normalisation."""
    qv, w = q[:3], q[3]
    t = cross(qv, v)
    t = t + t
    return v + w * t + cross(qv, t)


def qtoR(q):
    """Eigen's toRotationMatrix: no normalisation."""
    x, y, z, w = q
    tx, ty, tz = x + x, y + y, z + z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz, tyy, tyz, tzz = tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1 - (txx + tyy)]], dtype=q.dtype)


def qnormalized(m, q):
    n = m.sqrt(sum(x * x for x in q))
    return np.array([m.div(x, n) for x in q], dtype=q.dtype)


def qinverse(m, q):
    n2 = sum(x * x for x in q)
    return np.array([m.div(-q[0], n2), m.div(-q[1], n2), m.div(-q[2], n2), m.div(q[3], n2)], dtype=q.dtype)


def qident(m):
    return vec(m, (0, 0, 0, 1))


def axis2Quat(m, v):
    """math_utils.h:43-73"""
    theta = norm(m, v)
    if theta < 1e-10:
        return qident(m)
    ax = np.array([x / theta for x in v], dtype=v.dtype)
    s = m.sin(theta / 2)
    return np.array([ax[0] * s, ax[1] * s, ax[2] * s, m.cos(theta / 2)], dtype=v.dtype)


def rpy2Quat(m, rpy):
    """math_utils.h:131-148 (the normalized() result is discarded)"""
    hy, hp, hr = rpy[2] * m.f(0.5), rpy[1] * m.f(0.5), rpy[0] * m.f(0.5)
    cy, sy, cp, sp, cr, sr = m.cos(hy), m.sin(hy), m.cos(hp), m.sin(hp), m.cos(hr), m.sin(hr)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy,
                     cr * cp * cy + sr * sp * sy], dtype=m.dtype)


def R2rpy(m, R):
    """math_utils.h:184-190: divides by cos(pitch), so it is ill-conditioned near gimbal lock"""
    p = m.atan2(-R[2, 0], m.sqrt(R[2, 1] * R[2, 1] + R[2, 2] * R[2, 2]))
    c = m.cos(p)
    r = m.atan2(m.div(R[2, 1], c), m.div(R[2, 2], c))
    y = m.atan2(m.div(R[1, 0], c), m.div(R[0, 0], c))
    return np.array([r, p, y], dtype=m.dtype)


def Q2rpy(m, q):
    return R2rpy(m, qtoR(q))


# ---- the state ------------------------------------------------------------------------------------------------------
def split(s):
    s = np.asarray(s)
    return s[S_RN:S_RN + 3].copy(), s[S_VN:S_VN + 3].copy(), s[S_Q:S_Q + 4].copy(), s[S_BA:S_BA + 3].copy(), \
        s[S_BW:S_BW + 3].copy(), s[S_GN:S_GN + 3].copy()


def join(rn, vn, q, ba, bw, gn):
    return np.concatenate([rn, vn, q, ba, bw, gn])


def global_state(m, rn=None, vn=None, q=None, ba=None, bw=None):
    """GlobalState(rn, vn, qbn, ba, bw) (KalmanFilter.hpp:49-68): gn = (0, 0, -G0)"""
    z = vec(m, (0, 0, 0))
    return join(z if rn is None else rn, z if vn is None else vn, qident(m) if q is None else q, z if ba is None else ba,
                z if bw is None else bw, vec(m, (0, 0, -G0)))


# ---- StatePredictor (KalmanFilter.hpp) ------------------------------------------------------------------------------
def noise_diag(p=YAML):
    """initializeCovariance's noise_ (KalmanFilter.hpp:263-266, :307-311): (peba, pebg, pweba, pwebg)"""
    return (pow(p["acc_n"] * UG, 2), pow(p["gyr_n"] * DPH, 2), pow(p["acc_w"] * UGPSHZ, 2), pow(p["gyr_w"] * DPSH, 2))


def deg2rad(x):
    return x * math.pi / 180.0


def init_cov_diag(p=YAML):
    """initializeCovariance(0)'s diagonal (KalmanFilter.hpp:247-283)"""
    d = [v * v for v in p["init_pos_std"]] + [v * v for v in p["init_vel_std"]]
    d += [pow(deg2rad(v), 2) for v in p["init_att_std"]]
    d += [v * v for v in p["init_acc_std"]] + [v * v for v in p["init_gyr_std"]] + [0.01] * 3
    return d


def initialize_covariance(m, p=YAML):
    P = zeros(m, 18, 18)
    for i, v in enumerate(init_cov_diag(p)):
        P[i, i] = m.f(v)
    return P


def predict(m, s, P, acc_last, gyr_last, dt, acc, gyr, noise):
    """StatePredictor::predict(dt, acc, gyr, true) (KalmanFilter.hpp:125-186).  Returns (state, P); acc / gyr become the
    next call's acc_last / gyr_last."""
    rn, vn, q, ba, bw, gn = split(s)
    dt = m.f(dt)
    acc_last, gyr_last, acc, gyr = (vec(m, x) for x in (acc_last, gyr_last, acc, gyr))
    half = m.f(0.5)
    un_acc_0 = qrot(q, acc_last - ba) + gn
    un_gyr = half * (gyr_last + gyr) - bw
    q = qnormalized(m, qmul(q, axis2Quat(m, un_gyr * dt)))
    un_acc_1 = qrot(q, acc - ba) + gn
    un_acc = half * (un_acc_0 + un_acc_1)
    rn = rn + dt * vn + half * dt * dt * un_acc
    vn = vn + dt * un_acc

    R = qtoR(q)
    Ft = zeros(m, 18, 18)
    Ft[POS:POS + 3, VEL:VEL + 3] = eye(m, 3)
    Ft[VEL:VEL + 3, ATT:ATT + 3] = -R.dot(skew(m, acc - ba))
    Ft[VEL:VEL + 3, ACC:ACC + 3] = -R
    Ft[VEL:VEL + 3, GRA:GRA + 3] = eye(m, 3)
    Ft[ATT:ATT + 3, ATT:ATT + 3] = -skew(m, gyr - bw)
    Ft[ATT:ATT + 3, GYR:GYR + 3] = -eye(m, 3)
    Gt = zeros(m, 18, 12)
    Gt[VEL:VEL + 3, 0:3] = -R
    Gt[ATT:ATT + 3, 3:6] = -eye(m, 3)
    Gt[ACC:ACC + 3, 6:9] = eye(m, 3)
    Gt[GYR:GYR + 3, 9:12] = eye(m, 3)
    Gt = Gt * dt
    N = zeros(m, 12, 12)
    for b in range(4):
        for i in range(3):
            N[3 * b + i, 3 * b + i] = m.f(noise[b])
    F = eye(m, 18) + Ft * dt + half * Ft.dot(Ft) * dt * dt
    P = F.dot(np.asarray(P)).dot(F.T) + Gt.dot(N).dot(Gt.T)
    P = half * (P + P.T)
    return join(rn, vn, q, ba, bw, gn), P


def reset1(m, s, P, p=YAML):
    """StatePredictor::reset(1) (KalmanFilter.hpp:320-353)"""
    rn, vn, q, ba, bw, gn = split(s)
    P = np.asarray(P)
    Rinv, R = qtoR(qinverse(m, q)), qtoR(q)
    out = zeros(m, 18, 18)
    for i in range(3):
        out[POS + i, POS + i] = m.f(p["init_pos_std"][i] ** 2)
        out[ATT + i, ATT + i] = m.f(pow(deg2rad(p["init_att_std"][i]), 2))
    out[VEL:VEL + 3, VEL:VEL + 3] = Rinv.dot(P[VEL:VEL + 3, VEL:VEL + 3]).dot(R)
    out[ACC:ACC + 3, ACC:ACC + 3] = P[ACC:ACC + 3, ACC:ACC + 3]
    out[GYR:GYR + 3, GYR:GYR + 3] = P[GYR:GYR + 3, GYR:GYR + 3]
    out[GRA:GRA + 3, GRA:GRA + 3] = Rinv.dot(P[GRA:GRA + 3, GRA:GRA + 3]).dot(R)
    rn = vec(m, (0, 0, 0))
    vn = qrot(qinverse(m, q), vn)
    q = qident(m)
    gn = qrot(qinverse(m, q), gn)
    n = norm(m, gn)
    gn = np.array([m.div(x * m.f(9.81), n) for x in gn], dtype=m.dtype)
    return join(rn, vn, q, ba, bw, gn), out


# ---- StateEstimator (StateEstimator.hpp) ----------------------------------------------------------------------------
def integrate(m, g, f):
    """integrateTransformation (StateEstimator.hpp:608-617): g = globalState_, f = filter_->state_"""
    grn, gvn, gq, gba, gbw, ggn = split(g)
    frn, fvn, fq, fba, fbw, fgn = split(f)
    grn = qrot(gq, frn) + grn
    gq = qmul(gq, fq)
    gvn = qrot(qmul(gq, qinverse(m, fq)), fvn)
    return join(grn, gvn, gq, fba.copy(), fbw.copy(), qrot(gq, fgn))


def rp_from_gravity(m, fb):
    """calculateRPfromGravity (StateEstimator.hpp:602-605): (roll, pitch)"""
    sg = sign(fb[2])
    return sg * m.asin(fb[1] / m.f(G0)), -sg * m.asin(fb[0] / m.f(G0))


def correct_roll_pitch(m, g, roll, pitch):
    """correctRollPitch (StateEstimator.hpp:427-431)"""
    rn, vn, q, ba, bw, gn = split(g)
    rpy = Q2rpy(m, q)
    return join(rn, vn, rpy2Quat(m, np.array([roll, pitch, rpy[2]], dtype=m.dtype)), ba, bw, gn)


def post_step(m, g, f, P, p=YAML):
    """processScan after performIESKF (StateEstimator.hpp:443-453): `f`, `P` = what filter_->update received (the
    IESKF posterior, or after divergence the prior with estimateTransform's rn / qbn and the prior covariance,
    :585-598).  Returns (globalState_, filter_->state_, filter_->covariance_)."""
    g = integrate(m, g, f)
    f, P = reset1(m, f, P, p)
    roll, pitch = rp_from_gravity(m, f[S_GN:S_GN + 3])
    return correct_roll_pitch(m, g, roll, pitch), f, P


def icp_prior(s, t, q_xyzw):
    """The filter state performIESKF hands to update() after divergence: the prior with estimateTransform's pose."""
    s = np.array(s, copy=True)
    s[S_RN:S_RN + 3] = t
    s[S_Q:S_Q + 4] = q_xyzw
    return s


# ---- IntegrationBase (integrationBase.h) ----------------------------------------------------------------------------
class Preint:
    """IntegrationBase(acc_0, gyr_0, linearized_ba, linearized_bg) and its propagate (integrationBase.h:35-51,
    :61-80, :161-188); the Jacobian is not needed by processSecondScan's estimateInitialState."""

    def __init__(self, m, acc0, gyr0, ba, bg):
        self.m = m
        self.acc_0, self.gyr_0, self.ba, self.bg = vec(m, acc0), vec(m, gyr0), vec(m, ba), vec(m, bg)
        self.delta_p, self.delta_v, self.delta_q = vec(m, (0, 0, 0)), vec(m, (0, 0, 0)), qident(m)
        self.sum_dt = m.f(0)

    def push_back(self, dt, acc, gyr):
        m = self.m
        dt, acc1, gyr1 = m.f(dt), vec(m, acc), vec(m, gyr)
        half, two = m.f(0.5), m.f(2)
        un_acc_0 = qrot(self.delta_q, self.acc_0 - self.ba)
        un_gyr = half * (self.gyr_0 + gyr1) - self.bg
        rq = qmul(self.delta_q, np.array([un_gyr[0] * dt / two, un_gyr[1] * dt / two, un_gyr[2] * dt / two, m.f(1)], dtype=m.dtype))
        un_acc_1 = qrot(rq, acc1 - self.ba)  # the unnormalised result_delta_q
        un_acc = half * (un_acc_0 + un_acc_1)
        self.delta_p = self.delta_p + self.delta_v * dt + half * un_acc * dt * dt
        self.delta_v = self.delta_v + un_acc * dt
        self.delta_q = qnormalized(m, rq)
        self.sum_dt = self.sum_dt + dt
        self.acc_0, self.gyr_0 = acc1, gyr1


def first_scan(m, imu, p=YAML):
    """processFirstScan once its gate passed (StateEstimator.hpp:331-375): returns (filter state, P, preintegration,
    acc_last, gyr_last); globalState_ is left as it was."""
    imu = vec(m, imu)
    pre = Preint(m, imu[:3], imu[3:], p["init_ba"], p["init_bw"])
    z = vec(m, (0, 0, 0))
    f = global_state(m, z, z, rpy2Quat(m, z), z, z)
    return f, initialize_covariance(m, p), pre, imu[:3].copy(), imu[3:].copy()


def second_scan_start(m, pre):
    """processSecondScan's start pose of estimateTransform (StateEstimator.hpp:388-396): (pl, ql); ba0 = 0 and
    linState_.gn_ = (0, 0, -G0) here"""
    ba0 = vec(m, (0, 0, 0))
    gn = vec(m, (0, 0, -G0))
    s2 = pre.sum_dt * pre.sum_dt
    half = m.f(0.5)
    pl = pre.delta_p + half * gn * s2 - half * ba0 * s2
    return pl, pre.delta_q.copy()


def second_scan(m, pre, pl, ql, imu, p=YAML):
    """processSecondScan after estimateTransform returned (pl, ql) (StateEstimator.hpp:399-415) with
    estimateInitialState (:1408-1419; v = p / sum_dt, no guard): returns (globalState_, filter state, P, acc_last,
    gyr_last)."""
    imu = vec(m, imu)
    pl = vec(m, pl)
    v1 = np.array([m.div(x, pre.sum_dt) for x in pl], dtype=m.dtype)
    ba0, bw0 = vec(m, p["init_ba"]), vec(m, p["init_bw"])
    z = vec(m, (0, 0, 0))
    f = global_state(m, pl, v1, rpy2Quat(m, z), ba0, bw0)
    roll, pitch = rp_from_gravity(m, imu[:3] - ba0)
    g = global_state(m, pl, v1, rpy2Quat(m, np.array([roll, pitch, m.f(0)], dtype=m.dtype)), ba0, bw0)
    return g, f, initialize_covariance(m, p), imu[:3].copy(), imu[3:].copy()


# ---- processImu (StateEstimator.hpp:242-257) ------------------------------------------------------------------------
STATUS_INIT, STATUS_FIRST_SCAN, STATUS_RUNNING = 0, 1, 3


def process_imu(m, status, dt, acc, gyr, filt=None, pre=None, noise=None):
    """One IMU row: nothing in INIT, pre-integration only (no predict) in FIRST_SCAN, predict in RUNNING.
    `filt` = dict(state, P, acc_last, gyr_last), updated in place in RUNNING; `pre` = the Preint, in FIRST_SCAN."""
    if status == STATUS_FIRST_SCAN:
        pre.push_back(dt, acc, gyr)
    elif status == STATUS_RUNNING:
        filt["state"], filt["P"] = predict(m, filt["state"], filt["P"], filt["acc_last"], filt["gyr_last"], dt, acc, gyr, noise)
        filt["acc_last"], filt["gyr_last"] = vec(m, acc), vec(m, gyr)


# ---- comparison bars ------------------------------------------------------------------------------------------------
STATE_RTOL = 1e-13    # relative to max(|x|, 1): the floor keeps entries near zero from failing on rounding noise
COV_RTOL = 1e-12      # relative to max(|x|, 1e-3 max|P|)
COS_PITCH_MIN = 1e-3  # R2rpy divides by cos(pitch): below this the attitude is not compared


def nan_pattern(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isinf(a) & (a > 0), np.isinf(b) & (b > 0)) \
        and np.array_equal(np.isinf(a) & (a < 0), np.isinf(b) & (b < 0))


def check_state(got, want, what, skip=()):
    got, want = np.asarray(got, float), np.asarray(want, float)
    assert nan_pattern(got, want), (what, got, want)
    ok = np.isfinite(want)
    if len(skip):
        ok[list(skip)] = False
    err = np.abs(got[ok] - want[ok])
    tol = STATE_RTOL * np.maximum(np.abs(want[ok]), 1.0)
    assert (err <= tol).all(), (what, np.abs(got - want).max(), got, want)


def check_cov(got_colmajor, want, what):
    got = np.asarray(got_colmajor, float).reshape(18, 18).T  # column-major on the C side
    want = np.asarray(want, float)
    assert nan_pattern(got, want), (what,)
    ok = np.isfinite(want)
    if not ok.any():
        return
    floor = 1e-3 * np.abs(want[ok]).max()
    err = np.abs(got[ok] - want[ok])
    tol = COV_RTOL * np.maximum(np.abs(want[ok]), floor)
    assert (err <= tol).all(), (what, (err - tol).max())
