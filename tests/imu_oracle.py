"""gb_imu_preintegrate's rule and the navigation terms of gb_nav_graph_optimize (include/glim_b200.h) restated in fp64 numpy:
IMUIntegration::integrate_imu's window, one step of GTSAM's tangent preintegration with its A, B, C, the IMU term
(ImuFactor's residual at state j) and the vector terms, each with its Jacobian in the solver's charts.  Also an analytic
trajectory with closed-form acceleration and angular rate, and its exact IMU samples.  Test infrastructure, written
independently of glim_b200/csrc/gb_imu_math.cuh."""
import numpy as np
from scipy.spatial.transform import Rotation

DEFAULT_PARAMS = dict(acc_noise=0.05, gyro_noise=0.02, int_noise=0.001, gravity=np.array([0.0, 0.0, -9.81]))


def hat(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def exp3(w):
    return Rotation.from_rotvec(np.asarray(w, dtype=np.float64)).as_matrix()


def log3(R):
    return Rotation.from_matrix(R).as_rotvec()


def jr(w):
    """J_r(w) = I - (1 - cos t) / t^2 [w]x + (t - sin t) / t^3 [w]x^2"""
    t = np.linalg.norm(w)
    K = hat(w)
    if t < 1e-4:
        return np.eye(3) - 0.5 * K + K @ K / 6.0
    return np.eye(3) - (1.0 - np.cos(t)) / t**2 * K + (t - np.sin(t)) / t**3 * K @ K


def jr_inv(w):
    """J_r(w)^-1 = I + [w]x / 2 + (1 / t^2 - (1 + cos t) / (2 t sin t)) [w]x^2"""
    t = np.linalg.norm(w)
    K = hat(w)
    c = 1.0 / 12.0 + t**2 / 720.0 if t < 1e-3 else 1.0 / t**2 - (1.0 + np.cos(t)) / (2.0 * t * np.sin(t))
    return np.eye(3) + 0.5 * K + c * K @ K


def d_jr_inv_w(th, w):
    """d (J_r(th)^-1 w) / d th, exactly: with J_r^-1 w = w + th x w / 2 + c(t) th x (th x w)"""
    t = np.linalg.norm(th)
    if t < 0.05:
        c = 1.0 / 12.0 + t**2 / 720.0 + t**4 / 30240.0
        dc_t = 1.0 / 360.0 + t**2 / 7560.0 + t**4 / 201600.0
    else:
        c = 1.0 / t**2 - (1.0 + np.cos(t)) / (2.0 * t * np.sin(t))
        h = 1e-4 * t  # c'(t) / t by a fourth-order difference of the closed form: independent of the device's series
        cf = lambda s: 1.0 / s**2 - (1.0 + np.cos(s)) / (2.0 * s * np.sin(s))
        dc_t = (-cf(t + 2 * h) + 8 * cf(t + h) - 8 * cf(t - h) + cf(t - 2 * h)) / (12 * h) / t
    tw = th @ w
    u = np.cross(th, np.cross(th, w))
    return -0.5 * hat(w) + c * (tw * np.eye(3) + np.outer(th, w) - 2.0 * np.outer(w, th)) + dc_t * np.outer(u, th)


def step(x, a, w, dt):
    """one step of TangentPreintegration::UpdatePreintegrated: -> (x_new, A 9x9, B 9x3, C 9x3)"""
    th, p, v = x[:3], x[3:6], x[6:]
    R = exp3(th)
    an = R @ a
    xn = np.concatenate([th + jr_inv(th) @ w * dt, p + v * dt + 0.5 * an * dt * dt, v + an * dt])
    M = R @ hat(-a) @ jr(th)
    A = np.eye(9)
    A[:3, :3] += d_jr_inv_w(th, w) * dt
    A[3:6, :3] = M * 0.5 * dt * dt
    A[3:6, 6:] = np.eye(3) * dt
    A[6:, :3] = M * dt
    B = np.zeros((9, 3))
    B[3:6] = R * 0.5 * dt * dt
    B[6:] = R * dt
    C = np.zeros((9, 3))
    C[:3] = jr_inv(th) * dt
    return xn, A, B, C


def new_record(bias, params=None):
    P = dict(DEFAULT_PARAMS, **(params or {}))
    return dict(delta_t=0.0, preintegrated=np.zeros(9), H_bias_acc=np.zeros((9, 3)), H_bias_omega=np.zeros((9, 3)), covariance=np.zeros((9, 9)),
                bias_hat=np.asarray(bias, dtype=np.float64).copy(), gravity=np.asarray(P["gravity"], dtype=np.float64).copy(), num_integrated=0)


def integrate(rec, acc, omega, dt, params=None):
    """PreintegratedImuMeasurements::integrateMeasurement on the record dict"""
    P = dict(DEFAULT_PARAMS, **(params or {}))
    a = np.asarray(acc) - rec["bias_hat"][:3]
    w = np.asarray(omega) - rec["bias_hat"][3:]
    xn, A, B, C = step(rec["preintegrated"], a, w, dt)
    rec["delta_t"] += dt
    rec["preintegrated"] = xn
    rec["H_bias_acc"] = A @ rec["H_bias_acc"] - B
    rec["H_bias_omega"] = A @ rec["H_bias_omega"] - C
    S = A @ rec["covariance"] @ A.T + B @ (P["acc_noise"] ** 2 * np.eye(3) / dt) @ B.T + C @ (P["gyro_noise"] ** 2 * np.eye(3) / dt) @ C.T
    S[3:6, 3:6] += P["int_noise"] ** 2 * np.eye(3) * dt
    rec["covariance"] = 0.5 * (S + S.T)


def preintegrate(samples, start, end, bias, params=None):
    """IMUIntegration::integrate_imu(start, end, bias) over the sample rows (t, a, w), read from the first"""
    rec = new_record(bias, params)
    samples = np.asarray(samples, dtype=np.float64).reshape(-1, 7)
    if len(samples) == 0:
        return rec
    last, i = start, 0
    for i in range(len(samples) + 1):
        if i == len(samples):
            break
        t = samples[i, 0]
        if t > end:
            break
        dt = t - last
        if dt <= 0.0:
            continue
        integrate(rec, samples[i, 1:4], samples[i, 4:7], dt, params)
        last = t
        rec["num_integrated"] += 1
    if end - last > 0.0:
        s = samples[i] if i < len(samples) else samples[-1]
        integrate(rec, s[1:4], s[4:7], end - last, params)
    return rec


def integrate_imu_deque(samples, intervals, biases, params=None):
    """GLIM's IMUIntegration literally: a deque of samples, integrate_imu over the queue's front, then erase_imu_data(cursor)
    drops the samples the loop walked (the cursor stops at the first sample after the end), interval by interval.  An interval
    that finds the queue empty integrates nothing."""
    queue = [np.asarray(s, dtype=np.float64) for s in np.asarray(samples, dtype=np.float64).reshape(-1, 7)]
    out = []
    for (start, end), bias in zip(intervals, biases):
        rec = new_record(bias, params)
        cursor = 0
        if queue:
            last = start
            k = 0
            while k < len(queue):
                s = queue[k]
                if s[0] > end:
                    break
                dt = s[0] - last
                k += 1
                cursor += 1
                if dt <= 0.0:
                    continue
                integrate(rec, s[1:4], s[4:7], dt, params)
                last = s[0]
                rec["num_integrated"] += 1
            if end - last > 0.0:
                s = queue[k] if k < len(queue) else queue[-1]
                integrate(rec, s[1:4], s[4:7], end - last, params)
            del queue[:cursor]
        out.append(rec)
    return out


def record_of(r):
    """a capi.PREINTEGRATED_DTYPE record -> the dict the functions here take"""
    return dict(delta_t=float(r["delta_t"]), preintegrated=np.array(r["preintegrated"]), H_bias_acc=np.array(r["H_bias_acc"]), H_bias_omega=np.array(r["H_bias_omega"]),
                covariance=np.array(r["covariance"]), bias_hat=np.array(r["bias_hat"]), gravity=np.array(r["gravity"]), num_integrated=int(r["num_integrated"]))


def to_struct(rec, out):
    """the record dict into one capi.PREINTEGRATED_DTYPE element"""
    for k in ("delta_t", "preintegrated", "H_bias_acc", "H_bias_omega", "covariance", "bias_hat", "gravity", "num_integrated"):
        out[k] = rec[k]


# ---- the terms ----

def imu_residual(Ti, vi, Tj, vj, b, rec):
    """ImuFactor's residual at state j: -> (r 9, J 9 x 30 over pose_i [rot; trans] | vel_i (3 + 3 dead) | pose_j | vel_j | bias)"""
    d = rec["preintegrated"] + rec["H_bias_acc"] @ (b[:3] - rec["bias_hat"][:3]) + rec["H_bias_omega"] @ (b[3:] - rec["bias_hat"][3:])
    dt, g = rec["delta_t"], rec["gravity"]
    Ri, pi, Rj, pj = Ti[:3, :3], Ti[:3, 3], Tj[:3, :3], Tj[:3, 3]
    Ed = exp3(d[:3])
    E = Rj.T @ Ri @ Ed
    rt = log3(E)
    rp = Rj.T @ (pi + vi * dt + 0.5 * g * dt * dt + Ri @ d[3:6] - pj)
    rv = Rj.T @ (vi + g * dt + Ri @ d[6:] - vj)
    J = np.zeros((9, 30))
    Jri = jr_inv(rt)
    RR = Rj.T @ Ri
    J[:3, 0:3] = Jri @ Ed.T
    J[:3, 12:15] = -Jri @ E.T
    J[3:6, 0:3] = -RR @ hat(d[3:6])
    J[3:6, 3:6] = RR
    J[3:6, 6:9] = Rj.T * dt
    J[3:6, 12:15] = hat(rp)
    J[3:6, 15:18] = -np.eye(3)
    J[6:, 0:3] = -RR @ hat(d[6:])
    J[6:, 6:9] = Rj.T
    J[6:, 12:15] = hat(rv)
    J[6:, 18:21] = -Rj.T
    Hb = np.hstack([rec["H_bias_acc"], rec["H_bias_omega"]])
    J[:3, 24:] = Jri @ jr(d[:3]) @ Hb[:3]
    J[3:6, 24:] = RR @ Hb[3:6]
    J[6:, 24:] = RR @ Hb[6:]
    return np.concatenate([rt, rp, rv]), J


VELOCITY_PRIOR, BIAS_PRIOR, VELOCITY_BETWEEN, BIAS_BETWEEN, ROTATE_VELOCITY = range(5)


def vector_residual(kind, xa, xb, z):
    """-> (r, J rows x 12: the slot of key_a | the slot of key_b); xa / xb a 4x4 pose, a 3-velocity or a 6-bias"""
    z = np.asarray(z, dtype=np.float64)
    if kind == ROTATE_VELOCITY:
        R = xa[:3, :3]
        J = np.zeros((3, 12))
        J[:, :3] = -R @ hat(z[:3])
        J[:, 6:9] = -np.eye(3)
        return R @ z[:3] - xb, J
    d = 6 if kind in (BIAS_PRIOR, BIAS_BETWEEN) else 3
    J = np.zeros((d, 12))
    if kind in (VELOCITY_BETWEEN, BIAS_BETWEEN):
        J[:, :d] = -np.eye(d)
        J[:, 6:6 + d] = np.eye(d)
        return (xb[:d] - xa[:d]) - z[:d], J
    J[:, :d] = np.eye(d)
    return xa[:d] - z[:d], J


# ---- an analytic trajectory: p(t), R(t) = Rz(psi(t)) Rx(phi(t)) with closed-form derivatives ----

def _angles(t):
    psi, dpsi = 0.3 * t + 0.4 * np.sin(0.8 * t), 0.3 + 0.32 * np.cos(0.8 * t)
    phi, dphi = 0.2 * np.sin(1.3 * t), 0.26 * np.cos(1.3 * t)
    return psi, dpsi, phi, dphi


def _rz(a):
    return Rotation.from_rotvec([0.0, 0.0, a]).as_matrix()


def _rx(a):
    return Rotation.from_rotvec([a, 0.0, 0.0]).as_matrix()


def truth(t):
    """-> (T 4x4, v world 3, a world 3, w body 3) at time t"""
    psi, dpsi, phi, dphi = _angles(t)
    p = np.array([4.0 * np.sin(0.5 * t), 3.0 * np.cos(0.4 * t) - 3.0, 0.5 * np.sin(0.9 * t) + 0.1 * t])
    v = np.array([2.0 * np.cos(0.5 * t), -1.2 * np.sin(0.4 * t), 0.45 * np.cos(0.9 * t) + 0.1])
    a = np.array([-1.0 * np.sin(0.5 * t), -0.48 * np.cos(0.4 * t), -0.405 * np.sin(0.9 * t)])
    R = _rz(psi) @ _rx(phi)
    w = _rx(phi).T @ np.array([0.0, 0.0, dpsi]) + np.array([dphi, 0.0, 0.0])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, p
    return T, v, a, w


def samples(t0, t1, rate, bias, gravity=DEFAULT_PARAMS["gravity"]):
    """exact IMU rows (t, a_meas, w_meas) at `rate` Hz over [t0, t1]: a_meas = R^T (a - g) + b_a, w_meas = w + b_g"""
    ts = np.arange(t0, t1 + 0.5 / rate, 1.0 / rate)
    rows = []
    for t in ts:
        T, _, a, w = truth(t)
        rows.append(np.concatenate([[t], T[:3, :3].T @ (a - gravity) + bias[:3], w + bias[3:]]))
    return np.array(rows)
