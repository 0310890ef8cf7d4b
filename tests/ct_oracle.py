"""numpy restatement of the continuous-time GICP factor and its solve (gb_cloud_add_times, gb_ct_gicp_factor_create,
gb_ct_gicp_align), written from the rules in include/glim_b200.h and independently of the CUDA: the time table, SE(3) Exp / Log
(matrix exponential and logarithm), the right Jacobian as the series of the adjoint, the entry poses, the factor at the device
layout (fp32 lookup transform and fp32-cast residual pose per entry, as tests/ivox_oracle.py; fp64 after), the two small terms
of the objective and the Levenberg-Marquardt loop at 12 dof."""
import numpy as np
from scipy.linalg import expm

from tests import ivox_oracle as io

F32, F64 = np.float32, np.float64
TIME_EPS = 1e-3
CT_DEFAULTS = dict(max_iterations=8, lambda_initial=1e-10, lambda_factor=10.0, lambda_upper_bound=1e5, relative_error_tol=1e-5,
                   absolute_error_tol=1e-2, step_translation_tol=0.0, step_rotation_tol=0.0)
W_PRIOR, W_BETWEEN = 1e-3, 1e3  # config_odometry_ct.json:25-26


def time_table(times):
    """-> (starts (B+1,), tau (B,)): a point opens an entry iff later than the entry's time by more than TIME_EPS"""
    t = np.asarray(times, dtype=F64)
    starts, cur = [0], t[0]
    for i in range(1, len(t)):
        if t[i] - cur > TIME_EPS:
            starts.append(i)
            cur = t[i]
    B = len(starts)
    tb = t[starts]
    tau = np.zeros(B) if B == 1 else (tb - t[0]) / (tb[-1] - t[0])
    return np.array(starts + [len(t)], np.int64), tau


# ---------------------------------------------------------------------------------------------------------------------
# SE(3), tangent [w; v], right perturbations
# ---------------------------------------------------------------------------------------------------------------------
def hat3(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def twist(xi):
    M = np.zeros((4, 4))
    M[:3, :3] = hat3(xi[:3])
    M[:3, 3] = xi[3:]
    return M


def se3_exp(xi):
    return expm(twist(np.asarray(xi, dtype=F64)))


def se3_log(T):
    """closed-form SO(3) log, then v = J_l(w)^-1 t with J_l(w) = sum_k hat(w)^k / (k+1)!"""
    T = np.asarray(T, dtype=F64)
    R = T[:3, :3]
    c = np.clip((np.trace(R) - 1.0) / 2.0, -1.0, 1.0)
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    th = np.arctan2(0.5 * np.linalg.norm(v), c)
    if c > -0.99:
        w = v * (0.5 + th * th / 12.0 if th < 1e-4 else th / (2.0 * np.sin(th)))
    else:
        S = (R + R.T) / 2.0 - c * np.eye(3)
        k = int(np.argmax(np.diag(S)))
        a = S[:, k] / np.sqrt(S[k, k])
        a = a / np.linalg.norm(a)
        w = th * (a if a @ v >= 0 else -a)
    K = hat3(w)
    J = np.eye(3)
    P, f = np.eye(3), 1.0
    for k in range(1, 30):
        P = P @ K
        f *= k + 1
        J = J + P / f
    return np.concatenate([w, np.linalg.solve(J, T[:3, 3])])


def ad(xi):
    """ad_xi = [[hat(w), 0], [hat(v), hat(w)]]"""
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = hat3(xi[:3])
    A[3:, :3] = hat3(xi[3:])
    return A


def jr(xi):
    """SE(3) right Jacobian: sum_k (-ad_xi)^k / (k+1)!"""
    A = -ad(np.asarray(xi, dtype=F64))
    J, P, f = np.eye(6), np.eye(6), 1.0
    for k in range(1, 40):
        P = P @ A
        f *= k + 1
        J = J + P / f
    return J


def jr_inv(xi):
    return np.linalg.inv(jr(xi))


def adjoint(T):
    R, t = T[:3, :3], T[:3, 3]
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = R
    A[3:, :3] = hat3(t) @ R
    return A


def inv(T):
    Ti = np.eye(4)
    Ti[:3, :3] = T[:3, :3].T
    Ti[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return Ti


def motion(X, Y):
    return se3_log(inv(X) @ Y)


def entry_pose(X, Y, tau):
    return X @ se3_exp(tau * motion(X, Y))


def entry_blocks(X, Y, tau):
    """(D0, D1) of an entry pose: d T_b = D0 d_X + D1 d_Y"""
    xi = motion(X, Y)
    D1 = tau * jr(tau * xi) @ jr_inv(xi)
    D0 = adjoint(se3_exp(-tau * xi)) - D1 @ adjoint(inv(Y) @ X)
    return D0, D1


# ---------------------------------------------------------------------------------------------------------------------
# the factor
# ---------------------------------------------------------------------------------------------------------------------
def entry_indices(starts):
    return [np.arange(starts[b], starts[b + 1]) for b in range(len(starts) - 1)]


def correspondences(m, xyz, starts, tau, X, Y, max_corr):
    """per entry: the record index of each of its points' correspondence (-1: none), at the entry's pose"""
    return [io.correspondences(m, xyz[idx], entry_pose(X, Y, t), max_corr) for idx, t in zip(entry_indices(starts), tau)]


def entry_terms(m, xyz, cov6, T, corr, cast=True, M_pose=None):
    """(H_b, b_b, error, inliers) of the points of one entry at pose T: the GICP factor's H_ss / b_s (the fp32-cast pose when
    cast, as the device); M formed at M_pose (default T)"""
    Tc = np.asarray(T, dtype=F32).astype(F64) if cast else np.asarray(T, dtype=F64)
    Mp = Tc if M_pose is None else (np.asarray(M_pose, dtype=F32).astype(F64) if cast else np.asarray(M_pose, dtype=F64))
    R, t, Rm = Tc[:3, :3], Tc[:3, 3], Mp[:3, :3]
    k = corr >= 0
    a = np.asarray(xyz, dtype=F32)[k].astype(F64)
    CA = io.cov33(np.asarray(cov6, dtype=F32)[k])
    mu = m.xyz[corr[k]].astype(F64)
    CB = io.cov33(m.cov6[corr[k]])
    q = a @ R.T + t
    r = mu - q
    M = np.linalg.inv(CB + Rm @ CA @ Rm.T)
    n = a.shape[0]
    Js = np.concatenate([R @ io.hat(a), np.tile(-R, (n, 1, 1))], axis=2)
    Mr = np.einsum("nij,nj->ni", M, r)
    return np.einsum("nki,nkl,nlj->ij", Js, M, Js), np.einsum("nki,nk->i", Js, Mr), float(np.einsum("ni,ni->", r, Mr)), float(n)


def linearize(m, xyz, cov6, starts, tau, X, Y, max_corr, corr=None, cast=True):
    """-> (dict H (12,12), b (12,), error, num_inliers, and the record blocks H_tt .. b_s, corr)"""
    if corr is None:
        corr = correspondences(m, xyz, starts, tau, X, Y, max_corr)
    H, b, e, n = np.zeros((12, 12)), np.zeros(12), 0.0, 0.0
    for idx, t, c in zip(entry_indices(starts), tau, corr):
        Hb, bb, eb, nb = entry_terms(m, xyz[idx], cov6[idx], entry_pose(X, Y, t), c, cast)
        D0, D1 = entry_blocks(X, Y, t)
        J = np.concatenate([D0, D1], axis=1)
        H += J.T @ Hb @ J
        b += J.T @ bb
        e += eb
        n += nb
    out = {"H": H, "b": b, "error": e, "num_inliers": n, "H_tt": H[:6, :6], "H_ss": H[6:, 6:], "H_ts": H[:6, 6:], "b_t": b[:6], "b_s": b[6:]}
    return out, corr


def error(m, xyz, cov6, starts, tau, X_lin, Y_lin, X_eval, Y_eval, max_corr, cast=True, freeze_M=False):
    """error at (X_eval, Y_eval) with the correspondences of (X_lin, Y_lin); freeze_M: M formed at the lin entry poses"""
    corr = correspondences(m, xyz, starts, tau, X_lin, Y_lin, max_corr)
    e = 0.0
    for idx, t, c in zip(entry_indices(starts), tau, corr):
        Mp = entry_pose(X_lin, Y_lin, t) if freeze_M else None
        e += entry_terms(m, xyz[idx], cov6[idx], entry_pose(X_eval, Y_eval, t), c, cast, M_pose=Mp)[2]
    return e


def small_terms(X, Y, Xp, w_prior=W_PRIOR, w_between=W_BETWEEN):
    """-> (e, H (12,12), b (12,)) of w_prior |Log(Xp^-1 X)|^2 + w_between |Log(X^-1 Y)|^2 (no 1/2)"""
    r = se3_log(inv(Xp) @ X)
    Jp = np.concatenate([jr_inv(r), np.zeros((6, 6))], axis=1)
    xi = motion(X, Y)
    Ji = jr_inv(xi)
    Jb = np.concatenate([-Ji @ adjoint(inv(Y) @ X), Ji], axis=1)
    e = w_prior * r @ r + w_between * xi @ xi
    H = w_prior * Jp.T @ Jp + w_between * Jb.T @ Jb
    b = w_prior * Jp.T @ r + w_between * Jb.T @ xi
    return float(e), H, b


def align(m, xyz, cov6, starts, tau, X0, Y0, Xp, max_corr, params=None, w_prior=W_PRIOR, w_between=W_BETWEEN):
    """gb_ct_gicp_align's rule on one problem in fp64 -> dict(X, Y, error, num_inliers, lambda, iterations, trials, status)"""
    P = dict(CT_DEFAULTS, **(params or {}))
    X, Y = np.asarray(X0, dtype=F64).copy(), np.asarray(Y0, dtype=F64).copy()
    lam, need_lin, iterations, trials = P["lambda_initial"], True, 0, 0
    H, b, e, n, corr = None, None, 0.0, 0.0, None

    def result(status):
        return {"X": X, "Y": Y, "error": e, "num_inliers": n, "lambda": lam, "iterations": iterations, "trials": trials, "status": status}

    while True:
        if need_lin:
            r, corr = linearize(m, xyz, cov6, starts, tau, X, Y, max_corr)
            es, Hs, bs = small_terms(X, Y, Xp, w_prior, w_between)
            H, b, e, n = r["H"] + Hs, r["b"] + bs, r["error"] + es, r["num_inliers"]
            iterations += 1
            need_lin = False
            if n == 0 and iterations == 1:
                return result(io.ALIGN_DEGENERATE)
        trials += 1
        A = H + lam * np.eye(12)
        try:
            np.linalg.cholesky(A)
            d = np.linalg.solve(A, -b)
            solved = bool(np.isfinite(d).all())
        except np.linalg.LinAlgError:
            solved = False
        if solved:
            EX, EY = se3_exp(d[:6]), se3_exp(d[6:])
            Xn, Yn = X @ EX, Y @ EY
            dt = max(np.linalg.norm(EX[:3, 3]), np.linalg.norm(EY[:3, 3]))
            dr = max(np.linalg.norm(d[:3]), np.linalg.norm(d[6:9]))
            e_new = linearize(m, xyz, cov6, starts, tau, Xn, Yn, max_corr, corr=corr)[0]["error"] + small_terms(Xn, Yn, Xp, w_prior, w_between)[0]
        status = None
        if solved and e_new < e:
            X, Y, lam, need_lin = Xn, Yn, lam / P["lambda_factor"], True
            de = e - e_new
            if not (dt < 1e-10 and dr < 1e-10) and dt < P["step_translation_tol"] and dr < P["step_rotation_tol"]:
                status = io.ALIGN_CONVERGED
            elif de <= P["absolute_error_tol"] or de / e <= P["relative_error_tol"]:
                status = io.ALIGN_CONVERGED
            elif iterations >= P["max_iterations"]:
                status = io.ALIGN_MAX_ITERATIONS
            e = e_new
        else:
            lam *= P["lambda_factor"]
            if lam > P["lambda_upper_bound"]:
                status = io.ALIGN_LAMBDA_EXCEEDED
        if status is not None:
            return result(status)


# ---------------------------------------------------------------------------------------------------------------------
# motion-distorted hdl32 frames (test data): each ray group of <= 0.5 ms is cast from the ground-truth pose at its time
# ---------------------------------------------------------------------------------------------------------------------
SPEED, EXTRA_YAW_RATE, ARC_RADIUS, ARC_CENTER, SCAN_PERIOD, GROUP = 10.0, 0.35, 40.0, (0.0, -45.0), 0.1, 5e-4


def gt_pose(t):
    """T_world_sensor at time t (s): 10 m/s along the arc of synth.arc_trajectory (the hall's obstacle-free corridor), the
    heading turning 0.25 rad/s with the arc plus 0.35 rad/s of its own (0.6 rad/s in all)"""
    phi = -0.5 + SPEED * t / ARC_RADIUS
    x = ARC_CENTER[0] + ARC_RADIUS * np.sin(phi)
    y = ARC_CENTER[1] + ARC_RADIUS * np.cos(phi)
    from glim_b200 import synth

    return synth.pose(x, y, 0.0, yaw=-phi - EXTRA_YAW_RATE * t)


def distorted_frame(scene, k, n_rays, rng, noise=0.02):
    """frame k (scan start 0.1 k s) in the sensor frame of each point's capture time -> (points (N,4), times (N,) relative to
    the scan start, ascending)"""
    from glim_b200 import synth

    d, t = synth.sensor_pattern("hdl32", None, n_rays)
    g = np.floor(t / GROUP).astype(np.int64)
    pts, tms = [], []
    for gi in np.unique(g):
        sel = g == gi
        T = gt_pose(SCAN_PERIOD * k + gi * GROUP)
        dw = d[sel] @ T[:3, :3].T
        r = synth._raycast(scene, T[:3, 3], dw, 100.0)
        r = r + rng.normal(0.0, noise, r.shape)
        ok = np.isfinite(r) & (r > 0.5) & (r < 100.0)
        pts.append(d[sel][ok] * r[ok, None])
        tms.append(t[sel][ok])
    p = np.concatenate(pts)
    return np.ascontiguousarray(np.concatenate([p, np.ones((len(p), 1))], axis=1)), np.ascontiguousarray(np.concatenate(tms))
