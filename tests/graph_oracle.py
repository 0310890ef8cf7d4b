"""gb_graph_optimize's rule (include/glim_b200.h) restated in fp64 over tests/lm_oracle.py: the system assembled from the factors'
records and the priors, numpy's Cholesky and solve, synth.se3_exp for the retraction and scipy for Log.  Test infrastructure,
written independently of glim_b200/csrc/gb_graph_math.cuh.  Each factor's linearization and error come in as callables: the
fp64 oracles (oracle.GpuMap, tests/grid_oracle.py, tests/icp_oracle.py) or the device's own records."""
import numpy as np
from scipy.spatial.transform import Rotation

from glim_b200 import synth
from tests import lm_oracle as lm

GRAPH_DEFAULTS = lm.ALIGN_DEFAULTS


def hat3(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def se3_log(T):
    """[w; v]: w from scipy's rotation vector, v = J_l(w)^-1 t"""
    w = Rotation.from_matrix(T[:3, :3]).as_rotvec()
    th = np.linalg.norm(w)
    K = hat3(w)
    if th < 1e-6:
        Jl = np.eye(3) + K / 2.0 + K @ K / 6.0
    else:
        Jl = np.eye(3) + (1.0 - np.cos(th)) / th**2 * K + (th - np.sin(th)) / th**3 * K @ K
    return np.concatenate([w, np.linalg.solve(Jl, T[:3, 3])])


def jr_inv(xi):
    """SE(3) right Jacobian (sum_k (-ad_xi)^k / (k+1)!) inverted"""
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = hat3(xi[:3])
    A[3:, :3] = hat3(xi[3:])
    A = -A
    J, P, f = np.eye(6), np.eye(6), 1.0
    for k in range(1, 40):
        P = P @ A
        f *= k + 1
        J = J + P / f
    return np.linalg.inv(J)


def prior_term(T, Z, w):
    """-> (e, H (6,6), b (6,)) of w |Log(Z^-1 T)|^2 (no 1/2), Jacobian J_r^-1(r)"""
    r = se3_log(synth.inv_pose(Z) @ T)
    J = jr_inv(r)
    return float(w * r @ r), w * J.T @ J, w * J.T @ r


def assemble(K, keys, records):
    """the system of the records (dicts of H_tt, H_ss, H_ts, b_t, b_s, error, num_inliers, [row, col]) at factor keys
    (t, s), summed in record order; the lower triangle mirrored, as the Cholesky reads it -> (H, b, e, n)"""
    n = 6 * K
    H, b, e, m = np.zeros((n, n)), np.zeros(n), 0.0, 0.0
    for (t, s), r in zip(keys, records):
        T, S = slice(6 * t, 6 * t + 6), slice(6 * s, 6 * s + 6)
        H[T, T] += r["H_tt"]
        H[S, S] += r["H_ss"]
        H[T, S] += r["H_ts"]
        H[S, T] += r["H_ts"].T
        b[T] += r["b_t"]
        b[S] += r["b_s"]
        e += r["error"]
        m += r["num_inliers"]
    L = np.tril(H)
    return L + np.tril(H, -1).T, b, e, m


def optimize(linearize, error, keys, T0, priors=(), params=None):
    """The rule on one problem.  linearize(f, T_ts) -> (record dict, state) of factor f at T_t^-1 T_s; error(f, state, T_ts) ->
    its error at T_ts with the inliers of the linearization that returned state; keys: (t, s) per factor; T0: (K,4,4);
    priors: (key, Z, w).  -> dict(T (K,4,4), error, num_inliers, lambda, iterations, trials, status)"""
    K = len(T0)

    def rows(T):
        return [synth.inv_pose(T[t]) @ T[s] for t, s in keys]

    def lin(T):
        out = [linearize(f, d) for f, d in enumerate(rows(T))]
        H, b, e, m = assemble(K, keys, [r for r, _ in out])
        for k, Z, w in priors:
            ep, Hp, bp = prior_term(T[k], Z, w)
            H[6 * k:6 * k + 6, 6 * k:6 * k + 6] += Hp
            b[6 * k:6 * k + 6] += bp
            e += ep
        return H, b, e, m, [st for _, st in out]

    def err(states, Tn):
        e = 0.0
        for f, d in enumerate(rows(Tn)):
            e += error(f, states[f], d)
        for k, Z, w in priors:
            e += prior_term(Tn[k], Z, w)[0]
        return e

    def retract(T, delta):
        out, dt, dr = [], 0.0, 0.0
        for k in range(K):
            E = synth.se3_exp(delta[6 * k:6 * k + 6])
            out.append(T[k] @ E)
            dt, dr = max(dt, float(np.linalg.norm(E[:3, 3]))), max(dr, float(np.linalg.norm(delta[6 * k:6 * k + 3])))
        return np.stack(out), dt, dr

    r = lm.levenberg_marquardt(lin, err, retract, np.asarray(T0, dtype=np.float64).copy(), dict(GRAPH_DEFAULTS, **(params or {})))
    r["T"] = r.pop("x")
    return r
