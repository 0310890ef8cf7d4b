"""gb_pose_graph_optimize's rule (include/glim_b200.h) restated in fp64 over tests/lm_oracle.py and tests/graph_oracle.py: the
system of the factors' records, then the between terms, then the priors; numpy's Cholesky and solve; synth.se3_exp for the
retraction and scipy for Log.  Test infrastructure, written independently of glim_b200/csrc/gb_pose_graph_math.cuh."""
import numpy as np

from glim_b200 import synth
from tests import graph_oracle as go
from tests import lm_oracle as lm


def adjoint(T):
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = T[:3, :3]
    A[3:, :3] = go.hat3(T[:3, 3]) @ T[:3, :3]
    return A


def between_term(Ti, Tj, Z, L, k):
    """-> (error, w, J_i, J_j, r) of the between term: r = Log(Z^-1 T_i^-1 T_j), GTSAM's BetweenFactor Jacobians, the Huber
    IRLS weight on m = sqrt(r^T L r) and the error 2 rho(m) (r^T L r without Huber)"""
    D = synth.inv_pose(Ti) @ Tj
    r = go.se3_log(synth.inv_pose(Z) @ D)
    Jj = go.jr_inv(r)
    Ji = -Jj @ adjoint(synth.inv_pose(D))
    m2 = float(r @ L @ r)
    m = np.sqrt(max(m2, 0.0))
    if k and m > k:
        return 2.0 * k * m - k * k, k / m, Ji, Jj, r
    return m2, 1.0, Ji, Jj, r


def between_record(Ti, Tj, Z, L, k):
    """the term as a record dict (H_tt = H_ii, H_ss = H_jj, H_ts = H_ij, b_t, b_s, error, num_inliers = 0)"""
    e, w, Ji, Jj, r = between_term(Ti, Tj, Z, L, k)
    return {"H_tt": w * Ji.T @ L @ Ji, "H_ss": w * Jj.T @ L @ Jj, "H_ts": w * Ji.T @ L @ Jj, "b_t": w * Ji.T @ L @ r, "b_s": w * Jj.T @ L @ r,
            "error": e, "num_inliers": 0.0}


def assemble(K, fkeys, frecords, bkeys, brecords, qkeys, qblocks):
    """the system summed per entry in the rule's order: factor records in record order, then between records in term order
    (both dicts as graph_oracle.assemble reads), then each prior's (H 6x6, b 6, e) in prior order; the lower triangle
    mirrored -> (H, b, e, n)"""
    n = 6 * K
    H, b, e, m = np.zeros((n, n)), np.zeros(n), 0.0, 0.0
    for (t, s), r in list(zip(fkeys, frecords)) + list(zip(bkeys, brecords)):
        T, S = slice(6 * t, 6 * t + 6), slice(6 * s, 6 * s + 6)
        H[T, T] += r["H_tt"]
        H[S, S] += r["H_ss"]
        H[T, S] += r["H_ts"]
        H[S, T] += r["H_ts"].T
        b[T] += r["b_t"]
        b[S] += r["b_s"]
        e += r["error"]
        m += r["num_inliers"]
    for k, (Hp, bp, ep) in zip(qkeys, qblocks):
        H[6 * k:6 * k + 6, 6 * k:6 * k + 6] += Hp
        b[6 * k:6 * k + 6] += bp
        e += ep
    return np.tril(H) + np.tril(H, -1).T, b, e, m


def optimize(linearize, error, fkeys, T0, priors=(), betweens=(), params=None):
    """The rule on one graph.  linearize(f, T_ts) -> (record dict, state); error(f, state, T_ts) -> its error with the inliers of
    that linearization (graph_oracle.optimize's); fkeys: (t, s) per factor; T0: (K,4,4); priors: (key, Z, w); betweens: (i, j, Z,
    L 6x6, k).  -> dict(T (K,4,4), error, num_inliers, lambda, iterations, trials, status)"""
    K, F = len(T0), len(fkeys)

    def rows(T):
        return [synth.inv_pose(T[t]) @ T[s] for t, s in fkeys]

    def lin(T):
        out = [linearize(f, d) for f, d in enumerate(rows(T))]
        brecs = [between_record(T[i], T[j], Z, L, k) for i, j, Z, L, k in betweens]
        qblocks = [go.prior_term(T[k], Z, w)[1:] + (go.prior_term(T[k], Z, w)[0],) for k, Z, w in priors]
        H, b, e, m = assemble(K, fkeys, [r for r, _ in out], [(i, j) for i, j, _, _, _ in betweens], brecs, [k for k, _, _ in priors], qblocks)
        if F == 0:
            m = 1.0  # no factor: never DEGENERATE (the result's num_inliers is 0)
        return H, b, e, m, [st for _, st in out]

    def err(states, Tn):
        e = 0.0
        for f, d in enumerate(rows(Tn)):
            e += error(f, states[f], d)
        for i, j, Z, L, k in betweens:
            e += between_term(Tn[i], Tn[j], Z, L, k)[0]
        for k, Z, w in priors:
            e += go.prior_term(Tn[k], Z, w)[0]
        return e

    def retract(T, delta):
        out, dt, dr = [], 0.0, 0.0
        for k in range(K):
            E = synth.se3_exp(delta[6 * k:6 * k + 6])
            out.append(T[k] @ E)
            dt, dr = max(dt, float(np.linalg.norm(E[:3, 3]))), max(dr, float(np.linalg.norm(delta[6 * k:6 * k + 3])))
        return np.stack(out), dt, dr

    r = lm.levenberg_marquardt(lin, err, retract, np.asarray(T0, dtype=np.float64).copy(), dict(lm.ALIGN_DEFAULTS, **(params or {})))
    r["T"] = r.pop("x")
    if F == 0:
        r["num_inliers"] = 0.0
    return r


def huber_weights(T, betweens):
    """each between term's IRLS weight at poses T"""
    return [between_term(T[i], T[j], Z, L, k)[1] for i, j, Z, L, k in betweens]
