"""gb_nav_graph_optimize's rule (include/glim_b200.h) restated in fp64 over tests/pose_graph_oracle.py and tests/lm_oracle.py:
6-dof slots (poses, then velocities with three pinned dofs, then biases), the system summed in the stated order (factor
records, between terms, IMU terms, vector terms, priors), numpy's solve and the retraction by slot kind.  Test infrastructure,
written independently of glim_b200/csrc/gb_pose_graph_math.cuh."""
import numpy as np

from glim_b200 import synth
from tests import graph_oracle as go
from tests import imu_oracle as io
from tests import lm_oracle as lm
from tests import pose_graph_oracle as pgo


class Graph:
    """K_X poses, K_V velocities, K_B biases (local indices); imu: (xi, vi, xj, vj, bi, record dict); vec: (kind, a, b, z, w)
    with io's kind numbers"""

    def __init__(self, KX, KV, KB, priors=(), betweens=(), imu=(), vec=()):
        self.KX, self.KV, self.KB = KX, KV, KB
        self.priors, self.betweens, self.imu, self.vec = list(priors), list(betweens), list(imu), list(vec)
        self.K = KX + KV + KB

    def vslot(self, k):
        return self.KX + k

    def bslot(self, k):
        return self.KX + self.KV + k

    def slots(self):
        """each IMU then vector term's slots, in the order of its Jacobian's column blocks"""
        out = [[xi, self.vslot(vi), xj, self.vslot(vj), self.bslot(bi)] for xi, vi, xj, vj, bi, _ in self.imu]
        for kind, a, b, _, _ in self.vec:
            if kind == io.VELOCITY_PRIOR:
                out.append([self.vslot(a)])
            elif kind == io.BIAS_PRIOR:
                out.append([self.bslot(a)])
            elif kind == io.VELOCITY_BETWEEN:
                out.append([self.vslot(a), self.vslot(b)])
            elif kind == io.BIAS_BETWEEN:
                out.append([self.bslot(a), self.bslot(b)])
            else:
                out.append([a, self.vslot(b)])
        return out

    def terms(self, X):
        """-> [(slots, H 6m x 6m, b 6m, e)] of the IMU terms then the vector terms at state X = (poses, vels, biases)"""
        T, V, Bs = X
        out = []
        for (xi, vi, xj, vj, bi, rec), sl in zip(self.imu, self.slots()):
            r, J = io.imu_residual(T[xi], V[vi], T[xj], V[vj], Bs[bi], rec)
            L = np.linalg.inv(rec["covariance"])
            out.append((sl, J.T @ L @ J, J.T @ L @ r, float(r @ L @ r)))
        for (kind, a, b, z, w), sl in zip(self.vec, self.slots()[len(self.imu):]):
            xa = {io.VELOCITY_PRIOR: V, io.BIAS_PRIOR: Bs, io.VELOCITY_BETWEEN: V, io.BIAS_BETWEEN: Bs, io.ROTATE_VELOCITY: T}[kind][a]
            xb = None if kind in (io.VELOCITY_PRIOR, io.BIAS_PRIOR) else (V if kind != io.BIAS_BETWEEN else Bs)[b]
            r, J = io.vector_residual(kind, xa, xb, z)
            J = J[:, :6 * len(sl)]
            out.append((sl, w * J.T @ J, w * J.T @ r, float(w * r @ r)))
        return out


def assemble(K, fkeys, frecords, bkeys, brecords, nav, qkeys, qblocks):
    """the system summed per entry in the rule's order: factor records, between records (pose_graph_oracle's dicts), the nav
    terms [(slots, H, b, e)] in term order, then the priors (H 6x6, b 6, e); the lower triangle mirrored -> (H, b, e)"""
    n = 6 * K
    H, b, e = np.zeros((n, n)), np.zeros(n), 0.0
    for (t, s), r in list(zip(fkeys, frecords)) + list(zip(bkeys, brecords)):
        Ts, Ss = slice(6 * t, 6 * t + 6), slice(6 * s, 6 * s + 6)
        H[Ts, Ts] += r["H_tt"]
        H[Ss, Ss] += r["H_ss"]
        H[Ts, Ss] += r["H_ts"]
        H[Ss, Ts] += r["H_ts"].T
        b[Ts] += r["b_t"]
        b[Ss] += r["b_s"]
        e += r["error"]
    for sl, Hn, bn, en in nav:
        for a, sa in enumerate(sl):
            for c, sc in enumerate(sl):
                H[6 * sa:6 * sa + 6, 6 * sc:6 * sc + 6] += Hn[6 * a:6 * a + 6, 6 * c:6 * c + 6]
            b[6 * sa:6 * sa + 6] += bn[6 * a:6 * a + 6]
        e += en
    for k, (Hp, bp, ep) in zip(qkeys, qblocks):
        H[6 * k:6 * k + 6, 6 * k:6 * k + 6] += Hp
        b[6 * k:6 * k + 6] += bp
        e += ep
    return np.tril(H) + np.tril(H, -1).T, b, e


def pinned(g):
    """the dead dofs: the last three of every velocity slot"""
    return [6 * g.vslot(k) + d for k in range(g.KV) for d in (3, 4, 5)]


def optimize(g, X0, params=None, factors=None):
    """The rule on one graph.  X0 = (poses (K_X,4,4), velocities (K_V,3), biases (K_B,6)); factors: None or (fkeys, linearize,
    error) as pose_graph_oracle.optimize takes them.  -> dict(X, error, num_inliers, lambda, iterations, trials, status)"""
    fkeys, linearize, error = factors if factors else ([], None, None)
    F = len(fkeys)

    def rows(T):
        return [synth.inv_pose(T[t]) @ T[s] for t, s in fkeys]

    def lin(X):
        T = X[0]
        out = [linearize(f, d) for f, d in enumerate(rows(T))]
        brecs = [pgo.between_record(T[i], T[j], Z, L, k) for i, j, Z, L, k in g.betweens]
        qblocks = [go.prior_term(T[k], Z, w)[1:] + (go.prior_term(T[k], Z, w)[0],) for k, Z, w in g.priors]
        H, b, e = assemble(g.K, fkeys, [r for r, _ in out], [(i, j) for i, j, _, _, _ in g.betweens], brecs, g.terms(X), [k for k, _, _ in g.priors], qblocks)
        m = sum(r["num_inliers"] for r, _ in out) if F else 1.0  # no factor: never DEGENERATE
        return H, b, e, m, [st for _, st in out]

    def err(states, Xn):
        T = Xn[0]
        e = sum(error(f, states[f], d) for f, d in enumerate(rows(T))) if F else 0.0
        for i, j, Z, L, k in g.betweens:
            e += pgo.between_term(T[i], T[j], Z, L, k)[0]
        for _, _, _, en in g.terms(Xn):
            e += en
        for k, Z, w in g.priors:
            e += go.prior_term(T[k], Z, w)[0]
        return e

    def retract(X, delta):
        T, V, Bs = X
        Tn, dt, dr = [], 0.0, 0.0
        for k in range(g.KX):
            E = synth.se3_exp(delta[6 * k:6 * k + 6])
            Tn.append(T[k] @ E)
            dt, dr = max(dt, float(np.linalg.norm(E[:3, 3]))), max(dr, float(np.linalg.norm(delta[6 * k:6 * k + 3])))
        Vn = np.array([V[k] + delta[6 * g.vslot(k):6 * g.vslot(k) + 3] for k in range(g.KV)]).reshape(-1, 3)
        Bn = np.array([Bs[k] + delta[6 * g.bslot(k):6 * g.bslot(k) + 6] for k in range(g.KB)]).reshape(-1, 6)
        return (np.stack(Tn), Vn, Bn), dt, dr

    pins = pinned(g)

    def retract_pinned(X, delta):  # the pinned dofs step 0: their rows solve 1 x = 0
        delta = delta.copy()
        delta[pins] = 0.0
        return retract(X, delta)

    P = dict(lm.ALIGN_DEFAULTS, **(params or {}))
    X0 = (np.asarray(X0[0], dtype=np.float64), np.asarray(X0[1], dtype=np.float64).reshape(-1, 3), np.asarray(X0[2], dtype=np.float64).reshape(-1, 6))
    r = lm.levenberg_marquardt(lin, err, retract_pinned, X0, P)
    if F == 0:
        r["num_inliers"] = 0.0
    return r
