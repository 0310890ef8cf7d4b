"""numpy restatement of the plane bundle adjustment rules of include/glim_b200.h (gb_plane_patch, gb_plane_auto_radius,
gb_plane_evm_*), point by point: the selection, the patch statistics (eigenvalues through oracle.eigen_sym3, the solver the
device uses), the modal's auto-radius loop, the factor's keys and moments, and the PlaneEVMFactor error, gradient and exact
Hessian from the per-point formulas (eigenpairs from numpy's eigh)."""
import numpy as np

from glim_b200 import synth
from oracle import oracle

DEFAULTS = {"radius": 1.0, "max_frame_distance": 25.0, "min_radius": 0.1, "max_radius": 5.0, "plane_eps": 0.01}


def params(**kw):
    p = dict(DEFAULTS)
    p.update(kw)
    return p


def select(frames, poses, center, radius, max_frame_distance):
    """frames: K (N_k, 3) float32 local points in original order; poses K (4, 4) T_world_frame.  -> (ids uint64, q (n, 3),
    local (n, 3) fp64) of the selected points, frame-major and ascending"""
    c = np.asarray(center, np.float64)
    ids, qs, loc = [], [], []
    for k, (a, T) in enumerate(zip(frames, poses)):
        T = np.asarray(T, np.float64)
        u = T[:3, 3] - c
        if not (np.sqrt((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]) <= max_frame_distance):
            continue
        a64 = np.asarray(a, np.float32).astype(np.float64).reshape(-1, 3)
        R = T[:3, :3]
        q = ((a64[:, 0:1] * R[:, 0] + a64[:, 1:2] * R[:, 1]) + a64[:, 2:3] * R[:, 2]) + u
        with np.errstate(invalid="ignore"):
            sel = np.nonzero(((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) < radius * radius)[0]
        ids.append((np.uint64(k) << np.uint64(32)) | sel.astype(np.uint64))
        qs.append(q[sel])
        loc.append(a64[sel])
    if not ids:
        return np.zeros(0, np.uint64), np.zeros((0, 3)), np.zeros((0, 3))
    return np.concatenate(ids), np.concatenate(qs), np.concatenate(loc)


def margin(frames, poses, center, radius, max_frame_distance):
    """the smallest | |q| / radius - 1 | over the points of the participating frames (scenes keep it above 1e-6)"""
    c = np.asarray(center, np.float64)
    best = np.inf
    for a, T in zip(frames, poses):
        T = np.asarray(T, np.float64)
        u = T[:3, 3] - c
        if not (np.linalg.norm(u) <= max_frame_distance):
            continue
        q = np.asarray(a, np.float32).astype(np.float64) @ T[:3, :3].T + u
        d = np.linalg.norm(q, axis=1)
        best = min(best, float(np.min(np.abs(d / radius - 1.0))) if len(d) else np.inf)
    return best


def stats(q):
    """(n, eigenvalues ascending) of calc_eigenvalues over the points q (n, 3) about the centre"""
    n = len(q)
    if n == 0:
        return 0, np.full(3, np.nan)
    s = q.sum(0)
    S = q.T @ q
    mean = s / n
    A = np.empty((3, 3))
    for r in range(3):
        for c in range(r, 3):
            A[r, c] = A[c, r] = (S[r, c] - mean[r] * s[c]) / n
    ev, _ = oracle.eigen_sym3(A)
    return n, ev


def auto_radius_loop(stats_at, p):
    """the modal's Auto Radius loop over stats_at(r) -> (n, ev): (r, n, ev, trials [(radius, n)])"""
    r = p["radius"]
    n, ev = stats_at(r)
    trials = []
    for _ in range(10):
        with np.errstate(invalid="ignore", divide="ignore"):
            planar = ev[0] / ev[2] > p["plane_eps"]
        trial = r * 0.8 if planar else r * 1.1
        if trial < p["min_radius"] or trial > p["max_radius"]:
            break
        n2, ev2 = stats_at(trial)
        trials.append((trial, n2))
        if n2 < 10:
            break
        with np.errstate(invalid="ignore", divide="ignore"):
            if trial > p["radius"] and ev2[0] / ev2[2] > p["plane_eps"]:
                break
        r, n, ev = trial, n2, ev2
    return r, n, ev, trials


def auto_radius(frames, poses, center, **kw):
    p = params(**kw)
    return auto_radius_loop(lambda r: stats(select(frames, poses, center, r, p["max_frame_distance"])[1]), p)


def factor_keys(frames, poses, center, radius=1.0, max_frame_distance=25.0):
    """(keys: frame indices, per-key local points (fp64)) of the factor created at radius"""
    ids, _, loc = select(frames, poses, center, radius, max_frame_distance)
    fr = (ids >> np.uint64(32)).astype(np.int64)
    keys = [int(k) for k in np.unique(fr)]
    return keys, [loc[fr == k] for k in keys]


def moments(pts):
    """{N, mean, scatter (3, 3)} of one key's local points, two passes"""
    m = pts.mean(0)
    d = pts - m
    return len(pts), m, d.T @ d


def points_world(key_pts, X, o):
    return [a @ np.asarray(T)[:3, :3].T + (np.asarray(T)[:3, 3] - o) for a, T in zip(key_pts, X)]


def error(key_pts, X, o):
    p = np.concatenate(points_world(key_pts, X, o))
    d = p - p.mean(0)
    return np.linalg.eigvalsh(d.T @ d / len(p))[0]


def linearize(key_pts, X, o):
    """(e, b (6K,), H (6K, 6K), degenerate) of PlaneEVMFactor by the per-point formulas: b = 1/2 de/dxi, H = 1/2 d2e/dxi2 along
    X_k Exp(xi_k), the second-order term of Exp included"""
    K = len(key_pts)
    P = points_world(key_pts, X, o)
    p = np.concatenate(P)
    N = len(p)
    pbar = p.mean(0)
    lam, U = np.linalg.eigh((p - pbar).T @ (p - pbar) / N)
    e = lam[0]
    if not (lam[1] - lam[0] > 0):
        return e, np.zeros(6 * K), np.zeros((6 * K, 6 * K)), True
    u0 = U[:, 0]
    g = np.zeros(6 * K)
    He = np.zeros((6 * K, 6 * K))
    Zs, Ws = np.zeros((K, 6)), np.zeros((2, K, 6))
    for k, (a, T, pk) in enumerate(zip(key_pts, X, P)):
        R = np.asarray(T)[:3, :3]
        d = pk - pbar
        # J_i^T v = [a_i x (R^T v); R^T v] for J_i = R [-hat(a_i), I]
        JT = lambda vec: np.concatenate([np.cross(a, vec @ R), vec @ R], axis=1)
        s0 = d @ u0
        grad_p = (2.0 / N) * s0[:, None] * u0[None, :]
        gi = JT(grad_p)
        g[6 * k:6 * k + 6] = gi.sum(0)
        Z = JT(np.repeat(u0[None, :], len(a), 0))
        He[6 * k:6 * k + 6, 6 * k:6 * k + 6] += (2.0 / N) * Z.T @ Z
        Zs[k] = Z.sum(0)
        for j, m in enumerate((1, 2)):
            um = U[:, m]
            w = s0[:, None] * um[None, :] + (d @ um)[:, None] * u0[None, :]
            Ws[j, k] = JT(w).sum(0)
        h = grad_p @ R  # R^T dE/dp_i per row
        blk = np.zeros((6, 6))
        for hi, ai in zip(h, a):
            blk[:3, :3] += 0.5 * (np.outer(hi, ai) + np.outer(ai, hi)) - np.dot(hi, ai) * np.eye(3)
            blk[:3, 3:] += -0.5 * synth.hat(hi)
            blk[3:, :3] += 0.5 * synth.hat(hi)
        He[6 * k:6 * k + 6, 6 * k:6 * k + 6] += blk
    He -= (2.0 / N**2) * np.outer(Zs.reshape(-1), Zs.reshape(-1))
    for j, m in enumerate((1, 2)):
        He += (2.0 / N**2) * np.outer(Ws[j].reshape(-1), Ws[j].reshape(-1)) / (lam[0] - lam[m])
    return e, 0.5 * g, 0.5 * He, False


def perturbed(X, xi):
    """X_k Exp(xi_k) for xi (6K,)"""
    return [np.asarray(T) @ synth.se3_exp(xi[6 * k:6 * k + 6]) for k, T in enumerate(X)]


def adjoint(T):
    """Ad(T) on tangents [omega; nu]"""
    T = np.asarray(T)
    R, t = T[:3, :3], T[:3, 3]
    A = np.zeros((6, 6))
    A[:3, :3] = R
    A[3:, 3:] = R
    A[3:, :3] = synth.hat(t) @ R
    return A
