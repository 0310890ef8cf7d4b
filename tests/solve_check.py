"""The diagonally scaled backward error of one damped Levenberg-Marquardt step, for the dense fp64 solvers of gb_graph_optimize,
gb_pose_graph_optimize and gb_nav_graph_optimize.  Test infrastructure.

Cholesky is invariant to symmetric diagonal scaling, so a correct solve of A d = -b (A = H + lambda I) has

    eta = |D (A d + b)|_inf / (|D A D|_inf |D^-1 d|_inf + |D b|_inf),   D = diag(A)^-1/2,

of order n u whatever the precisions of the graph -- a 1e10 anchor beside 1e-2 betweens included -- where a forward error
can only be held to cond(A) u.  It needs no reference solve, only a product with A.

The device's step is read back from a max_iterations = 1 result (each pose's Log(T0^-1 T), each velocity's and bias's
difference).  Reading it back perturbs it by e, |e_i| <= eps_i = RECOVERY u (1 + |x0_i| + |x_i|) per entry (x the pose's
translation, the velocity or the bias), which moves eta by at most eta_rec = | |D A| eps |_inf / (its denominator): on a row
stiffened by the 1e10 anchor that is the largest term.  Records taken by two identical sweeps differ (their fp32 partial sums
are added by atomics), a backward perturbation of A measured as eta_rec_noise: a step solved exactly from one sweep's records
and checked against the other's.  The device is held to

    eta_dev <= FACTOR max(eta_ref, n u, eta_rec, eta_noise)

with eta_ref the restatement's own step (numpy's solve through the restatement's retraction, read back the same way)."""
import contextlib

import numpy as np
from scipy.linalg import lapack

from glim_b200 import synth
from tests import graph_oracle as go
from tests import imu_oracle as io
from tests import lm_oracle as lm
from tests import nav_graph_oracle as ngo

U = 2.0**-53
FACTOR = 16.0
RECOVERY = 4.0  # roundings of a read-back entry: the retraction's product and sum, the inverse and the Log
TILE = 64  # gb_pose_graph_optimize's tile: n is padded to a multiple of it


def padded(n):
    return -(-n // TILE) * TILE


def scaled_backward_error(A, delta, b, live=None, eps=None):
    """eta of the step delta for A delta = -b over the live rows (all when None); delta must be exactly 0 elsewhere (the
    pinned velocity dofs).  The residual is summed in extended precision, so its own rounding stays below the n u it is
    compared with.  With eps (per-entry read-back uncertainties) -> (eta, eta_rec), eta_rec = | |D A| eps |_inf over the
    same denominator."""
    n = len(b)
    live = np.ones(n, bool) if live is None else np.asarray(live, bool)
    assert np.all(delta[~live] == 0.0), "a pinned dof moved"
    idx = np.flatnonzero(live)
    d, bb = delta[idx], b[idx]
    D = 1.0 / np.sqrt(np.diag(A)[idx])
    dl = d.astype(np.longdouble)
    r = np.empty(len(idx))
    row_norm = np.empty(len(idx))
    spread = np.zeros(len(idx))
    for s in range(0, len(idx), 1024):  # row blocks: the extended-precision copy of A stays small
        blk = idx[s:s + 1024]
        Ab = A[np.ix_(blk, idx)]
        r[s:s + 1024] = (Ab.astype(np.longdouble) @ dl + bb[s:s + 1024]) * D[s:s + 1024]
        row_norm[s:s + 1024] = (np.abs(Ab) * D[None, :]).sum(axis=1) * D[s:s + 1024]
        if eps is not None:
            spread[s:s + 1024] = (np.abs(Ab) @ eps[idx]) * D[s:s + 1024]
    den = row_norm.max() * np.abs(d / D).max() + np.abs(D * bb).max()
    eta = float(np.abs(r).max() / den)
    return eta if eps is None else (eta, float(spread.max() / den))


def condition_1norm(A, live=None):
    """LAPACK's 1-norm condition estimate of A over the live rows, from its Cholesky factor"""
    if live is not None:
        idx = np.flatnonzero(live)
        A = A[np.ix_(idx, idx)]
    c, info = lapack.dpotrf(A, lower=1)
    assert info == 0
    rcond, info = lapack.dpocon(c, np.abs(A).sum(axis=0).max(), uplo="L")
    return 1.0 / rcond


@contextlib.contextmanager
def systems():
    """every (H, b, lambda_initial) the restatements linearize while the block runs (lm.levenberg_marquardt's linearize
    wrapped): the host system of a step is H + lambda I, b"""
    seen = []
    inner = lm.levenberg_marquardt

    def spy(linearize, error, retract, x0, params):
        def lin(x):
            out = linearize(x)
            seen.append((out[0], out[1], params["lambda_initial"]))
            return out

        return inner(lin, error, retract, x0, params)

    lm.levenberg_marquardt = spy
    try:
        yield seen
    finally:
        lm.levenberg_marquardt = inner


def pose_steps(T0, T):
    """each pose's step Log(T0^-1 T) in the chart of synth.se3_exp ([rot; trans]), concatenated"""
    return np.concatenate([go.se3_log(synth.inv_pose(a) @ b) for a, b in zip(T0, T)])


def pose_eps(T0, T):
    """the read-back uncertainty of pose_steps: RECOVERY u (1 + |t0| + |t|) on each of a pose's 6 entries"""
    return np.concatenate([np.full(6, RECOVERY * U * (1.0 + np.linalg.norm(a[:3, 3]) + np.linalg.norm(b[:3, 3]))) for a, b in zip(T0, T)])


def nav_steps(X0, X):
    """the step of a navigation graph's state X = (poses, velocities, biases) from X0, in slot order: 6 per pose, the 3
    velocity dofs per velocity followed by 3 zeros, 6 per bias.  The zeros stand for the pinned dofs: a result carries 3
    entries per velocity and pg_retract never reads the pinned rows of the step, so their exact 0 cannot be read back here
    (tests/test_graph_solve_check_host.py checks it on the host schedule)."""
    d = [pose_steps(X0[0], X[0])]
    d += [np.concatenate([np.asarray(v, float) - v0, np.zeros(3)]) for v0, v in zip(X0[1], X[1])]
    d += [np.asarray(b, float) - b0 for b0, b in zip(X0[2], X[2])]
    return np.concatenate(d)


def nav_eps(X0, X):
    """the read-back uncertainty of nav_steps: pose_eps, then RECOVERY u (1 + |x0| + |x|) per velocity and bias entry"""
    e = [pose_eps(X0[0], X[0])]
    e += [np.concatenate([RECOVERY * U * (1.0 + np.abs(v0) + np.abs(np.asarray(v, float))), np.zeros(3)]) for v0, v in zip(X0[1], X[1])]
    e += [RECOVERY * U * (1.0 + np.abs(b0) + np.abs(np.asarray(b, float))) for b0, b in zip(X0[2], X[2])]
    return np.concatenate(e)


def check(label, system, d_dev, d_ref, eps, live=None, noise=None, cond=True):
    """eta of the device's step and of the restatement's on the host system (H, b, lambda), eps the device step's read-back
    uncertainty (pose_eps / nav_eps), noise None or a second sweep's system (H', b') of the same records; asserts the bound
    and returns (eta_dev, the condition estimate or None)"""
    H, b, lam = system
    A = H + lam * np.eye(len(b))
    eta_dev, eta_rec = scaled_backward_error(A, d_dev, b, live, eps)
    eta_ref = scaled_backward_error(A, d_ref, b, live)
    eta_noise = 0.0
    if noise is not None:
        eta_noise = scaled_backward_error(noise[0] + lam * np.eye(len(b)), d_ref, noise[1], live)
    n = len(b) if live is None else int(np.count_nonzero(live))
    bound = FACTOR * max(eta_ref, n * U, eta_rec, eta_noise)
    kappa = condition_1norm(A, live) if cond else None
    print(f"[solve] {label}: n {n} (N {padded(len(b))}), cond_1 {kappa if kappa is None else f'{kappa:.3g}'}, eta_dev {eta_dev:.3g}, "
          f"eta_ref {eta_ref:.3g}, eta_rec {eta_rec:.3g}, eta_noise {eta_noise:.3g}, bound {bound:.3g}")
    assert eta_dev <= bound, (label, eta_dev, eta_ref, eta_rec, eta_noise, bound)
    return eta_dev, kappa


# ---- graphs shared by the host and device checks ----


def spd6(rng, scale):
    A = rng.normal(size=(6, 6))
    L = scale * (A @ A.T + 6.0 * np.eye(6))
    return np.triu(L) + np.triu(L, 1).T  # exactly symmetric


def between_graph(K, seed, spread=(0.0, 0.0), extra=None):
    """a chain plus random extra edges (K // 2 by default) with random SPD informations scaled by 10^U(spread), starts off the
    measurements; the 1e10 anchor at key 0 as GLIM sets it.  -> (T0, priors, betweens (i, j, Z, L, 0.0))"""
    rng = np.random.default_rng(seed)
    gt = [synth.se3_exp(np.concatenate([rng.normal(size=3) * 0.5, rng.normal(size=3) * 5.0])) for _ in range(K)]
    edges = [(k, k + 1) for k in range(K - 1)]
    edges += [tuple(int(x) for x in rng.choice(K, 2, replace=False)) for _ in range(K // 2 if extra is None else extra)] if K > 2 else []
    bts = []
    for i, j in edges:
        L = spd6(rng, 10.0 ** rng.uniform(*spread))
        bts.append((i, j, synth.perturb(synth.inv_pose(gt[i]) @ gt[j], rng, 0.005, 0.02), L, 0.0))
    T0 = [gt[0]] + [synth.perturb(T, rng, 0.01, 0.05) for T in gt[1:]]
    return T0, [(0, T0[0], 1e10)], bts


def ill_conditioned_graph():
    """K = 1024 betweens with informations spread from 1e-2 to 1e8 beside the 1e10 anchor"""
    return between_graph(1024, 4100, spread=(-2.0, 8.0))


def imu_chain(m, preintegrate, seed=4200):
    """an IMU-coupled chain of m frames on imu_oracle's analytic trajectory, as sub-mapping builds it (sub_mapping.cpp:218-243):
    X, V per frame, a bias per interval; an ImuFactor per interval (preintegrate(samples, intervals, biases) -> its records, each
    interval frame i to i + 1 with bias i), a
    1e3 velocity prior per frame, a 1e6 bias prior per bias and 1e6 bias betweens, 1e6 odometry betweens between the poses and
    the 1e10 anchor on X(0); drifted starts.  Slots: m poses, then m velocities, then m - 1 biases.
    -> dict(times, bias, graph (nav_graph_oracle.Graph), X0, priors, betweens, imu, vec (io kinds), live mask)"""
    rng = np.random.default_rng(seed)
    times = 1.0 + 0.2 * np.arange(m)
    bias = np.array([0.05, -0.04, 0.03, 0.004, 0.002, -0.003])
    T_gt = [io.truth(t)[0] for t in times]
    V_gt = [io.truth(t)[1] for t in times]
    est_bias = [bias + rng.normal(size=6) * 0.002 for _ in range(m - 1)]
    v_est = [v + rng.normal(size=3) * 0.05 for v in V_gt]
    records = preintegrate(io.samples(times[0] - 0.05, times[-1] + 0.05, 200, bias), list(zip(times[:-1], times[1:])), est_bias)
    drift = np.array([0.0, 0.0, 0.002, 0.01, -0.005, 0.0])
    T0 = [T_gt[0]] + [synth.perturb(T_gt[i] @ synth.se3_exp(i * drift), rng, 0.002, 0.02) for i in range(1, m)]
    priors = [(0, T0[0], 1e10)]
    betweens = [(i, i + 1, synth.perturb(synth.inv_pose(T_gt[i]) @ T_gt[i + 1], rng, 0.001, 0.005), 1e6) for i in range(m - 1)]
    imu = [(i, i, i + 1, i + 1, i, records[i]) for i in range(m - 1)]
    vec = [(io.VELOCITY_PRIOR, i, None, v_est[i], 1e3) for i in range(m)] + [(io.BIAS_PRIOR, i, None, est_bias[i], 1e6) for i in range(m - 1)]
    vec += [(io.BIAS_BETWEEN, i - 1, i, np.zeros(6), 1e6) for i in range(1, m - 1)]
    graph = ngo.Graph(m, m, m - 1, priors, [(i, j, Z, w * np.eye(6), 0.0) for i, j, Z, w in betweens],
                      [(a, b, c, d, e, io.record_of(r) if not isinstance(r, dict) else r) for a, b, c, d, e, r in imu], vec)
    live = np.ones(6 * graph.K, bool)
    live[ngo.pinned(graph)] = False
    X0 = (np.stack(T0), np.stack(v_est), np.stack(est_bias))
    return dict(times=times, bias=bias, est_bias=est_bias, graph=graph, X0=X0, priors=priors, betweens=betweens, imu=imu, vec=vec, live=live)
