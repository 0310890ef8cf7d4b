"""The Levenberg-Marquardt rule of gb_vgicp_align and gb_ct_gicp_align (include/glim_b200.h) restated once, in fp64 -- the
reference the CPU tests of the host-compiled rule and the GPU tests compare against.  Test infrastructure: written
independently of glim_b200/csrc/gb_align_math.cuh (numpy Cholesky / solve, synth.se3_exp).  Each problem's restatement
(tests/align_oracle.py, ivox_oracle.py, grid_oracle.py, ct_oracle.py) passes in what is its own: the linearization, the error
with the inliers of the last linearization and the retraction."""
import numpy as np

from glim_b200 import synth

ALIGN_CONVERGED, ALIGN_MAX_ITERATIONS, ALIGN_LAMBDA_EXCEEDED, ALIGN_DEGENERATE = 0, 1, 2, 3
ALIGN_DEFAULTS = dict(max_iterations=8, lambda_initial=1e-5, lambda_factor=10.0, lambda_upper_bound=1e5, relative_error_tol=1e-5,
                      absolute_error_tol=0.1, step_translation_tol=1e-3, step_rotation_tol=1e-3 * np.pi / 180.0)
CT_DEFAULTS = dict(max_iterations=8, lambda_initial=1e-10, lambda_factor=10.0, lambda_upper_bound=1e5, relative_error_tol=1e-5,
                   absolute_error_tol=1e-2, step_translation_tol=0.0, step_rotation_tol=0.0)


def levenberg_marquardt(linearize, error, retract, x0, params):
    """The rule on one problem.  linearize(x) -> (H, b, e, n, state): the system, error and inlier count at x, and whatever
    error() needs of that linearization; error(state, x_new) -> the error at x_new with the inliers of the linearization that
    returned state; retract(x, delta) -> (x_new, dt, dr): the trial and its step size (translation norm, rotation angle).
    params: every gb_align_params field.  -> dict(x, error, num_inliers, lambda, iterations, trials, status)"""
    P = params
    x = x0
    lam, need_lin, iterations, trials = P["lambda_initial"], True, 0, 0
    H, b, e, n, state = None, None, 0.0, 0.0, None

    def result(status):
        return {"x": x, "error": e, "num_inliers": n, "lambda": lam, "iterations": iterations, "trials": trials, "status": status}

    while True:
        if need_lin:  # 1. linearize at x
            H, b, e, n, state = linearize(x)
            iterations += 1
            need_lin = False
            if n == 0 and iterations == 1:
                return result(ALIGN_DEGENERATE)
        # 2. (H + lambda I) delta = -b by Cholesky
        trials += 1
        A = H + lam * np.eye(len(b))
        try:
            np.linalg.cholesky(A)
            delta = np.linalg.solve(A, -b)
            solved = bool(np.isfinite(delta).all())
        except np.linalg.LinAlgError:
            solved = False
        if solved:
            xn, dt, dr = retract(x, delta)
            e_new = error(state, xn)  # 3. error at x' with the inliers of x
        status = None
        if solved and e_new < e:  # 4. accept
            x, lam, need_lin = xn, lam / P["lambda_factor"], True
            de = e - e_new
            if not (dt < 1e-10 and dr < 1e-10) and dt < P["step_translation_tol"] and dr < P["step_rotation_tol"]:
                status = ALIGN_CONVERGED
            elif de <= P["absolute_error_tol"] or de / e <= P["relative_error_tol"]:
                status = ALIGN_CONVERGED
            elif iterations >= P["max_iterations"]:
                status = ALIGN_MAX_ITERATIONS
            e = e_new
        else:  # 5. reject
            lam *= P["lambda_factor"]
            if lam > P["lambda_upper_bound"]:
                status = ALIGN_LAMBDA_EXCEEDED
        if status is not None:
            return result(status)


def retract_pose(T, delta):
    """T Exp(delta) and the size of the step Exp(delta)"""
    E = synth.se3_exp(delta)
    return T @ E, float(np.linalg.norm(E[:3, 3])), float(np.linalg.norm(delta[:3]))


def align_pose(linearize, error, T0, params=None):
    """gb_vgicp_align's rule on one pose problem (linearize, error as levenberg_marquardt's, over a 4x4 pose); params: dict of
    gb_align_params fields (missing ones take ALIGN_DEFAULTS).  -> dict(T, error, num_inliers, lambda, iterations, trials,
    status)"""
    r = levenberg_marquardt(linearize, error, retract_pose, np.asarray(T0, dtype=np.float64).copy(), dict(ALIGN_DEFAULTS, **(params or {})))
    r["T"] = r.pop("x")
    return r
