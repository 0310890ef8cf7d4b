"""gb_vgicp_align's Levenberg-Marquardt rule (include/glim_b200.h) restated in fp64 on the oracle's linearize_gpumap /
error_gpumap -- the reference the CPU test of the host-compiled rule and the GPU tests compare against.  Test
infrastructure: written independently of glim_b200/csrc/gb_align_math.cuh (numpy Cholesky / solve, synth.se3_exp)."""
import numpy as np

from glim_b200 import synth
from oracle import oracle

ALIGN_CONVERGED, ALIGN_MAX_ITERATIONS, ALIGN_LAMBDA_EXCEEDED, ALIGN_DEGENERATE = 0, 1, 2, 3
ALIGN_DEFAULTS = dict(max_iterations=8, lambda_initial=1e-5, lambda_factor=10.0, lambda_upper_bound=1e5, relative_error_tol=1e-5,
                      absolute_error_tol=0.1, step_translation_tol=1e-3, step_rotation_tol=1e-3 * np.pi / 180.0)


def align_gpumap(maps, xyz, cov6, T0, params=None, normals=None):
    """maps: the problem's levels (oracle.GpuMap), all with the same source (xyz, cov6 in the device's fp32 layout);
    params: dict of gb_align_params fields (missing ones take ALIGN_DEFAULTS); normals: surface validation on every level.
    -> dict(T, error, num_inliers, lambda, iterations, trials, status)"""
    P = dict(ALIGN_DEFAULTS, **(params or {}))
    xyz, cov6 = np.ascontiguousarray(xyz, dtype=np.float32), np.ascontiguousarray(cov6, dtype=np.float32)
    T = np.asarray(T0, dtype=np.float64).copy()
    lam, need_lin, iterations, trials = P["lambda_initial"], True, 0, 0
    H, b, e, n, keep = None, None, 0.0, 0.0, []

    def result(status):
        return {"T": T, "error": e, "num_inliers": n, "lambda": lam, "iterations": iterations, "trials": trials, "status": status}

    while True:
        if need_lin:  # 1. linearize every level at T, sums in level order
            H, b, e, n, keep = np.zeros((6, 6)), np.zeros(6), 0.0, 0.0, []
            for m in maps:
                raw, corr = oracle.linearize_gpumap(m, xyz, cov6, T, normals=normals)
                r = oracle.split122(raw)
                H, b, e, n = H + r["H_ss"], b + r["b_s"], e + r["error"], n + r["num_inliers"]
                keep.append(corr != -2)  # points the surface gate turned away at T do not count in error() either
            iterations += 1
            need_lin = False
            if n == 0 and iterations == 1:
                return result(ALIGN_DEGENERATE)
        # 2. (H + lambda I) delta = -b by Cholesky
        trials += 1
        A = H + lam * np.eye(6)
        try:
            np.linalg.cholesky(A)
            delta = np.linalg.solve(A, -b)
            solved = bool(np.isfinite(delta).all())
        except np.linalg.LinAlgError:
            solved = False
        if solved:
            E = synth.se3_exp(delta)
            Tn = T @ E
            dt, dr = float(np.linalg.norm(E[:3, 3])), float(np.linalg.norm(delta[:3]))
            # 3. error at T' with the inliers of T
            e_new = sum(oracle.error_gpumap(m, xyz[k], cov6[k], T, Tn) for m, k in zip(maps, keep))
        status = None
        if solved and e_new < e:  # 4. accept
            T, lam, need_lin = Tn, lam / P["lambda_factor"], True
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
