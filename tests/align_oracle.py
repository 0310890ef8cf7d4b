"""gb_vgicp_align's Levenberg-Marquardt problem on the oracle's linearize_gpumap / error_gpumap: the levels of one problem and
their surface gate, driven by the rule's restatement in tests/lm_oracle.py -- the reference the CPU test of the host-compiled
rule and the GPU tests compare against."""
import numpy as np

from oracle import oracle
from tests import lm_oracle as lm


def align_gpumap(maps, xyz, cov6, T0, params=None, normals=None):
    """maps: the problem's levels (oracle.GpuMap), all with the same source (xyz, cov6 in the device's fp32 layout);
    params: dict of gb_align_params fields (missing ones take lm_oracle.ALIGN_DEFAULTS); normals: surface validation on every level.
    -> dict(T, error, num_inliers, lambda, iterations, trials, status)"""
    xyz, cov6 = np.ascontiguousarray(xyz, dtype=np.float32), np.ascontiguousarray(cov6, dtype=np.float32)

    def linearize(T):  # every level at T, sums in level order
        H, b, e, n, keep = np.zeros((6, 6)), np.zeros(6), 0.0, 0.0, []
        for m in maps:
            raw, corr = oracle.linearize_gpumap(m, xyz, cov6, T, normals=normals)
            r = oracle.split122(raw)
            H, b, e, n = H + r["H_ss"], b + r["b_s"], e + r["error"], n + r["num_inliers"]
            keep.append(corr != -2)  # points the surface gate turned away at T do not count in error() either
        return H, b, e, n, (T, keep)

    def error(state, Tn):
        T, keep = state
        return sum(oracle.error_gpumap(m, xyz[k], cov6[k], T, Tn) for m, k in zip(maps, keep))

    return lm.align_pose(linearize, error, T0, params)
