"""numpy restatement of gb_find_overlapping_submaps' candidate rule (include/glim_b200.h): the candidate pairs in lexicographic
order, delta = T_i^-1 T_j with every dot product ((a0 b0 + a1 b1) + a2 b2) (numpy rounds each operation, no FMA), and the
distance gate (t0 t0 + t1 t1) + t2 t2 <= max_distance^2."""
import numpy as np


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def deltas(Ti, Tj):
    """T_i^-1 T_j of (..., 4, 4) poses, as the device computes it"""
    Ti, Tj = np.asarray(Ti, np.float64), np.asarray(Tj, np.float64)
    Ri, Rj = np.swapaxes(Ti[..., :3, :3], -1, -2), np.swapaxes(Tj[..., :3, :3], -1, -2)  # rows = columns of R
    D = np.zeros(np.broadcast_shapes(Ti.shape, Tj.shape))
    for r in range(3):
        for c in range(3):
            D[..., r, c] = _dot(Ri[..., r, :], Rj[..., c, :])
        D[..., r, 3] = _dot(Ri[..., r, :], Tj[..., :3, 3]) + (-_dot(Ri[..., r, :], Ti[..., :3, 3]))
    D[..., 3, 3] = 1.0
    return D


def gate(D, max_distance):
    return _dot(D[..., :3, 3], D[..., :3, 3]) <= max_distance * max_distance


def slots(S, first_source):
    """every (i, j) with i < j, j >= first_source, in lexicographic order"""
    return [(i, j) for i in range(S) for j in range(max(i + 1, first_source), S)]


def candidates(T, first_source=0, existing=(), max_distance=100.0):
    """[(i, j, delta)] of the gated candidates; `existing` is looked up as ordered pairs"""
    ex = {(int(a), int(b)) for a, b in existing}
    out = []
    for i, j in slots(len(T), first_source):
        if (i, j) in ex:
            continue
        D = deltas(T[i], T[j])
        if gate(D, max_distance):
            out.append((i, j, D))
    return out
