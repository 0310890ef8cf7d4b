"""Degenerate-neighbourhood battery for the covariance / normal estimation (CloudCovarianceEstimation::estimate with PLANE
regularisation) and its exact reference.

The battery is deterministic: a list of cases, each a small point set with the neighbour lists the k-NN returns for it
(oracle.knn_bruteforce, self-filled when the set has fewer than k_correspondences points), k_correspondences and
k_neighbors.  Every point of a case is one row.  Families: duplicates, k_neighbors = 1, self-filled lists, collinear and
near-collinear points, exact / tilted / lattice planes, discs and needles, cube corners and octahedra, generic blobs and
planes through the origin; at spreads from 1e-4 m to 10 m, offsets from 0 to 10 km and k from 1 to 32.

The exact reference of a row: A = the population covariance of its k_neighbors points, exact in rationals; its eigen
decomposition at 60 digits; C = I - (1 - 1e-3) v0 v0^T and the normal v0 oriented so that p . v0 <= 0.  A row is posed
when the gap lambda_1 - lambda_0 clears the rounding of the one-pass covariance sum(p p^T) / k - mean mean^T, whose error is
about u R^2 (u = 2^-53, R = the largest |p| of the neighbourhood): the error bar of a posed row is
POSED_C * u * R^2 / (lambda_1 - lambda_0), and a row is posed when that bar is below POSED_MAX.
"""
import functools
from fractions import Fraction

import mpmath
import numpy as np

from oracle import oracle

U = 2.0**-53
POSED_C = 16.0  # the oracle's worst error on the battery is 0.17 of this bar (test_cov_degenerate.py prints it)
POSED_MAX = 1e-3
INV_C = 4.0  # the oracle's worst invariant error on the battery is 0.09 of invariant_tol

SPREADS = (1e-4, 1e-2, 1.0, 10.0)
OFFSETS = (0.0, 10.0, 1.0e3, 1.0e4)
KS = (1, 2, 3, 5, 10, 20, 32)


def _rot(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def _place(local, spread, offset, rng, rotate=True):
    """local points (m, 3) of unit size -> (m, 4) homogeneous, rotated, scaled by spread, moved by offset in a random
    direction.  Duplicates stay exact duplicates (the same arithmetic on the same input)."""
    R = _rot(rng) if rotate else np.eye(3)
    d = rng.normal(size=3)
    o = offset * d / np.linalg.norm(d)
    P = (local @ R.T) * spread + o
    return np.concatenate([P, np.ones((len(P), 1))], axis=1)


def _families(rng):
    """(family, local points (m, 3), rotate?) of unit size"""
    g = rng.normal(size=3)
    yield "duplicates", lambda k: np.tile(g, (k, 1)), True
    yield "collinear", lambda k: np.outer(np.arange(k) - (k - 1) / 2.0, [1.0, 0.0, 0.0]), False  # exact: y and z constant
    yield "collinear_tilted", lambda k: np.outer(np.arange(k) * 0.05, [1.0, 0.0, 0.0]), True
    for lat in (1e-3, 1e-6, 1e-9, 1e-12):
        yield f"near_collinear_{lat:g}", (lambda lat: lambda k: np.concatenate([np.linspace(-1, 1, k)[:, None], lat * rng.normal(size=(k, 2))], axis=1))(lat), True
    yield "plane_axis", lambda k: np.concatenate([rng.uniform(-1, 1, (k, 2)), np.zeros((k, 1))], axis=1), False
    yield "plane_tilted", lambda k: np.concatenate([rng.uniform(-1, 1, (k, 2)), np.zeros((k, 1))], axis=1), True
    yield "plane_origin", lambda k: np.concatenate([rng.uniform(-1, 1, (k, 2)), np.zeros((k, 1))], axis=1), "origin"
    yield "blob", lambda k: rng.normal(size=(k, 3)) * [1.0, 0.5, 0.2], True


def _lattice(nx, ny):
    x, y = np.meshgrid(np.arange(nx) - (nx - 1) / 2.0, np.arange(ny) - (ny - 1) / 2.0)
    return np.stack([x.ravel(), y.ravel(), np.zeros(nx * ny)], axis=1)


def _polygon(m, z=0.0):
    a = 2 * np.pi * np.arange(m) / m
    return np.stack([np.cos(a), np.sin(a), np.full(m, z)], axis=1)


# fixed shapes whose neighbourhood is the whole set (k_correspondences = number of points)
SHAPES = {
    "lattice_4x3": _lattice(4, 3),
    "lattice_3x3": _lattice(3, 3),  # square lattice: isotropic in the plane (two equal eigenvalues above the third)
    "lattice_4x4": _lattice(4, 4),
    "disc_thin": _polygon(8),
    "disc_thick": np.concatenate([_polygon(6, 0.1), _polygon(6, -0.1)]),
    "needle": np.concatenate([_polygon(4, z) * [0.05, 0.05, 0] + [0, 0, z] for z in (-1.0, -0.5, 0.0, 0.5, 1.0)]),  # two equal eigenvalues below the third
    "cube": np.array([[x, y, z] for x in (-1.0, 1.0) for y in (-1.0, 1.0) for z in (-1.0, 1.0)]),
    "cube_centre": np.array([[x, y, z] for x in (-1.0, 1.0) for y in (-1.0, 1.0) for z in (-1.0, 1.0)] + [[0.0, 0.0, 0.0]]),
    "octahedron": np.concatenate([np.eye(3), -np.eye(3)]),
}


@functools.lru_cache(maxsize=None)
def battery():
    """-> list of cases {family, points (m, 4), nb (m, kc) int32, kc, k}; deterministic."""
    rng = np.random.default_rng(20261015)
    cases = []

    def add(family, P, kc, k):
        nb, _ = oracle.knn_bruteforce(P, kc)
        cases.append({"family": family, "points": np.ascontiguousarray(P), "nb": np.ascontiguousarray(nb, np.int32), "kc": kc, "k": k})

    for spread in SPREADS:
        for offset in OFFSETS:
            for family, make, rotate in _families(rng):
                for k in KS:
                    local = make(k)
                    if rotate == "origin":  # a plane through the origin: p . n = 0 up to rounding, the sign is decided by noise
                        P = _place(local, spread, 0.0, rng) if offset == 0.0 else _place(local, spread, 0.0, rng, rotate=False)
                    else:
                        P = _place(local, spread, offset, rng, rotate=bool(rotate))
                    add(family, P, k, k)
            for name, local in SHAPES.items():
                add(name, _place(local, spread, offset, rng), len(local), len(local))
            # k_neighbors = 1 and k_neighbors < k_correspondences (the stride of the neighbour list)
            blob = _place(rng.normal(size=(12, 3)), spread, offset, rng)
            add("k_neighbors_1", blob, 5, 1)
            add("k_neighbors_lt_kc", blob, 10, 5)
            add("k_neighbors_lt_kc", blob, 12, 7)
            # fewer points than k: the k-NN fills the missing neighbours with the query itself
            for k in (5, 10, 20):
                for n in sorted({1, 2, 3, k - 1}):
                    add("self_filled", _place(rng.normal(size=(n, 3)), spread, offset, rng), k, k)
    return cases


def rows(cases):
    """-> per row: (case index, row index in the case)"""
    return [(c, i) for c, case in enumerate(cases) for i in range(len(case["points"]))]


def oracle_outputs(case):
    n, c = oracle.covariance_estimate(case["points"], case["nb"], k_neighbors=case["k"])
    return n, c


def oracle_A(case):
    """the covariance A (m, 3, 3) that the oracle hands to its eigen solver, reproduced with the same IEEE operations
    (sum of rounded products, mean = S / k, (X - mean S) / k)"""
    P, nb, k = case["points"][:, :3], case["nb"][:, : case["k"]], case["k"]
    S = np.zeros((len(P), 3))
    X = np.zeros((len(P), 3, 3))
    for j in range(k):
        q = P[nb[:, j]]
        S = S + q
        X = X + q[:, :, None] * q[:, None, :]
    mean = S / k
    return (X - mean[:, :, None] * S[:, None, :]) / k


def solver_gaps(A):
    """gaps lambda_1 - lambda_0 and lambda_2 - lambda_1 of the shifted, scaled matrix the eigen solver works on (its own
    arithmetic for the shift and scale), for A (m, 3, 3)"""
    shift = ((A[:, 0, 0] + A[:, 1, 1]) + A[:, 2, 2]) / 3.0
    m = A - shift[:, None, None] * np.eye(3)  # off the diagonal: A - 0, exact
    scale = np.abs(m).reshape(len(m), 9).max(axis=1)
    m = np.where(scale[:, None, None] > 0, m / np.where(scale > 0, scale, 1.0)[:, None, None], m)
    w = np.linalg.eigvalsh(m)
    return w[:, 1] - w[:, 0], w[:, 2] - w[:, 1]


def invariant_tol(A):
    """tolerance of the invariants of C (symmetric, eigenvalues {1e-3, 1, 1}, normal = the 1e-3 eigenvector) for the oracle's
    A (m, 3, 3).  The eigen solver reads the characteristic polynomial from the lower triangle and the eigenvectors from whole
    columns of A - lambda I, so V is orthonormal only to the asymmetry of A (the rounding of mean[r] S[c] vs mean[c] S[r],
    which is O(1) after scaling when A is rounding noise) over the gaps, plus u / gap^2 from the roots: 1e-12 where the gaps
    and the symmetry are clean"""
    shift = ((A[:, 0, 0] + A[:, 1, 1]) + A[:, 2, 2]) / 3.0
    scale = np.abs(A - shift[:, None, None] * np.eye(3)).reshape(len(A), 9).max(axis=1)
    asym = np.abs(A - A.transpose(0, 2, 1)).reshape(len(A), 9).max(axis=1) / np.where(scale > 0, scale, 1.0)
    g01, g12 = solver_gaps(A)
    with np.errstate(divide="ignore"):
        return 1e-12 + INV_C * ((asym + U) * (1 / g01 + 1 / g12) + U * (1 / (g01 * g01) + 1 / (g12 * g12)))


def _frac_cov(P):
    """population covariance of the rows of P (k, 3), exact"""
    F = [[Fraction(float(x)) for x in p] for p in P]
    k = len(F)
    mean = [sum(p[r] for p in F) / k for r in range(3)]
    return [[sum((p[r] - mean[r]) * (p[c] - mean[c]) for p in F) / k for c in range(3)] for r in range(3)]


@functools.lru_cache(maxsize=None)
def _exact_eig(key):
    """key: the neighbourhood's points as a tuple of coordinate tuples -> (eigenvalues ascending, eigenvectors 3x3 columns)
    at 60 digits, as mpf"""
    A = _frac_cov(np.array(key))
    with mpmath.workdps(60):
        M = mpmath.matrix(3, 3)
        for r in range(3):
            for c in range(3):
                M[r, c] = mpmath.mpf(A[r][c].numerator) / A[r][c].denominator
        E, Q = mpmath.eigsy(M)
        order = sorted(range(3), key=lambda i: E[i])
        return [E[i] for i in order], [[Q[r, i] for r in range(3)] for i in order]


def exact_row(case, i):
    """exact reference of row i: dict(C (3,3), n (3,), gap, R, dot = p . n / |p| (0 for p = 0))"""
    k = case["k"]
    P = case["points"][case["nb"][i, :k], :3]
    E, vecs = _exact_eig(tuple(sorted(map(tuple, P.tolist()))))
    p = case["points"][i, :3]
    with mpmath.workdps(60):
        v0 = vecs[0]
        pn = sum(mpmath.mpf(float(p[r])) * v0[r] for r in range(3))
        if pn > 0:
            v0 = [-x for x in v0]
            pn = -pn
        n = np.array([float(x) for x in v0])
        C = np.array([[float((1 if r == c else 0) - (1 - mpmath.mpf(1e-3)) * v0[r] * v0[c]) for c in range(3)] for r in range(3)])
        lam = np.array([float(x) for x in E])
        g01, g12 = float(E[1] - E[0]), float(E[2] - E[1])
        pnorm = float(mpmath.sqrt(sum(mpmath.mpf(float(x)) ** 2 for x in p)))
        dot = float(pn) / pnorm if pnorm > 0 else 0.0
    R = float(np.sqrt((P * P).sum(axis=1)).max())
    return {"C": C, "n": n, "lam": lam, "g01": g01, "g12": g12, "R": R, "dot": dot}


def posed_bar(ex):
    """error bar of the oracle's C and normal against the exact reference (inf when an eigen gap is zero).
    The covariance carries an absolute rounding error of about u R^2, which moves the eigenvectors by u R^2 / gap.  The solver
    takes its eigenvalues from the roots of the characteristic polynomial of the shifted matrix scaled by s (its largest
    entry): a coefficient error u s^3 moves the root lambda_i by u s^3 / |p'(lambda_i)|, and the kernel of A - lambda_i I turns
    by that over the gap.  C = V diag(1e-3, 1, 1) V^T depends on both gaps, because V's columns are computed separately."""
    g01, g12 = ex["g01"], ex["g12"]
    if not (g01 > 0 and g12 > 0):
        return np.inf
    g02 = g01 + g12
    s = float(np.abs(ex["lam"] - ex["lam"].mean()).max())
    return POSED_C * U * (ex["R"] ** 2 * (1 / g01 + 1 / g12) + s**3 * (1 / (g01 * g01) + 1 / (g12 * g12)) / g02)
