"""Covariance / normal estimation on degenerate neighbourhoods, on the CPU.

tests/cov_reference.py builds the battery (duplicates, collinear, planar, isotropic, self-filled neighbour lists, far offsets)
and its exact reference.  Here: the oracle against the exact reference on every posed row, the invariants of the
regularised covariance on every row, and the kernels' own arithmetic text (glim_b200/csrc/gb_cov_math.cuh, compiled for the
host by tests/cpp/cov_math_host.cpp) bit for bit against the oracle on every row.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import cov_reference as cr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cm(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cm") / "libcov_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "cov_math_host.cpp")])
    L = C.CDLL(so)
    L.cm_covariance_estimate.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return L


def host_estimate(cm, case):
    n = len(case["points"])
    normals, covs = np.zeros((n, 4)), np.zeros((n, 16))
    cm.cm_covariance_estimate(n, case["points"].ctypes.data, case["nb"].ctypes.data, case["kc"], case["k"], normals.ctypes.data, covs.ctypes.data)
    return normals, covs.reshape(n, 4, 4).transpose(0, 2, 1)


def test_battery_covers_the_families():
    cases = cr.battery()
    fam = {c["family"] for c in cases}
    for f in ("duplicates", "k_neighbors_1", "self_filled", "collinear", "near_collinear_1e-12", "plane_axis", "plane_tilted", "lattice_3x3", "disc_thin", "needle", "cube", "octahedron", "blob", "plane_origin", "k_neighbors_lt_kc"):
        assert f in fam
    assert {c["kc"] for c in cases} >= set(cr.KS)
    assert any(c["k"] < c["kc"] for c in cases)
    assert any((c["nb"] == np.arange(len(c["points"]))[:, None]).all(axis=1).any() and len(c["points"]) < c["kc"] for c in cases)  # self-filled rows
    assert 3000 < len(cr.rows(cases)) < 20000


def test_host_build_of_the_kernel_arithmetic_is_bit_exact_with_oracle(cm):
    for case in cr.battery():
        n_o, c_o = cr.oracle_outputs(case)
        n_h, c_h = host_estimate(cm, case)
        assert np.array_equal(n_h, n_o) and np.array_equal(c_h, c_o), case["family"]


def test_invariants_on_every_row():
    for case in cr.battery():
        n_o, c_o = cr.oracle_outputs(case)
        tol = cr.invariant_tol(cr.oracle_A(case))
        C3 = c_o[:, :3, :3]
        assert not c_o[:, 3, :].any() and not c_o[:, :, 3].any() and not n_o[:, 3].any()
        assert (np.abs(C3 - C3.transpose(0, 2, 1)).max(axis=(1, 2)) <= tol).all(), case["family"]
        w = np.linalg.eigvalsh(C3)
        assert (np.abs(w - [1e-3, 1.0, 1.0]).max(axis=1) <= tol).all(), case["family"]
        n = n_o[:, :3]
        assert (np.abs(np.linalg.norm(n, axis=1) - 1.0) <= 1e-12).all()
        assert (np.abs(np.einsum("nij,nj->ni", C3, n) - 1e-3 * n).max(axis=1) <= tol).all(), case["family"]
        P = case["points"]
        pn = ((P[:, 0] * n_o[:, 0] + P[:, 1] * n_o[:, 1]) + P[:, 2] * n_o[:, 2]) + P[:, 3] * n_o[:, 3]  # the oracle's own evaluation
        assert (pn <= 0.0).all(), case["family"]
    # the tolerance is 1e-12 wherever the solver's gaps and the symmetry of A are clean: most rows
    tight = sum(int((cr.invariant_tol(cr.oracle_A(c)) < 1e-9).sum()) for c in cr.battery())
    assert tight > 0.4 * len(cr.rows(cr.battery()))


def _exact_error(n, C3, ex, bar):
    """largest entry difference of C and of the normal; either sign of the normal counts when p . n is within the bar"""
    en = np.abs(n - ex["n"]).max()
    if abs(ex["dot"]) <= bar:
        en = min(en, np.abs(n + ex["n"]).max())
    return max(np.abs(C3 - ex["C"]).max(), en)


def test_oracle_matches_exact_reference_on_posed_rows():
    worst, posed, fams = 0.0, 0, set()
    for case in cr.battery():
        n_o, c_o = cr.oracle_outputs(case)
        for i in range(len(case["points"])):
            ex = cr.exact_row(case, i)
            bar = cr.posed_bar(ex)
            if bar >= cr.POSED_MAX:
                continue
            posed += 1
            fams.add(case["family"])
            err = _exact_error(n_o[i, :3], c_o[i, :3, :3], ex, bar)
            worst = max(worst, err / bar)
            assert err <= bar, (case["family"], i, err, bar)
    print(f"oracle vs exact reference: {posed} posed rows, worst error / bar {worst:.3f} (POSED_C = {cr.POSED_C})")
    assert posed > 2000 and {"blob", "plane_axis", "plane_tilted", "plane_origin", "lattice_4x3", "self_filled", "k_neighbors_lt_kc"} <= fams
    assert worst > 0.05  # the constant is not loose by orders of magnitude


def test_exact_bar_rejects_a_small_rotation_of_the_normal():
    """rotating v0 by 1e-6 rad on a posed row fails the bar: it is not vacuous"""
    rng = np.random.default_rng(3)
    checked = 0
    for case in cr.battery():
        if case["family"] not in ("blob", "plane_tilted"):
            continue
        for i in range(len(case["points"])):
            ex = cr.exact_row(case, i)
            bar = cr.posed_bar(ex)
            if bar >= 1e-7:
                continue
            axis = np.cross(ex["n"], rng.normal(size=3))
            axis /= np.linalg.norm(axis)
            t = 1e-6
            n = ex["n"] * np.cos(t) + np.cross(axis, ex["n"]) * np.sin(t)
            C3 = np.eye(3) - (1 - 1e-3) * np.outer(n, n)
            assert _exact_error(n, C3, ex, bar) > bar
            checked += 1
    assert checked > 500
