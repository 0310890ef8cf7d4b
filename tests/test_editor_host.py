"""CPU-only checks of the map editor's selection tools and point removal (no GPU needed):
  * the per-point rules of glim_b200/csrc/gb_editor_math.cuh, compiled for the host (tests/cpp/editor_math_host.cpp), against
    the numpy restatement (tests/editor_oracle.py) on adversarial inputs: points exactly on the box's faces and on the unit
    sphere, NaN and inf, a scaled and sheared T_local_world, d_i equal to the threshold;
  * the removal oracle's bookkeeping on duplicates, out-of-range ids and whole frames;
  * the arguments gb_select_gizmo, gb_select_radius and gb_remove_points reject before they touch a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import editor_oracle as eo
from tests import segment_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64


@pytest.fixture(scope="module")
def hl(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("editor") / "libeditor_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "editor_math_host.cpp")])
    L = C.CDLL(out)
    vp = C.c_void_p
    L.compose.argtypes = [C.c_int, vp, vp, vp]
    L.inside.argtypes = [C.c_int, vp, C.c_int, C.c_double, vp]
    L.radius_flags.argtypes = [C.c_int, vp, vp, C.c_double, C.c_double, vp]
    L.outliers.argtypes = [C.c_int, C.c_double, C.c_double, C.c_int, C.c_double, vp, vp, vp, vp]
    return L


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def sheared_gizmo(rng):
    """T_local_world: the inverse of a rotated, anisotropically scaled and sheared model matrix, bottom row (0, 0, 0, 1)"""
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    S = np.diag([2.5, 0.7, 4.0])
    S[0, 1] = 0.6
    model = np.eye(4)
    model[:3, :3] = q @ S
    model[:3, 3] = rng.uniform(-30, 30, 3)
    A = np.linalg.inv(model)
    A[3] = [0, 0, 0, 1]
    return A


def random_pose(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    T = np.eye(4)
    T[:3, :3] = q * np.sign(np.linalg.det(q))
    T[:3, 3] = rng.uniform(-50, 50, 3)
    return T


def test_compose_matches_oracle(hl):
    rng = np.random.default_rng(1)
    A = sheared_gizmo(rng)
    Bs = [random_pose(rng) for _ in range(50)]
    M = np.empty((50, 16))
    B16 = np.ascontiguousarray(np.stack([b.T.reshape(16) for b in Bs]))
    hl.compose(50, p(np.ascontiguousarray(A.T.reshape(16))), p(B16), p(M))
    for i, b in enumerate(Bs):
        assert np.array_equal(M[i].reshape(4, 4).T, eo.compose(A, b))


def test_box_and_sphere_match_oracle_on_faces_and_non_finite(hl):
    rng = np.random.default_rng(2)
    q = rng.uniform(-0.7, 0.7, (4000, 3))
    faces = rng.uniform(-0.4, 0.4, (600, 3))
    for a in range(3):  # exactly on a face: never inside the box
        faces[200 * a: 200 * a + 100, a] = 0.5
        faces[200 * a + 100: 200 * a + 200, a] = -0.5
    nxt = np.nextafter(0.5, 0.0)
    inner = np.array([[nxt, 0, 0], [-nxt, nxt, -nxt], [0.0, 0.0, 0.0]])
    v = rng.normal(size=(500, 3))
    sphere = v / np.linalg.norm(v, axis=1, keepdims=True)  # on (or within an ulp of) the unit sphere
    axes = np.array([[1.0, 0, 0], [0, -1.0, 0], [0, 0, 1.0], [np.nextafter(1.0, 0.0), 0, 0]])
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan, np.nan, np.nan]])
    q = np.ascontiguousarray(np.concatenate([q, faces, inner, sphere, axes, bad]))
    out = np.empty(len(q), np.int32)
    hl.inside(len(q), p(q), 1, 0.0, p(out))
    ref = eo.in_box(q)
    assert np.array_equal(out.astype(bool), ref)
    assert not ref[4000:4600].any() and ref[4600:4603].all() and not ref[-4:].any()
    hl.inside(len(q), p(q), 0, 1.0, p(out))
    ref = eo.in_sphere(q, 1.0)
    assert np.array_equal(out.astype(bool), ref)
    assert not ref[-8:-5].any() and ref[-5] and not ref[-4:].any()  # exactly on the sphere along an axis: not inside


def test_gizmo_transform_of_a_sheared_model_matches_oracle(hl):
    rng = np.random.default_rng(3)
    A = sheared_gizmo(rng)
    T = random_pose(rng)
    model = np.linalg.inv(A)
    # points around the gizmo, in the submap's local frame, including the images of the faces' centres
    local_gizmo = rng.uniform(-0.9, 0.9, (3000, 3))
    world = local_gizmo @ model[:3, :3].T + model[:3, 3]
    a = ((world - T[:3, 3]) @ T[:3, :3]).astype(F32)
    M = np.empty(16)
    hl.compose(1, p(np.ascontiguousarray(A.T.reshape(16))), p(np.ascontiguousarray(T.T.reshape(16))), p(M))
    M = M.reshape(4, 4).T
    q = np.ascontiguousarray(so.transform_points(M, a))
    for box in (1, 0):
        out = np.empty(len(q), np.int32)
        hl.inside(len(q), p(q), box, 1.0, p(out))
        ref = eo.in_box(q) if box else eo.in_sphere(q, 1.0)
        assert np.array_equal(out.astype(bool), ref) and 100 < ref.sum() < 2900


def test_radius_flags_match_oracle(hl):
    rng = np.random.default_rng(4)
    c = np.array([10.25, -3.5, 1.0])
    xyz = (c + rng.uniform(-4, 4, (5000, 3))).astype(F32)
    # exactly at the radii along an axis (d2 == radius^2 is not inside), and non-finite points
    xyz[:4] = (c + np.array([[2.0, 0, 0], [0, -3.0, 0], [0, 0, 1.0], [0, 0, 0]])).astype(F32)
    xyz[4:7] = [[np.nan, 0, 0], [np.inf, 1, 1], [0, 0, -np.inf]]
    xyz = np.ascontiguousarray(xyz)
    out = np.empty(len(xyz), np.int32)
    hl.radius_flags(len(xyz), p(xyz), p(c), 4.0, 9.0, p(out))
    inside, part = eo.radius_flags(xyz, c, 4.0, 9.0)
    assert np.array_equal((out & 1).astype(bool), inside) and np.array_equal((out >> 1).astype(bool), part)
    assert not inside[0] and inside[2] and not part[1] and not (out[4:7]).any()


def test_outlier_threshold_and_selection_match_oracle_at_the_threshold(hl):
    rng = np.random.default_rng(5)
    d = rng.uniform(0.05, 0.3, 400)
    S, S2 = float(np.sum(d)), float(np.sum(d * d))
    th_ref = eo.threshold(S, S2, len(d), 2.0)
    d[:5] = th_ref                      # exactly at the threshold: an outlier (not d < threshold)
    d[5] = np.nextafter(th_ref, 0.0)    # just below: an inlier
    d[6] = np.nan                       # NaN is never an inlier
    inside = np.ones(len(d), np.int32)
    inside[7] = 0                       # an outlier outside the radius is not selected
    d[7] = 10.0
    th = np.empty(1)
    out = np.empty(len(d), np.int32)
    hl.outliers(len(d), S, S2, len(d), 2.0, p(d), p(inside), p(th), p(out))
    assert th[0] == th_ref
    with np.errstate(invalid="ignore"):
        ref = inside.astype(bool) & ~(d < th_ref)
    assert np.array_equal(out.astype(bool), ref)
    assert out[:5].all() and not out[5] and out[6] and not out[7]
    # a zero or negative variance clamps to 0: the threshold is the mean
    hl.outliers(0, 3.0, 1.0, 3, 2.0, p(d), p(inside), p(th), p(out))
    assert th[0] == 1.0 == eo.threshold(3.0, 1.0, 3, 2.0)


def test_oracle_knn_distances_are_order_free_under_ties():
    # a square lattice: every point's neighbours tie; d_i does not depend on which tied neighbour is taken
    g = np.stack(np.meshgrid(np.arange(6.0), np.arange(6.0), [0.0]), -1).reshape(-1, 3)
    d = eo.mean_knn_dists(g, 4)
    assert np.all(d[(g[:, 0] > 0) & (g[:, 0] < 5) & (g[:, 1] > 0) & (g[:, 1] < 5)] == 0.75)


def test_removal_oracle_bookkeeping():
    sizes = [5, 0, 3, 4]
    ids = np.array([(0 << 32) | 1, (0 << 32) | 1, (0 << 32) | 4, (1 << 32) | 0, (2 << 32) | 0, (2 << 32) | 1, (2 << 32) | 2,
                    (2 << 32) | 3, (7 << 32) | 0, (3 << 32) | 0xFFFFFFFF], np.uint64)
    out, removed, ignored = eo.remove_points(sizes, ids)
    assert np.array_equal(out[0], [0, 2, 3]) and out[1] is None and len(out[2]) == 0 and out[3] is None
    assert removed == 5 and ignored == 4  # frame 1 is empty, index 3 == size of frame 2, frame 7 >= K, 2^32 - 1 >= size


def test_refusals_before_any_device_work():
    from glim_b200 import capi

    L = capi.lib()
    prm = capi.SelectRadiusParams()
    assert L.gb_select_radius_default_params(C.byref(prm)) == 0
    assert (prm.radius, prm.radius_offset, prm.stddev_thresh, prm.mode, prm.k) == (2.0, 1.0, 2.0, capi.RADIUS_INSIDE, 10)
    res = capi.SelectRadiusResult()
    q = np.zeros(3)
    # a null context or cloud is refused before anything else (every other refusal needs a device and is checked there)
    assert L.gb_select_radius(None, None, p(q), C.byref(prm), C.byref(res), None) == 1
    A = np.eye(4).reshape(16)
    m = C.c_size_t(7)
    assert L.gb_select_gizmo(None, 0, None, None, p(A), capi.GIZMO_BOX, None, C.byref(m)) == 1
    r = capi.RemovePointsResult()
    assert L.gb_remove_points(None, 0, None, 0, None, None, C.byref(r), None) == 1
