"""The map editor's min-cut segmentation on the device (gb_min_cut) against the numpy / scipy restatement
(tests/mincut_oracle.py): the graph (edges, participants, roles) exactly and capacities within 1; scipy's maximum flow on the
device's own graph bit for bit (selection and cut value), and the sequential host driver of the same rounds on it (rounds
included); the end-to-end selection where the capacities agree; the one semantic bar (a pole cut from its floor and wall);
the editor recipe end to end; refusals and launch counts."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import mincut_oracle as mo
from tests import segment_oracle as so

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULTS = dict(distance_sigma=0.25, angle_sigma=math.radians(10), foreground_mask_radius=0.5, background_mask_radius=5.0, foreground_weight=10.0,
                k_neighbors=20)


@pytest.fixture(scope="module")
def ctx():
    return gpu.Context(0)


@pytest.fixture(scope="module")
def hl(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mincut_gpu") / "libmincut_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "cpp", "mincut_math_host.cpp")])
    L = C.CDLL(out)
    L.solve.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_int] + [C.c_void_p] * 3
    return L


def upload(ctx, xyz, nrm):
    xyz = np.asarray(xyz, F64)
    h = np.concatenate([xyz, np.ones((len(xyz), 1))], axis=1)
    n4 = np.concatenate([np.asarray(nrm, F64), np.zeros((len(nrm), 1))], axis=1)
    return gpu.PointCloudGPU.clone(h, None, n4, ctx=ctx)


def plane(rng, lo, hi, step, axis, at, noise=0.005):
    u, v = np.arange(lo[0], hi[0], step), np.arange(lo[1], hi[1], step)
    U, V = np.meshgrid(u, v, indexing="ij")
    P = np.zeros((U.size, 3))
    o = [a for a in range(3) if a != axis]
    P[:, o[0]], P[:, o[1]], P[:, axis] = U.ravel(), V.ravel(), at
    P += rng.normal(scale=noise, size=P.shape)
    N = np.zeros_like(P)
    N[:, axis] = 1.0
    return P, N


def box(rng, lo, hi, step=0.05):
    """the five visible faces (no bottom) of an axis-aligned box"""
    parts = [plane(rng, (lo[0], lo[1]), (hi[0], hi[1]), step, 2, hi[2], 0.002)]
    for a in (0, 1):
        o = [b for b in (0, 1, 2) if b != a]
        for at in (lo[a], hi[a]):
            P, N = plane(rng, (lo[o[0]], lo[o[1]]), (hi[o[0]], hi[o[1]]), step, a, at, 0.002)
            parts.append((P, N if at == hi[a] else -N))
    return parts


def pole(rng, centre, radius=0.15, height=2.0, rings=0.05, per_ring=24):
    z = np.arange(0.0, height, rings)
    t = np.arange(per_ring) * 2 * np.pi / per_ring
    Z, T = np.meshgrid(z, t, indexing="ij")
    N = np.stack([np.cos(T.ravel()), np.sin(T.ravel()), np.zeros(T.size)], axis=1)
    P = N * radius + [centre[0], centre[1], 0.0]
    P[:, 2] = Z.ravel()
    return P + rng.normal(scale=0.002, size=P.shape), N


def scene(parts, rng, shuffle=True):
    P = np.concatenate([p for p, _ in parts]).astype(F32)
    N = np.concatenate([n for _, n in parts]).astype(F32)
    lab = np.concatenate([np.full(len(p), i) for i, (p, _) in enumerate(parts)])
    if shuffle:
        o = rng.permutation(len(P))
        P, N, lab = P[o], N[o], lab[o]
    return P, N, lab


def box_scene(rng):
    parts = [plane(rng, (-7, -7), (7, 7), 0.1, 2, 0.0), plane(rng, (-7, 0), (7, 3), 0.1, 0, -2.5), plane(rng, (-7, 0), (7, 3), 0.1, 0, 2.5)]
    return scene(parts + box(rng, (-0.5, -0.5, 0.0), (0.5, 0.5, 1.0)), rng)


def pole_scene(rng, gap=0.6):
    parts = [plane(rng, (-7, -7), (7, 7), 0.1, 2, 0.0), plane(rng, (-7, 0), (7, 3), 0.1, 0, 0.15 + gap)]
    return scene(parts + [pole(rng, (0.0, 0.0))], rng)


def run(ctx, hl, P, N, c, **params):
    """the device's cut against the oracle's graph and against scipy and the host driver on the device's own graph"""
    prm = dict(DEFAULTS, **params)
    cloud = upload(ctx, P, N)
    got = gpu.min_cut(cloud, c, ctx=ctx, graph=True, **prm)
    ref = mo.min_cut(P, N, c, **prm)
    for k in ("seed", "status", "num_points", "num_foreground", "num_background", "num_edges"):
        assert got[k] == ref[k], k
    assert np.array_equal(got["edges"], ref["edges"])
    diff = np.abs(got["capacities"].astype(np.int64) - ref["capacities"])
    assert diff.max(initial=0) <= 1
    if got["status"] != capi.MINCUT_FOUND:
        return got, ref
    # scipy on the device's own graph: the combinatorial solve, bit for bit
    sel, cut = mo.cut_on_graph(len(P), ref["nodes"], ref["role"], got["edges"], got["capacities"], prm["foreground_weight"])
    assert np.array_equal(got["selected"], sel) and got["cut_value"] == cut
    # the same synchronous rounds run sequentially on the host
    m = len(ref["nodes"])
    pos = np.full(len(P), -1, np.int64)
    pos[ref["nodes"]] = np.arange(m)
    e = pos[got["edges"].astype(np.int64)]
    row, head, rev, q = csr(m, e, got["capacities"])
    role = np.ascontiguousarray(ref["role"], np.int32)
    hsel = np.zeros(max(m, 1), np.int32)
    hcut, hrounds = C.c_longlong(), C.c_int()
    st = hl.solve(m, *(a.ctypes.data for a in (row, head, rev, q, role)), int(math.floor(prm["foreground_weight"] * 65536.0)), 65536, hsel.ctypes.data,
                  C.byref(hcut), C.byref(hrounds))
    assert st == 0 and hcut.value == got["cut_value"] and hrounds.value == got["rounds"]
    assert np.array_equal(ref["nodes"][hsel[:m].astype(bool)], got["selected"])
    # end to end where the capacities agree
    assert diff.max(initial=0) == 0
    assert np.array_equal(got["selected"], ref["selected"]) and got["cut_value"] == ref["cut_value"]
    again = gpu.min_cut(cloud, c, ctx=ctx, graph=True, **prm)
    for k in ("selected", "edges", "capacities"):
        assert np.array_equal(again[k], got[k]), k
    for k in ("cut_value", "rounds", "num_selected", "seed"):
        assert again[k] == got[k], k
    return got, ref


def csr(m, e, caps):
    u = np.concatenate([e[:, 0], e[:, 1]])
    v = np.concatenate([e[:, 1], e[:, 0]])
    q = np.concatenate([caps, caps]).astype(np.int32)
    key = u * (m + 1) + v
    o = np.argsort(key, kind="stable")
    u, v, q, key = u[o], v[o], q[o], key[o]
    return (np.searchsorted(u, np.arange(m + 1)).astype(np.int32), v.astype(np.int32), np.searchsorted(key, v * (m + 1) + u).astype(np.int32), q)


def test_box_between_walls(ctx, hl):
    rng = np.random.default_rng(1)
    P, N, _ = box_scene(rng)
    got, _ = run(ctx, hl, P, N, [0.0, 0.0, 1.0])
    assert got["num_selected"] > 100 and got["num_background"] > 0


def test_pole_is_cut_from_floor_and_wall(ctx, hl):
    """the one semantic bar: a 2 m pole 0.6 m from a wall, picked at mid-height with the editor's defaults"""
    rng = np.random.default_rng(2)
    P, N, lab = pole_scene(rng)
    picked = [0.15, 0.0, 1.0]
    got, _ = run(ctx, hl, P, N, picked)
    sel = np.zeros(len(P), bool)
    sel[got["selected"]] = True
    assert sel[lab == 2].mean() >= 0.95
    assert sel[lab == 0].mean() < 0.01 and sel[lab == 1].mean() < 0.01
    # a foreground radius that covers the whole pole
    got, _ = run(ctx, hl, P, N, picked, foreground_mask_radius=1.2)
    sel[:] = False
    sel[got["selected"]] = True
    assert sel[lab == 2].mean() >= 0.95 and got["cut_value"] > 0  # the floor inside the radius pulls flow through its rim


def test_two_touching_boxes(ctx, hl):
    rng = np.random.default_rng(3)
    parts = [plane(rng, (-7, -7), (7, 7), 0.1, 2, 0.0)] + box(rng, (-0.5, -0.5, 0.0), (0.5, 0.5, 1.0)) + box(rng, (0.5, -0.4, 0.0), (1.3, 0.4, 0.8))
    P, N, _ = scene(parts, rng)
    run(ctx, hl, P, N, [0.0, 0.0, 1.0])
    run(ctx, hl, P, N, [0.9, 0.0, 0.8], foreground_weight=0.5)


def test_nan_points_normals_and_duplicates(ctx, hl):
    rng = np.random.default_rng(4)
    P, N, _ = pole_scene(rng)
    P[rng.choice(len(P), 50, replace=False)] = np.nan
    N[rng.choice(len(P), 50, replace=False)] = np.nan
    N[rng.choice(len(P), 50, replace=False)] = 0
    run(ctx, hl, P, N, [0.15, 0.0, 1.0])
    D = np.concatenate([P, P[:3000], P[:40]])  # coincident duplicates, some three deep
    M = np.concatenate([N, N[:3000], -N[:40]])
    run(ctx, hl, D, M, [0.15, 0.0, 1.0])


def test_tiny_angle_sigma_and_no_seed(ctx, hl):
    rng = np.random.default_rng(5)
    P, N, _ = box_scene(rng)
    Nn = N + rng.normal(scale=0.05, size=N.shape)  # a few degrees apart: at 1e-3 rad almost every capacity is 0
    Nn = (Nn / np.linalg.norm(Nn, axis=1, keepdims=True)).astype(F32)
    got, _ = run(ctx, hl, P, Nn, [0.0, 0.0, 1.0], angle_sigma=1e-3)
    assert (got["capacities"] == 0).mean() > 0.9
    got, _ = run(ctx, hl, P, N, [500.0, 0.0, 0.0])
    assert got["status"] == capi.MINCUT_NO_SEED and got["seed"] == -1 and got["num_selected"] == 0 and got["num_points"] == 0


def test_large_scene(ctx, hl):
    """about 200 k participants: a dense floor, two walls and a pole"""
    rng = np.random.default_rng(6)
    parts = [plane(rng, (-4.0, -4.0), (4.0, 4.0), 0.02, 2, 0.0), plane(rng, (-4.0, 0), (4.0, 3), 0.04, 0, 1.2), plane(rng, (-4.0, 0), (4.0, 3), 0.04, 1, -3.0),
             pole(rng, (0.0, 0.0), rings=0.02, per_ring=48)]
    P, N, _ = scene(parts, rng)
    got, _ = run(ctx, hl, P, N, [0.15, 0.0, 1.0], k_neighbors=10)
    assert got["num_points"] > 180_000


def test_editor_recipe_end_to_end(ctx):
    """submaps with covariances -> concat_frames with a 2 m x +-5-cell window -> estimate_normals -> min_cut -> ids[selected],
    against the oracle on the host-gathered window with the same normals"""
    rng = np.random.default_rng(7)
    poses, host, frames = [], [], []
    for k in range(6):
        T = np.eye(4)
        yaw = rng.uniform(-np.pi, np.pi)
        T[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
        T[:3, 3] = [6.0 * (k % 3), 6.0 * (k // 3), 0.0]
        parts = [plane(rng, (T[0, 3] - 4, T[1, 3] - 4), (T[0, 3] + 4, T[1, 3] + 4), 0.12, 2, 0.0)]
        if k == 1:
            parts.append(pole(rng, (6.0, 0.0)))
        Pw = np.concatenate([q for q, _ in parts])
        local = ((Pw - T[:3, 3]) @ T[:3, :3]).astype(F32)
        h4 = np.concatenate([local.astype(F64), np.ones((len(local), 1))], axis=1)
        _, covs = synth.with_covariances(h4, 10)
        poses.append(T)
        host.append((local, covs[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(F32), None))
        frames.append(gpu.PointCloudGPU.clone(h4, covs, ctx=ctx))
    picked = np.array([6.15, 0.0, 1.0])
    cell, w = 2.0, 5
    c = np.floor(picked / cell).astype(int)
    window = (cell, tuple(c - w), tuple(c + w))
    cloud, ids = gpu.concat_frames(poses, frames, window=window, ctx=ctx)
    cloud.estimate_normals()
    got = gpu.min_cut(cloud, picked, ctx=ctx)
    ref_cat = so.concat_frames(poses, host, window)
    assert np.array_equal(ids, ref_cat["ids"])
    ref = mo.min_cut(ref_cat["xyz"], cloud.normals(), picked, **DEFAULTS)
    assert np.array_equal(ids[got["selected"]], ref_cat["ids"][ref["selected"]])
    assert got["status"] == capi.MINCUT_FOUND and got["num_selected"] > 500


def launches(ctx, fn):
    before = ctx.kernel_launches
    fn()
    return ctx.kernel_launches - before


def test_refusals_make_no_launch(ctx):
    rng = np.random.default_rng(8)
    P, N = plane(rng, (0, 0), (2, 2), 0.1, 2, 0.0)
    cloud = upload(ctx, P, N)
    bare = gpu.PointCloudGPU.clone(np.concatenate([P, np.ones((len(P), 1))], axis=1), ctx=ctx)
    bad = [dict(cloud=bare), dict(seed=[np.nan, 0, 0]), dict(distance_sigma=0.0), dict(distance_sigma=np.inf), dict(angle_sigma=0.0),
           dict(angle_sigma=3.2), dict(angle_sigma=np.nan), dict(foreground_mask_radius=0.0), dict(foreground_mask_radius=np.nan),
           dict(background_mask_radius=0.5), dict(background_mask_radius=np.inf), dict(foreground_weight=-1.0), dict(foreground_weight=1001.0),
           dict(foreground_weight=np.nan), dict(k_neighbors=11), dict(k_neighbors=0)]
    for b in bad:
        c = b.pop("cloud", cloud)
        s = b.pop("seed", [0, 0, 0])

        def call():
            with pytest.raises(capi.GlimB200Error):
                gpu.min_cut(c, s, ctx=ctx, **b)
        assert launches(ctx, call) == 0, b


@pytest.mark.parametrize("n", [1000, 100_000])
def test_launch_counts_are_constant(ctx, n):
    rng = np.random.default_rng(n)
    N = np.tile(np.array([0, 0, 1], F32), (n, 1))
    for P in (np.stack([0.05 * np.arange(n), np.zeros(n), np.zeros(n)], axis=1), rng.normal(size=(n, 3))):
        cloud = upload(ctx, P.astype(F32), N)
        assert launches(ctx, lambda: gpu.min_cut(cloud, P[0], ctx=ctx)) == 17
        assert launches(ctx, lambda: gpu.min_cut(cloud, P[0], ctx=ctx, graph=True, k_neighbors=5)) == 17
        assert launches(ctx, lambda: gpu.min_cut(cloud, [1e4, 0, 0], ctx=ctx)) == 17  # NO_SEED: the same kernels, with no node
    empty = upload(ctx, np.zeros((0, 3), F32), np.zeros((0, 3), F32))
    assert launches(ctx, lambda: gpu.min_cut(empty, [0, 0, 0], ctx=ctx)) == 0
