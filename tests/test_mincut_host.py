"""CPU-only checks of the min-cut segmentation (no GPU needed):
  * the per-node steps of glim_b200/csrc/gb_mincut_math.cuh, compiled for the host (tests/cpp/mincut_math_host.cpp) and driven
    through the same synchronous rounds and global relabels as k_mc_solve, agree with scipy's maximum flow and a search of its
    residual graph (tests/mincut_oracle.py) on the cut value and the selection: seeded random graphs and adversarial ones;
  * the round cap gives NOT_CONVERGED with nothing selected;
  * the host build of the capacity is within 1 of numpy's, and the roles are exact;
  * the arguments gb_min_cut rejects before it touches a device."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from tests import mincut_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F64 = np.float32, np.float64
FREE, FG, BG, SEED = mo.FREE, mo.FOREGROUND, mo.BACKGROUND, mo.SEED


@pytest.fixture(scope="module")
def hl(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mincut") / "libmincut_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", out,
                           os.path.join(ROOT, "tests", "cpp", "mincut_math_host.cpp")])
    L = C.CDLL(out)
    vp = C.c_void_p
    L.edge_capacity.argtypes = [C.c_int, vp, vp, vp, vp, C.c_double, C.c_double, vp]
    L.roles.argtypes = [C.c_int, vp, vp, C.c_double, C.c_double, vp]
    L.solve.argtypes = [C.c_int, vp, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp]
    return L


def p(a):
    return a.ctypes.data_as(C.c_void_p)


def csr(m, edges, caps):
    """both arcs of every edge in (u, v) order: row offsets, heads, reverse arcs, capacities"""
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    u = np.concatenate([e[:, 0], e[:, 1]])
    v = np.concatenate([e[:, 1], e[:, 0]])
    q = np.concatenate([caps, caps]).astype(np.int32)
    key = u * (m + 1) + v
    o = np.argsort(key, kind="stable")
    u, v, q, key = u[o], v[o], q[o], key[o]
    row = np.searchsorted(u, np.arange(m + 1)).astype(np.int32)
    rev = np.searchsorted(key, v * (m + 1) + u).astype(np.int32)
    return row, v.astype(np.int32), rev, q


def host_solve(hl, m, edges, caps, role, fw, max_rounds=None):
    row, head, rev, q = csr(m, edges, caps)
    rl = np.ascontiguousarray(role, np.int32)
    sel = np.zeros(max(m, 1), np.int32)
    cut, rounds = C.c_longlong(), C.c_int()
    st = hl.solve(m, p(row), p(head), p(rev), p(q), p(rl), int(math.floor(fw * 65536.0)), hl.max_rounds() if max_rounds is None else max_rounds,
                  p(sel), C.byref(cut), C.byref(rounds))
    return st, sel[:m].astype(bool), cut.value, rounds.value


def check(hl, m, edges, caps, role, fw):
    edges = np.asarray(edges, np.int64).reshape(-1, 2)
    caps = np.asarray(caps, np.int32)
    st, sel, cut, rounds = host_solve(hl, m, edges, caps, role, fw)
    ref_sel, ref_cut = mo.solve(m, edges, caps, np.asarray(role), fw)
    assert st == 0
    assert cut == ref_cut
    assert np.array_equal(sel, ref_sel)
    again = host_solve(hl, m, edges, caps, role, fw)
    assert again[2:] == (cut, rounds) and np.array_equal(again[1], sel)
    return sel, cut, rounds


def random_graph(rng):
    m = int(rng.integers(2, 300))
    E = int(rng.integers(0, 4 * m))
    e = rng.integers(0, m, (E, 2))
    e = e[e[:, 0] != e[:, 1]]
    e = np.unique(np.stack([e.min(axis=1), e.max(axis=1)], axis=1), axis=0) if len(e) else np.zeros((0, 2), np.int64)
    scale = int(rng.choice([2, 5, 65537]))
    caps = rng.integers(0, scale, len(e)).astype(np.int32)
    caps[rng.random(len(e)) < 0.2] = 0
    role = rng.choice([FREE, FG, BG], m, p=[0.6, 0.2, 0.2]).astype(np.int32)
    role[int(rng.integers(0, m))] = SEED
    fw = float(rng.choice([0.0, 1e-4, 0.5, 10.0, 1000.0]))
    return m, e, caps, role, fw


@pytest.mark.parametrize("seed", range(200))
def test_random_graphs_agree_with_scipy(hl, seed):
    m, e, caps, role, fw = random_graph(np.random.default_rng(1000 + seed))
    check(hl, m, e, caps, role, fw)


def test_equal_parallel_cuts_select_the_minimal_side(hl):
    """seed - a - b - bg with equal capacities: every one of the three cuts is minimum; the smallest source side wins"""
    sel, cut, _ = check(hl, 4, [[0, 1], [1, 2], [2, 3]], [7, 7, 7], [SEED, FREE, FREE, BG], 10.0)
    assert cut == 7 and sel.tolist() == [True, False, False, False]
    # a cheaper cut further out moves the side outwards
    sel, cut, _ = check(hl, 4, [[0, 1], [1, 2], [2, 3]], [9, 8, 7], [SEED, FREE, FREE, BG], 10.0)
    assert cut == 7 and sel.tolist() == [True, True, True, False]


def test_all_zero_capacities(hl):
    rng = np.random.default_rng(5)
    m = 50
    e = np.array([[i, i + 1] for i in range(m - 1)])
    role = np.full(m, FREE, np.int32)
    role[0], role[10:15], role[40:] = SEED, FG, BG
    sel, cut, _ = check(hl, m, e, np.zeros(len(e), np.int32), role, 10.0)
    assert cut == 0 and set(np.flatnonzero(sel)) == {0, *range(10, 15)}  # unsaturated foreground arcs only
    sel, cut, _ = check(hl, m, e, np.zeros(len(e), np.int32), role, 0.0)
    assert cut == 0 and np.flatnonzero(sel).tolist() == [0]
    check(hl, m, e, rng.integers(0, 2, len(e)), role, 0.0)


def test_isolated_components(hl):
    rng = np.random.default_rng(6)
    parts, role, off = [], [], 0
    for c in range(6):
        k = int(rng.integers(3, 30))
        parts.append(np.array([[off + i, off + i + 1] for i in range(k - 1)]))
        r = rng.choice([FREE, FG, BG], k)
        role.extend(r.tolist())
        off += k
    role = np.array(role, np.int32)
    role[0] = SEED
    e = np.concatenate(parts)
    check(hl, off, e, rng.integers(0, 100, len(e)), role, 1.0)


def test_long_chain(hl):
    """10 k nodes: the excess crosses the whole chain, many global relabels"""
    m = 10_000
    e = np.array([[i, i + 1] for i in range(m - 1)])
    caps = np.full(m - 1, 1000, np.int32)
    caps[m // 2] = 999
    role = np.full(m, FREE, np.int32)
    role[0], role[-1] = SEED, BG
    sel, cut, rounds = check(hl, m, e, caps, role, 10.0)
    assert cut == 999 and sel.sum() == m // 2 + 1 and rounds > 1


def test_bipartite_bottleneck(hl):
    """many sources into a narrow middle: the cut is the middle layer"""
    rng = np.random.default_rng(7)
    A, B = 40, 3
    m = 1 + A + B + A
    left = np.arange(1, 1 + A)
    mid = np.arange(1 + A, 1 + A + B)
    right = np.arange(1 + A + B, m)
    e = [[0, a] for a in left] + [[a, b] for a in left for b in mid] + [[b, r] for b in mid for r in right]
    caps = [1000] * A + list(rng.integers(50, 100, A * B)) + [5] * (B * A)
    role = np.full(m, FREE, np.int32)
    role[0], role[right] = SEED, BG
    sel, cut, _ = check(hl, m, e, caps, role, 1.0)
    assert cut == 5 * B * A and sel[mid].all()


def test_foreground_next_to_background(hl):
    """a foreground node joined only to a background node: its foreground arc carries the flow"""
    role = np.array([SEED, FG, BG, FREE], np.int32)
    for q, fw, on in ((100, 10.0, True), (10 * 65536 + 5, 10.0, False), (100, 0.0, False)):
        sel, cut, _ = check(hl, 4, [[1, 2], [0, 3]], [q, 40], role, fw)
        assert cut == min(q, int(fw * 65536)) and sel[1] == on and sel[3]


def test_round_cap_gives_not_converged(hl):
    m = 200
    e = np.array([[i, i + 1] for i in range(m - 1)])
    role = np.full(m, FREE, np.int32)
    role[0], role[-1] = SEED, BG
    st, sel, cut, rounds = host_solve(hl, m, e, np.full(m - 1, 10, np.int32), role, 1.0, max_rounds=3)
    assert st == 2 and rounds == 3 and not sel.any() and cut == 0
    st, _, cut, rounds = host_solve(hl, m, e, np.full(m - 1, 10, np.int32), role, 1.0)
    assert st == 0 and cut == 10 and rounds > 3


def test_capacity_and_roles_match_oracle(hl):
    rng = np.random.default_rng(8)
    n = 20000
    a = rng.uniform(-5, 5, (n, 3)).astype(F32)
    b = (a + rng.normal(scale=0.3, size=(n, 3))).astype(F32)
    na = rng.normal(size=(n, 3)).astype(F32)
    nb = rng.normal(size=(n, 3)).astype(F32)
    na /= np.linalg.norm(na, axis=1, keepdims=True)
    nb /= np.linalg.norm(nb, axis=1, keepdims=True)
    nb[:2000] = na[:2000]       # parallel
    nb[2000:2100] = -na[2000:2100]  # opposite: the same weight
    na[3000:3010] = np.nan
    na[3010:3020] = 0
    nb[3020:3030] = 0
    b[4000:4010] = a[4000:4010]  # coincident
    for sd, sa in ((0.25, math.radians(10)), (0.05, 1e-4), (2.0, math.pi)):
        out = np.empty(n, np.int32)
        hl.edge_capacity(n, p(a), p(na), p(b), p(nb), 2.0 * sd * sd, 2.0 * sa * sa, p(out))
        ref = mo.capacity(a, na, b, nb, sd, sa)
        assert np.abs(out.astype(np.int64) - ref).max() <= 1
        assert not out[3000:3030].any() and (out >= 0).all()
        back = np.empty(n, np.int32)
        hl.edge_capacity(n, p(b), p(nb), p(a), p(na), 2.0 * sd * sd, 2.0 * sa * sa, p(back))
        assert np.array_equal(out, back)
    assert (out > 0).sum() > n // 2
    c = np.array([0.3, -0.2, 0.1])
    xyz = np.concatenate([rng.uniform(-7, 7, (n, 3)), [c + [0.5, 0, 0], c + [5.0, 0, 0], c + [0, 0, 0.25]]]).astype(F32)
    out = np.empty(len(xyz), np.int32)
    hl.roles(len(xyz), p(xyz), p(c), 0.5 * 0.5, 5.0 * 5.0, p(out))
    ref = mo.roles(xyz, c, -1, 0.5, 5.0)
    assert np.array_equal(out, ref)
    assert {FREE, FG, BG} <= set(out.tolist())


def test_oracle_graph_rows_are_brute_force():
    """the oracle's k-NN rows (candidates re-ranked, ties re-done by brute force) equal a brute-force ranking, coincident and
    lattice points included"""
    rng = np.random.default_rng(9)
    g = np.stack(np.meshgrid(*[np.arange(6) * 0.1] * 3, indexing="ij"), -1).reshape(-1, 3)
    xyz = np.concatenate([g, g[:20], rng.uniform(0, 0.5, (100, 3))]).astype(F32)
    for k in (1, 6, 20):
        rows = mo.knn_rows(xyz, k)
        P = xyz.astype(F64)
        for i in range(len(xyz)):
            dd = mo.d2(xyz, P[i])
            assert rows[i].tolist() == np.lexsort((np.arange(len(xyz)), dd))[:k].tolist()


def test_min_cut_refusals_before_any_device_work():
    from glim_b200 import capi

    L = capi.lib()
    prm = capi.MinCutParams()
    assert L.gb_min_cut_default_params(C.byref(prm)) == 0
    assert (prm.distance_sigma, prm.foreground_mask_radius, prm.background_mask_radius, prm.foreground_weight, prm.k_neighbors) == (0.25, 0.5, 5.0, 10.0, 20)
    assert abs(prm.angle_sigma - math.radians(10)) < 1e-15
    res = capi.MinCutResult()
    q = np.zeros(3)
    # a null context or cloud is refused before anything else (every other refusal needs a device and is checked there)
    assert L.gb_min_cut(None, None, p(q), C.byref(prm), C.byref(res), None, None, None) == 1
    assert L.gb_min_cut_default_params(None) == 1
