"""CPU-only: the scaled backward error of tests/solve_check.py has teeth.  A numpy restatement of pg_cholesky_solve's schedule
(gb_pose_graph_math.cuh: the damped padded copy over 64-row tiles, the diagonal tile's factor, the panel, the trailing tile
updates, the tile-blocked forward and backward substitution) solves host systems GLIM's graphs produce; the faithful schedule
must pass the device's bound, and each of the faults a device solve could make must miss it by three orders of magnitude."""
import numpy as np
import pytest
from scipy.linalg import solve_triangular

from tests import graph_oracle as go
from tests import imu_oracle as io
from tests import nav_graph_oracle as ngo
from tests import pose_graph_oracle as pgo
from tests import solve_check as sc

T = sc.TILE
MUTATIONS = ["skip_update", "stale_panel_tile", "transposed_fragment", "wrong_triangle_copy", "short_trsv"]


def tiles(i):
    return slice(T * i, T * i + T)


def tiled_solve(H, b, lam, live, mutation=None):
    """pg_damped_copy and pg_cholesky_solve in numpy, with one fault when mutation is given:
    skip_update          one trailing-tile update is not applied
    stale_panel_tile     one update reads its row tile as it was before the panel's triangular solve
    transposed_fragment  one 8 x 8 fragment of one update's product lands transposed
    wrong_triangle_copy  one off-diagonal tile of the damped copy is read from the other triangle of H
    short_trsv           the last diagonal tile's backward trsv stops one column short
    The faulted update is the one of the middle tile step with the largest scaled product (off the diagonal but for a skip), the
    faulted copy tile the largest scaled off-diagonal tile: a fault where the product is ~0 changes nothing any check could
    see.  -> the step (n,) or None (failed pivot)"""
    n = len(b)
    N = sc.padded(n)
    nt = N // T
    dead = np.ones(N, bool)
    dead[:n] = ~live
    # the device's H holds the lower 6 x 6 blocks only
    blk = np.arange(n) // 6
    Hl = np.zeros((N, N))
    Hl[:n, :n] = np.where(blk[:, None] >= blk[None, :], H, 0.0)
    A = np.tril(Hl) + lam * np.eye(N)
    A[dead, :] = 0.0
    A[:, dead] = 0.0
    A[dead, dead] = 1.0
    x = np.where(dead, 0.0, -np.concatenate([b, np.zeros(N - n)]))
    D = 1.0 / np.sqrt(np.diag(A))
    if mutation == "wrong_triangle_copy":
        S = np.abs(D[:, None] * A * D[None, :])
        it, jt = max(((i, j) for i in range(nt) for j in range(i)), key=lambda t: S[tiles(t[0]), tiles(t[1])].max())
        i0, j0 = tiles(it), tiles(jt)
        A[i0, j0] = Hl[j0, i0].T  # A_ij = H_ji: the unwritten upper blocks
    at = None  # (kt, it, jt) of the faulted update
    for kt in range(nt):
        K = tiles(kt)
        try:
            L = np.linalg.cholesky(np.tril(A[K, K]) + np.tril(A[K, K], -1).T)
        except np.linalg.LinAlgError:
            return None
        A[K, K] = L
        R = slice(T * (kt + 1), N)
        pre = A[R, K].copy()
        A[R, K] = solve_triangular(L, A[R, K].T, lower=True).T
        if kt == nt // 2 and mutation in ("skip_update", "stale_panel_tile", "transposed_fragment"):
            s = {t: np.abs(D[tiles(t), None] * A[tiles(t), K]).max() for t in range(kt + 1, nt)}
            diag = mutation == "skip_update"  # a skipped diagonal update keeps A positive definite; the others go off the diagonal
            at = (kt,) + max(((i, j) for i in s for j in s if kt < j < i + diag), key=lambda t: s[t[0]] * s[t[1]])
        for it in range(kt + 1, nt):  # the lower tiles of row it: (it, kt + 1 .. it)
            I, C = tiles(it), slice(T * (kt + 1), T * (it + 1))
            P = A[I, K] @ A[C, K].T
            if at is not None and at[0] == kt and at[1] == it:
                jc = tiles(at[2] - kt - 1)
                if mutation == "skip_update":
                    P[:, jc] = 0.0
                elif mutation == "stale_panel_tile":
                    P[:, jc] = pre[tiles(it - kt - 1)] @ A[tiles(at[2]), K].T
                else:
                    F = P[:, jc]  # a view: the 8 x 8 fragment whose transpose changes the most, below the diagonal
                    sd = D[I][:, None] * F * D[tiles(at[2])][None, :]
                    r0, c0 = max(((r, c) for r in range(0, T, 8) for c in range(0, T, 8) if at[1] != at[2] or r > c),
                                 key=lambda rc: np.abs(sd[rc[0]:rc[0] + 8, rc[1]:rc[1] + 8] - sd[rc[0]:rc[0] + 8, rc[1]:rc[1] + 8].T).max())
                    F[r0:r0 + 8, c0:c0 + 8] = F[r0:r0 + 8, c0:c0 + 8].T.copy()
            A[I, C] -= P
    for kt in range(nt):
        K = tiles(kt)
        x[K] = solve_triangular(A[K, K], x[K], lower=True)
        x[T * (kt + 1):] -= A[T * (kt + 1):, K] @ x[K]
    for kt in reversed(range(nt)):
        K = tiles(kt)
        L = A[K, K]
        if mutation == "short_trsv" and kt == nt - 1:
            xk = x[K]
            for c in range(T - 1, 0, -1):  # column 0 never taken
                xk[c] /= L[c, c]
                xk[:c] -= L[c, :c] * xk[c]
        else:
            x[K] = solve_triangular(L.T, x[K], lower=False)
        x[:T * kt] -= A[K, :T * kt].T @ x[K]
    return x[:n]


def pose_system():
    T0, priors, bts = sc.ill_conditioned_graph()
    recs = [pgo.between_record(T0[i], T0[j], Z, L, k) for i, j, Z, L, k in bts]
    qblocks = [go.prior_term(T0[k], Z, w)[1:] + (0.0,) for k, Z, w in priors]
    H, b, _, _ = pgo.assemble(len(T0), [], [], [(i, j) for i, j, _, _, _ in bts], recs, [k for k, _, _ in priors], qblocks)
    return H, b, np.ones(len(b), bool), sc.pose_eps(T0, T0)


def nav_system():
    ch = sc.imu_chain(40, io.integrate_imu_deque)
    g, X0 = ch["graph"], ch["X0"]
    T = X0[0]
    brecs = [pgo.between_record(T[i], T[j], Z, L, k) for i, j, Z, L, k in g.betweens]
    qblocks = [go.prior_term(T[k], Z, w)[1:] + (0.0,) for k, Z, w in g.priors]
    H, b, _ = ngo.assemble(g.K, [], [], [(i, j) for i, j, _, _, _ in g.betweens], brecs, g.terms(X0), [k for k, _, _ in g.priors], qblocks)
    return H, b, ch["live"], sc.nav_eps(X0, X0)


@pytest.fixture(scope="module", params=["pose_graph_1024", "nav_chain_40"])
def system(request):
    H, b, live, eps = pose_system() if request.param == "pose_graph_1024" else nav_system()
    lam = 1e-5
    A = H + lam * np.eye(len(b))
    idx = np.flatnonzero(live)
    d_np = np.zeros(len(b))
    d_np[idx] = np.linalg.solve(A[np.ix_(idx, idx)], -b[idx])
    eta_np, eta_rec = sc.scaled_backward_error(A, d_np, b, live, eps)
    bound = sc.FACTOR * max(eta_np, len(idx) * sc.U, eta_rec)  # the device's bound, its read-back floor at the start poses
    return dict(name=request.param, H=H, b=b, live=live, lam=lam, A=A, bound=bound, cond=sc.condition_1norm(A, live))


def test_the_graphs_are_what_the_device_solves(system):
    s = system
    print(f"{s['name']}: n {int(s['live'].sum())}, N {sc.padded(len(s['b']))}, cond_1 {s['cond']:.3g}, bound {s['bound']:.3g}")
    if s["name"] == "pose_graph_1024":
        assert len(s["b"]) == 6144 and s["cond"] >= 1e12
    else:
        assert sc.padded(len(s["b"])) > len(s["b"]) and not s["live"].all()  # padded rows and pinned dofs both


def test_faithful_schedule_passes(system):
    s = system
    d = tiled_solve(s["H"], s["b"], s["lam"], s["live"])
    eta = sc.scaled_backward_error(s["A"], d, s["b"], s["live"])
    print(f"{s['name']}: faithful eta {eta:.3g}, bound {s['bound']:.3g}")
    assert eta <= s["bound"]
    assert np.all(d[~s["live"]] == 0.0)


# On the K = 1024 graph (cond_1 2e14) these faults perturb the scaled system by more than its smallest eigenvalue: a later pivot
# turns non-positive, the device rejects the trial, and every device check sees (iterations, trials) != (1, 1).  Faulting a
# smaller update instead leaves a perturbation below 1e3 x the bound (the next largest transposed fragment: 5.7 x).
PIVOT_FAILURES = {("pose_graph_1024", "stale_panel_tile"), ("pose_graph_1024", "transposed_fragment")}


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_every_fault_is_caught_by_three_orders(system, mutation):
    """each fault misses the bound by 1e3, or fails a pivot where PIVOT_FAILURES says so"""
    s = system
    d = tiled_solve(s["H"], s["b"], s["lam"], s["live"], mutation)
    if (s["name"], mutation) in PIVOT_FAILURES:
        assert d is None, mutation
        return
    assert d is not None, mutation
    d[~s["live"]] = 0.0  # what the device could read back
    eta = sc.scaled_backward_error(s["A"], d, s["b"], s["live"])
    print(f"{s['name']} {mutation}: eta {eta:.3g} = {eta / s['bound']:.3g} x the bound")
    assert eta >= 1e3 * s["bound"], (mutation, eta, s["bound"])
