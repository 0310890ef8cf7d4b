"""The dense fp64 solves of gb_pose_graph_optimize, gb_nav_graph_optimize and gb_graph_optimize on the H100, held to the
diagonally scaled backward error of tests/solve_check.py: one max_iterations = 1 round whose first trial is accepted, the
device's step read back from its result and checked against the restatement's host system -- at every tile shape, at the
size limits, on GLIM's graphs with their 1e10 anchor -- and the failed-pivot path of the tiled Cholesky."""
import numpy as np
import pytest

from glim_b200 import capi, gpu, synth, workloads
from tests import graph_oracle as go
from tests import lm_oracle as lm
from tests import nav_graph_oracle as ngo
from tests import pose_graph_oracle as pgo
from tests import solve_check as sc

pytestmark = pytest.mark.gpu

ONE = {"max_iterations": 1}
KIND_NAMES = {v: k for k, v in capi.VECTOR_KINDS.items()}


def between_round(ctx, T0, priors, bts, params=ONE):
    """one device round on a between graph and the restatement's; -> (device result, restatement result, host systems)"""
    got = gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=priors, betweens=[(i, j, Z, L, None) for i, j, Z, L, _ in bts], params=params, ctx=ctx)
    with sc.systems() as seen:
        ref = pgo.optimize(None, None, [], T0, priors, bts, params)
    return got, ref, seen


def rel(A, B):
    return synth.inv_pose(A) @ B


def check_round(label, got_T, got, ref, seen, T0, noise=None, cond=True):
    assert (got["iterations"], got["trials"]) == (ref["iterations"], ref["trials"]) == (1, 1), (label, got, ref["trials"])
    assert got["status"] == ref["status"]
    return sc.check(label, seen[0], sc.pose_steps(T0, got_T), sc.pose_steps(T0, ref["T"]), sc.pose_eps(T0, got_T), noise=noise, cond=cond)


@pytest.mark.parametrize("K", range(2, 66))
def test_pose_graph_every_tile_shape(ctx, K):
    """K = 2 .. 65: one tile (K <= 10), exactly two tiles, n = 192 unpadded and every residue of n = 6K mod 64"""
    T0, priors, bts = sc.between_graph(K, 4000 + K)
    got, ref, seen = between_round(ctx, T0, priors, bts)
    check_round(f"pose graph K {K}", [got["values"][k] for k in range(K)], got, ref, seen, T0)


def test_pose_graph_at_its_limit_ill_conditioned(ctx):
    T0, priors, bts = sc.ill_conditioned_graph()
    got, ref, seen = between_round(ctx, T0, priors, bts)
    _, cond = check_round("pose graph K 1024, informations 1e-2 .. 1e8", [got["values"][k] for k in range(1024)], got, ref, seen, T0)
    assert cond >= 1e12


@pytest.fixture(scope="module")
def gm64(ctx):
    """global mapping scaled down as tests/test_pose_graph_gpu.py builds it: 64 submaps on two laps, drifted starts"""
    w = workloads.global_mapping(ctx, n_submaps=64, laps=2, n_rays=64 * 128)
    facs = w.gpu_factors(w.sets[0])
    rng = synth.rng_for(2100)
    drift = np.array([0.0, 0.0, 0.001, 0.01, -0.005, 0.0])
    T0 = [w.poses[0]] + [synth.perturb(w.poses[k] @ synth.se3_exp(k * drift), rng, 0.002, 0.02) for k in range(1, len(w.poses))]
    return dict(facs=facs, T0=T0, keys=[(f.target, f.source) for f in w.sets[0].factors])


def sweep_records(ctx, facs, rows0, sel=None):
    """the restatement's linearize callables on the records of two identical gpu.Sweep runs over facs at rows0 -- the factors of
    the device call, as its sweep holds them -- restricted to the factors sel (all when None), and its error"""
    sel = range(len(facs)) if sel is None else sel
    out = []
    for _ in range(2):
        recs = gpu.Sweep(ctx, facs).linearize(rows0)[list(sel)]
        out.append(lambda f, d, recs=recs: (gpu.unpack_linearized(recs[f]), d))
    sub = [facs[i] for i in sel]

    def err(f, dl, d):
        return float(gpu.NonlinearFactorSetGPU(ctx).add([sub[f]]).error_deltas(dl[None], d[None])[0])

    return out, err


def restate_twice(optimize, lins, err, *args):
    """the restatement on the first sweep's records (result and system) and the second sweep's system"""
    with sc.systems() as seen:
        ref = optimize(lins[0], err, *args)
    with sc.systems() as again:
        optimize(lins[1], err, *args)
    return ref, seen, again[0][:2]


def test_pose_graph_global_mapping_vgicp(ctx, gm64):
    g = gm64
    T0, facs, K = g["T0"], g["facs"], len(g["T0"])
    priors = [(0, T0[0], 1e10)]
    call = lambda: gpu.optimize_pose_graph(facs, dict(enumerate(T0)), priors=priors, params=ONE, ctx=ctx)
    call()  # the factors learn their inlier fractions, as in the call below
    lins, err = sweep_records(ctx, facs, np.stack([rel(T0[t], T0[s]) for t, s in g["keys"]]))
    ref, seen, noise = restate_twice(pgo.optimize, lins, err, g["keys"], T0, priors, [], ONE)
    got = call()
    check_round(f"pose graph gm64 VGICP ({len(facs)} factors)", [got["values"][k] for k in range(K)], got, ref, seen, T0, noise)


def graph_problem(g, first, K, priors):
    keys = list(range(first, first + K))
    sel = [i for i, (t, s) in enumerate(g["keys"]) if first <= t < first + K and first <= s < first + K]
    return dict(keys=keys, sel=sel, prob=dict(factors=[g["facs"][i] for i in sel], values={k: g["T0"][k] for k in keys}, priors=priors))


def local_rows(g, p):
    first = p["keys"][0]
    lkeys = [(g["keys"][i][0] - first, g["keys"][i][1] - first) for i in p["sel"]]
    T0 = [g["T0"][k] for k in p["keys"]]
    return lkeys, T0, np.stack([rel(T0[t], T0[s]) for t, s in lkeys])


def graph_check(g, label, p, got, lins, err):
    """one gb_graph_optimize problem against the restatement on the records of its call's sweep, in local keys"""
    first = p["keys"][0]
    lkeys, T0, _ = local_rows(g, p)
    ref, seen, noise = restate_twice(go.optimize, lins, err, lkeys, T0, [(k - first, Z, w) for k, Z, w in p["prob"]["priors"]], ONE)
    return check_round(label, [got["values"][k] for k in p["keys"]], got, ref, seen, T0, noise)


def test_graph_batch_of_every_size(ctx, gm64):
    """31 problems of K = 2 .. 32 keys over gm64's submap ranges in one call, each against its own host system.  The records
    come from a sweep over the call's factors: a factor's fp32 partial sums are added in an order that depends on the sweep
    it is in."""
    g = gm64
    ps = [graph_problem(g, K - 2, K, [(K - 2, g["T0"][K - 2], 1e6)]) for K in range(2, 33)]
    assert all(p["sel"] for p in ps)
    gpu.optimize_graphs([p["prob"] for p in ps], params=ONE)  # the inlier fractions, as in the call below
    out = gpu.optimize_graphs([p["prob"] for p in ps], params=ONE)
    facs = [f for p in ps for f in p["prob"]["factors"]]
    rows = np.concatenate([local_rows(g, p)[2] for p in ps])
    off = np.cumsum([0] + [len(p["sel"]) for p in ps])
    for i, (p, got) in enumerate(zip(ps, out)):
        lins, err = sweep_records(ctx, facs, rows, range(off[i], off[i + 1]))
        graph_check(g, f"graph K {len(p['keys'])}", p, got, lins, err)


def test_graph_32_keys_with_1e10_and_1e8_priors(ctx, gm64):
    g = gm64
    p = graph_problem(g, 0, 32, [(0, g["T0"][0], 1e10), (31, g["T0"][31], 1e8)])
    gpu.optimize_graphs([p["prob"]], params=ONE)
    got = gpu.optimize_graphs([p["prob"]], params=ONE)[0]
    graph_check(g, "graph K 32, priors 1e10 / 1e8", p, got, *sweep_records(ctx, p["prob"]["factors"], local_rows(g, p)[2]))


def nav_round(ctx, label, m):
    ch = sc.imu_chain(m, lambda s, iv, bs: gpu.imu_preintegrate(s, iv, bs, ctx=ctx))
    T0, V0, B0 = ch["X0"]
    got = gpu.optimize_nav_graph([], dict(enumerate(T0)), dict(enumerate(V0)), dict(enumerate(B0)), priors=ch["priors"],
                                 betweens=[(i, j, Z, w, None) for i, j, Z, w in ch["betweens"]], imu_terms=ch["imu"],
                                 vector_terms=[(KIND_NAMES[k], a, b, z, w) for k, a, b, z, w in ch["vec"]], params=ONE, ctx=ctx)
    with sc.systems() as seen:
        ref = ngo.optimize(ch["graph"], ch["X0"], ONE)
    assert (got["iterations"], got["trials"]) == (ref["iterations"], ref["trials"]) == (1, 1), (label, got)
    assert got["status"] == ref["status"]
    X = ([got["poses"][k] for k in range(m)], [got["velocities"][k] for k in range(m)], [got["biases"][k] for k in range(m - 1)])
    return sc.check(label, seen[0], sc.nav_steps(ch["X0"], X), sc.nav_steps(ch["X0"], ref["x"]), sc.nav_eps(ch["X0"], X), live=ch["live"]), ch


def test_nav_graph_pinned_dofs_across_the_first_tile_edge(ctx):
    """K_X = 10 poses, then the velocities: the first velocity's pinned dofs are rows 63, 64, 65"""
    _, ch = nav_round(ctx, "nav chain of 10 frames", 10)
    assert [i for i in range(66) if not ch["live"][i]] == [63, 64, 65]


def test_nav_graph_at_its_limit(ctx):
    """683 poses, 683 velocities and 682 biases: 2048 slots, n = N = 12288, 192 tiles"""
    _, ch = nav_round(ctx, "nav chain of 2048 slots", 683)
    assert ch["graph"].K == 2048 and len(ch["live"]) == 12288


# ---- the failed-pivot path: a pair of keys joined by 2^50 I and nothing else ----


def pair_graph(K, pair, w):
    """a well-conditioned between graph over every key but the pair (the 1e10 anchor on key 0), started off its optimum, and the
    pair at identity joined by a between of information w I with its measurement identity"""
    rest = [k for k in range(K) if k not in pair]
    T0r, priors, bts = sc.between_graph(K - 2, 4300 + pair[0])
    T0 = [np.eye(4)] * K
    for r, k in enumerate(rest):
        T0[k] = T0r[r]
    bts = [(rest[i], rest[j], Z, L, k) for i, j, Z, L, k in bts] + [(pair[0], pair[1], np.eye(4), w * np.eye(6), 0.0)]
    return T0, [(rest[k], Z, wq) for k, Z, wq in priors], bts


@pytest.mark.parametrize("pair", [(1, 2), (1022, 1023)], ids=["tile0", "last_tile"])
def test_pose_graph_failed_pivots_reject_trials(ctx, pair):
    K, w = 1024, 2.0**50
    T0, priors, bts = pair_graph(K, pair, w)
    rec = pgo.between_record(np.eye(4), np.eye(4), np.eye(4), w * np.eye(6), 0.0)
    # every operand exact: blocks +-2^50 I, b = 0, so for lambda <= 0.1 (2^50 + lambda == 2^50) the second key's pivots are 0
    assert np.array_equal(rec["H_tt"], w * np.eye(6)) and np.array_equal(rec["H_ss"], w * np.eye(6)) and np.array_equal(rec["H_ts"], -w * np.eye(6))
    assert not rec["b_t"].any() and not rec["b_s"].any() and rec["error"] == 0.0
    got, ref, seen = between_round(ctx, T0, priors, bts)
    H, b, _ = seen[0]
    pr = np.r_[6 * pair[0]:6 * pair[0] + 6, 6 * pair[1]:6 * pair[1] + 6]
    rest = np.setdiff1d(np.arange(len(b)), pr)
    assert not H[np.ix_(pr, rest)].any() and not b[pr].any()  # the pair's rows stand alone: its block decides its pivots
    Hp = H[np.ix_(pr, pr)]

    def fails(Hb, lam):
        try:
            np.linalg.cholesky(Hb + lam * np.eye(len(Hb)))
            return False
        except np.linalg.LinAlgError:
            return True

    # numpy's verdicts: the five trials up to 0.1 fail, 1 solves; the restatement took them on the whole system
    assert [fails(Hp, 1e-5 * 10.0**k) for k in range(6)] == [True] * 5 + [False]
    assert (got["iterations"], got["trials"], got["status"], got["lambda"]) == (ref["iterations"], ref["trials"], ref["status"], ref["lambda"])
    assert (got["iterations"], got["trials"], got["status"]) == (1, 6, lm.ALIGN_MAX_ITERATIONS)
    Tg = [got["values"][k] for k in range(K)]
    assert all(np.array_equal(Tg[k], T0[k]) for k in pair)  # the pair's rows solve to exactly 0
    eps = sc.pose_eps(T0, Tg)
    eps[pr] = 0.0  # read back exactly: the pair's step is 0 and its poses are the identity, unchanged
    sc.check(f"pose graph K 1024, 2^50 pair at {pair}, lambda 1", (H, b, 1.0), sc.pose_steps(T0, Tg), sc.pose_steps(T0, ref["T"]), eps, cond=False)
    # the rejected trials leave the poses alone: stopped before lambda = 1 they come back as they went in
    stop = dict(ONE, lambda_upper_bound=0.5)
    got = gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=priors, betweens=[(i, j, Z, L, None) for i, j, Z, L, _ in bts], params=stop, ctx=ctx)
    assert (got["iterations"], got["trials"], got["status"]) == (1, 5, lm.ALIGN_LAMBDA_EXCEEDED)
    assert all(np.array_equal(got["values"][k], T0[k]) for k in range(K))
    # at 2^100 I every lambda up to the bound rounds away: LAMBDA_EXCEEDED after the 11 trials of 1e-5 .. 1e5
    big = bts[:-1] + [(pair[0], pair[1], np.eye(4), 2.0**100 * np.eye(6), 0.0)]
    assert all(fails(Hp * 2.0**50, 1e-5 * 10.0**k) for k in range(11))
    got = gpu.optimize_pose_graph([], dict(enumerate(T0)), priors=priors, betweens=[(i, j, Z, L, None) for i, j, Z, L, _ in big], params=ONE, ctx=ctx)
    assert (got["iterations"], got["trials"], got["status"]) == (1, 11, lm.ALIGN_LAMBDA_EXCEEDED)
    assert got["lambda"] > 1e5
    assert all(np.array_equal(got["values"][k], T0[k]) for k in range(K))
