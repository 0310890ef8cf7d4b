"""The entry-wise bound of tests/util.check_entrywise on the CPU: its per-hit data reproduce the fp64 oracle's record, and it
rejects defects of the kind a sweep's reduction or its fp64 epilogue could introduce, which the relative Frobenius bar of
check_linearized lets through when they land outside the rotation-rotation sub-block.

Each defect is applied to the oracle's own record (the target-side sums, then factor_epilogue's identities in fp64), on
util.scan_pair() at 0.5 m and the ground-truth pose."""
import numpy as np
import pytest

from glim_b200 import synth
from oracle import oracle
from tests import util

DROPPED = 32  # one warp's worth of hits


@pytest.fixture(scope="module")
def case():
    sp = util.scan_pair()
    tgt, src = (oracle.pack_cloud(sp["points"][k], util.cov_colmajor16(sp["covs"][k])) for k in (0, 1))
    T = synth.inv_pose(sp["poses"][0]) @ sp["poses"][1]
    m = oracle.GpuMap(*tgt, 0.5)
    rec, corr = oracle.linearize_gpumap(m, *src, T)
    hits = util.factor_hits(m.vmean, m.vcov, *src, T, corr)
    return oracle.split122(rec), hits, T


def old_bar_accepts(got, ref):
    try:
        util.check_linearized(got, ref)
        return True
    except AssertionError:
        return False


def new_bar_accepts(got, ref, hits):
    try:
        util.check_entrywise(got, ref, util.record_scale(hits))
        return True
    except AssertionError:
        return False


def test_hits_sum_to_the_oracle_record(case):
    """the numpy sum of the per-hit terms is the C oracle's record to fp64 rounding, and the epilogue's identities give its
    source blocks to the orthogonality of the fp32-cast rotation (R^T R = I within fp32 rounding, so Ad^T H_tt Ad and the
    oracle's sum over J_s agree to ~1e-7, far inside the bound)"""
    ref, hits, T = case
    assert len(hits) == ref["num_inliers"] > 6000
    s = util.hit_sums(hits)
    assert util.rel_err(s["H_tt"], ref["H_tt"]) < 1e-13
    assert np.linalg.norm(s["b_t"] - ref["b_t"]) < 1e-12 * np.linalg.norm(ref["b_t"])
    assert abs(s["error"] - ref["error"]) < 1e-12 * ref["error"]
    full = util.epilogue(s["H_tt"], s["b_t"], s["error"], s["num_inliers"], util.adjoint_f32(T))
    for k in ("H_ss", "H_ts"):
        assert util.rel_err(full[k], ref[k]) < 1e-6, k
    assert np.linalg.norm(full["b_s"] - ref["b_s"]) < 1e-6 * np.linalg.norm(ref["b_s"])
    # the exact record passes with room to spare
    assert util.check_linearized(full, ref, hits=hits) < 0.01


def mutated(hits, T, kind):
    """the oracle's record with one defect"""
    s = util.hit_sums(hits)
    Ad = util.adjoint_f32(T)
    if kind == "d":  # hat(t) R in Ad's upper-right block
        Ad = Ad.copy()
        Ad[:3, 3:] = Ad[3:, :3]
    out = util.epilogue(s["H_tt"].copy(), s["b_t"].copy(), s["error"], s["num_inliers"], Ad)
    k = slice(0, DROPPED)
    if kind == "a":  # a reduction that drops one warp's hits from the M sums (H_tt's translation block) only
        out["H_tt"][3:, 3:] -= hits.M[k].sum(0)
    elif kind == "b":  # ... from b_t's translation half only
        out["b_t"][3:] -= np.einsum("nij,nj->i", hits.M[k], hits.r[k])
    elif kind == "c":  # H_ts's column-major storage read as row-major
        out["H_ts"] = out["H_ts"].T.copy()
    elif kind == "e":  # the sign of H_ss's rotation-translation block
        out["H_ss"][:3, 3:] *= -1.0
        out["H_ss"][3:, :3] *= -1.0
    return out


@pytest.mark.parametrize("kind", ["a", "b", "c", "d", "e"])
def test_entrywise_bound_rejects_each_defect(case, kind):
    """(a) 32 hits dropped from H_tt's translation block, (b) from b_t's translation half, (c) H_ts transposed, (d) hat(t) R in
    Ad's upper-right block, (e) H_ss's rotation-translation block negated: the entry-wise bound rejects every one.  The
    relative Frobenius bar accepts (a) and (b)."""
    ref, hits, T = case
    got = mutated(hits, T, kind)
    old = old_bar_accepts(got, ref)
    print(f"defect ({kind}): the relative Frobenius bar {'accepts' if old else 'rejects'} it")
    assert not new_bar_accepts(got, ref, hits)
    if kind in ("a", "b"):
        assert old, "the old bar was expected to let this defect through"
