"""CPU-only checks of gb_find_overlapping_submaps (no GPU needed):
  * gb_overlap_math.cuh compiled for the host (tests/cpp/overlap_math_host.cpp): the candidate slots decode to the lexicographic
    pair list, and the relative pose and gate equal the numpy restatement (tests/overlap_search_oracle.py) bit for bit, also
    for poses 1e5 m from the origin;
  * every argument rule of the header is refused before any launch, with gb_last_error naming the argument."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from glim_b200 import capi, synth
from tests import overlap_search_oracle as oso

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def om(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("om") / "liboverlap_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so, os.path.join(ROOT, "tests", "cpp", "overlap_math_host.cpp")])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.om_num_slots.argtypes, L.om_num_slots.restype = [C.c_longlong, C.c_longlong], C.c_longlong
    L.om_pairs.argtypes = [C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong, vp]
    L.om_deltas.argtypes = [C.c_int, vp, vp, C.c_double, vp, vp]
    L.om_chunks.argtypes = [C.c_int, vp, vp]
    L.om_items.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("S", [1, 2, 3, 7, 64, 257])
def test_slots_decode_to_the_lexicographic_pairs(om, S):
    for f in sorted({0, 1, S // 2, max(0, S - 2), S - 1}):
        want = oso.slots(S, f)
        N = om.om_num_slots(S, f)
        assert N == len(want) == (S * (S - 1) - f * (f - 1)) // 2, (S, f)
        got = np.zeros((max(N, 1), 2), np.int32)
        om.om_pairs(S, f, 0, N, _p(got))
        assert [tuple(x) for x in got[:N]] == want, (S, f)


def test_largest_slot_count(om):
    """S = GB_OVERLAP_SEARCH_MAX_SUBMAPS: 8.4 M slots; the first and last rows and slots around row boundaries decode right"""
    S = capi.GB_OVERLAP_SEARCH_MAX_SUBMAPS
    for f in (0, 1000, S - 1):
        want = oso.slots(S, f) if f == S - 1 else None
        N = om.om_num_slots(S, f)
        assert N == (S * (S - 1) - f * (f - 1)) // 2
        if want is not None:
            got = np.zeros((N, 2), np.int32)
            om.om_pairs(S, f, 0, N, _p(got))
            assert [tuple(x) for x in got] == want
    assert om.om_num_slots(S, 0) == 8386560
    for k, want in ((0, (0, 1)), (S - 2, (0, S - 1)), (S - 1, (1, 2)), (2 * S - 4, (1, S - 1)), (2 * S - 3, (2, 3)), (8386560 - 1, (S - 2, S - 1))):
        got = np.zeros((1, 2), np.int32)
        om.om_pairs(S, 0, k, 1, _p(got))
        assert tuple(got[0]) == want, k


def test_work_items_are_counted_in_64_bits(om):
    """k_overlap's items: a search over 4096 submaps of up to 2^30 points each has up to 8.4 M x 2^22 items.  The chunk counts,
    the query of an item and its first point are exact far beyond 2^31 items (query of item k: the first q with
    item_end[q] > k, queries without points skipped)."""
    rng = np.random.default_rng(9)
    nq = 20000
    sizes = rng.integers(0, 70000, nq).astype(np.int32)
    sizes[rng.random(nq) < 0.05] = 0                        # empty sources: no items
    sizes[rng.choice(nq, 3000, replace=False)] = (1 << 30) - 1  # the largest clouds
    chunks = np.zeros(nq, np.int64)
    om.om_chunks(nq, _p(sizes), _p(chunks))
    assert np.array_equal(chunks, (sizes.astype(np.int64) + 255) // 256)
    item_end = np.cumsum(chunks)
    assert item_end[-1] > 1 << 33
    items = np.unique(np.concatenate([rng.integers(0, item_end[-1], 200000), item_end[:-1], item_end - 1, [0, (1 << 31) - 1, 1 << 31, (1 << 32) + 5, item_end[-1] - 1]]))
    items = items[(items >= 0) & (items < item_end[-1])]
    q = np.zeros(len(items), np.int32)
    pt = np.zeros(len(items), np.int32)
    om.om_items(_p(item_end), nq, len(items), _p(items), _p(q), _p(pt))
    want_q = np.searchsorted(item_end, items, side="right")
    start = np.where(want_q > 0, item_end[np.maximum(want_q - 1, 0)], 0)
    assert np.array_equal(q, want_q)
    assert np.array_equal(pt, (items - start) * 256)
    assert (pt >= 0).all() and (pt < sizes[q]).all()


def random_poses(rng, n, offset):
    T = np.stack([synth.pose(*(rng.uniform(-50, 50, 3) + offset), rng.uniform(-np.pi, np.pi), *rng.uniform(-0.3, 0.3, 2)) for _ in range(n)])
    return T


@pytest.mark.parametrize("offset", [0.0, 1e5, -3e5])
def test_host_build_delta_and_gate_equal_the_restatement(om, offset):
    rng = np.random.default_rng(int(abs(offset)) + 5)
    n = 4000
    Ti, Tj = random_poses(rng, n, offset), random_poses(rng, n, offset)
    Tj[:50] = Ti[:50]  # identical poses: t = 0 exactly
    for md in (0.0, 30.0, 60.0, 1e300):
        D = np.zeros((n, 16))
        g = np.zeros(n, np.int32)
        om.om_deltas(n, _p(capi.pose16(Ti)), _p(capi.pose16(Tj)), md * md, _p(D), _p(g))
        want = oso.deltas(Ti, Tj)
        assert np.array_equal(D, capi.pose16(want))
        assert np.array_equal(g.astype(bool), oso.gate(want, md))
        if md == 0.0:
            assert g[:50].all() and g.sum() == 50 + int((np.abs(want[50:, :3, 3]).sum(1) == 0).sum())
        if md == 1e300:
            assert g.all()
    # the restatement is T_i^-1 T_j to rounding
    ref = np.linalg.inv(Ti) @ Tj
    assert np.abs(want - ref).max() < 1e-9 * max(1.0, abs(offset))


# ---------------------------------------------------------------------------------------------------------------------
# argument rules
# ---------------------------------------------------------------------------------------------------------------------
def refusal(**kw):
    """gb_find_overlapping_submaps with valid-looking dummy arguments (never dereferenced: validation comes first) and kw
    replaced; -> (status, gb_last_error)"""
    L = capi.lib()
    S = kw.get("S", 3)
    dummy = C.c_void_p(1)
    handles = (C.c_void_p * max(1, S))(*([1] * max(1, S)))
    T = kw.get("T", capi.pose16(np.stack([np.eye(4)] * max(1, S))))
    ex = kw.get("existing", np.zeros((0, 2), np.int32))
    found = C.c_size_t(7)
    pairs, ovs = np.zeros((4, 2), np.int32), np.zeros(4)
    args = dict(ctx=dummy, S=S, maps=C.cast(handles, C.c_void_p), sources=C.cast(handles, C.c_void_p), T=capi.ptr(T) if T is not None else None, first_source=0, E=len(ex),
                existing=capi.ptr(ex) if len(ex) else None, max_distance=100.0, min_overlap=0.2, capacity=4, num_found=C.byref(found), pairs=capi.ptr(pairs),
                overlaps=capi.ptr(ovs))
    args.update({k: v for k, v in kw.items() if k in args})
    if "T" in kw:
        args["T"] = capi.ptr(T)
    if "existing" in kw:
        args["existing"] = capi.ptr(ex) if len(ex) else None
        args["E"] = kw.get("E", len(ex))
    st = L.gb_find_overlapping_submaps(*args.values())
    return st, L.gb_last_error().decode(), found.value


@pytest.mark.parametrize("kw, names", [
    (dict(ctx=None), "ctx"),
    (dict(num_found=None), "num_found"),
    (dict(maps=None), "maps"),
    (dict(sources=None), "sources"),
    (dict(T=None), "T_world_submap"),
    (dict(S=0), "num_submaps"),
    (dict(S=capi.GB_OVERLAP_SEARCH_MAX_SUBMAPS + 1), "num_submaps"),
    (dict(first_source=3), "first_source"),
    (dict(first_source=10), "first_source"),
    (dict(T=np.where(np.arange(48) == 13, np.nan, np.tile(capi.pose16(np.eye(4)), 3)).reshape(3, 16)), "T_world_submap"),
    (dict(T=np.where(np.arange(48) == 40, np.inf, np.tile(capi.pose16(np.eye(4)), 3)).reshape(3, 16)), "T_world_submap"),
    (dict(max_distance=-1.0), "max_distance"),
    (dict(max_distance=float("nan")), "max_distance"),
    (dict(max_distance=float("inf")), "max_distance"),
    (dict(min_overlap=float("nan")), "min_overlap"),
    (dict(min_overlap=float("-inf")), "min_overlap"),
    (dict(E=2, existing=np.zeros((0, 2), np.int32)), "existing"),
    (dict(existing=np.array([[0, 1], [1, 3]], np.int32)), "existing"),
    (dict(existing=np.array([[-1, 2]], np.int32)), "existing"),
    (dict(pairs=None), "pairs"),
    (dict(overlaps=None), "overlaps"),
])
def test_invalid_arguments_are_refused_before_any_launch(kw, names):
    st, err, found = refusal(**kw)
    assert st == 1, (kw, err)
    assert names in err, (kw, err)
    if "num_found" not in kw:
        assert found == 0  # cleared before the first rule that reads the arrays


def test_capacity_zero_with_null_arrays_passes_the_array_rule():
    """capacity 0 with NULL pairs / overlaps is allowed: such a call with an out-of-range existing key is refused for the key,
    and with every earlier rule met it gets past the array rule to the handles (here refused for a NULL map entry)."""
    st, err, _ = refusal(capacity=0, pairs=None, overlaps=None, existing=np.array([[0, 5]], np.int32))
    assert st == 1 and "existing" in err
    L = capi.lib()
    handles = (C.c_void_p * 3)(None, None, None)
    T = capi.pose16(np.stack([np.eye(4)] * 3))
    found = C.c_size_t(7)
    st = L.gb_find_overlapping_submaps(C.c_void_p(1), 3, C.cast(handles, C.c_void_p), C.cast(handles, C.c_void_p), capi.ptr(T), 0, 0, None, 100.0, 0.2, 0,
                                       C.byref(found), None, None)
    assert st == 1 and "null entry of maps" in L.gb_last_error().decode() and found.value == 0


def test_signature_and_limit():
    assert capi.GB_OVERLAP_SEARCH_MAX_SUBMAPS == 4096
    hdr = open(os.path.join(ROOT, "include", "glim_b200.h")).read()
    assert "#define GB_OVERLAP_SEARCH_MAX_SUBMAPS 4096" in hdr
