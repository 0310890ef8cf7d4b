"""The Python binding of the C-ABI without a GPU:
  * capi's signature table declares, for every GB_API prototype of include/glim_b200.h, the ctypes argument and return types
    that prototype implies, in order -- a wrong float width or a dropped argument would otherwise pass every CPU test and
    corrupt the call on the device;
  * every handle class of gpu.py releases its handle through its own gb_*_destroy exactly once: on close(), not again on a
    second close() or on garbage collection, and also when its Context was closed first (clouds and maps hold no context,
    factors, sweeps and peer slabs hold a reference to theirs).  The library is replaced by a stub that records each call."""
import ctypes as C
import gc
import os
import re

import numpy as np
import pytest

from glim_b200 import capi, gpu
from tests.test_boundary import header_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCALARS = {"double": C.c_double, "float": C.c_float, "int": C.c_int, "int32_t": C.c_int, "gb_status": C.c_int, "size_t": C.c_size_t,
            "uint64_t": C.c_uint64}


def _ctype(decl: str):
    """a parameter declaration or a return type -> the ctypes type the binding must use"""
    if "*" in decl or "[" in decl:
        return C.c_char_p if decl.replace(" ", "") == "constchar*" else C.c_void_p
    words = decl.replace("const", "").split()
    return _SCALARS[words[0]]


def header_prototypes() -> dict:
    """name -> (argtypes, restype) of every GB_API function of include/glim_b200.h"""
    src = open(os.path.join(ROOT, "include", "glim_b200.h")).read()
    src = re.sub(r"/\*.*?\*/|//[^\n]*", "", src, flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"GB_API\s+([\w\s\*]+?)\s*\b(gb_\w+)\s*\(([^)]*)\)\s*;", src):
        params = [p.strip() for p in params.split(",")]
        args = [] if params == ["void"] else [_ctype(p) for p in params]
        out[name] = (args, _ctype(ret))
    return out


def test_signature_table_matches_the_header():
    declared = header_prototypes()
    assert len(declared) >= 85 and sorted(declared) == sorted(header_functions())  # every declaration was parsed
    assert capi.SYMBOLS == tuple(capi._SIGNATURES)
    assert sorted(declared) == sorted(capi.SYMBOLS)
    drift = {n: (capi._SIGNATURES[n], want) for n, want in declared.items() if (list(capi._SIGNATURES[n][0]), capi._SIGNATURES[n][1]) != want}
    assert not drift, drift


class _StubLib:
    """Records every call; a creator's trailing C.byref(c_void_p) receives a fresh fake handle."""

    def __init__(self):
        self.calls = []
        self.issued = set()

    def __getattr__(self, name):
        def call(*args):
            first = args[0] if args else None
            self.calls.append((name, first.value if isinstance(first, C.c_void_p) else first))
            if args and isinstance(getattr(args[-1], "_obj", None), C.c_void_p):
                args[-1]._obj.value = 0x1000 + 0x10 * len(self.issued)
                self.issued.add(args[-1]._obj.value)
            return 0

        return call

    def destroys(self, handle):
        return [n for n, h in self.calls if n.endswith("_destroy") and h == handle.value]


@pytest.fixture
def stub(monkeypatch):
    L = _StubLib()
    monkeypatch.setattr(capi, "lib", lambda: L)
    monkeypatch.setattr(gpu, "lib", lambda: L)
    yield L
    # objects a failed test left alive must not hand their fake handles to the real library later
    for o in gc.get_objects():
        if type(o).__module__ == gpu.__name__ and isinstance(getattr(o, "h", None), C.c_void_p) and o.h.value in L.issued:
            o.h = None


def _build_all(ctx):
    """one live object of every handle class -> [(object, its destroy function)]"""
    pts = np.hstack([np.zeros((4, 3)), np.ones((4, 1))])
    cloud = gpu.PointCloudGPU.clone(pts, ctx=ctx)
    vmap = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(cloud)
    incr = gpu.IncrementalVoxelMapGPU(0.5, ctx=ctx)
    ivox = gpu.IVoxGPU(1.0, ctx=ctx)
    grid = gpu.PointGridGPU(cloud, 1.0, ctx=ctx)
    vgicp = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, vmap, cloud, ctx=ctx)
    gicp = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, grid, cloud, 1.0, ctx=ctx)
    gicp._handle()  # factors create their handle on first use
    ct = gpu.IntegratedCT_GICPFactorGPU(0, 1, ivox, cloud, 1.0, ctx=ctx)
    sweep = gpu.Sweep(ctx, [vgicp])
    slab = gpu.PeerSlab(ctx, 4)
    return [(cloud, "gb_cloud_destroy"), (vmap, "gb_voxelmap_destroy"), (incr, "gb_voxelmap_destroy"), (ivox, "gb_ivox_destroy"),
            (grid, "gb_point_grid_destroy"), (vgicp, "gb_vgicp_factor_destroy"), (gicp, "gb_vgicp_factor_destroy"),
            (ct, "gb_vgicp_factor_destroy"), (sweep, "gb_sweep_destroy"), (slab, "gb_peer_slab_destroy")]


@pytest.mark.parametrize("context_closed_first", [False, True])
def test_every_handle_is_destroyed_exactly_once(stub, context_closed_first):
    ctx = gpu.Context(0)
    ctx_h = ctx.h
    objs = _build_all(ctx)
    handles = [(type(o).__name__, o.h, destroy) for o, destroy in objs]
    assert all(h.value for _, h, _ in handles)
    if context_closed_first:
        ctx.close()
    for o, _ in objs:
        o.close()
        assert o.h is None
        o.close()
    del o, objs
    gc.collect()
    for cls, h, destroy in handles:
        assert stub.destroys(h) == [destroy], cls
    ctx.close()
    del ctx
    gc.collect()
    assert stub.destroys(ctx_h) == ["gb_ctx_destroy"]
