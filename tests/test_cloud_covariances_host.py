"""gb_cloud_estimate_covariances without a GPU: its binding matches include/glim_b200.h, and the two PointCloudGPU methods that
reach it (estimate_covariances, estimate_normals with an integer k) pass the right k and outputs flags, while estimate_normals()
without k still calls gb_cloud_estimate_normals.  The library is replaced by a recorder."""
import ctypes as C

import pytest

from glim_b200 import capi, gpu
from tests.test_binding_host import header_prototypes


def test_binding_matches_the_header():
    want = header_prototypes()["gb_cloud_estimate_covariances"]
    assert want == ([C.c_void_p, C.c_void_p, C.c_int, C.c_int], C.c_int)
    args, res = capi._SIGNATURES["gb_cloud_estimate_covariances"]
    assert (list(args), res) == want


def test_output_flags_match_the_header():
    import os
    import re

    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "glim_b200.h")).read()
    flags = dict((n, int(v)) for n, v in re.findall(r"#define (GB_CLOUD_\w+)\s+(\d+)", src))
    assert flags == {"GB_CLOUD_COVARIANCES": capi.GB_CLOUD_COVARIANCES, "GB_CLOUD_NORMALS": capi.GB_CLOUD_NORMALS}


@pytest.fixture
def recorded(monkeypatch):
    calls = []

    class Lib:
        def gb_cloud_estimate_covariances(self, ctx, cloud, k, outputs):
            assert isinstance(k, int) and isinstance(outputs, int)
            calls.append(("gb_cloud_estimate_covariances", ctx, cloud, k, outputs))
            return 0

        def gb_cloud_estimate_normals(self, ctx, cloud):
            calls.append(("gb_cloud_estimate_normals", ctx, cloud))
            return 0

    monkeypatch.setattr(gpu, "lib", lambda: Lib())
    ctx = object.__new__(gpu.Context)
    ctx.h = "ctx"
    cloud = object.__new__(gpu.PointCloudGPU)
    cloud.ctx, cloud.h, cloud.n = ctx, "cloud", 5
    yield cloud, calls
    cloud.h = ctx.h = None  # the fake handles must never reach the real library's destroy functions


def test_methods_pass_k_and_outputs(recorded):
    cloud, calls = recorded
    COV, NRM = capi.GB_CLOUD_COVARIANCES, capi.GB_CLOUD_NORMALS
    assert cloud.estimate_covariances() is cloud
    assert cloud.estimate_covariances(20) is cloud
    assert cloud.estimate_covariances(10, normals=True) is cloud
    assert cloud.estimate_covariances(k=32, normals=False) is cloud
    assert cloud.estimate_normals(20) is cloud
    assert cloud.estimate_normals(k=1) is cloud
    assert cloud.estimate_normals() is cloud
    assert cloud.estimate_normals(None) is cloud
    E = "gb_cloud_estimate_covariances"
    assert calls == [(E, "ctx", "cloud", 10, COV), (E, "ctx", "cloud", 20, COV), (E, "ctx", "cloud", 10, COV | NRM), (E, "ctx", "cloud", 32, COV),
                     (E, "ctx", "cloud", 20, NRM), (E, "ctx", "cloud", 1, NRM),
                     ("gb_cloud_estimate_normals", "ctx", "cloud"), ("gb_cloud_estimate_normals", "ctx", "cloud")]
