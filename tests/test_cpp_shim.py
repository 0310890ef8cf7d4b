"""The C++ side of the drop-in boundary: include/glim_b200.h is valid C, the gtsam_points-compatible shims compile in both
modes (stand-alone, and -DGLIM_B200_WITH_GTSAM against signature stubs -- GTSAM itself is not installed here), and on a
GPU a C++ program that drives the shims the way OdometryEstimationGPU does reproduces the oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
CPP = os.path.join(ROOT, "tests", "cpp")
GXX = "/usr/bin/g++"
GCC = "/usr/bin/gcc"


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "c_abi.c"
    src.write_text('#include "glim_b200.h"\nint main(void) { gb_linearized6 l; (void)l; return sizeof(gb_linearized6) == 122 * sizeof(double) ? 0 : 1; }\n')
    exe = tmp_path / "c_abi"
    subprocess.check_call([GCC, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{INC}", str(src), "-o", str(exe)])
    assert subprocess.call([str(exe)]) == 0


def test_plain_c_consumer_dlopens_the_library_and_resolves_every_entry_point(tmp_path):
    """SURVEY section 4, boundary tier: a C99 program (what a cgo / JNI stub would be) dlopen()s libglim_b200.so, resolves every
    symbol the header declares and drives the device-free part of the protocol; without a device gb_ctx_create must fail with
    GB_ERR_NO_DEVICE (no CPU fallback), with one it must succeed.  Runs on both boxes."""
    from glim_b200 import capi

    exe = tmp_path / "cabi_smoke"
    subprocess.check_call([GCC, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{INC}", os.path.join(CPP, "cabi_smoke.c"), "-o", str(exe), "-ldl"])
    r = subprocess.run([str(exe), capi.SO_PATH, *capi.SYMBOLS], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert f"{len(capi.SYMBOLS)} symbols" in r.stdout


def test_shims_compile_standalone_and_gtsam_mode(tmp_path):
    subprocess.check_call([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{INC}", "-c", os.path.join(CPP, "shim_main.cpp"), "-o", str(tmp_path / "a.o")])
    subprocess.check_call([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{INC}", f"-I{os.path.join(CPP, 'gtsam_stub')}", "-c", os.path.join(CPP, "gtsam_mode_check.cpp"), "-o", str(tmp_path / "b.o")])
    subprocess.check_call([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-pthread", f"-I{INC}", "-c", os.path.join(CPP, "replay_glim.cpp"), "-o", str(tmp_path / "c.o")])
    subprocess.check_call([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{INC}", "-c", os.path.join(CPP, "preprocess_main.cpp"), "-o", str(tmp_path / "d.o")])
    # GTSAM mode with Eigen-TYPED frames (the Eigen stand-in of oracle/ref_shim + the GTSAM signature stubs): the statements of GLIM's
    # GPU call sites (odometry_estimation_gpu.cpp:76-106, :128-165, :224-248, :383-386; sub_mapping.cpp:165-169; global_mapping.cpp:252-266)
    subprocess.check_call([GXX, "-std=c++17", "-Wall", "-Wextra", "-Werror", f"-I{INC}", f"-I{os.path.join(CPP, 'gtsam_stub')}", f"-I{os.path.join(ROOT, 'oracle', 'ref_shim')}",
                           "-c", os.path.join(CPP, "gtsam_eigen_mode_callsites.cpp"), "-o", str(tmp_path / "e.o")])


def test_cloud_deskewing_shim_host_half_matches_oracle_and_reference(tmp_path):
    """glim::CloudDeskewing shim (glim_preprocess_compat.hpp): its host half -- time table + pose per slot, the arguments exactly as
    deskew() marshals them -- built against the library and RUN on this box; applied on the host it must reproduce the oracle and,
    on a fixed sample of the points, the reference's own cloud_deskewing.cpp.  Without a device deskew() itself must throw."""
    import struct

    from oracle import oracle
    from tests.test_deskew import IMU_P, IMU_T, T_IL, V, W, scan_like

    lib_dir = os.path.join(ROOT, "glim_b200")
    exe = tmp_path / "deskew_host"
    subprocess.check_call([GXX, "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{INC}", os.path.join(CPP, "deskew_host_main.cpp"), "-o", str(exe),
                           f"-L{lib_dir}", "-lglim_b200", f"-Wl,-rpath,{lib_dir}"])
    times, pts = scan_like(n=5000, seed=7)
    n = len(pts)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    poses = np.ascontiguousarray(np.swapaxes(IMU_P, 1, 2)).reshape(-1, 16)
    with open(inp, "wb") as f:
        f.write(struct.pack("i", n) + times.tobytes() + np.ascontiguousarray(pts).tobytes() + oracle.pose_colmajor(T_IL).tobytes() + V.tobytes() + W.tobytes())
        f.write(struct.pack("i", len(IMU_T)) + np.ascontiguousarray(IMU_T).tobytes() + poses.tobytes() + struct.pack("d", 100.0))
    r = subprocess.run([str(exe), str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    raw = open(out, "rb").read()
    a = np.frombuffer(raw, np.float64, 4 * n).reshape(n, 4)
    b = np.frombuffer(raw, np.float64, 4 * n, offset=32 * n).reshape(n, 4)
    slots, threw = struct.unpack("ii", raw[64 * n:])
    assert slots > 100
    assert np.abs(a - oracle.deskew_const_vel(T_IL, V, W, times, pts)).max() < 1e-11
    assert np.abs(b - oracle.deskew_imu(T_IL, IMU_T, IMU_P, 100.0, times, pts)).max() < 1e-11
    from glim_b200 import capi

    if capi.lib().gb_device_count() == 0:
        assert threw == 1, "deskew() must fail loudly without a device (no CPU fallback)"
    # the original's own cloud_deskewing.cpp on the same scan (tests/golden/reference_tu_golden.npz)
    from tests.test_oracle_vs_reference_tu import GOLDEN, sample_rows

    rows = sample_rows(n)
    with np.load(GOLDEN) as g:
        assert np.abs(a[rows] - g["deskew7/cv_vw"]).max() < 1e-11
        assert np.abs(b[rows] - g["deskew7/imu_full"]).max() < 1e-11


def test_host_side_helpers_run_without_a_device(tmp_path):
    """random_sampling / sample (sub_mapping.cpp:385, global_mapping.cpp:248), the factor-set hook (offline_viewer.cpp:29) and
    VoxelBucket: host code of the shim, built against the library and run here (no device call is made)."""
    lib_dir = os.path.join(ROOT, "glim_b200")
    exe = tmp_path / "host_helpers"
    subprocess.check_call([GXX, "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{INC}", os.path.join(CPP, "host_helpers_main.cpp"), "-o", str(exe),
                           f"-L{lib_dir}", "-lglim_b200", f"-Wl,-rpath,{lib_dir}"])
    out = tmp_path / "out.bin"
    n, rate = 5000, 0.1
    assert subprocess.call([str(exe), str(n), str(rate), str(out)]) == 0
    raw = out.read_bytes()
    m = int(np.frombuffer(raw[:4], np.int32)[0])
    idx = np.frombuffer(raw[4:4 + 4 * m], np.int32)
    assert m == int(n * rate) and raw[-1] == 1
    assert (np.diff(idx) > 0).all() and idx.min() >= 0 and idx.max() < n
    # a uniform draw: the sample's mean index is near the middle, every decile is hit
    assert abs(idx.mean() - n / 2) < 0.1 * n and len(set(idx // (n // 10))) == 10


def test_solver_handoff_blocks_host_only():
    """gb_hessian_blocks / gb_slab_row_hessian_blocks (SURVEY A.3, global_mapping.cpp:492-501): HessianFactor(k_t, k_s, H_tt, H_ts,
    -b_t, H_ss, -b_s, scale * error) from a record and from a pair-slab row; host-only helpers, no device needed."""
    from glim_b200 import capi, gpu, multi_gpu

    rng = np.random.default_rng(3)
    rec = np.zeros(1, gpu.LIN_DTYPE)
    A = rng.normal(size=(12, 12))
    H = A @ A.T
    rec[0]["H_tt"] = H[:6, :6].T.reshape(36)
    rec[0]["H_ts"] = H[:6, 6:].T.reshape(36)
    rec[0]["H_ss"] = H[6:, 6:].T.reshape(36)
    rec[0]["b_t"], rec[0]["b_s"] = rng.normal(size=6), rng.normal(size=6)
    rec[0]["error"], rec[0]["num_inliers"] = 3.5, 1234.0
    outs = [np.zeros(36), np.zeros(36), np.zeros(6), np.zeros(36), np.zeros(6), np.zeros(1)]
    capi.check(capi.lib().gb_hessian_blocks(capi.ptr(rec), 0.5, *[capi.ptr(o) for o in outs]))
    assert np.array_equal(outs[0].reshape(6, 6).T, H[:6, :6]) and np.array_equal(outs[1].reshape(6, 6).T, H[:6, 6:]) and np.array_equal(outs[3].reshape(6, 6).T, H[6:, 6:])
    assert np.array_equal(outs[2], -rec[0]["b_t"]) and np.array_equal(outs[4], -rec[0]["b_s"]) and outs[5][0] == 0.5 * 3.5
    row = multi_gpu.pack_slab_row(gpu.unpack_linearized(rec[0]))
    outs2 = [np.zeros(36), np.zeros(36), np.zeros(6), np.zeros(36), np.zeros(6), np.zeros(1), np.zeros(1)]
    capi.check(capi.lib().gb_slab_row_hessian_blocks(capi.ptr(row), 0.5, *[capi.ptr(o) for o in outs2]))
    for a, b in zip(outs, outs2[:6]):
        assert np.allclose(a, b, rtol=1e-6, atol=1e-6)
    assert outs2[6][0] == 1234.0


@pytest.mark.gpu
def test_cpp_shim_reproduces_oracle(tmp_path):
    from glim_b200 import capi, synth
    from oracle import oracle
    from tests import util

    exe = tmp_path / "shim_main"
    libdir = os.path.dirname(capi.SO_PATH)
    subprocess.check_call([GXX, "-std=c++17", "-O2", f"-I{INC}", os.path.join(CPP, "shim_main.cpp"), "-o", str(exe), f"-L{libdir}", "-lglim_b200", f"-Wl,-rpath,{libdir}"])
    pair = util.scan_pair()
    Tt = synth.pose(3.0, -1.0, 0.2, 0.4, 0.01, -0.02)
    T = synth.perturb(synth.inv_pose(pair["poses"][0]) @ pair["poses"][1], synth.rng_for(21), 0.01, 0.05)
    Ts = Tt @ T
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([len(pair["points"][0]), len(pair["points"][1])], np.int32).tofile(f)
        for k in (0, 1):
            np.ascontiguousarray(pair["points"][k]).tofile(f)
            util.cov_colmajor16(pair["covs"][k]).tofile(f)
        capi.pose16(Tt).tofile(f)
        capi.pose16(Ts).tofile(f)
    out = tmp_path / "out.bin"
    subprocess.check_call([str(exe), str(inp), str(out)])
    raw = np.fromfile(out, dtype=np.uint8)
    recs = np.frombuffer(raw[: 4 * 976].tobytes(), dtype=np.float64).reshape(4, 122)
    err, ov = np.frombuffer(raw[4 * 976 : 4 * 976 + 16].tobytes(), dtype=np.float64)
    nv = np.frombuffer(raw[4 * 976 + 16 : 4 * 976 + 32].tobytes(), dtype=np.int32)

    xyz0, cov0 = oracle.pack_cloud(pair["points"][0], util.cov_colmajor16(pair["covs"][0]))
    xyz1, cov1 = oracle.pack_cloud(pair["points"][1], util.cov_colmajor16(pair["covs"][1]))
    delta = synth.inv_pose(Tt) @ Ts
    for level, res in enumerate((0.25, 0.5)):
        m = oracle.GpuMap(xyz0, cov0, res)
        assert (nv[level], nv[2 + level]) == (m.num_voxels, m.num_buckets)
        ref = oracle.split122(oracle.linearize_gpumap(m, xyz1, cov1, delta)[0])
        for rec in (recs[level], recs[2 + level]):  # binary and unary forms see the same delta
            got = oracle.split122(rec)
            assert got["num_inliers"] == ref["num_inliers"] > 0
            for k in ("H_tt", "H_ss", "H_ts"):
                assert util.rel_err(got[k], ref[k]) < util.REL_TOL
            assert abs(got["error"] - ref["error"]) < util.REL_TOL * ref["error"]
        if level == 1:
            assert abs(err - ref["error"]) < util.REL_TOL * ref["error"]
            assert ov == oracle.overlap_gpumap([m], xyz1, [delta])


@pytest.mark.gpu
def test_replay_glim_modules_across_threads_under_asan(tmp_path):
    """The exact statements of odometry_estimation_gpu.cpp:96-104, sub_mapping.cpp:165-169 / :393-399 and
    global_mapping.cpp:239-266 / :322-335, one module per thread, frames handed from module to module, built with
    AddressSanitizer: clones own their host data (reading frame->points after `frame = clone(*frame)` is legal), work runs on
    the stream each module passes, factor sets mix clouds / maps uploaded by different module threads."""
    from glim_b200 import capi, synth
    from oracle import oracle
    from tests import util

    exe = tmp_path / "replay_glim"
    libdir = os.path.dirname(capi.SO_PATH)
    subprocess.check_call([GXX, "-std=c++17", "-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer", "-pthread", f"-I{INC}", os.path.join(CPP, "replay_glim.cpp"), "-o", str(exe), f"-L{libdir}", "-lglim_b200", f"-Wl,-rpath,{libdir}"])
    pair = util.scan_pair()
    Tt = synth.pose(3.0, -1.0, 0.2, 0.4, 0.01, -0.02)
    T = synth.perturb(synth.inv_pose(pair["poses"][0]) @ pair["poses"][1], synth.rng_for(22), 0.01, 0.05)
    Ts = Tt @ T
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([len(pair["points"][0]), len(pair["points"][1])], np.int32).tofile(f)
        for k in (0, 1):
            np.ascontiguousarray(pair["points"][k]).tofile(f)
            util.cov_colmajor16(pair["covs"][k]).tofile(f)
        capi.pose16(Tt).tofile(f)
        capi.pose16(Ts).tofile(f)
    out = tmp_path / "out.bin"
    env = dict(os.environ, ASAN_OPTIONS="protect_shadow_gap=0:detect_leaks=0:abort_on_error=0")
    r = subprocess.run([str(exe), str(inp), str(out)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
    assert "AddressSanitizer" not in r.stderr
    raw = np.fromfile(out, dtype=np.uint8)
    recs = np.frombuffer(raw[: 6 * 976].tobytes(), dtype=np.float64).reshape(6, 122)
    ov = np.frombuffer(raw[6 * 976 : 6 * 976 + 24].tobytes(), dtype=np.float64)
    md = np.frombuffer(raw[6 * 976 + 24 : 6 * 976 + 40].tobytes(), dtype=np.float64)
    assert md[0] == md[1] > 0  # host data survived clone-of-clone and the death of every earlier owner
    xyz0, cov0 = oracle.pack_cloud(pair["points"][0], util.cov_colmajor16(pair["covs"][0]))
    xyz1, cov1 = oracle.pack_cloud(pair["points"][1], util.cov_colmajor16(pair["covs"][1]))
    delta = synth.inv_pose(Tt) @ Ts
    for level, res in enumerate((0.25, 0.5)):
        m = oracle.GpuMap(xyz0, cov0, res)
        ref = oracle.split122(oracle.linearize_gpumap(m, xyz1, cov1, delta)[0])
        for module in range(3):  # odometry / sub-mapping (mixed contexts) / global mapping
            got = oracle.split122(recs[2 * module + level])
            assert got["num_inliers"] == ref["num_inliers"] > 0
            for k in ("H_tt", "H_ss", "H_ts"):
                assert util.rel_err(got[k], ref[k]) < util.REL_TOL
        if level == 1:
            assert ov[0] == ov[1] == ov[2] == oracle.overlap_gpumap([m], xyz1, [delta])


@pytest.mark.gpu
def test_cpp_preprocess_shims_match_oracle(tmp_path):
    """glim::CloudPreprocessor / CloudCovarianceEstimation shims (C++, include/glim_b200/glim_preprocess_compat.hpp) and the
    fused preprocess_to_gpu_frame against the oracle composition of the reference pipeline; merge_frames_gpu on the result."""
    from glim_b200 import capi, synth
    from oracle import oracle

    exe = tmp_path / "preprocess_main"
    libdir = os.path.dirname(capi.SO_PATH)
    subprocess.check_call([GXX, "-std=c++17", "-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer", f"-I{INC}", os.path.join(CPP, "preprocess_main.cpp"), "-o", str(exe), f"-L{libdir}", "-lglim_b200", f"-Wl,-rpath,{libdir}"])
    sc = synth.make_hall_scene()
    P, T = synth.scan(sc, "hdl32", synth.arc_trajectory(8)[2], synth.rng_for(43), n_rays=32 * 500)
    k, res, near, far = 10, 0.2, 1.0, 60.0
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        np.array([len(P)], np.int32).tofile(f)
        np.ascontiguousarray(P).tofile(f)
        np.ascontiguousarray(T).tofile(f)
        np.array([res, near, far]).tofile(f)
        np.array([k], np.int32).tofile(f)
    env = dict(os.environ, ASAN_OPTIONS="protect_shadow_gap=0:detect_leaks=0")
    r = subprocess.run([str(exe), str(inp), str(out)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "AddressSanitizer" not in r.stderr, r.stderr[-3000:]
    raw = open(out, "rb").read()
    m = int(np.frombuffer(raw[:4], np.int32)[0])
    o = 4
    pts = np.frombuffer(raw[o : o + 32 * m], np.float64).reshape(m, 4); o += 32 * m
    tms = np.frombuffer(raw[o : o + 8 * m], np.float64); o += 8 * m
    nb = np.frombuffer(raw[o : o + 4 * m * k], np.int32).reshape(m, k); o += 4 * m * k
    cov_a = np.frombuffer(raw[o : o + 128 * m], np.float64).reshape(m, 4, 4).transpose(0, 2, 1); o += 128 * m
    cov_b = np.frombuffer(raw[o : o + 128 * m], np.float64).reshape(m, 4, 4).transpose(0, 2, 1); o += 128 * m
    merged, has_gpu = np.frombuffer(raw[o : o + 8], np.int32)
    rp, rt, _ = oracle.voxelgrid_sampling(P, res, times=T)
    sq = (rp[:, :3] ** 2).sum(1)
    idx = np.nonzero((sq > near * near) & (sq < far * far))[0]
    idx = idx[np.argsort(rt[idx], kind="stable")]
    rp, rt = np.ascontiguousarray(rp[idx]), rt[idx]
    assert m == len(rp) and np.array_equal(pts, rp) and np.array_equal(tms, rt)
    rnb, _ = oracle.knn_bruteforce(rp, k)
    assert np.array_equal(nb, rnb)
    _, rc = oracle.covariance_estimate(rp, rnb)
    assert np.allclose(cov_a, rc, atol=1e-9) and np.allclose(cov_b, rc, atol=1e-9)
    assert has_gpu == 1 and 0 < merged <= 2 * m
