"""Global registration on the device (gb_cloud_estimate_fpfh, gb_fpfh_match, gb_ransac_align, gb_gnc_align) with the manual
loop-closure modal's defaults (manual_loop_close_modal.cpp:42-52: fpfh_radius 5.0, 5000 iterations, early stop at 0.9, 1.0 m
inlier voxels, 4-DoF, 10000 GNC samples), on two overlapping maps of the hall scene at 30 k and 100 k points each, the source expressed under a pose 120 degrees
of yaw and 18 m away:

  fpfh      gb_cloud_estimate_fpfh of one map (its point grid included);
  match     gb_fpfh_match of the source's features against the target's;
  ransac    gb_ransac_align with early stop at 0.9 (the default) and without (rate 2: every hypothesis is scored);
  gnc       gb_gnc_align (reciprocal matches of 10000 samples, the Geman-McClure schedule, the score);
  e2e       both maps' features, RANSAC and the fine registration (LM on a grid GICP factor, r = 1.0), from device clouds;
  gnc_e2e   the same with GNC as the global method;
  normals   gb_cloud_estimate_normals of one merged submap (gb_merge_frames of the map: covariances, no normals);
  icp       one linearization of a point-to-point ICP factor on a point grid (r = 1.0) between the two maps uploaded without
            covariances, and the modal's 200-iteration align (GTSAM's LM defaults, no step tests) from 0.1 m / 0.01 rad off;
  submap_e2e  the right-click recipe from two merged device submaps: normals, features, RANSAC and the fine registration
            (20 iterations);
  host      the numpy restatement of the match (tests/global_oracle.py) on 2 k x 2 k of the same features; the restatement of
            the FPFH and of RANSAC takes minutes at these sizes and is not run.

Times are a host clock around synchronised calls after one warm-up pass, median of --repeats passes.  Prints one JSON line per
size with the card's name and power limit, read in the same run.

    python scripts/bench_global.py [--repeats 3] [--sizes 30000,100000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from glim_b200 import gpu, preprocess, synth  # noqa: E402
from tests import global_oracle as gl  # noqa: E402


def world_points(frames_idx, n, seed):
    """n points of the hall seen from the arc frames frames_idx, in the world frame, with PLANE normals and covariances"""
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(24)
    pts = []
    for i in frames_idx:
        p, _ = synth.scan(sc, "hdl32", traj[i], synth.rng_for(700, i), n_rays=32 * 1200)
        p = p[np.isfinite(p).all(1)]
        p[:, :3] = p[:, :3] @ traj[i][:3, :3].T + traj[i][:3, 3]
        pts.append(p)
    p = np.concatenate(pts)
    p = p[np.random.default_rng(seed).choice(len(p), size=min(n, len(p)), replace=False)]
    nb = preprocess.find_neighbors(p, 10)
    normals, covs = preprocess.CloudCovarianceEstimation().estimate(p, nb)
    return p, covs, normals


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sizes", default="30000,100000")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    ctx = gpu.default_context()
    T_gt = synth.pose(15.0, -10.0, 0.5, np.radians(120))
    Ti = synth.inv_pose(T_gt)
    def error(T):
        D = Ti @ T
        return float(np.linalg.norm(D[:3, 3])), float(np.degrees(np.arccos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1))))

    for n in [int(s) for s in args.sizes.split(",")]:
        tp, tc, tn = world_points(range(0, 12), n, 1)
        sp, sc, sn = world_points(range(6, 18), n, 2)
        sp = np.c_[sp[:, :3] @ Ti[:3, :3].T + Ti[:3, 3], np.ones(len(sp))]
        sc = np.einsum("ij,njk,lk->nil", Ti, sc, Ti)
        sn = np.c_[sn[:, :3] @ Ti[:3, :3].T, np.zeros(len(sn))]
        tgt = gpu.PointCloudGPU.clone(tp, tc, tn, ctx=ctx)
        src = gpu.PointCloudGPU.clone(sp, sc, sn, ctx=ctx)
        out = {"points": n, "card": card}
        out["fpfh_ms"] = timed(lambda: tgt.estimate_fpfh(5.0), args.repeats)
        src.estimate_fpfh(5.0)
        out["match_ms"] = timed(lambda: gpu.fpfh_match(tgt, src), args.repeats)
        res = {}

        def ransac(rate):
            res[rate] = gpu.estimate_pose_ransac(tgt, src, early_stop_inlier_rate=rate)

        out["ransac_early_stop_ms"] = timed(lambda: ransac(0.9), args.repeats)
        out["ransac_all_ms"] = timed(lambda: ransac(2.0), args.repeats)
        for rate, key in ((0.9, "ransac_early_stop"), (2.0, "ransac_all")):
            r = res[rate]
            et, er = np.linalg.norm((Ti @ r["T_target_source"])[:3, 3]), np.degrees(np.arccos(np.clip((np.trace((Ti @ r["T_target_source"])[:3, :3]) - 1) / 2, -1, 1)))
            out[key + "_result"] = {"status": r["status_name"], "evaluated": r["evaluated"], "inlier_rate": round(r["inlier_rate"], 4),
                                    "err_m": round(float(et), 3), "err_deg": round(float(er), 3)}
        gnc = {}

        def run_gnc():
            gnc["r"] = gpu.estimate_pose_gnc(tgt, src)

        out["gnc_ms"] = timed(run_gnc, args.repeats)
        r = gnc["r"]
        et, er = error(r["T_target_source"])
        out["gnc_result"] = {"status": r["status_name"], "samples": r["samples"], "correspondences": r["correspondences"], "iterations": r["iterations"],
                             "inlier_rate": round(r["inlier_rate"], 4), "err_m": round(et, 3), "err_deg": round(er, 3)}
        fine = {}

        def e2e(estimate):
            a = gpu.PointCloudGPU.clone(tp, tc, tn, ctx=ctx).estimate_fpfh(5.0)
            b = gpu.PointCloudGPU.clone(sp, sc, sn, ctx=ctx).estimate_fpfh(5.0)
            r = estimate(a, b)
            g = gpu.PointGridGPU(a, 1.05, ctx=ctx)
            f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, g, b, 1.0, ctx=ctx)
            fine["r"] = gpu.align_vgicp([[f]], [r["T_target_source"]], params={"max_iterations": 30})[0]

        for key, estimate in (("e2e", gpu.estimate_pose_ransac), ("gnc_e2e", gpu.estimate_pose_gnc)):
            out[key + "_ms"] = timed(lambda: e2e(estimate), args.repeats)
            et, er = error(fine["r"]["T_target_source"])
            out[key + "_err_m"] = round(et, 4)
            out[key + "_err_deg"] = round(er, 4)
        def merged(p, c):
            return gpu.merge_frames_gpu([np.eye(4)], [gpu.PointCloudGPU.clone(p, c, ctx=ctx)], 0.01, ctx=ctx, host_outputs=False)[2]

        ta = merged(tp, tc)
        out["normals_ms"] = timed(ta.estimate_normals, args.repeats)
        out["normals_points"] = ta.n
        ti, si = gpu.PointCloudGPU.clone(tp, ctx=ctx), gpu.PointCloudGPU.clone(sp, ctx=ctx)
        fi = gpu.IntegratedICPFactorGPU(np.eye(4), 0, gpu.PointGridGPU(ti, 1.05, ctx=ctx), si, 1.0, ctx=ctx)
        out["icp_linearize_ms"] = timed(lambda: fi.linearize({0: T_gt}), args.repeats)
        T0 = synth.perturb(T_gt, np.random.default_rng(3), 0.01, 0.1)
        modal = {"max_iterations": 200, "lambda_initial": 1e-5, "lambda_factor": 10.0, "lambda_upper_bound": 1e5, "relative_error_tol": 1e-5,
                 "absolute_error_tol": 1e-5, "step_translation_tol": 0.0, "step_rotation_tol": 0.0}
        icp = {}

        def icp_align():
            icp["r"] = gpu.align_vgicp([[fi]], [T0], params=modal)[0]

        out["icp_align_ms"] = timed(icp_align, args.repeats)
        et, er = error(icp["r"]["T_target_source"])
        out["icp_align_result"] = {"status": icp["r"]["status_name"], "iterations": icp["r"]["iterations"], "err_m": round(et, 4), "err_deg": round(er, 4)}

        def submap_e2e():
            a = merged(tp, tc).estimate_normals().estimate_fpfh(5.0)
            b = merged(sp, sc).estimate_normals().estimate_fpfh(5.0)
            r = gpu.estimate_pose_ransac(a, b)
            f = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, gpu.PointGridGPU(a, 1.05, ctx=ctx), b, 1.0, ctx=ctx)
            fine["r"] = gpu.align_vgicp([[f]], [r["T_target_source"]], params=dict(modal, max_iterations=20))[0]

        out["submap_e2e_ms"] = timed(submap_e2e, args.repeats)
        et, er = error(fine["r"]["T_target_source"])
        out["submap_e2e_err_m"] = round(et, 4)
        out["submap_e2e_err_deg"] = round(er, 4)
        ft, fs = tgt.fpfh()[:2000], src.fpfh()[:2000]
        t0 = time.perf_counter()
        gl.match(ft, fs)
        out["host_match_2k_ms"] = (time.perf_counter() - t0) * 1e3
        out["points_actual"] = [tgt.n, src.n]
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
