"""The incremental device voxel map (gb_voxelmap_insert) on GLIM's scan-to-map odometry loop (odometry_estimation_cpu.cpp:105-191):

  (a) insert: hdl32 frames (60 000 rays) along the M2 arc into maps at 0.2 / 0.4 m with LRU horizon 100 / clear cycle 10,
      rate 1 for the first five frames and 0.1 after (update_target); the first --warm frames grow the maps to a realistic
      size, then every further insert is timed;
  (b) insert of one 500 k-point MID-360-shaped frame at rate 1 into an empty 0.2 m map;
  (c) one odometry frame on the device -- two-level gb_vgicp_align (max_iterations 5) plus two inserts -- against the same
      frame with the maps kept on the host: the frame is sampled and transformed on the host, inserted into the oracle's
      GaussianVoxelMapCPU (go_cpumap), and the map is uploaded again as a cloud of its voxels and rebuilt with
      gb_voxelmap_build.  The uploaded content is the device map's voxel set, which is the host map's up to key rounding:
      the upload and build costs depend only on its size;
  (d) the GICP configuration GLIM ships (registration_type "GICP"): a 1.0 m device iVox grown over the warm frames, then per
      frame one device odometry frame -- gb_vgicp_align on one GICP factor (max_iterations 8) plus the insert at rate 0.1 --
      with the insert also reported on its own;
  (e) the CT configuration GLIM ships for LiDAR-only odometry (odometry_estimation_ct.cpp, config_odometry_ct.json):
      motion-distorted hdl32 frames (60 000 rays, 10 m/s, 0.6 rad/s; tests/ct_oracle.distorted_frame), a 1.0 m iVox (min_dist
      0.1, mode 1, LRU 200) grown over --ct-warm frames deskewed at ground truth, then per frame gb_cloud_add_times, the CT
      factor, gb_ct_gicp_align (default gb_ct_params, max_correspondence_distance 2.0), gb_ct_deskew and the insert of every
      deskewed point at X.  The twist prediction is host arithmetic outside the timed span; frames are uploaded beforehand.

Times are a host clock around synchronised calls, median over the timed frames.  Launch counts come from
gb_ctx_kernel_launches.  Every line carries the card's name and power limit, read in the same run.

    python scripts/bench_odometry.py [--warm 40] [--frames 20] [--ct-warm 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from glim_b200 import gpu, synth, workloads  # noqa: E402

CARD = "unknown"


def emit(**kv):
    print(json.dumps(dict(card=CARD, **kv)), flush=True)


def rate_of(k):
    return 1.0 if k < 5 else 0.1


def main():
    global CARD
    ap = argparse.ArgumentParser()
    ap.add_argument("--warm", type=int, default=40)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--ct-warm", type=int, default=10)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    CARD = card[0] if card else "unknown"
    ctx = gpu.Context(0)
    n_frames = args.warm + args.frames
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(n_frames)
    world0 = synth.inv_pose(traj[0])
    gt = [world0 @ T for T in traj]
    host = [workloads.make_scan(sc, "hdl32", traj[k], synth.rng_for(520, k), ctx=ctx, use_gpu=True) for k in range(n_frames)]
    clouds = [gpu.PointCloudGPU.clone(p, c, ctx=ctx) for p, c in host]

    # (a) inserts into maps of realistic size
    maps = [gpu.IncrementalVoxelMapGPU(r, lru_horizon=100, lru_clear_cycle=10, ctx=ctx) for r in (0.2, 0.4)]
    for k in range(args.warm):
        for m in maps:
            m.insert(clouds[k], gt[k], rate_of(k), seed=k)
    for li, m in enumerate(maps):
        ts, launches = [], []
        for k in range(args.warm, n_frames):
            l0 = ctx.kernel_launches
            t0 = time.perf_counter()
            m.insert(clouds[k], gt[k], 0.1, seed=k)
            ts.append(time.perf_counter() - t0)
            launches.append(ctx.kernel_launches - l0)
        emit(leg=f"insert/hdl32/{m.resolution}m", median_ms=round(float(np.median(ts)) * 1e3, 3), runs_ms=[round(t * 1e3, 3) for t in ts], kernel_launches=int(np.median(launches)),
             map_voxels=m.num_voxels, map_buckets=m.num_buckets, frame_points=int(clouds[-1].n), sampling_rate=0.1)

    # (b) one 500 k-point MID-360 frame at rate 1
    pts, cov = workloads.make_scan(sc, "mid360", traj[0], synth.rng_for(521), n_rays=500_000, ctx=ctx, use_gpu=True)
    big = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
    ts = []
    for rep in range(6):
        m = gpu.IncrementalVoxelMapGPU(0.2, ctx=ctx)
        l0 = ctx.kernel_launches
        t0 = time.perf_counter()
        m.insert(big, None, 1.0)
        ts.append(time.perf_counter() - t0)
        launches = ctx.kernel_launches - l0
    ts = ts[1:]  # the first call sizes the scratch arena
    emit(leg="insert/mid360_500k/0.2m/empty_map", median_ms=round(float(np.median(ts)) * 1e3, 3), runs_ms=[round(t * 1e3, 3) for t in ts], kernel_launches=launches,
         map_voxels=m.num_voxels, frame_points=int(big.n), sampling_rate=1.0)

    # (c) one odometry frame: device maps against host maps
    from oracle import oracle

    P = gpu.align_params(max_iterations=5)
    rng = synth.rng_for(522)
    cpumaps = []
    for r in (0.2, 0.4):
        cm = oracle.CpuMap(float(np.float32(r)))
        cm.set_lru_horizon(100, clear_cycle=10)
        cpumaps.append(cm)
    dev_ms, host_ms, dev_launches = [], [], []
    est = gt[args.warm - 1]
    for k in range(args.warm, n_frames):
        inc = synth.perturb(synth.inv_pose(gt[k - 1]) @ gt[k], rng, 0.01, 0.1)
        T0 = est @ inc
        # device: align + two inserts
        l0 = ctx.kernel_launches
        t0 = time.perf_counter()
        facs = [gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, clouds[k], ctx=ctx) for m in maps]
        T = gpu.align_vgicp([facs], [T0], params=P)[0]["T_target_source"]
        for m in maps:
            m.insert(clouds[k], T, 0.1, seed=k)
        dev_ms.append(time.perf_counter() - t0)
        dev_launches.append(ctx.kernel_launches - l0)
        est = T
        # host-kept maps: the same align on maps rebuilt from the host, then the host insert + rebuild + upload
        p, c = host[k]
        t0 = time.perf_counter()
        facs = [gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, clouds[k], ctx=ctx) for m in maps]
        gpu.align_vgicp([facs], [T0], params=P)
        keep = np.sort(np.random.default_rng(k).choice(len(p), int(len(p) * 0.1), replace=False))
        q = p[keep] @ T.T
        Ck = np.einsum("ij,njk,lk->nil", T, c[keep], T)
        for cm, m in zip(cpumaps, maps):
            cm.insert(q, np.ascontiguousarray(np.swapaxes(Ck, 1, 2)).reshape(-1, 16))
            _, _, vmean, vcov = m.download()
            V = len(vmean)
            vp = np.concatenate([vmean.astype(np.float64), np.ones((V, 1))], 1)
            vc = np.zeros((V, 4, 4))
            vc[:, :3, :3] = vcov.astype(np.float64)[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
            vcl = gpu.PointCloudGPU.clone(vp, vc, ctx=ctx)
            gpu.GaussianVoxelMapGPU(m.resolution, ctx=ctx).insert(vcl)
        host_ms.append(time.perf_counter() - t0)
    d, h = float(np.median(dev_ms[1:])) * 1e3, float(np.median(host_ms[1:])) * 1e3
    emit(leg="odometry_frame/device_maps", median_ms=round(d, 3), runs_ms=[round(t * 1e3, 3) for t in dev_ms], kernel_launches=int(np.median(dev_launches)))
    emit(leg="odometry_frame/host_maps", median_ms=round(h, 3), runs_ms=[round(t * 1e3, 3) for t in host_ms])
    emit(odometry_frame_speedup_device_vs_host=round(h / d, 2))

    # (d) the GICP configuration GLIM ships: a 1.0 m iVox (min_dist 0.1, mode 1, LRU 100 / 10) grown over the warm frames,
    #     then per frame one device odometry frame (GICP align, max_iterations 8, max_correspondence_distance 2.0, then the
    #     insert at rate 0.1), with the insert also timed on its own
    ivox = gpu.IVoxGPU(1.0, 0.1, 10, 1, 100, 10, ctx=ctx)
    for k in range(args.warm):
        ivox.insert(clouds[k], gt[k], rate_of(k), seed=k)
    ins_ms, ins_launches, frame_ms, frame_launches = [], [], [], []
    est = gt[args.warm - 1]
    rng = synth.rng_for(523)
    for k in range(args.warm, n_frames):
        inc = synth.perturb(synth.inv_pose(gt[k - 1]) @ gt[k], rng, 0.01, 0.1)
        l0 = ctx.kernel_launches
        t0 = time.perf_counter()
        fac = gpu.IntegratedGICPFactorGPU(np.eye(4), 0, ivox, clouds[k], 2.0, ctx=ctx)
        T = gpu.align_vgicp([[fac]], [est @ inc], params=gpu.align_params(max_iterations=8))[0]["T_target_source"]
        l1 = ctx.kernel_launches
        t1 = time.perf_counter()
        ivox.insert(clouds[k], T, 0.1, seed=k)
        t2 = time.perf_counter()
        ins_ms.append(t2 - t1)
        ins_launches.append(ctx.kernel_launches - l1)
        frame_ms.append(t2 - t0)
        frame_launches.append(ctx.kernel_launches - l0)
        est = T
    emit(leg="gicp/insert/hdl32/1.0m", median_ms=round(float(np.median(ins_ms[1:])) * 1e3, 3), runs_ms=[round(t * 1e3, 3) for t in ins_ms],
         kernel_launches=int(np.median(ins_launches)), frame_points=int(clouds[-1].n), sampling_rate=0.1)
    emit(leg="gicp/odometry_frame/device_ivox", median_ms=round(float(np.median(frame_ms[1:])) * 1e3, 3), runs_ms=[round(t * 1e3, 3) for t in frame_ms],
         kernel_launches=int(np.median(frame_launches)), ivox_voxels=ivox.num_voxels, ivox_points=ivox.num_points)

    # (e) the CT configuration: per frame add_times + CT factor + gb_ct_gicp_align + gb_ct_deskew + insert
    from tests import ct_oracle as co

    n_ct = args.ct_warm + args.frames
    frames = []
    for k in range(n_ct):
        pts, tms = co.distorted_frame(sc, k, 32 * 1875, synth.rng_for(524, k))
        nb = synth.knn(pts, 10)
        cov = synth.plane_covariances(pts, nb)[1]
        frames.append((gpu.PointCloudGPU.clone(pts, cov, ctx=ctx), nb, tms))
    ivox = gpu.IVoxGPU(1.0, 0.1, 10, 1, 200, 10, ctx=ctx)
    ms, launches, iters = [], [], []
    X_last = Y_last = span = None
    for k, (cloud, nb, tms) in enumerate(frames):
        t_first, t_last = 0.1 * k + tms[0], 0.1 * k + tms[co.time_table(tms)[0][-2]]  # t_0 and t_{B-1}
        if k < args.ct_warm:
            X, Y = co.gt_pose(t_first), co.gt_pose(t_last)
            cloud.add_times(tms)
            ivox.insert(gpu.deskew_ct(cloud, X, Y, nb, 10, host_outputs=False)[3], X, 1.0, seed=k)
        else:
            v = co.motion(X_last, Y_last) / (span[1] - span[0])
            X0 = Y_last @ co.se3_exp(v * (t_first - span[1]))
            Y0 = X0 @ co.se3_exp(v * (t_last - t_first))
            l0 = ctx.kernel_launches
            t0 = time.perf_counter()
            cloud.add_times(tms)
            fac = gpu.IntegratedCT_GICPFactorGPU(0, 1, ivox, cloud, 2.0, ctx=ctx)
            r = gpu.align_ct_gicp([fac], [X0], [Y0], [Y_last])[0]
            X, Y = r["X"], r["Y"]
            ivox.insert(gpu.deskew_ct(cloud, X, Y, nb, 10, host_outputs=False)[3], X, 1.0, seed=k)
            ms.append(time.perf_counter() - t0)
            launches.append(ctx.kernel_launches - l0)
            iters.append(r["iterations"])
        X_last, Y_last, span = X, Y, (t_first, t_last)
    emit(leg="ct/odometry_frame/device_ivox", median_ms=round(float(np.median(ms[1:])) * 1e3, 3), runs_ms=[round(t * 1e3, 3) for t in ms],
         kernel_launches=int(np.median(launches)), lm_iterations=int(np.median(iters)), frame_points=int(frames[-1][0].n), ivox_voxels=ivox.num_voxels,
         ivox_points=ivox.num_points)


if __name__ == "__main__":
    main()
