"""bench.py --workload preprocess: the per-frame preprocess of north_star (voxel downsample + k-NN + covariance estimation, ending
in the device cloud the VGICP factors read) on one HDL-32e-shaped 60 k-point frame, next to the CPU path.  Bench plumbing next to
bench.py (its cpu_baseline leg executes oracle/, which nothing under glim_b200/ may), not part of the drop-in surface."""
import time

import numpy as np


def cpu_preprocess(points, times, params, threads):
    """The reference's host pipeline with the tools available here: oracle voxel grid (the restatement of
    gtsam_points::voxelgrid_sampling), numpy gates + stable time sort, scipy cKDTree k-NN on all threads (gtsam_points::KdTree),
    oracle covariance estimation (OpenMP, all threads)."""
    from scipy.spatial import cKDTree

    from oracle import oracle

    pts, tms, _ = oracle.voxelgrid_sampling(points, params.downsample_resolution, times=times)
    sq = np.einsum("ij,ij->i", pts[:, :3], pts[:, :3])
    keep = np.nonzero((sq > params.distance_near_thresh**2) & (sq < params.distance_far_thresh**2) & np.isfinite(pts).all(axis=1))[0]
    keep = keep[np.argsort(tms[keep], kind="stable")]
    pts, tms = np.ascontiguousarray(pts[keep]), tms[keep]
    _, nb = cKDTree(pts[:, :3]).query(pts[:, :3], k=params.k_correspondences, workers=threads)
    normals, covs = oracle.covariance_estimate(pts, nb.astype(np.int32), num_threads=threads)
    return pts, tms, nb, normals, covs


def run(env, args, metric_name):
    import bench
    from glim_b200 import preprocess, synth

    torch = env.torch
    sampler = bench.ClockSampler(env.local_rank) if env.rank == 0 else None  # nvidia-smi clocks / throttle reasons during the timed region
    sc = synth.make_hall_scene()
    pts, tms = synth.scan(sc, "hdl32", synth.arc_trajectory(8)[2], synth.rng_for(32))
    n = len(pts)
    params = preprocess.CloudPreprocessorParams(distance_near_thresh=0.5, distance_far_thresh=100.0, downsample_resolution=0.1, k_correspondences=10)
    g = preprocess.FramePreprocessorGPU(params, env.ctx)
    pinned = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy() for a in (pts, tms)]

    def step_device():  # raw scan H2D from pinned memory, every stage on the device, result = the device cloud
        _, _, _, cloud = g.preprocess(0.0, pinned[1], pinned[0], host_outputs=False)
        return cloud

    def step_e2e():  # + the PreprocessedFrame fields and fp64 covariances / normals copied back to host arrays
        return g.preprocess(0.0, pinned[1], pinned[0], host_outputs=True)

    for _ in range(max(3, args.warmup)):
        step_device()
    steps = args.steps
    l0 = env.ctx.kernel_launches
    ms, _, t0, t1 = env.timed(step_device, steps, False)
    launches = env.ctx.kernel_launches - l0
    for _ in range(3):
        step_e2e()
    ems, _, _, t1e = env.timed(step_e2e, steps, False)
    clocks = None
    if sampler:
        time.sleep(0.15)
        sampler.stop()
        clocks = sampler.summary(t0, t1e)
    fr, normals, covs, cloud = step_e2e()
    m = fr.size()
    if args.dump_outputs and env.rank == 0:
        bench.dump_outputs(args.dump_outputs, {"points": fr.points, "times": fr.times, "neighbors": fr.neighbors.reshape(m, -1), "normals": normals, "covs": covs})
    # parity spot check against the CPU pipeline (indices exact, covariances 1e-9)
    threads = bench.host_threads()
    ref = cpu_preprocess(pts, tms, params, threads)
    ok = bool(m == len(ref[0]) and np.array_equal(fr.points, ref[0]) and np.array_equal(np.sort(fr.neighbors.reshape(m, -1), axis=1), np.sort(ref[2], axis=1)) and np.allclose(covs, ref[4], atol=1e-9))
    # the strongest CPU number: best over thread counts (all threads is not the fastest on a 128-thread host) and repetitions
    t_cpu = {}
    for th in sorted({t for t in (2, 8, 16, 32, 64, threads) if t <= threads}):
        best = 1e9
        for _ in range(2):
            tc = time.perf_counter()
            cpu_preprocess(pts, tms, params, th)
            best = min(best, time.perf_counter() - tc)
        t_cpu[th] = best
    threads = min(t_cpu, key=lambda t: t_cpu[t])
    cpu_ms = 1e3 * t_cpu[threads]
    peaks = bench.load_peaks()
    peak = float(peaks.get("hbm_gbs", bench.HBM_PEAK_GBS))
    # algorithmic bytes: raw point + time in (40 B), frame products out (point 32 + time 8 + k neighbours 4k + cov 128 + normal 32), device cloud planes (52 B)
    alg = n * 40 + m * (32 + 8 + 4 * params.k_correspondences + 128 + 32 + 52)
    per = ms / steps
    return {
        "metric": "per-frame preprocess throughput (voxel grid + range gate + time order + exact k-NN + covariances + device cloud)", "value": n / (per * 1e-3) / 1e6, "unit": "M raw points/s",
        "n_gpus": env.world, "steps": steps, "warmup": max(3, args.warmup), "ms_per_step": per, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": {"workload": "preprocess", "raw_points": n, "frame_points": int(m), "sensor": "HDL-32e-shaped, 60 000 rays", "downsample_resolution_m": 0.1, "k_correspondences": 10,
                   "note": "value: raw scan H2D from pinned memory + all stages on the device, result = the device cloud (no host products); e2e: the same + PreprocessedFrame fields, fp64 covariances and normals copied back"},
        "e2e": {"value": n / (ems / steps * 1e-3) / 1e6, "unit": "M raw points/s", "ms_per_step": ems / steps, "h2d_bytes_per_step": int(n * 40), "d2h_bytes_per_step": int(m * (32 + 8 + 4 * params.k_correspondences + 128 + 32))},
        "gpu_launches": int(launches), "clocks": clocks,
        "roofline": {"bound": "hbm", "achieved": alg / (per * 1e-3) / 1e9, "peak": peak, "unit": "GB/s", "frac": alg / (per * 1e-3) / 1e9 / peak, "traffic": None,
                     "note": "a 60 k-point frame is ~20 short launches (sorts, scans, hash build, k-NN, covariances, reorder): launch- and latency-bound, far from the HBM roofline by construction"},
        "cpu_baseline": {"value": n / (cpu_ms * 1e-3) / 1e6, "unit": "M raw points/s", "ms_per_frame": cpu_ms, "cores": threads, "kind": "port", "ms_by_threads": {str(t): round(1e3 * v, 2) for t, v in t_cpu.items()},
                         "sample": "the same frame: oracle voxel grid + numpy gates / time sort + scipy cKDTree k-NN (all threads) + oracle covariance estimation (OpenMP); best thread count, best of 2"},
        "speedup_vs_cpu": cpu_ms / per, "speedup_vs_cpu_e2e": cpu_ms / (ems / steps), "parity_check": {"ok": ok, "what": "points exact, neighbour sets exact, covariances 1e-9 vs the CPU pipeline"},
    }
