#!/usr/bin/env python
"""bench.py -- VGICP linearize throughput (M points.factors / s) on H100, next to the CPU path.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload NAME] [--impl reference] [--verify K] [--dump-outputs DIR]

A "step" is one relinearization pass of the hot path over the workload's whole factor set (every
NonlinearFactorSetGPU::linearize call the workload contains, back to back).  Default workload:
global_mapping_gpu (BASELINE.json configs[3]: 256 submaps x 50 k points, 0.5 / 1.0 m voxels), the one
configuration BASELINE.json defines at 1 / 2 / 4 / 8 GPUs -- total work is fixed, the pair list is sharded
over the ranks and the per-pair Hessian slab is exchanged ("scaling": "strong").  The other BASELINE
configurations (single_pair, odometry_gpu, sub_mapping_gpu, livox_stress) run with --workload; the default
N = 1 line also carries a short measurement of each of them in `roofline_by_workload`.  `--workload preprocess`
times the per-frame preprocess (voxel grid -> k-NN -> covariances -> device cloud) instead.

value      whole-job points.factors / s, inputs resident in HBM, CUDA events on the launching stream, max over ranks
e2e        the same through the C-ABI with HOST buffers: poses H2D from pinned memory + launch (+ exchange) + the result
           (pair slab for the sharded global-mapping sweep, gb_linearized6 records otherwise) D2H, every step
roofline   algorithmic bytes per launch (SURVEY 8(d) B_sweep, from gb_sweep_stats) / measured launch duration vs
           MEASURED_PEAKS.json hbm_gbs (else the H100 SXM data sheet's 3.35 TB/s); next to it the miss-aware byte count
parity_check   --verify K (default 4): after the timed region K random pairs are recomputed with the fp64 CPU oracle and
           compared with the rows of the exchanged pair slab (at N > 1 that includes rows produced by other ranks)
--impl reference   the CPU path (oracle port of gtsam_points::IntegratedVGICPFactor, fp64, all host threads) on a
           bounded sample of the same workload.  The only place besides cpu_baseline / parity_check where bench.py
           executes oracle/.  Builds its sample on the host (numpy / scipy): libglim_b200.so is not loaded.
--dump-outputs DIR   what the last timed step computed (pair slab or records; the frame for preprocess) as DIR/<name>.npy;
           inputs are seeded, so two builds run with the same arguments can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "VGICP linearize throughput"
UNIT = "M points*factors/s"
WORKLOADS = ["single_pair", "odometry_gpu", "sub_mapping_gpu", "global_mapping_gpu", "livox_stress"]
L2_BYTES = 50e6  # H100: inputs that fit are re-read from L2 across steps, so the L2 is flushed between timed steps
HBM_PEAK_GBS = 3350.0  # H100 SXM data sheet (HBM3), used when MEASURED_PEAKS.json gives no measured figure
DUMP_BYTES = 64_000_000


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="global_mapping_gpu", choices=WORKLOADS + ["preprocess"])
    ap.add_argument("--scale", type=float, default=1.0, help="shrink the workload (debug only; a scaled run is not a bench value)")
    ap.add_argument("--collective", default="fused", choices=["fused", "nccl"], help="multi-GPU result exchange: rows pushed into peer memory by the sweep kernel (fused) or fp32 atomics + NCCL all-reduce (nccl)")
    ap.add_argument("--verify", type=int, default=4, help="pairs re-computed with the CPU oracle after the timed region and compared with the exchanged slab rows (0 = off)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-other-workloads", action="store_true", help="skip roofline_by_workload in the default N = 1 line")
    ap.add_argument("--cpu-seconds", type=float, default=12.0, help="CPU work budget for the cpu_baseline sample")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's outputs to DIR/<name>.npy")
    return ap.parse_args()


def host_threads():
    """Hardware threads this process may use.  NOT omp_get_max_threads(): torchrun exports OMP_NUM_THREADS=1, which made
    round 1's N > 1 reference arm single threaded."""
    try:
        return max(1, len(os.sched_getaffinity(0)))
    except Exception:
        return max(1, os.cpu_count() or 1)


def cpu_model():
    """CPU model string of the host (SURVEY 8(d): state the host the CPU arm ran on, never assume it)."""
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.lower().startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except Exception:
        pass
    return None


# --------------------------------------------------------------------------------------------------------------
# workload construction (identical on every rank: seeded)
# --------------------------------------------------------------------------------------------------------------
def workload_args(name, scale):
    s = scale
    if name == "global_mapping_gpu":
        from glim_b200 import workloads

        n = max(8, int(round(256 * s)) // 4 * 4)
        return dict(n_submaps=n, laps=4, side=300.0, n_rays=None if s >= 1 else 64 * max(64, int(2048 * s)), params=workloads.GlobalMappingParams(submap_target_num_points=max(2000, int(50000 * s))))
    if name == "odometry_gpu":
        n = max(6, int(round(64 * s)))
        return dict(n_frames=n, first_bench_frame=max(1, n // 4), n_rays=None if s >= 1 else 32 * max(64, int(1875 * s)))
    if name == "sub_mapping_gpu":
        return dict(n_keyframes=max(3, int(round(15 * s))), n_rays=None if s >= 1 else 64 * max(64, int(2048 * s)))
    if name == "single_pair":
        return dict(n_rays=None if s >= 1 else 64 * max(64, int(1563 * s)))
    if name == "livox_stress":
        return dict(n_rays=max(5000, int(500_000 * s)))
    raise ValueError(name)


def build_workload(name, ctx, scale, use_gpu):
    from glim_b200 import workloads

    return workloads.BUILDERS[name](ctx, use_gpu=use_gpu, **workload_args(name, scale))


def workload_config(name, w, extra):
    cfg = {
        "workload": name,
        "clouds": len(w.host_clouds),
        "points_per_cloud": int(np.median([len(c[0]) for c in w.host_clouds if c is not None])),
        "voxel_resolutions_m": w.resolutions,
        "factor_sets_per_step": len(w.sets),
        "factors_per_step": int(sum(len(s.factors) for s in w.sets)),
        "point_factors_per_step": int(w.point_factors),
        "l2": "inputs larger than L2 (no flush)" if sum(len(c[0]) for c in w.host_clouds if c is not None) * 36 > L2_BYTES else "L2 flushed between steps (256 MB write)",
    }
    cfg.update({k: v for k, v in w.notes.items() if not k.startswith("_")})
    cfg.update(extra)
    return cfg


# --------------------------------------------------------------------------------------------------------------
# clocks
# --------------------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, device):
        self.samples = []
        self.proc = None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100", "-i", str(device)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.samples.append((time.monotonic(), line.strip()))

    def stop(self):
        if self.proc:
            self.proc.terminate()

    def summary(self, t0, t1):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "note": "nvidia-smi not available"}
        sel = [l for (t, l) in self.samples if t0 <= t <= t1] or [l for (_, l) in self.samples[-3:]]
        mhz, mx, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for l in sel:
            f = [x.strip() for x in l.split(",")]
            try:
                mhz.append(float(f[0]))
                mx = float(f[1])
            except Exception:
                continue
            for nm, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": float(np.median(mhz)) if mhz else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(mhz)}


# --------------------------------------------------------------------------------------------------------------
# CPU path (oracle port of gtsam_points::IntegratedVGICPFactor), used by cpu_baseline and --impl reference
# --------------------------------------------------------------------------------------------------------------
def c16(cov):
    return np.ascontiguousarray(np.swapaxes(cov, 1, 2)).reshape(len(cov), 16)


class CpuSample:
    """A bounded sample of the workload for the CPU path: factors of ONE source cloud (one 'insert_submap' worth of factors
    in global mapping, one frame's factors in odometry), capped at `max_factors`.  One source cloud re-used by all its
    factors is cache-friendly for the CPU -- a conservative choice for the GPU / CPU ratio."""

    def __init__(self, name, resolutions, host_clouds, picked, desc_tail=""):
        """picked: list of (target, level, source, delta 4x4) sharing one source."""
        from oracle import oracle

        self.oracle = oracle
        self.threads = host_threads()
        self.items = []
        maps = {}
        src = picked[0][2]
        pts, cov = host_clouds[src]
        src16 = c16(cov)
        for (t, lvl, s, delta) in picked:
            assert s == src
            if (t, lvl) not in maps:
                m = oracle.CpuMap(resolutions[lvl])
                tp, tc = host_clouds[t]
                m.insert(tp, c16(tc))
                maps[(t, lvl)] = m
            fac = oracle.CpuFactor(maps[(t, lvl)], pts, src16, num_threads=self.threads)
            self.items.append((fac, oracle.pose_colmajor(delta)))
        self.point_factors = len(pts) * len(self.items)
        self.out = np.zeros(122)
        self.desc = f"{len(self.items)} factors x {len(pts)} source points of one {name} source cloud{desc_tail}"

    @staticmethod
    def from_workload(w, max_factors=16):
        fset = w.sets[len(w.sets) // 2]
        by_src = {}
        for k, f in enumerate(fset.factors):
            by_src.setdefault(f.source, []).append(k)
        src = max(by_src, key=lambda s: (len(by_src[s]), -s))
        idx = by_src[src][:max_factors]
        picked = [(fset.factors[k].target, fset.factors[k].level, src, fset.deltas[k]) for k in idx]
        return CpuSample(w.name, w.resolutions, w.host_clouds, picked, f" (the source with most factors, first {max_factors})")

    def set_threads(self, t):
        for fac, _ in self.items:
            fac.num_threads = t

    def run_once(self):
        for fac, Tc in self.items:
            fac.linearize_raw(Tc, self.out)


def cpu_thread_sweep(s, seconds):
    """Time the sample at the shipped thread count (2, config_odometry_cpu.json:36) and at 8 / 16 / 32 / all host
    threads; the baseline reported is the FASTEST of them (OpenMP fork/join can make 'all threads' slower on small
    clouds -- the strongest CPU number is the honest one to compare against)."""
    allt = s.threads
    cands = sorted({t for t in (2, 8, 16, 32, allt) if t <= allt})
    per = {}
    budget = seconds / len(cands)
    s.spread = {}
    for t in cands:
        s.set_threads(t)
        s.run_once()
        t0 = time.perf_counter()
        reps, laps, last = 0, [], t0
        while True:
            s.run_once()
            reps += 1
            now = time.perf_counter()
            laps.append(now - last)
            last = now
            el = now - t0
            if el >= budget or reps >= 100000:
                break
        per[t] = s.point_factors * reps / el / 1e6
        q = np.percentile(np.asarray(laps), [90, 50, 10])  # slow laps = low throughput: p10 of the throughput is the p90 lap
        s.spread[t] = [round(float(s.point_factors / x / 1e6), 2) for x in q]
    best = max(per, key=lambda t: per[t])
    s.set_threads(best)
    return best, per


def cpu_baseline(w, seconds):
    s = CpuSample.from_workload(w)
    best, per = cpu_thread_sweep(s, seconds)
    return {"value": per[best], "unit": UNIT, "cores": best, "kind": "port", "host_threads_available": s.threads, "cpu_model": cpu_model(),
            "by_threads": {str(t): round(v, 2) for t, v in per.items()}, "p10_median_p90_at_best": s.spread.get(best),
            "sample": f"{s.desc}; ~{seconds:.0f} s of CPU work split over thread counts {sorted(per)}; fp64, update_correspondences + evaluate (OpenMP); value = fastest thread count ({best})"}


def reference_sample_global_mapping(scale, max_factors=16):
    """The reference arm's sample for global_mapping_gpu, built WITHOUT libglim_b200 and without a GPU: one source submap
    (a fixed index on the third lap) and the first `max_factors` factors GlobalMapping::insert_submap would create for it
    (candidates in ascending index within max_implicit_loop_distance, overlap gate evaluated by the host twin of its
    definition) -- only the clouds that are needed are generated (numpy ray casting, scipy k-NN, oracle covariances)."""
    from glim_b200 import synth, workloads

    a = workload_args("global_mapping_gpu", scale)
    p = a["params"]
    n = a["n_submaps"]
    w = workloads.Workload("global_mapping_gpu", None)
    sc = synth.make_blocks_scene()
    traj = synth.loop_trajectory(n // a["laps"], a["laps"], side=a["side"])
    w.poses = list(traj)
    w.host_clouds = [None] * n
    w.resolutions = [p.submap_voxel_resolution * p.submap_voxelmap_scaling_factor**l for l in range(p.submap_voxelmap_levels)]

    def need(i):
        if w.host_clouds[i] is None:
            w.host_clouds[i] = workloads.make_scan(sc, "os1_64", traj[i], synth.rng_for(401, i), n_rays=a["n_rays"], max_points=p.submap_target_num_points, ctx=None, use_gpu=False)

    picked = []
    # the fixed source submap of the full-size workload; a scaled-down (debug) layout may give it no partner: try later ones
    for cur in [n // 2 + n // 8] + list(range(n - 1, 0, -1)):
        need(cur)
        rng = synth.rng_for(402)
        for i in range(cur):
            if np.sum((traj[i][:3, 3] - traj[cur][:3, 3]) ** 2) > p.max_implicit_loop_distance**2:
                continue
            need(i)
            gt = w.gt_delta(i, cur)
            if w.overlap([i], len(w.resolutions) - 1, cur, [gt]) < p.min_implicit_loop_overlap:
                continue
            delta = synth.perturb(gt, rng, 0.02, 0.2)
            for l in range(p.submap_voxelmap_levels):
                picked.append((i, l, cur, delta))
            if len(picked) >= max_factors:
                break
        if picked:
            break
    if not picked:
        raise SystemExit("reference arm: the scaled layout has no overlapping submap pair (use a larger --scale)")
    s = CpuSample("global_mapping_gpu", w.resolutions, w.host_clouds, picked[:max_factors], f" (submap {cur}; its first {max_factors} factors in GlobalMapping::insert_submap order)")
    w.host_clouds = [c for c in w.host_clouds if c is not None]
    return s, w


def run_reference(args, rank):
    """--impl reference: the CPU VGICP path on the box's host cores, bounded sample of the same workload.  Nothing of
    libglim_b200 is loaded: the sample is built on the host."""
    if rank != 0:
        return
    t_build = time.perf_counter()
    if args.workload == "global_mapping_gpu":
        s, w = reference_sample_global_mapping(args.scale)
        cfg = {"workload": args.workload, "clouds_generated_for_the_sample": len(w.host_clouds), "points_per_cloud": int(np.median([len(c[0]) for c in w.host_clouds])),
               "voxel_resolutions_m": w.resolutions, "reference_step": s.desc}
    else:
        w = build_workload(args.workload, None, args.scale, use_gpu=False)
        s = CpuSample.from_workload(w)
        cfg = workload_config(args.workload, w, {"reference_step": s.desc})
    cfg["sample_build_seconds"] = round(time.perf_counter() - t_build, 1)
    cfg["same_config"] = "bounded sample: the factors of ONE source cloud of the workload (cache-friendly for the CPU), not the whole factor set"
    best, per = cpu_thread_sweep(s, min(10.0, args.cpu_seconds))  # pick the fastest thread count for this host, then time K steps with it
    for _ in range(max(1, min(args.warmup, 3))):
        s.run_once()
    # bound the run: at most ~60 s of CPU work
    t_probe = time.perf_counter()
    s.run_once()
    per_step = time.perf_counter() - t_probe
    steps = max(1, min(args.steps, int(60.0 / max(per_step, 1e-6))))
    t0 = time.perf_counter()
    for _ in range(steps):
        s.run_once()
    el = time.perf_counter() - t0
    val = s.point_factors * steps / el / 1e6
    line = {
        "impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": steps, "warmup": args.warmup,
        "ms_per_step": el / steps * 1e3, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": cfg,
        "cpu_baseline": {"value": val, "unit": UNIT, "cores": best, "kind": "port", "host_threads_available": s.threads, "cpu_model": cpu_model(), "omp_num_threads_env": os.environ.get("OMP_NUM_THREADS"),
                         "by_threads": {str(t): round(v, 2) for t, v in per.items()}, "p10_median_p90_at_best": s.spread.get(best),
                         "sample": s.desc + f"; one step = one pass over the sample with the fastest thread count ({best}); thread count from sched_getaffinity, OMP_NUM_THREADS ignored"},
        "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "note": "GLIM's own CPU path (gtsam_points::IntegratedVGICPFactor) cannot be built here (GTSAM / gtsam_points / Eigen absent); this is the oracle port, fp64, all host threads",
    }
    print(json.dumps(line))


# --------------------------------------------------------------------------------------------------------------
# our arm
# --------------------------------------------------------------------------------------------------------------
class Env:
    """torch / distributed / stream plumbing of one rank."""

    def __init__(self):
        import torch
        import torch.distributed as dist

        from glim_b200 import gpu

        self.torch, self.dist = torch, dist
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        if not torch.cuda.is_available():
            raise SystemExit("bench.py needs an H100: no CUDA device visible (there is no CPU fallback)")
        torch.cuda.set_device(self.local_rank)
        if self.world > 1:
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            dist.init_process_group("nccl", device_id=torch.device("cuda", self.local_rank))
        self.stream = torch.cuda.Stream()
        torch.cuda.set_stream(self.stream)
        self.ctx = gpu.Context(self.local_rank, cuda_stream=self.stream.cuda_stream)
        self.dev = f"cuda:{self.local_rank}"
        self.flush = None

    def flush_buf(self):
        if self.flush is None:
            self.flush = self.torch.empty(256 << 20, dtype=self.torch.uint8, device=self.dev)
        return self.flush

    def timed(self, fn, steps, flush_l2):
        """K steps bracketed by barrier + synchronize; device time from CUDA events on the launching stream; max over ranks.
        Returns (max-over-ranks ms, this rank's ms, t0, t1)."""
        torch, dist = self.torch, self.dist
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)] if flush_l2 else None
        if self.world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        t0 = time.monotonic()
        if flush_l2:
            fl = self.flush_buf()
            for a, b in ev:
                fl.fill_(1)
                a.record(self.stream)
                fn()
                b.record(self.stream)
            torch.cuda.synchronize()
            ms = sum(a.elapsed_time(b) for a, b in ev)
        else:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(self.stream)
            for _ in range(steps):
                fn()
            b.record(self.stream)
            torch.cuda.synchronize()
            ms = a.elapsed_time(b)
        if self.world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        t1 = time.monotonic()
        mine = ms
        if self.world > 1:
            t = torch.tensor([ms], dtype=torch.float64, device=self.dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms, mine, t0, t1

    def gather_floats(self, x):
        if self.world == 1:
            return [float(x)]
        t = self.torch.tensor([x], dtype=self.torch.float64, device=self.dev)
        outs = [self.torch.empty_like(t) for _ in range(self.world)]
        self.dist.all_gather(outs, t)
        return [float(o.item()) for o in outs]

    def exchange(self, handle: bytes):
        t = self.torch.tensor(list(handle), dtype=self.torch.uint8, device=self.dev)
        outs = [self.torch.empty_like(t) for _ in range(self.world)]
        self.dist.all_gather(outs, t)
        return [bytes(o.cpu().numpy().tobytes()) for o in outs]


def load_peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        return {}


def dump_outputs(out_dir, arrays):
    """--dump-outputs: every array as out_dir/<name>.npy, float32 kept, anything else as float64; an array larger than its share of
    DUMP_BYTES is cut to a fixed, seeded sample of its rows."""
    os.makedirs(out_dir, exist_ok=True)
    share = DUMP_BYTES // max(1, len(arrays))
    for name, a in arrays.items():
        a = np.atleast_1d(np.asarray(a))
        a = a.astype(np.float32 if a.dtype == np.float32 else np.float64)
        if a.nbytes > share:
            keep = max(1, share // (a.nbytes // len(a)))
            a = a[np.sort(np.random.default_rng(0).choice(len(a), keep, replace=False))]
        np.save(os.path.join(out_dir, f"{name}.npy"), a)


def roofline_of(name, my_bytes, miss_bytes, k_launches, kernel_ms_per_launch, world, scale):
    peaks = load_peaks()
    peak = float(peaks.get("hbm_gbs", HBM_PEAK_GBS))
    achieved = my_bytes / max(1, k_launches) / (kernel_ms_per_launch * 1e-3) / 1e9
    r = {"bound": "hbm", "kernel": "k_vgicp_sweep3 / k_vgicp_sweep5 <LINEARIZE>", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
         "peak_source": "MEASURED_PEAKS.json hbm_gbs (measured)" if peaks else f"H100 SXM data sheet, {HBM_PEAK_GBS:.0f} GB/s",
         "algorithmic_bytes_per_launch": my_bytes / max(1, k_launches), "launch_ms": kernel_ms_per_launch,
         # what the kernel must actually fetch: a miss reads 16 B of the point, not 48
         "miss_aware_bytes_per_launch": miss_bytes / max(1, k_launches) if miss_bytes is not None else None,
         "miss_aware_frac": (miss_bytes / max(1, k_launches) / (kernel_ms_per_launch * 1e-3) / 1e9 / peak) if miss_bytes is not None else None,
         "note": "frac = SURVEY 8(d) B_sweep (48 B per point.factor + 48 B per target voxel + 16 B per bucket + 552 B per factor, no credit for reuse) / CUDA-event launch time / peak: the CONTRACT figure, not a DRAM utilisation -- clouds shared by consecutive factors are served from L2 and misses read 16 B, so B_sweep can exceed what HBM delivers (frac > 1 is possible)"}
    return r


def measure_simple(env, name, w, steps, warmup):
    """Single-GPU measurement of a non-sharded workload: device value, kernel-only launch time, roofline, e2e."""
    from glim_b200 import gpu

    ctx = env.ctx
    sweeps = []
    for fset in w.sets:
        sw = gpu.Sweep(ctx, w.gpu_factors(fset))
        sw.set_poses(fset.deltas)
        sw._deltas = fset.deltas
        sweeps.append(sw)
    ctx.synchronize()
    sizes = [len(c[0]) for c in w.host_clouds]
    small = sum(sizes) * 36 <= L2_BYTES
    my_pf = sum(sw.point_factors for sw in sweeps)
    my_bytes = sum(sw.algorithmic_bytes for sw in sweeps)

    def step():
        for sw in sweeps:
            sw.launch()

    step()
    for sw in sweeps:  # a real caller fetches every linearization: the first fetch lets small sweeps size their items from measured inlier fractions
        sw.fetch()
    for _ in range(max(3, warmup)):
        step()
    l0 = ctx.kernel_launches
    ms, _, t0, t1 = env.timed(step, steps, small)
    launches = ctx.kernel_launches - l0
    # inlier counts (for the miss-aware byte figure)
    inl = sum(float(sw.fetch()["num_inliers"].sum()) for sw in sweeps)
    miss_bytes = my_bytes - 32.0 * (my_pf - inl)
    kms = ms / steps / len(sweeps)

    from glim_b200.capi import pose16

    for sw in sweeps:
        sw._p16, sw._out = pose16(sw._deltas), np.zeros(sw.F, gpu.LIN_DTYPE)

    def step_e2e():
        for sw in sweeps:
            sw.linearize_raw(sw._p16, sw._out)  # gb_sweep_linearize with host buffers: poses H2D + launch + records D2H (one CUDA-graph launch for small sweeps)

    for _ in range(3):
        step_e2e()
    e_steps = steps
    ems, _, _, _ = env.timed(step_e2e, e_steps, False)
    F = sum(sw.F for sw in sweeps)
    out = {
        "value": my_pf / (ms / steps * 1e-3) / 1e6, "ms_per_step": ms / steps, "launches_per_step": len(sweeps), "gpu_launches": int(launches),
        "roofline": roofline_of(name, my_bytes, miss_bytes, len(sweeps), kms, 1, 1.0),
        "e2e": {"value": my_pf / (ems / e_steps * 1e-3) / 1e6, "unit": UNIT, "h2d_bytes_per_step": F * 128, "d2h_bytes_per_step": F * 976, "ms_per_step": ems / e_steps},
        "inlier_fraction": inl / max(1, my_pf), "t0": t0, "t1": t1,
    }
    del sweeps
    return out


def parity_check(env, w, fset, peers_row_fetch, K, seed=7):
    """K random pairs of the factor set: recompute their factors with the fp64 oracle on the device-layout inputs and
    compare with the fp32 slab rows (sum of the pair's levels) the sweep exchanged.  rank 0 only."""
    from glim_b200 import multi_gpu
    from oracle import oracle

    rows = peers_row_fetch()
    pairs = sorted({f.pair for f in fset.factors})
    rng = np.random.default_rng(seed)
    chosen = sorted(rng.choice(len(pairs), min(K, len(pairs)), replace=False).tolist())
    packed, maps = {}, {}
    max_h, max_b, max_b_raw, max_e, exact = 0.0, 0.0, 0.0, 0.0, True
    for pi in chosen:
        pair = pairs[pi]
        ks = [k for k, f in enumerate(fset.factors) if f.pair == pair]
        tot = np.zeros(122)
        for k in ks:
            f = fset.factors[k]
            for c in (f.target, f.source):
                if c not in packed:
                    packed[c] = oracle.pack_cloud(w.host_clouds[c][0], c16(w.host_clouds[c][1]))
            if (f.target, f.level) not in maps:
                maps[(f.target, f.level)] = oracle.GpuMap(*packed[f.target], w.resolutions[f.level])
            ref, _ = oracle.linearize_gpumap(maps[(f.target, f.level)], *packed[f.source], fset.deltas[k], normals=w.host_normals[f.source] if w.surface_validation else None)
            tot += ref
        ref = oracle.split122(tot)
        got = multi_gpu.unpack_slab_row(rows[pair])
        exact = exact and (got["num_inliers"] == ref["num_inliers"])
        for kk in ("H_tt", "H_ss", "H_ts"):
            max_h = max(max_h, float(np.linalg.norm(got[kk] - ref[kk]) / max(np.linalg.norm(ref[kk]), 1e-300)))
        for kk, hk in (("b_t", "H_tt"), ("b_s", "H_ss")):
            d = float(np.linalg.norm(got[kk] - ref[kk]))
            max_b_raw = max(max_b_raw, d / max(np.linalg.norm(ref[kk]), 1e-300))
            max_b = max(max_b, d / max(np.linalg.norm(ref[kk]), 0.1 * np.sqrt(np.trace(ref[hk]) * max(ref["error"], 1e-30))))
        max_e = max(max_e, abs(got["error"] - ref["error"]) / max(abs(ref["error"]), 1e-300))
    ok = bool(exact and max_h < 1e-4 and max_b < 1e-4 and max_e < 1e-4)
    return {"pairs": len(chosen), "pair_ids": [int(pairs[i]) for i in chosen], "max_rel_H": max_h, "max_rel_b": max_b, "max_rel_b_raw": max_b_raw, "max_rel_error": max_e,
            "inliers_exact": bool(exact), "tolerance": 1e-4, "ok": ok,
            "what": "fp32 slab rows after the exchange vs fp64 oracle (go_vgicp_linearize_gpumap) summed over the pair's levels; max_rel_b is relative to max(|b|, 0.1 sqrt(tr(H) error)) (a cancelling sum), max_rel_b_raw to |b| itself"}


def run_preprocess(args, env):
    """--workload preprocess: one 60 k-point HDL-32e-shaped frame through the per-frame preprocess."""
    import bench_preprocess

    line = bench_preprocess.run(env, args, METRIC)
    if env.rank == 0:
        print(json.dumps(line))


def main():
    args = parse_args()
    if args.impl == "reference":
        run_reference(args, int(os.environ.get("RANK", "0")))
        return

    env = Env()
    torch, dist = env.torch, env.dist
    rank, world, local_rank, ctx = env.rank, env.world, env.local_rank, env.ctx
    from glim_b200 import gpu, multi_gpu
    from glim_b200.capi import GB_SLAB_STRIDE

    if args.workload == "preprocess":
        run_preprocess(args, env)
        return

    sampler = ClockSampler(local_rank) if rank == 0 else None  # started early: nvidia-smi takes ~1 s to produce its first line
    t_build = time.perf_counter()
    w = build_workload(args.workload, ctx, args.scale, use_gpu=True)
    build_s = time.perf_counter() - t_build

    # ---- shard: pairs over ranks for global mapping; every other workload is a single online stream (replicas only) ----
    sharded = args.workload == "global_mapping_gpu"
    sizes = [len(c[0]) for c in w.host_clouds]
    fused = args.collective == "fused"

    def make_sweeps(inliers_by_set=None, reuse_peers=None, scale_by_set=None):
        """Partition every factor set over the ranks and prepare this rank's sweeps.  inliers_by_set: measured inlier counts per
        factor (from a calibration sweep) for the cost-balanced partition; None -> the overlap estimate of the gate."""
        sweeps, slabs, peers, my_pf, my_bytes, all_pf = [], [], [], 0, 0, 0
        for si, fset in enumerate(w.sets):
            if sharded:
                f_rank, _ = multi_gpu.shard_factors(fset.factors, sizes, world, pair_cost=w.notes.get("_pair_overlap"),
                                                    factor_inliers=None if inliers_by_set is None else inliers_by_set[si],
                                                    factor_scale=None if scale_by_set is None else scale_by_set[si])
                mine = [k for k in range(len(fset.factors)) if f_rank[k] == rank]
            else:
                mine = list(range(len(fset.factors)))
            sub = type(fset)([fset.factors[k] for k in mine], fset.deltas[mine] if len(mine) else np.zeros((0, 4, 4)))
            gf = w.gpu_factors(sub)
            num_pairs = max((f.pair for f in fset.factors), default=-1) + 1
            sw = gpu.Sweep(ctx, gf, pair_index=[f.pair for f in sub.factors])
            slab = None
            ps = None
            if sharded and fused:
                ps = reuse_peers[si] if reuse_peers is not None else gpu.PeerSlab(ctx, max(1, num_pairs), world, rank, env.exchange)
                sw.attach_peer_slab(ps)
            elif sharded:
                slab = torch.zeros((max(1, num_pairs), GB_SLAB_STRIDE), dtype=torch.float32, device=env.dev)
                sw.attach_slab(slab.data_ptr(), max(1, num_pairs))
            peers.append(ps)
            sw.set_poses(sub.deltas)
            sw._sub = sub
            sw._mine = mine
            sw._f_rank = f_rank if sharded else None
            sweeps.append(sw)
            slabs.append(slab)
            my_pf += sw.point_factors
            my_bytes += sw.algorithmic_bytes
            all_pf += sum(sizes[f.source] for f in fset.factors)
        return sweeps, slabs, peers, my_pf, my_bytes, all_pf

    sweeps, slabs, peers, my_pf, my_bytes, all_pf = make_sweeps()
    calibrated = False
    feedback_history = []
    if sharded and world > 1:
        # Calibration sweep: a relinearizing back-end knows every factor's inlier count from its previous sweep; use it to
        # balance the partition by measured cost instead of the gate's overlap estimate, then rebuild this rank's sweeps.
        inl = []
        for si, (sw, ps) in enumerate(zip(sweeps, peers)):
            sw.launch()
            if fused:
                ps.signal_wait()
            rec = sw.fetch()
            full = torch.zeros(len(w.sets[si].factors), dtype=torch.float64, device=env.dev)
            if len(sw._mine):
                full[torch.tensor(sw._mine, device=full.device)] = torch.from_numpy(np.ascontiguousarray(rec["num_inliers"])).to(full.device)
            dist.all_reduce(full, op=dist.ReduceOp.SUM)
            inl.append(full.cpu().numpy())
        old = sweeps
        sweeps, slabs, peers, my_pf, my_bytes, all_pf = make_sweeps(inl, reuse_peers=peers if fused else None)
        del old
        calibrated = True
        # Time feedback (<= 2 rounds): every rank times its own kernel (CUDA events, all ranks sweeping at once as in a step);
        # the factors a rank held get their weight scaled by t_rank / mean(t) and the list is cut again.  A back-end that
        # re-linearizes the same factor set every solver iteration gets these times for free.
        scale = [np.ones(len(fs.factors)) for fs in w.sets]
        for _ in range(2):
            def kernels_only():
                for sw in sweeps:
                    sw.launch()
            for _w in range(3):
                kernels_only()
            _, t_mine, _, _ = env.timed(kernels_only, 8, False)
            t_all = np.array(env.gather_floats(t_mine), dtype=np.float64)
            feedback_history.append([round(float(x) / 8, 4) for x in t_all])
            if fused:
                for sw, ps in zip(sweeps, peers):  # re-sync the exchange state after the kernel-only launches
                    sw.launch()
                    ps.signal_wait()
            if t_all.max() <= 1.012 * t_all.mean():
                break
            for si, sw in enumerate(sweeps):
                scale[si] *= (t_all / t_all.mean())[np.asarray(sw._f_rank)]
            old = sweeps
            sweeps, slabs, peers, my_pf, my_bytes, all_pf = make_sweeps(inl, reuse_peers=peers if fused else None, scale_by_set=scale)
            del old
    total_pf = all_pf if sharded else all_pf * world  # replicas: every rank processes the whole stream
    ctx.synchronize()

    small_inputs = sum(sizes) * 36 <= L2_BYTES

    def step_device():
        for sw, slab, ps in zip(sweeps, slabs, peers):
            if ps is not None:
                sw.launch()  # epilogue stores finished pair rows into every rank's slab
                ps.signal_wait()  # completion flags: publish ours, wait for the peers'
            elif slab is not None:
                slab.zero_()
                sw.launch()
                if world > 1:
                    dist.all_reduce(slab, op=dist.ReduceOp.SUM)
            else:
                sw.launch()

    step_device()
    for sw in sweeps:  # a real caller fetches every linearization: the first fetch lets small sweeps size their items from measured inlier fractions
        if sw.F:
            sw.fetch()
    for _ in range(max(3, args.warmup)):
        step_device()
    launches0 = ctx.kernel_launches
    profiling = bool(os.environ.get("GB_PROFILE"))  # ncu --profile-from-start off: capture only the timed region
    if profiling:
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
    ms, _, t0, t1 = env.timed(step_device, args.steps, small_inputs)
    if profiling:
        torch.cuda.profiler.stop()
    gpu_launches = (ctx.kernel_launches - launches0) * world  # every rank launches the same sequence
    if args.dump_outputs and rank == 0:
        outs = {}
        for si, (sw, slab, ps) in enumerate(zip(sweeps, slabs, peers)):
            if ps is not None or slab is not None:
                outs[f"pair_slab{si}"] = ps.fetch() if ps is not None else slab.cpu().numpy()
            elif sw.F:
                rec = sw.fetch()
                outs[f"linearized{si}"] = rec.view(np.float64).reshape(len(rec), -1)
        dump_outputs(args.dump_outputs, outs)
    ms_per_step = ms / args.steps
    value = total_pf / (ms_per_step * 1e-3) / 1e6

    # ---- kernel-only duration for the roofline (same launches, no memset / collective in the bracket) ----
    def step_kernels():
        for sw in sweeps:
            sw.launch()

    for s in slabs:
        if s is not None:
            s.zero_()
    kms, kms_mine, _, _ = env.timed(step_kernels, args.steps, small_inputs)
    if sharded and fused:  # the kernel-only bracket advanced the ping-pong-free sweeps only; re-sync the exchange state
        step_device()
    k_launches = len(sweeps)
    kernel_ms_per_launch = kms / args.steps / max(1, k_launches)
    per_rank_kernel_ms = env.gather_floats(kms_mine / args.steps)
    # inlier counts of this rank's factors -> miss-aware bytes
    inl_mine = sum(float(sw.fetch()["num_inliers"].sum()) for sw in sweeps if sw.F)
    miss_bytes = my_bytes - 32.0 * (my_pf - inl_mine)
    roofline = roofline_of(args.workload, my_bytes, miss_bytes, k_launches, kernel_ms_per_launch, world, args.scale)

    # ---- end to end through the C-ABI with host buffers ----
    host_deltas = [sw._sub.deltas.copy() for sw in sweeps]
    h2d = sum(d.shape[0] * 128 for d in host_deltas)
    if sharded:  # the solver needs the pair slab only (levels pre-summed on the device): no per-factor records D2H
        d2h = sum((ps.num_pairs if ps is not None else s.shape[0]) * GB_SLAB_STRIDE * 4 for ps, s in zip(peers, slabs))
    else:
        d2h = sum(d.shape[0] * 976 for d in host_deltas)
    host_slabs = [torch.empty(s.shape, dtype=torch.float32, pin_memory=True) if s is not None else None for s in slabs]
    from glim_b200.capi import pose16

    host_p16 = [pose16(d) for d in host_deltas]
    host_out = [np.zeros(len(d), gpu.LIN_DTYPE) for d in host_deltas]

    def step_e2e():
        for k, (sw, slab, ps) in enumerate(zip(sweeps, slabs, peers)):
            if ps is None and slab is None:
                sw.linearize_raw(host_p16[k], host_out[k])  # gb_sweep_linearize with host buffers: poses H2D + launch + records D2H (one CUDA-graph launch for small sweeps)
                continue
            sw.set_poses(host_deltas[k])  # gb_sweep_set_poses: pinned staging + H2D (double buffered, no stream sync)
            if ps is not None:
                sw.launch()
                ps.signal_wait()
                ps.fetch_async()  # D2H of the complete slab into pinned memory
                ctx.synchronize()
            elif slab is not None:
                slab.zero_()
                sw.launch()
                if world > 1:
                    dist.all_reduce(slab, op=dist.ReduceOp.SUM)
                host_slabs[k].copy_(slab, non_blocking=True)
                ctx.synchronize()

    for _ in range(3):
        step_e2e()
    e_steps = args.steps
    ems, _, _, _ = env.timed(step_e2e, e_steps, False)
    e2e_val = total_pf / (ems / e_steps * 1e-3) / 1e6

    # ---- the exchanged slab of one step: checksum (identical at every N) and the oracle parity check of random rows ----
    step_device()
    torch.cuda.synchronize()
    slab_checksum, parity = None, None
    if sharded:
        rows_all = [ps.fetch() if ps is not None else s.cpu().numpy() for ps, s in zip(peers, slabs)]
        slab_checksum = float(sum(np.abs(r.astype(np.float64)).sum() for r in rows_all))
        if args.verify > 0 and rank == 0:
            parity = parity_check(env, w, w.sets[0], lambda: rows_all[0], args.verify)
    elif args.verify > 0 and rank == 0:
        # non-sharded workloads: records of the first factor set, summed per pair on the host
        rec = sweeps[0].fetch()
        rows = {}
        for k, f in enumerate(w.sets[0].factors):
            r = gpu.unpack_linearized(rec[k])
            if f.pair in rows:
                for kk in ("H_tt", "H_ss", "H_ts", "b_t", "b_s"):
                    rows[f.pair][kk] = rows[f.pair][kk] + r[kk]
                rows[f.pair]["error"] += r["error"]
                rows[f.pair]["num_inliers"] += r["num_inliers"]
            else:
                rows[f.pair] = r
        packed_rows = {p: multi_gpu.pack_slab_row(r).astype(np.float64) for p, r in rows.items()}
        parity = parity_check(env, w, w.sets[0], lambda: packed_rows, args.verify)
    if sampler:
        time.sleep(0.15)
        sampler.stop()

    line = None
    if rank == 0:
        push_fused = os.environ.get("GB_PEER_PUSH") == "fused" or (os.environ.get("GB_PEER_PUSH") != "deferred" and world <= 4)  # the library's policy
        how = ("are stored into every rank's buffer by the sweep kernel's epilogue over NVLink (CUDA IPC peer memory) + completion flags" if push_fused else
               "are written to the rank's own buffer by the sweep kernel's epilogue; the exchange kernel that follows (four CTAs per peer) copies the rank's rows into every peer's buffer over NVLink (CUDA IPC peer memory) and publishes / awaits the completion flags")
        par = (f"pairs sharded over {world} rank(s); finished pair rows of the [{peers[0].num_pairs} x {GB_SLAB_STRIDE}] fp32 Hessian slab {how}; no NCCL in the step"
               if (sharded and fused) else (f"pairs sharded over {world} rank(s), NCCL all-reduce of the [{slabs[0].shape[0]} x {GB_SLAB_STRIDE}] fp32 Hessian slab" if sharded else f"replicas x{world} (single online stream does not shard)"))
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms_per_step,
            "higher_is_better": True, "scaling": "strong" if sharded else "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(args.workload, w, {"parallelism": par,
                                                       "tiles_grid_first_sweep": [int(sweeps[0].num_tiles), int(sweeps[0].grid)], "partition": ("contiguous, cost = n_source + 1.25 * measured inliers (calibration sweep), then <= 2 rounds of per-rank kernel-time feedback" if calibrated else "contiguous, cost = n_source * (1 + 1.25 * gate overlap)") if sharded else None, "partition_feedback_kernel_ms": feedback_history or None, "build_seconds": round(build_s, 1), "scale": args.scale,
                                                       "kernel": os.environ.get("GB_KERNEL", "auto: k_vgicp_sweep5 + strided items for small sweeps, k_vgicp_sweep3 for large ones")}),
            "e2e": {"value": e2e_val, "unit": UNIT, "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h), "ms_per_step": ems / e_steps,
                    "result": "pair slab (levels pre-summed on the device)" if sharded else "gb_linearized6 records"},
            "gpu_launches": int(gpu_launches),
            "clocks": sampler.summary(t0, t1) if sampler else None,
            "roofline": roofline,
            "kernel_ms_per_rank": {"min": min(per_rank_kernel_ms), "median": float(np.median(per_rank_kernel_ms)), "max": max(per_rank_kernel_ms), "all": [round(x, 4) for x in per_rank_kernel_ms],
                                   "note": "k_vgicp_sweep only, per step, CUDA events on each rank (imbalance = max / median)"},
            "slab_checksum": slab_checksum,
            "parity_check": parity,
        }
        # the other BASELINE configurations, measured in the same process (each is ms-scale): SURVEY 8(d) sets the >= 60 % bar on M3 / M5
        if world == 1 and args.workload == "global_mapping_gpu" and args.scale == 1.0 and not args.no_other_workloads:
            del sweeps, slabs, peers
            others = {}
            names = {"single_pair": "M1", "odometry_gpu": "M2", "sub_mapping_gpu": "M3", "livox_stress": "M5"}
            others["M4 global_mapping_gpu"] = {"value": value, "launch_ms": roofline["launch_ms"], "frac": roofline["frac"], "miss_aware_frac": roofline["miss_aware_frac"], "e2e": e2e_val}
            for nm, tag in names.items():
                try:
                    wo = build_workload(nm, ctx, 1.0, use_gpu=True)
                    r = measure_simple(env, nm, wo, args.steps, 3)
                    others[f"{tag} {nm}"] = {"value": r["value"], "launch_ms": r["roofline"]["launch_ms"], "frac": r["roofline"]["frac"], "miss_aware_frac": r["roofline"]["miss_aware_frac"],
                                             "e2e": r["e2e"]["value"], "inlier_fraction": round(r["inlier_fraction"], 3),
                                             "factors_per_launch": int(sum(len(s.factors) for s in wo.sets) / len(wo.sets))}
                    del wo
                except Exception as ex:  # never lose the headline line to a secondary measurement
                    others[f"{tag} {nm}"] = {"error": repr(ex)[:200]}
            line["roofline_by_workload"] = others
        if world == 1 and not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_baseline(w, args.cpu_seconds)
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
