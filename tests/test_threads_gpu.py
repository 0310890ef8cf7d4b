"""The library under GLIM's threading (the rules of the boundary in include/glim_b200.h): one context per module thread,
clouds and maps that move between contexts, factors whose sweeps are cached by other contexts, caller-owned streams, a
pooled-block free while another thread captures a CUDA graph, and the per-thread error message.

ctypes releases the GIL around every C call, so the Python threads below really are inside the library at the same time.
Every thread is joined with a timeout: a deadlock fails the test instead of hanging it.  The reference for every result is
the same script run serially on one thread.  Results the header or another test calls exact (map downloads, merges, the CT
align batch, deskew, the graph solves, overlaps) are compared bit for bit; so are the sweep records, because two serial runs
of the scripts below give bit-identical records on the H100 (test_serial_runs_repeat_bit_for_bit)."""
import ctypes as C
import queue
import threading

import numpy as np
import pytest

from glim_b200 import capi, gpu, synth
from tests import util
from tests import voxelmap_oracle as vo

pytestmark = pytest.mark.gpu

TIMEOUT = 120.0  # seconds: every join and every handshake
N_FRAMES, N_RAYS = 20, 32 * 150
GROUP = 4  # frames per submap
MAX_CORR = 2.0
# Two serial runs of these scripts give bit-identical sweep records (test_serial_runs_repeat_bit_for_bit), so sweep
# linearizations are compared bit for bit as well.  The fp64 atomics add few fp32 item sums per factor in these small
# sweeps, and those adds come out exact whatever their order.  False would hold the records to util.check_linearized.
SWEEPS_BIT_EQUAL = True


@pytest.fixture(scope="module")
def frames():
    """arc frames 1 m apart with PLANE covariances, their k = 10 neighbours and scan times over 0.1 s"""
    fr = vo.arc_frames(N_FRAMES, N_RAYS)
    nbs = [np.ascontiguousarray(synth.knn(p, 10), dtype=np.int32) for p, _, _ in fr]
    return fr, nbs


# ---------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------
class Records:
    """sweep records (a LIN_DTYPE array): bit for bit when SWEEPS_BIT_EQUAL, else within util.check_linearized"""

    def __init__(self, a):
        self.a = np.array(a, copy=True)


def compare(got, want, where, out, stats):
    """append to `out` every difference between two results (nested dicts / lists / tuples of arrays and scalars)"""
    if isinstance(want, Records):
        same = got.a.tobytes() == want.a.tobytes()
        stats["records"] += 1
        stats["records_bit_equal"] += same
        if same:
            return
        if SWEEPS_BIT_EQUAL:
            out.append(f"{where}: sweep records differ in their bits")
            return
        for i, (g, w) in enumerate(zip(got.a, want.a)):
            try:
                util.check_linearized(gpu.unpack_linearized(g), gpu.unpack_linearized(w))
            except AssertionError as e:
                out.append(f"{where}[{i}]: {e}")
    elif isinstance(want, dict):
        if set(got) != set(want):
            out.append(f"{where}: keys {sorted(got)} != {sorted(want)}")
        for k in want:
            if k in got:
                compare(got[k], want[k], f"{where}.{k}", out, stats)
    elif isinstance(want, (list, tuple)):
        if len(got) != len(want):
            out.append(f"{where}: {len(got)} entries != {len(want)}")
        for i, (g, w) in enumerate(zip(got, want)):
            compare(g, w, f"{where}[{i}]", out, stats)
    else:
        g, w = np.asarray(got), np.asarray(want)
        if g.shape != w.shape or g.dtype != w.dtype or g.tobytes() != w.tobytes():
            out.append(f"{where}: {g.ravel()[:4]} != {w.ravel()[:4]} (shape {g.shape} / {w.shape})")


def assert_same(got, want, what):
    out, stats = [], {"records": 0, "records_bit_equal": 0}
    compare(got, want, what, out, stats)
    print(f"{what}: {stats['records_bit_equal']} of {stats['records']} sweep-record sets bit-equal, {len(out)} differences")
    assert not out, "\n".join(out[:20])
    return stats


def run_threads(targets, timeout=TIMEOUT):
    """start one daemon thread per callable, join each with a timeout; -> the exceptions they raised"""
    errors = []

    def wrap(fn):
        def run():
            try:
                fn()
            except BaseException as e:  # noqa: BLE001 -- reported by the caller
                errors.append(e)
        return run

    threads = [threading.Thread(target=wrap(fn), daemon=True) for fn in targets]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout)
    assert not any(t.is_alive() for t in threads), "a thread did not finish: deadlock or hang"
    return errors


def assert_no_errors(errors):
    assert not errors, "\n".join(f"{type(e).__name__}: {e}" for e in errors)


def rel(A, B):
    return synth.inv_pose(A) @ B


class Closing:
    """closes a handle at the end of a with block"""

    def __init__(self, h):
        self.h = h

    def __enter__(self):
        return self.h

    def __exit__(self, *exc):
        self.h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 1. three module threads, three contexts
# ---------------------------------------------------------------------------------------------------------------------
def odometry(ctx, frames, out_q, log):
    """per frame: VGICP against the previous frame's map through a fresh factor set (its first linearization captures a
    sweep graph, the others replay it), CT-GICP align (a batch of two) against an iVox of the previous frame, deskew; the
    previous frame's cloud then goes on to sub-mapping"""
    fr, nbs = frames
    prev = None
    try:
        for k, (pts, cov, T) in enumerate(fr):
            src = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx)
            if prev is not None:
                T_rel = rel(fr[k - 1][2], T)
                rng = synth.rng_for(7100, k)
                m = gpu.GaussianVoxelMapGPU(1.0, ctx=ctx).insert(prev)
                f = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, src, ctx=ctx)
                fs = gpu.NonlinearFactorSetGPU(ctx).add([f])
                lins = [Records(fs.linearize_deltas(synth.perturb(T_rel, rng, 0.01, 0.1)[None])) for _ in range(3)]
                ivox = gpu.IVoxGPU(1.0, 0.1, 10, 7, 100, 10, ctx=ctx)
                ivox.insert(prev)
                timed = gpu.PointCloudGPU.clone(pts, cov, ctx=ctx).add_times(np.linspace(0.0, 0.1, len(pts)))
                ct = gpu.IntegratedCT_GICPFactorGPU(0, 1, ivox, timed, MAX_CORR, ctx=ctx)
                X0 = [synth.perturb(T_rel, rng, 0.005, 0.05) for _ in range(2)]
                aligned = gpu.align_ct_gicp([ct, ct], X0, X0, [T_rel, T_rel], ctx=ctx)
                dp, dc, dn, dcloud = gpu.deskew_ct(timed, aligned[0]["X"], aligned[0]["Y"], nbs[k], 10, ctx=ctx)
                log.append({"map": m.download(), "lin": lins, "ct": aligned, "deskew": (dp, dc, dn)})
                for h in (dcloud, ct, timed, ivox, f, m):
                    h.close()
                out_q.put((k - 1, prev))
            prev = src
        out_q.put((len(fr) - 1, prev))
    finally:
        out_q.put(None)


def sub_mapping(ctx, frames, in_q, out_q, log):
    """per GROUP frames (clouds made by the odometry context): merge into a submap, build its map, optimize the frames' poses
    over VGICP factors between consecutive frames; the submap and its frame clouds then go on to global mapping"""
    fr, _ = frames
    group = []
    try:
        while True:
            item = in_q.get(timeout=TIMEOUT)
            if item is None:
                break
            group.append(item)
            if len(group) < GROUP:
                continue
            ids, clouds = [k for k, _ in group], [c for _, c in group]
            T0 = fr[ids[0]][2]
            poses = [rel(T0, fr[k][2]) for k in ids]
            pts, cov, sub = gpu.merge_frames_gpu(poses, clouds, 0.1, ctx=ctx)
            m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(sub)
            fmaps = [gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(c) for c in clouds]
            facs = [gpu.IntegratedVGICPFactorGPU(i, i + 1, fmaps[i], clouds[i + 1], ctx=ctx) for i in range(GROUP - 1)]
            rng = synth.rng_for(7200, ids[0])
            values = {i: (poses[i] if i == 0 else synth.perturb(poses[i], rng, 0.005, 0.05)) for i in range(GROUP)}
            res = gpu.optimize_graphs([dict(factors=facs, values=values, priors=[(0, poses[0], 1e8)])], params=dict(max_iterations=5), ctx=ctx)
            log.append({"merge": (pts, cov), "map": m.download(), "graph": res})
            for h in facs + fmaps:
                h.close()
            out_q.put((sub, m, T0, clouds))
            group = []
    finally:
        out_q.put(None)


def global_mapping(ctx, in_q, log):
    """per submap: find the overlapping submaps among all so far, optimize the pose graph over VGICP factors on the pairs
    found, then destroy the submap's frame clouds (made by the odometry context, used by the sub-mapping context)"""
    maps, sources, T = [], [], []
    try:
        while True:
            item = in_q.get(timeout=TIMEOUT)
            if item is None:
                break
            sub, m, T0, clouds = item
            sources.append(sub)
            maps.append(m)
            T.append(T0)
            pairs, ovs = gpu.find_overlapping_submaps(maps, sources, T, max_distance=100.0, min_overlap=0.0, ctx=ctx)
            entry = {"pairs": pairs, "overlaps": ovs}
            if len(pairs):
                facs = [gpu.IntegratedVGICPFactorGPU(int(i), int(j), maps[i], sources[j], ctx=ctx) for i, j in pairs]
                rng = synth.rng_for(7300, len(T))
                values = {i: (T[i] if i == 0 else synth.perturb(T[i], rng, 0.002, 0.02)) for i in range(len(T))}
                entry["graph"] = gpu.optimize_pose_graph(facs, values, priors=[(0, T[0], 1e10)], params=dict(max_iterations=5), ctx=ctx)
                for h in facs:
                    h.close()
            log.append(entry)
            for c in clouds:
                c.close()
    finally:
        for h in maps + sources:
            h.close()


def pipeline(frames, threaded):
    """odometry -> sub-mapping -> global mapping on three fresh contexts, as three threads or one after the other on this one.
    -> ({module: step outputs}, {module: launch count delta})"""
    names = ("odometry", "sub_mapping", "global_mapping")
    ctxs = {n: gpu.Context(0) for n in names}
    q_sub, q_glob = queue.Queue(), queue.Queue()
    logs = {n: [] for n in names}
    l0 = {n: ctxs[n].kernel_launches for n in names}
    steps = [lambda: odometry(ctxs["odometry"], frames, q_sub, logs["odometry"]),
             lambda: sub_mapping(ctxs["sub_mapping"], frames, q_sub, q_glob, logs["sub_mapping"]),
             lambda: global_mapping(ctxs["global_mapping"], q_glob, logs["global_mapping"])]
    if threaded:
        assert_no_errors(run_threads(steps))
    else:
        for s in steps:
            s()
    launches = {n: ctxs[n].kernel_launches - l0[n] for n in names}
    for c in ctxs.values():
        c.close()
    assert len(logs["odometry"]) == N_FRAMES - 1 and len(logs["sub_mapping"]) == N_FRAMES // GROUP == len(logs["global_mapping"])
    return logs, launches


@pytest.fixture(scope="module")
def serial(frames):
    return pipeline(frames, threaded=False)


def test_serial_runs_repeat_bit_for_bit(frames, serial):
    """Two serial runs of the pipeline: every output, the sweep records included, and every launch count are bit-identical.
    This is what lets the threaded runs be held to bit equality."""
    logs, launches = pipeline(frames, threaded=False)
    stats = assert_same(logs, serial[0], "second serial run")
    assert stats["records"] == 3 * (N_FRAMES - 1)
    assert launches == serial[1]


def test_three_module_threads_match_the_serial_run(frames, serial):
    """Odometry, sub-mapping and global mapping each on its own thread and context, at once: the global thread destroys frame
    clouds while odometry captures and replays sweep graphs.  Every step's output equals the serial run's, and each context's
    launch count does too (the counter is per context: another thread's work does not move it)."""
    ref_logs, ref_launches = serial
    assert ref_launches["odometry"] > 0 and ref_launches["sub_mapping"] > 0 and ref_launches["global_mapping"] > 0
    assert any("graph" in e for e in ref_logs["global_mapping"])
    logs, launches = pipeline(frames, threaded=True)
    assert_same(logs, ref_logs, "threaded run")
    assert launches == ref_launches, (launches, ref_launches)


# ---------------------------------------------------------------------------------------------------------------------
# 2. objects that cross contexts
# ---------------------------------------------------------------------------------------------------------------------
def deltas_for(fr, a, b, n, key):
    rng = synth.rng_for(7400, key)
    return [synth.perturb(rel(fr[a][2], fr[b][2]), rng, 0.01, 0.1) for _ in range(n)]


def test_objects_shared_across_contexts(frames):
    """One cloud read at once by factors of two contexts on two threads while a third context's thread runs overlap on a map
    built by a fourth context; then every object is destroyed from a thread that did not make it.  Results equal the same
    calls made serially beforehand, and the making context still works afterwards."""
    fr, _ = frames
    A, B, C, D = (gpu.Context(0) for _ in range(4))
    tgt = gpu.PointCloudGPU.clone(fr[5][0], fr[5][1], ctx=A)
    src = gpu.PointCloudGPU.clone(fr[6][0], fr[6][1], ctx=A)
    m1 = gpu.GaussianVoxelMapGPU(0.5, ctx=A).insert(tgt)
    m2 = gpu.GaussianVoxelMapGPU(1.0, ctx=A).insert(tgt)
    fB = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m1, src, ctx=B)
    fC = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m2, src, ctx=C)
    sets = {"B": gpu.NonlinearFactorSetGPU(B).add([fB]), "C": gpu.NonlinearFactorSetGPU(C).add([fC])}
    ds = deltas_for(fr, 5, 6, 8, 0)

    def work(name, out):
        if name == "D":
            out[name] = [gpu.overlap_gpu([m1, m2], src, [d, d], ctx=D) for d in ds]
        else:
            out[name] = [Records(sets[name].linearize_deltas(d[None])) for d in ds]

    want, got = {}, {}
    for name in ("B", "C", "D"):
        work(name, want)
    assert_no_errors(run_threads([lambda n=n: work(n, got) for n in ("B", "C", "D")]))
    assert_same(got, want, "shared cloud")
    assert min(want["D"]) > 0.5

    # destroyed from threads that did not make them (the factors first: they borrow the maps and the cloud)
    assert_no_errors(run_threads([fB.close, fC.close]))
    assert_no_errors(run_threads([lambda: [h.close() for h in (m1, m2, src)]]))
    again = gpu.GaussianVoxelMapGPU(0.5, ctx=A).insert(tgt)
    assert again.num_voxels > 0
    assert_no_errors(run_threads([again.close, tgt.close]))
    for c in (A, B, C, D):
        c.close()


def test_factors_outlive_their_context(frames):
    """A context destroyed while its factors are alive: they still linearize from another thread, equal to the same factor
    made on a live context, and the last factor's destroy (on yet another thread) tears the context down."""
    fr, _ = frames
    A, D = gpu.Context(0), gpu.Context(0)
    tgt = gpu.PointCloudGPU.clone(fr[8][0], fr[8][1], ctx=A)
    src = gpu.PointCloudGPU.clone(fr[9][0], fr[9][1], ctx=A)
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=A).insert(tgt)
    ds = deltas_for(fr, 8, 9, 3, 1)
    fA = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, src, ctx=A)
    fD = [gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, src, ctx=D) for _ in range(2)]
    for f in fD:
        f._handle()
    want = [Records(gpu.NonlinearFactorSetGPU(A).add([fA]).linearize_deltas(d[None])) for d in ds]
    D.close()  # gb_ctx_destroy: the owner lets go; the factors keep the context alive
    got = {}

    def use(k):
        one = []
        for d in ds:
            out = np.zeros(1, gpu.LIN_DTYPE)
            capi.check(capi.lib().gb_vgicp_linearize(fD[k].h, capi.ptr(capi.pose16(d)), capi.ptr(out)))
            one.append(Records(out))
        got[k] = one

    assert_no_errors(run_threads([lambda: use(0), lambda: use(1)]))
    assert_same(got, {0: want, 1: want}, "factors of a destroyed context")
    assert_no_errors(run_threads([fD[0].close]) + run_threads([fD[1].close]))
    for h in (fA, m, src, tgt, A):
        h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. cached sweeps across contexts
# ---------------------------------------------------------------------------------------------------------------------
def test_cached_sweeps_of_a_factor_destroyed_elsewhere(frames):
    """A factor made on A, linearized in factor sets of B and of C (both cache a sweep naming it), destroyed from a third
    thread.  The next linearization of another set on B and on C (each context drops its stale sweep on the way in) succeeds
    and equals its value from before, and a caller-owned sweep that still names the dead factor is refused."""
    fr, _ = frames
    A, B, C = (gpu.Context(0) for _ in range(3))
    clouds = [gpu.PointCloudGPU.clone(fr[k][0], fr[k][1], ctx=A) for k in (10, 11, 12)]
    maps = [gpu.GaussianVoxelMapGPU(0.5, ctx=A).insert(c) for c in clouds[:2]]
    f = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, maps[0], clouds[1], ctx=A)
    gB = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, maps[1], clouds[2], ctx=B)
    gC = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, maps[1], clouds[2], ctx=C)
    d_f, d_g = deltas_for(fr, 10, 11, 1, 2)[0], deltas_for(fr, 11, 12, 1, 3)[0]
    both = {n: gpu.NonlinearFactorSetGPU(c).add([f, g]) for n, c, g in (("B", B, gB), ("C", C, gC))}
    alone = {n: gpu.NonlinearFactorSetGPU(c).add([g]) for n, c, g in (("B", B, gB), ("C", C, gC))}
    owned = gpu.Sweep(B, [f, gB])
    want = {n: Records(alone[n].linearize_deltas(d_g[None])) for n in alone}
    pair = {}
    assert_no_errors(run_threads([lambda n=n: pair.__setitem__(n, Records(both[n].linearize_deltas(np.stack([d_f, d_g])))) for n in both]))
    assert_same(pair["B"].a[1:], pair["C"].a[1:], "gB and gC in sets with the factor")
    owned.linearize(np.stack([d_f, d_g]))

    assert_no_errors(run_threads([f.close]))
    got = {}
    assert_no_errors(run_threads([lambda n=n: got.__setitem__(n, Records(alone[n].linearize_deltas(d_g[None]))) for n in alone]))
    assert_same(got, want, "sets of B and C after the factor died")
    with pytest.raises(capi.GlimB200Error, match="a factor of this sweep has been destroyed"):
        owned.linearize(np.stack([d_f, d_g]))
    for h in [owned, gB, gC] + maps + clouds + [A, B, C]:
        h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. caller-owned streams
# ---------------------------------------------------------------------------------------------------------------------
class DeviceArray:
    """a device pointer as a __cuda_array_interface__ (version 2: no stream, so torch reads it on its current stream)"""

    def __init__(self, p, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (p, False), "version": 2}


def stream_script(ctx, fr):
    """upload, build, a factor set linearized three times (its first call captures a sweep graph where the stream allows),
    merge and overlap -> outputs"""
    a = gpu.PointCloudGPU.clone(fr[13][0], fr[13][1], ctx=ctx)
    b = gpu.PointCloudGPU.clone(fr[14][0], fr[14][1], ctx=ctx)
    m = gpu.GaussianVoxelMapGPU(0.5, ctx=ctx).insert(a)
    f = gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, m, b, ctx=ctx)
    fs = gpu.NonlinearFactorSetGPU(ctx).add([f])
    out = {"cloud": b.download(), "map": m.download(), "lin": [Records(fs.linearize_deltas(d[None])) for d in deltas_for(fr, 13, 14, 3, 4)]}
    pts, cov, merged = gpu.merge_frames_gpu([np.eye(4), rel(fr[13][2], fr[14][2])], [a, b], 0.1, ctx=ctx)
    out["merge"] = (pts, cov)
    out["overlap"] = gpu.overlap_gpu(m, b, rel(fr[13][2], fr[14][2]), ctx=ctx)
    for h in (merged, f, m, b, a):
        h.close()
    return out


def test_caller_owned_streams(frames):
    """gb_ctx_create_on_stream on a torch side stream and on the legacy default stream (0): every result equals an owned-stream
    context's, bit for bit.  On the legacy stream no graph capture can begin, so the factor set falls back to plain launches
    and still succeeds.  gb_sweep_results_device read by torch on the same stream right after gb_sweep_launch, with no host
    synchronisation between, equals gb_sweep_fetch."""
    import torch

    fr, _ = frames
    owned = gpu.Context(0)
    side_stream = torch.cuda.Stream()
    side = gpu.Context(0, side_stream.cuda_stream)
    legacy = gpu.Context(0, 0)
    assert side.stream == side_stream.cuda_stream and legacy.stream == 0
    want = stream_script(owned, fr)
    assert_same(stream_script(side, fr), want, "side stream")
    assert_same(stream_script(legacy, fr), want, "legacy stream")

    a = gpu.PointCloudGPU.clone(fr[15][0], fr[15][1], ctx=side)
    b = gpu.PointCloudGPU.clone(fr[16][0], fr[16][1], ctx=side)
    maps = [gpu.GaussianVoxelMapGPU(r, ctx=side).insert(a) for r in (0.25, 0.5, 1.0)]
    facs = [gpu.IntegratedVGICPFactorGPU(np.eye(4), 0, mm, b, ctx=side) for mm in maps]
    sw = gpu.Sweep(side, facs)
    sw.set_poses(np.stack(deltas_for(fr, 15, 16, 3, 5)))
    sw.launch()
    with torch.cuda.stream(side_stream):
        read = torch.as_tensor(DeviceArray(sw.results_device_ptr(), sw.F * 122), device="cuda").clone()
    side_stream.synchronize()
    fetched = sw.fetch()
    assert (fetched["num_inliers"] > 0).all()
    assert read.cpu().numpy().tobytes() == fetched.tobytes()
    for h in [sw] + facs + maps + [b, a, legacy, side, owned]:
        h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. a pooled-block free during another thread's capture
# ---------------------------------------------------------------------------------------------------------------------
def test_free_during_another_threads_capture(frames):
    """Thread B captures a torch graph (thread-local mode) on the caller-owned stream of its context.  Meanwhile thread A
    destroys a cloud, whose pooled blocks are recycled only after every live context's stream has drained, and then makes
    one launching call (gb_voxelmap_build): that call succeeds and builds the same map as before, and B's capture ends valid
    and replays correctly.  Deterministic: Event handshakes order the steps, nothing is retried."""
    import torch

    fr, _ = frames
    s = torch.cuda.Stream()
    ctx_b = gpu.Context(0, s.cuda_stream)
    ctx_a = gpu.Context(0)
    keep = gpu.PointCloudGPU.clone(fr[17][0], fr[17][1], ctx=ctx_a)
    victim = gpu.PointCloudGPU.clone(fr[18][0], fr[18][1], ctx=ctx_a)
    with Closing(gpu.GaussianVoxelMapGPU(0.5, ctx=ctx_a).insert(keep)) as m0:
        want = m0.download()
    x = torch.arange(4096, device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    capturing, freed = threading.Event(), threading.Event()
    res = {}

    def thread_b():
        try:
            with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
                y = x * 2.0 + 1.0
                capturing.set()
                assert freed.wait(TIMEOUT), "thread A did not finish"
            res["y"] = y
        finally:
            capturing.set()

    def thread_a():
        try:
            assert capturing.wait(TIMEOUT), "thread B did not begin its capture"
            victim.close()
            with Closing(gpu.GaussianVoxelMapGPU(0.5, ctx=ctx_a).insert(keep)) as m:
                res["map"] = m.download()
        finally:
            freed.set()

    assert_no_errors(run_threads([thread_b, thread_a]))
    assert_same(res["map"], want, "map built right after the free")
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(res["y"], x * 2.0 + 1.0)
    for h in (keep, ctx_a, ctx_b):
        h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. gb_last_error is per thread
# ---------------------------------------------------------------------------------------------------------------------
def test_last_error_is_per_thread():
    """A refused call in thread A leaves thread B's message as B's own refused call left it."""
    L = capi.lib()
    b_failed, a_failed = threading.Event(), threading.Event()
    res = {}

    def thread_b():
        try:
            res["b_status"] = L.gb_cloud_size(None, None)
            res["b_before"] = L.gb_last_error().decode()
            b_failed.set()
            assert a_failed.wait(TIMEOUT)
            res["b_after"] = L.gb_last_error().decode()
        finally:
            b_failed.set()

    def thread_a():
        assert b_failed.wait(TIMEOUT)
        try:
            h = C.c_void_p()
            res["a_status"] = L.gb_cloud_upload(None, 0, None, None, None, C.byref(h))
            res["a"] = L.gb_last_error().decode()
        finally:
            a_failed.set()

    assert_no_errors(run_threads([thread_b, thread_a]))
    assert res["a_status"] == 1 and res["a"] == "invalid argument: null ctx / output"
    assert res["b_status"] == 1 and res["b_before"] == "invalid argument: null argument"
    assert res["b_after"] == res["b_before"]
