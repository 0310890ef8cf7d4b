"""numpy restatement of the incremental device voxel map (gb_voxelmap_create_incremental / gb_voxelmap_insert), written from
the rule in include/glim_b200.h and independently of the CUDA: sampling pick, fp64 transform, fp64 keys, sequential sums,
stamps and LRU eviction, ascending-key numbering, fp32 records and the open-addressing table (sequential first-free-slot
insertion in ascending voxel order, the build's sizing rule)."""
import functools

import numpy as np

from glim_b200 import synth

KEY_OFFSET = 1 << 20
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


@functools.lru_cache(maxsize=None)
def arc_frames(n_frames, n_rays, sensor="hdl32", nan_frame=None):
    """hdl32 scans along the M2 arc (1 m apart) in the sensor frame, with PLANE covariances (k = 10), and their world poses.
    Frame `nan_frame` gets every 7th point replaced by NaN.  -> list of (points (N,4), covs (N,4,4), T_world_sensor)"""
    sc = synth.make_hall_scene()
    traj = synth.arc_trajectory(n_frames)
    out = []
    for i, T in enumerate(traj):
        pts, _ = synth.scan(sc, sensor, T, synth.rng_for(510, i), n_rays=n_rays)
        _, cov = synth.with_covariances(pts, 10)
        if i == nan_frame:
            pts = pts.copy()
            pts[::7, :3] = np.nan
        out.append((np.ascontiguousarray(pts), np.ascontiguousarray(cov), T))
    return out


def rg_hash(seed, idx):
    """splitmix64 finalizer of seed + golden * (i + 1), in wrapping uint64 arithmetic."""
    with np.errstate(over="ignore"):
        i = np.asarray(idx, dtype=np.uint64)
        z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * ((i + np.uint64(1)) & np.uint64(0xFFFFFFFF))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def sample_mask(n, rate, seed):
    """rate = 1: every point; otherwise the (size_t)(n * rate) points with the smallest rg_hash(seed, index)."""
    keep = np.zeros(n, bool)
    if rate >= 1.0:
        keep[:] = True
        return keep
    m = int(n * rate)
    if m > 0:
        keep[np.argsort(rg_hash(seed, np.arange(n)), kind="stable")[:m]] = True
    return keep


def transform(T, xyz, cov6):
    """q = R a + t and the upper triangle of R C R^T in fp64, with the association order of the device transform."""
    T = np.asarray(T, dtype=np.float64)
    a = np.asarray(xyz, dtype=np.float32).astype(np.float64)
    c = np.asarray(cov6, dtype=np.float32).astype(np.float64)
    x, y, z = a[:, 0], a[:, 1], a[:, 2]
    q = np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], 1)
    C = [[c[:, 0], c[:, 1], c[:, 2]], [c[:, 1], c[:, 3], c[:, 4]], [c[:, 2], c[:, 4], c[:, 5]]]
    RC = [[(T[r, 0] * C[0][k] + T[r, 1] * C[1][k]) + T[r, 2] * C[2][k] for k in range(3)] for r in range(3)]
    out = [(RC[r][0] * T[k, 0] + RC[r][1] * T[k, 1]) + RC[r][2] * T[k, 2] for r in range(3) for k in range(r, 3)]
    return q, np.stack(out, 1)


def coords(q, resolution):
    """floor(q * (1.0 / (double)resolution)) in fp64 -> (int64 coords (n,3), valid mask: finite and inside the 21-bit range)."""
    inv = 1.0 / float(np.float32(resolution))
    fin = np.isfinite(q).all(1)
    with np.errstate(invalid="ignore"):
        f = np.floor(np.where(fin[:, None], q, 0.0) * inv)
    ok = fin & (f >= -KEY_OFFSET).all(1) & (f < KEY_OFFSET).all(1)
    return np.where(ok[:, None], f, 0).astype(np.int64), ok


def pack(c):
    c = np.asarray(c, dtype=np.int64) + KEY_OFFSET
    return (c[:, 0].astype(np.uint64) << np.uint64(42)) | (c[:, 1].astype(np.uint64) << np.uint64(21)) | c[:, 2].astype(np.uint64)


def unpack(k):
    k = np.asarray(k, dtype=np.uint64)
    m = np.uint64(0x1FFFFF)
    return np.stack([((k >> np.uint64(42)) & m).astype(np.int64), ((k >> np.uint64(21)) & m).astype(np.int64), (k & m).astype(np.int64)], 1) - KEY_OFFSET


def voxel_hash(c):
    with np.errstate(over="ignore"):
        c = np.asarray(c, dtype=np.int64).astype(np.uint64)
        return (c[:, 0] * np.uint64(73856093)) ^ (c[:, 1] * np.uint64(19349669)) ^ (c[:, 2] * np.uint64(83492791))


def build_table(vcoord, vn, init_buckets, max_scan, drop_rate, total_points):
    """Sequential first-free-slot insertion in ascending voxel order; init_buckets doubled until >= 8 V, then doubled while
    more than drop_rate * total_points points are dropped.  -> (buckets (nb,4) int32, dropped points)"""
    V = len(vcoord)
    nb = int(init_buckets)
    while nb < 8 * V:
        nb *= 2
    home = voxel_hash(vcoord) if V else np.zeros(0, np.uint64)
    while True:
        mask = nb - 1
        owner = np.full(nb, -1, np.int64)
        dropped = 0
        h = (home & np.uint64(mask)).astype(np.int64)
        for v in range(V):
            for d in range(max_scan):
                s = (h[v] + d) & mask
                if owner[s] < 0:
                    owner[s] = v
                    break
            else:
                dropped += int(vn[v])
        if dropped <= drop_rate * total_points or nb >= (1 << 28):
            break
        nb *= 2
    buckets = np.zeros((nb, 4), np.int32)
    buckets[:, 3] = -1
    occ = owner >= 0
    buckets[occ, :3] = vcoord[owner[occ]]
    buckets[occ, 3] = owner[occ]
    return buckets, dropped


class IncrementalMap:
    """The map state of the rule: per voxel key, n, fp64 sums (q: 3, C: 6) and stamp; per map the insert counter."""

    def __init__(self, resolution, lru_horizon=0, lru_clear_cycle=10, init_buckets=16384, max_scan=10, drop_rate=1e-3):
        self.resolution = float(np.float32(resolution))
        self.h, self.k = int(lru_horizon), int(lru_clear_cycle)
        self.init_buckets, self.max_scan, self.drop_rate = init_buckets, max_scan, drop_rate
        self.counter = 0
        self.keys = np.zeros(0, np.uint64)
        self.n = np.zeros(0, np.int64)
        self.stamp = np.zeros(0, np.int64)
        self.sums = np.zeros((0, 9))
        self.last_points = (np.zeros((0, 3)), np.zeros((0, 6)))  # the fp64 points of the last insert that entered the map
        self.finalize()

    def insert(self, xyz, cov6, T=None, rate=1.0, seed=0):
        T = np.eye(4) if T is None else np.asarray(T, dtype=np.float64)
        n = len(xyz)
        keep = sample_mask(n, rate, seed)
        q, c6 = transform(T, xyz, cov6)
        cc, ok = coords(q, self.resolution)
        sel = keep & ok
        self.last_points = (q[sel], c6[sel])
        nk = pack(cc[sel])
        allk = np.unique(np.concatenate([self.keys, nk]))
        sums = np.zeros((len(allk), 9))
        cnt = np.zeros(len(allk), np.int64)
        stamp = np.zeros(len(allk), np.int64)
        old = np.searchsorted(allk, self.keys)
        sums[old], cnt[old], stamp[old] = self.sums, self.n, self.stamp
        pos = np.searchsorted(allk, nk)
        np.add.at(sums, pos, np.concatenate([q[sel], c6[sel]], 1))  # sequential, in point order
        np.add.at(cnt, pos, 1)
        stamp[np.unique(pos)] = self.counter
        self.counter += 1
        alive = np.ones(len(allk), bool)
        if self.h > 0 and self.counter % self.k == 0:
            alive = ~(stamp + self.h < self.counter)
        self.keys, self.n, self.stamp, self.sums = allk[alive], cnt[alive], stamp[alive], sums[alive]
        self.finalize()
        return self

    def finalize(self):
        d = self.n.astype(np.float64)[:, None]
        rec = (self.sums / d).astype(np.float32) if len(self.n) else np.zeros((0, 9), np.float32)
        self.means, self.covs = rec[:, :3], rec[:, 3:]
        self.vcoord = unpack(self.keys)
        self.buckets, self.dropped = build_table(self.vcoord, self.n, self.init_buckets, self.max_scan, self.drop_rate, float(self.n.sum()))

    @property
    def num_voxels(self):
        return len(self.keys)

    def mean_cov64(self):
        """fp64 mean (V,3) and covariance (V,3,3) of every voxel"""
        d = self.n.astype(np.float64)[:, None]
        m = self.sums[:, :3] / d
        c = self.sums[:, 3:] / d
        C = np.stack([c[:, [0, 1, 2]], c[:, [1, 3, 4]], c[:, [2, 4, 5]]], 1)
        return m, C
