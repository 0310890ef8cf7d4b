"""The host rules that schedule a linearization sweep (gb_sweep_create, build_items, sweep_learn_inliers, graph_eligible and the
launchers' ctr_base advance in glim_b200/csrc), restated in Python, and the factor sizes of every regime that
tests/test_sweep_schedules_gpu.py runs.  Written from the rules, not derived from the CUDA: the GPU tests compare what this
module predicts with gb_sweep_stats, so a changed rule fails on the regime a test asked for instead of quietly testing another.
Every size follows from the device's SM count."""
import math

import numpy as np

CTAS_PER_SM = 2
WARPS_PER_CTA = 8
DESC_CACHE = 40  # sweep5's shared-memory descriptor cache (kDescCache)
ROUND3 = 480  # sweep3's points per round (kRound3)
MAX_PREFIX = 100_000  # the largest source prefix any regime takes (the test clouds hold more points)
POINT_FACTOR_BUDGET = 32_000_000  # the most point-factors one regime may sweep

N_POSES = 8  # poses cycled over the factors of a regime
N_MAPS = 3  # voxel levels cycled over the factors of a regime


def warps(sms):
    return sms * CTAS_PER_SM * WARPS_PER_CTA


def plan(sizes, sms, kernel=0, gicp=False, inlier_frac=None):
    """gb_sweep_create's schedule of a sweep over factors with `sizes` source points.  kernel: GB_KERNEL (0 = unset); gicp: a
    GICP / ICP sweep; inlier_frac: each factor's learned inlier fraction (None or < 0: unknown)."""
    sizes = [int(n) for n in sizes]
    F = len(sizes)
    capacity = sms * CTAS_PER_SM
    W = warps(sms)
    total = sum(sizes)
    small = F > 0 and total <= W * 2048
    kv = kernel if kernel in (3, 5) else (5 if small else 3)
    if gicp:
        kv = 5
    want = total // (W * 6) + 1
    tile = min(2048, max(128, want))
    tile = (tile + 31) // 32 * 32
    frac = [-1.0] * F if inlier_frac is None else [float(r) for r in inlier_frac]
    p = {"kernel": kv, "tile_size": tile, "F": F, "sizes": sizes, "sms": sms, "capacity": capacity, "gicp": gicp, "calibrated": False}
    items = _items(p, frac)
    p.update(items)
    p["tiles_cap"] = max(p["num_tiles"], W + F if kv == 5 else 0)
    p["grid"] = max(1, min((p["num_tiles"] + 7) // 8, capacity))
    acc = 1
    while F > 0 and acc < 16 and p["num_tiles"] > F * 64 * acc:
        acc *= 2
    p["acc_slots"] = acc
    _derive(p)
    return p


def _items(p, frac):
    """build_items: per factor its item count J and (sweep3) its item size"""
    sizes, F, W = p["sizes"], p["F"], p["capacity"] * WARPS_PER_CTA
    if p["kernel"] == 3:
        tile = p["tile_size"]
        total = sum(sizes)
        tail16 = int(W * tile * 0.4)
        tail4 = int(W * tile * 1.5)
        chunks, J = [], []
        before = 0
        for n in sizes:
            remaining = total - before
            chunk = tile
            if remaining <= tail16:
                chunk = max(128, tile // 16)
            elif remaining <= tail4:
                chunk = max(128, tile // 4)
            if total <= int(W * tile * 3.0):
                chunk = tile
            chunks.append(chunk)
            J.append(max(1, (n + chunk - 1) // chunk))
            before += n
        return {"J": J, "chunks": chunks, "num_tiles": sum(J)}
    cost = []
    tot = 0.0
    for n, r in zip(sizes, frac):
        rr = r if r >= 0.0 else 0.5
        c = float(n) * (1.0 + 1.25 * rr) + 64.0
        cost.append(c)
        tot += c
    budget = float(W)
    J = [0] * F
    for _ in range(64):
        s = 0
        for f, n in enumerate(sizes):
            rows = (n + 31) // 32
            jmax = max(1, rows // 4)
            J[f] = min(jmax, max(1, int(cost[f] / tot * budget + 0.5)))
            s += J[f]
        if s <= W:
            break
        budget *= 0.95
    return {"J": J, "chunks": [0] * F, "num_tiles": sum(J)}


def _derive(p):
    """what the launch does with the table: the queue, sweep5's descriptor cache, the captured graph"""
    W = p["grid"] * WARPS_PER_CTA
    p["dynamic"] = p["num_tiles"] > W
    p["cached"] = p["kernel"] == 5 and not p["gicp"] and p["F"] <= DESC_CACHE
    p["graph"] = p["kernel"] == 5 and p["num_tiles"] <= p["grid"] * 8 and p["F"] > 0  # without a slab attached
    # the queue counter's advance per launch: one draw per item, plus one look-ahead draw per warp in sweep5
    p["ctr_advance"] = (p["num_tiles"] + (W if p["kernel"] == 5 and not p["gicp"] else 0)) if p["dynamic"] else 0


def learn(p, inliers):
    """sweep_learn_inliers after a fetch of the records' `inliers`: each factor's inlier fraction (fp32), and, once per sweep5
    sweep, the item table re-sized from them when some factor's item count moves by more than an eighth.  -> (new plan, fractions)"""
    frac = [float(np.float32(float(k) / n)) if n else -1.0 for k, n in zip(inliers, p["sizes"])]
    q = dict(p)
    if p["kernel"] != 5 or p["calibrated"]:
        return q, frac
    q["calibrated"] = True
    new = _items(p, frac)
    changed = any(abs(a - b) * 8 > a for a, b in zip(p["J"], new["J"]))
    if changed and new["num_tiles"] <= p["tiles_cap"]:
        q.update(new)
        q["grid"] = max(1, min((q["num_tiles"] + 7) // 8, p["capacity"]))
        _derive(q)
    return q, frac


def chunk_sizes(p):
    """the distinct item sizes of a sweep3 plan"""
    return sorted(set(p["chunks"]))


# ---------------------------------------------------------------------------------------------------------------------
# the regimes: factor sizes (source prefix lengths) by SM count
# ---------------------------------------------------------------------------------------------------------------------
# Prefix cycles have lengths coprime to N_POSES * N_MAPS = 24: factor f takes prefix f % len, pose f % 8 and level f % 3, so
# neighbouring factors differ in all three and any misrouted item or row changes some factor's exact inlier count.
RAGGED = [0, 1, 31, 33, 5000, 777, 12000, 2047, 64, 9001, 3000]
TINY = [1, 7, 31, 32, 33, 64, 97]
BOUNDARY = [479, 480, 481, 991, 2047, 2048, 2049]
QUEUE3 = [1000, 2500, 4000, 700, 3300]
LARGE = [100000, 0, 479, 70000, 1, 480, 85000, 31, 481, 95000, 33, 991, 60000, 2047, 2048, 2049, 90000]
SV_SET = [100000, 83000, 91000, 77000, 65536]
GICP_WAVE = [0, 1, 31, 33, 700, 1500, 2600]
ACC_ITEMS = {1: 60, 2: 100, 4: 200, 8: 300, 16: 600}  # acc_slots -> a single factor's item count that selects it
# near-full (even) and near-empty (odd) factors: after the first fetch the near-full ones reach their most items (rows / 4),
# so the re-sized table leaves part of the item budget unused and num_tiles changes
CALIB = [15000 + 100 * f if f % 2 == 0 else 60000 + 1000 * f for f in range(8)]
CALIB_FRACTIONS = [0.65 if f % 2 == 0 else 0.1 for f in range(8)]  # the least / most the GPU test lets them be


def cycle(base, F):
    return [base[f % len(base)] for f in range(F)]


def regimes(sms):
    """regime -> dict(sizes (one list per sweep), kernel (GB_KERNEL, 0 = unset), gicp)"""
    W = warps(sms)
    per_cycle5 = sum(-(-n // 128) for n in BOUNDARY)  # BOUNDARY's 128-point items
    per_cycle6 = sum(-(-n // 128) for n in QUEUE3)
    large_target = 1.1 * 6 * W * 2048
    sv_target = 1.2 * W * 2048
    return {
        "R1": {"sizes": [cycle(RAGGED, 40), cycle(RAGGED, 41)], "kernel": 0},
        "R2": {"sizes": [cycle(TINY, W + 300)], "kernel": 0},
        "R3": {"sizes": [[128 * ACC_ITEMS[a]] for a in sorted(ACC_ITEMS)], "kernel": 0},
        "R4": {"sizes": [CALIB], "kernel": 0},
        "R5": {"sizes": [cycle(BOUNDARY, len(BOUNDARY) * (W // per_cycle5))], "kernel": 3},
        "R6": {"sizes": [cycle(QUEUE3, len(QUEUE3) * math.ceil(3 * W / per_cycle6))], "kernel": 3},
        "R7": {"sizes": [cycle(LARGE, len(LARGE) * math.ceil(large_target / sum(LARGE)))], "kernel": 0},
        "R8": {"sizes": [cycle(SV_SET, math.ceil(sv_target / (sum(SV_SET) / len(SV_SET))))], "kernel": 0},
        "R9": {"sizes": [cycle(SV_SET, math.ceil(sv_target / (sum(SV_SET) / len(SV_SET))))], "kernel": 0},
        "R10": {"sizes": [cycle(GICP_WAVE, 21), cycle(TINY, W + 100)], "kernel": 0, "gicp": True},
    }


def plans_of(name, sms):
    """the restated plan of every sweep of a regime, as built (no learned inlier fractions)"""
    r = regimes(sms)[name]
    return [plan(s, sms, kernel=r["kernel"], gicp=r.get("gicp", False)) for s in r["sizes"]]


def check_regime(name, plans, sms):
    """asserts that the plans of a regime's sweeps are the regime the name stands for, within the size budget"""
    W = warps(sms)
    for p in plans:
        assert sum(p["sizes"]) <= POINT_FACTOR_BUDGET and max(p["sizes"]) <= MAX_PREFIX, name
    if name == "R1":
        a, b = plans
        assert (a["F"], b["F"]) == (40, 41)
        assert a["kernel"] == b["kernel"] == 5 and a["cached"] and not b["cached"]
        assert not a["dynamic"] and not b["dynamic"]
        assert {0, 1, 31, 33} <= set(a["sizes"]) and {0, 1, 31, 33} <= set(b["sizes"])
    elif name == "R2":
        (p,) = plans
        assert p["kernel"] == 5 and p["F"] > W and p["dynamic"] and not p["cached"] and max(p["sizes"]) <= 97
        assert p["ctr_advance"] == p["num_tiles"] + p["grid"] * WARPS_PER_CTA
    elif name == "R3":
        assert [p["acc_slots"] for p in plans] == [1, 2, 4, 8, 16]
        assert all(p["kernel"] == 5 and p["F"] == 1 and not p["dynamic"] for p in plans)
    elif name == "R4":
        (p,) = plans
        assert p["kernel"] == 5 and p["graph"] and not p["dynamic"]
        assert sum(max(1, -(-n // 32) // 4) for n in p["sizes"]) > W  # the item budget binds: the inlier fractions size the items
        q, _ = learn(p, [r * n for r, n in zip(CALIB_FRACTIONS, p["sizes"])])
        assert q["num_tiles"] != p["num_tiles"] and q["graph"] and not q["dynamic"]
    elif name == "R5":
        (p,) = plans
        assert p["kernel"] == 3 and p["tile_size"] == 128 and chunk_sizes(p) == [128] and not p["dynamic"]
    elif name == "R6":
        (p,) = plans
        assert p["kernel"] == 3 and p["tile_size"] == 128 and p["dynamic"]
        assert p["ctr_advance"] == p["num_tiles"]
    elif name == "R7":
        (p,) = plans
        assert p["kernel"] == 3 and p["tile_size"] == 2048 and chunk_sizes(p) == [128, 512, 2048] and p["dynamic"]
        assert sum(p["sizes"]) > 6 * W * 2048
        assert set(BOUNDARY) | {0, 1, 31, 33} <= set(p["sizes"])
        # the round boundary is crossed inside 2048-point items: factors of 481..2049 points in the head of the sweep
        head = [n for n, c in zip(p["sizes"], p["chunks"]) if c == 2048]
        assert {481, 991, 2049} <= set(head)
    elif name in ("R8", "R9"):
        (p,) = plans
        assert p["kernel"] == 3 and p["dynamic"]
    elif name == "R10":
        wave, queue = plans
        assert wave["kernel"] == queue["kernel"] == 5 and wave["gicp"] and queue["gicp"]
        assert not wave["dynamic"] and queue["dynamic"] and queue["F"] > W
        assert queue["ctr_advance"] == queue["num_tiles"]
    else:
        raise KeyError(name)
