"""numpy / scipy restatement of gb_min_cut's rule (include/glim_b200.h): participants, seed, roles, the k-NN graph and its
capacities, the network with the hard terminals contracted, scipy's maximum flow and a breadth-first search of its residual
graph from the seed.

numpy float64 operations round each operation and never fuse, which is the uncontracted fp64 rule of the device.  The
weights go through numpy's exp and acos, which may differ from the device's by an ulp, and so a capacity by 1."""
import math

import numpy as np
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import breadth_first_order, maximum_flow
from scipy.spatial import cKDTree

from tests import segment_oracle as so

F32, F64 = np.float32, np.float64
FREE, FOREGROUND, BACKGROUND, SEED = 0, 1, 2, 3
SCALE = 65536.0
KNN_CELL = 0.25
KEY_HALF = 1 << 20


def d2(p, c):
    """fp64 (dx^2 + dy^2) + dz^2 of fp32 points p (.., 3) to c"""
    e = np.asarray(p, F32).astype(F64) - np.asarray(c, F64)
    return (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]


def participants(xyz, c, background_mask_radius):
    """the finite points with fp64 d2 to c below (background_mask_radius + 1)^2, ascending"""
    xyz = np.asarray(xyz, F32)
    r1 = background_mask_radius + 1.0
    with np.errstate(invalid="ignore", over="ignore"):
        ok = so.finite(xyz) & (d2(xyz, c) < r1 * r1)
    return np.flatnonzero(ok)


def roles(xyz, c, seed_node, fg_r, bg_r):
    """the role of each node (fp32 positions of the participants, in node order)"""
    dd = d2(xyz, c)
    r = np.where(dd < fg_r * fg_r, FOREGROUND, np.where(dd > bg_r * bg_r, BACKGROUND, FREE))
    if seed_node >= 0:
        r[seed_node] = SEED
    return r


def knn_keyed(xyz):
    """the 0.25 m cell of the k-NN lies in the 21-bit range: floor(x * 4) + 2^20 in [0, 2^21) on every axis (fp64)"""
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(np.asarray(xyz, F32).astype(F64) * (1.0 / KNN_CELL)) + KEY_HALF
        return ((f >= 0) & (f < 2 * KEY_HALF)).all(axis=1)


def knn_rows(xyz, k):
    """row i = the k nearest keyed nodes of keyed node i by (exact fp64 d2, index), the query included; -1 pads; an unkeyed
    node's row is all -1.  cKDTree gives candidates, re-ranked exactly; a row whose candidates might cut a tie at the k-th
    distance is redone by brute force."""
    P = np.asarray(xyz, F32).astype(F64)
    m = len(P)
    rows = np.full((m, k), -1, np.int64)
    keyed = np.flatnonzero(knn_keyed(xyz))
    if len(keyed) == 0:
        return rows
    Q = P[keyed]
    kk = min(len(keyed), k + 8)
    _, cand = cKDTree(Q).query(Q, kk)
    C = keyed[np.asarray(cand).reshape(len(keyed), kk)]
    dd = d2(P[C].astype(F32), Q[:, None, :])
    order = np.lexsort((C, dd), axis=-1)
    C, dd = np.take_along_axis(C, order, -1), np.take_along_axis(dd, order, -1)
    kt = min(k, kk)
    rows[keyed, :kt] = C[:, :kt]
    if kk < len(keyed):  # a row whose candidate list may cut the k-th distance's tie is redone by brute force
        for r in np.flatnonzero(dd[:, kt - 1] >= dd[:, -1] * (1 - 1e-9)):
            i = keyed[r]
            di = d2(Q.astype(F32), P[i])
            rows[i] = keyed[np.lexsort((keyed, di))[:k]]
    return rows


def capacity(pa, na, pb, nb, distance_sigma, angle_sigma):
    """floor(2^16 exp(-d2 / (2 s_d^2)) exp(-theta^2 / (2 s_a^2))) per row of fp32 positions / normals; 0 for a NaN dot or a
    zero normal"""
    na64, nb64 = np.asarray(na, F32).astype(F64), np.asarray(nb, F32).astype(F64)
    with np.errstate(invalid="ignore"):
        dot = (na64[:, 0] * nb64[:, 0] + na64[:, 1] * nb64[:, 1]) + na64[:, 2] * nb64[:, 2]
    zero = (np.asarray(na, F32) == 0).all(axis=1) | (np.asarray(nb, F32) == 0).all(axis=1) | np.isnan(dot)
    th = np.arccos(np.minimum(np.abs(np.where(zero, 0.0, dot)), 1.0))
    e = np.asarray(pa, F32).astype(F64) - np.asarray(pb, F32).astype(F64)
    dd = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
    w = np.exp(-(dd / (2.0 * distance_sigma * distance_sigma))) * np.exp(-((th * th) / (2.0 * angle_sigma * angle_sigma)))
    q = np.floor(w * SCALE).astype(np.int64)
    return np.where(zero, 0, q).astype(np.int32)


def graph(xyz, nrm, k, distance_sigma, angle_sigma):
    """the undirected edges (E, 2) of node indices i < j, ascending, and their capacities"""
    rows = knn_rows(xyz, k)
    i = np.repeat(np.arange(len(rows)), k)
    j = rows.ravel()
    ok = (j >= 0) & (j != i)
    i, j = i[ok], j[ok]
    e = np.unique(np.stack([np.minimum(i, j), np.maximum(i, j)], axis=1), axis=0) if len(i) else np.zeros((0, 2), np.int64)
    xyz, nrm = np.asarray(xyz, F32), np.asarray(nrm, F32)
    q = capacity(xyz[e[:, 0]], nrm[e[:, 0]], xyz[e[:, 1]], nrm[e[:, 1]], distance_sigma, angle_sigma) if len(e) else np.zeros(0, np.int32)
    return e.astype(np.int64), q


def solve(m, edges, caps, role, foreground_weight):
    """the cut of rule 5-6 on m nodes: -> (selected node mask, cut_value).  The background nodes are contracted into one sink;
    scipy's maximum flow from the seed, then a breadth-first search of the residual graph from the seed."""
    seed = int(np.flatnonzero(role == SEED)[0])
    bg = role == BACKGROUND
    t = m  # the contracted sink
    node = np.where(bg, t, np.arange(m))
    u, v = node[edges[:, 0]], node[edges[:, 1]]
    keep = (u != v) & (caps > 0)
    u, v, q = u[keep], v[keep], caps[keep].astype(np.int64)
    fg = np.flatnonzero(role == FOREGROUND)
    F = int(math.floor(foreground_weight * SCALE))
    src = np.concatenate([u, v, np.full(len(fg) if F > 0 else 0, seed)])
    dst = np.concatenate([v, u, fg if F > 0 else np.zeros(0, np.int64)])
    cap = np.concatenate([q, q, np.full(len(fg) if F > 0 else 0, F, np.int64)])
    G = csr_matrix((cap.astype(np.int32), (src, dst)), shape=(m + 1, m + 1))
    G.sum_duplicates()
    if not bg.any():
        flow_value, R = 0, G
    else:
        r = maximum_flow(G, seed, t, method="dinic")
        flow_value = int(r.flow_value)
        F_ = r.flow.tocsr()
        R = (G - F_).tocsr()  # residual capacities (a reverse arc of G with flow f holds -(-f) = f)
    R.eliminate_zeros()
    R.data = np.where(R.data > 0, R.data, 0)
    R.eliminate_zeros()
    seen = np.zeros(m + 1, bool)
    seen[breadth_first_order(R, seed, directed=True, return_predecessors=False)] = True
    sel = seen[:m] & ~bg
    return sel, flow_value


def min_cut(xyz, nrm, c, distance_sigma=0.25, angle_sigma=math.radians(10), foreground_mask_radius=0.5, background_mask_radius=5.0,
            foreground_weight=10.0, k_neighbors=20):
    """-> dict(seed, status, num_points, num_foreground, num_background, num_edges, num_selected, cut_value, selected, edges,
    capacities) by the rule of gb_min_cut (edges as original indices)"""
    xyz, nrm = np.asarray(xyz, F32), np.asarray(nrm, F32)
    c = np.asarray(c, F64)
    idx = participants(xyz, c, background_mask_radius)
    m = len(idx)
    s = so.seed_of(xyz[idx], c) if m else -1
    out = {"seed": int(idx[s]) if s >= 0 else -1, "status": 0 if s >= 0 else 1, "num_points": m}
    P, N = xyz[idx], nrm[idx]
    role = roles(P, c, s, foreground_mask_radius, background_mask_radius)
    e, q = graph(P, N, k_neighbors, distance_sigma, angle_sigma)
    out.update(num_foreground=int((role == FOREGROUND).sum()), num_background=int((role == BACKGROUND).sum()), num_edges=len(e),
               edges=idx[e].astype(np.int32).reshape(-1, 2), capacities=q, role=role, nodes=idx)
    if s < 0:
        out.update(num_selected=0, cut_value=0, selected=np.zeros(0, np.int32))
        return out
    sel, flow = solve(m, e, q, role, foreground_weight)
    out.update(num_selected=int(sel.sum()), cut_value=flow, selected=idx[sel].astype(np.int32))
    return out


def cut_on_graph(n, nodes, role, edges, caps, foreground_weight):
    """the cut of rule 5-6 on a given graph: edges (E, 2) original indices, nodes the participants' original indices
    (ascending) with their roles -> (selected original indices, cut_value)"""
    pos = np.full(n, -1, np.int64)
    pos[nodes] = np.arange(len(nodes))
    e = pos[np.asarray(edges, np.int64).reshape(-1, 2)]
    sel, flow = solve(len(nodes), e, np.asarray(caps, np.int32), role, foreground_weight)
    return nodes[sel].astype(np.int32), flow
