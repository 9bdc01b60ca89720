"""Numpy restatement of K10's contract (discregrid_b200/csrc/k10_distance_grad.cu, DESIGN §3 "Mesh distance gradients"): the barycentric
weights of the nearest point (tri_dist2's (s, t) on the winning leaf, k1_sdf.cu), the gradient with respect to the points, the contributions
to the vertex slots, the stable sort of the queries by triangle and the fixed summation shape of the vertex gradient.  IEEE fp64 operations
in the kernels' order, no FMA, so the device and the CPU emulation must equal these arrays bit for bit."""
import numpy as np

FAN = 32


def leaf_params(V, F, tri, x):
    """(s, t, entity) of tri_dist2 (k1_sdf.cu) for points x (n, 3) on the leaf records (bvh_records.h make_leaf_record) of triangles
    tri (n,); NaN and -1 where tri = -1"""
    V = np.asarray(V, np.float64); F = np.asarray(F, np.int64); x = np.asarray(x, np.float64); tri = np.asarray(tri)
    ok = tri >= 0
    T = F[np.where(ok, tri, 0)]
    v0, v1, v2 = V[T[:, 0]], V[T[:, 1]], V[T[:, 2]]
    with np.errstate(all="ignore"):
        e0, e1 = v1 - v0, v2 - v0
        a00 = e0[:, 0] * e0[:, 0] + e0[:, 1] * e0[:, 1] + e0[:, 2] * e0[:, 2]
        a01 = e0[:, 0] * e1[:, 0] + e0[:, 1] * e1[:, 1] + e0[:, 2] * e1[:, 2]
        a11 = e1[:, 0] * e1[:, 0] + e1[:, 1] * e1[:, 1] + e1[:, 2] * e1[:, 2]
        det = np.abs(a00 * a11 - a01 * a01)
        inv_det = 1 / det
        denom = a00 - 2 * a01 + a11
        d = v0 - x
        b0 = d[:, 0] * e0[:, 0] + d[:, 1] * e0[:, 1] + d[:, 2] * e0[:, 2]
        b1 = d[:, 0] * e1[:, 0] + d[:, 1] * e1[:, 1] + d[:, 2] * e1[:, 2]
        s0 = a01 * b1 - a11 * b0
        t0 = a01 * b0 - a00 * b1
        lower = s0 + t0 <= det
        sneg, tneg = s0 < 0, t0 < 0
        tmp1_2, tmp0_2 = a11 + b1, a01 + b0
        tmp1_6, tmp0_6 = a00 + b0, a01 + b1
        numer_2, numer_6 = tmp1_2 - tmp0_2, tmp1_6 - tmp0_6
        numer_1 = tmp1_2 - a01 - b0
        W = np.where
        chain_b1 = W(b1 >= 0, 0, W(-b1 >= a11, 2, 5))
        chain_b0 = W(b0 >= 0, 0, W(-b0 >= a00, 1, 3))
        ent_r4 = W(b0 < 0, W(-b0 >= a00, 1, 3), chain_b1)
        ent_r2 = W(tmp1_2 > tmp0_2, W(numer_2 >= denom, 1, 4), W(tmp1_2 <= 0, 2, W(b1 >= 0, 0, 5)))
        ent_r6 = W(tmp1_6 > tmp0_6, W(numer_6 >= denom, 2, 4), W(tmp1_6 <= 0, 1, W(b0 >= 0, 0, 3)))
        ent_r1 = W(numer_1 <= 0, 2, W(numer_1 >= denom, 1, 4))
        ent = W(lower, W(sneg, W(tneg, ent_r4, chain_b1), W(tneg, chain_b0, 6)), W(sneg, ent_r2, W(tneg, ent_r6, ent_r1)))
        region6 = ~lower & ~sneg & tneg
        numer = W(sneg, numer_2, W(tneg, numer_6, numer_1))
        num = W(ent == 3, -b0, W(ent == 5, -b1, W(ent == 4, numer, 0.0)))
        den = W(ent == 3, a00, W(ent == 5, a11, W(ent == 4, denom, 1.0)))
        q = num / den
        sF, tF = s0 * inv_det, t0 * inv_det
        omq = 1 - q
        s = W(ent == 6, sF, W(ent == 4, W(region6, omq, q), W(ent == 1, 1.0, W(ent == 3, q, 0.0))))
        t = W(ent == 6, tF, W(ent == 4, W(region6, q, omq), W(ent == 2, 1.0, W(ent == 5, q, 0.0))))
    s = W(ok, s, np.nan); t = W(ok, t, np.nan); ent = W(ok, ent, -1)
    return s, t, ent


def nearest_point(V, F, tri, s, t):
    """finish_query's v0 + s e0 + t e1 (left to right); rows with tri = -1 are NaN"""
    V = np.asarray(V, np.float64); F = np.asarray(F, np.int64); tri = np.asarray(tri)
    T = F[np.where(tri >= 0, tri, 0)]
    v0 = V[T[:, 0]]
    with np.errstate(all="ignore"):
        e0, e1 = V[T[:, 1]] - v0, V[T[:, 2]] - v0
        p = v0 + s[:, None] * e0 + t[:, None] * e1
    return np.where((tri >= 0)[:, None], p, np.nan)


def weights(s, t):
    """w = (fl(fl(1 - s) - t), s, t); NaN where s, t are"""
    with np.errstate(all="ignore"):
        return np.stack([(1.0 - s) - t, s, t], axis=1)


def grad_points(x, dist, near, tri, g):
    """gx = fl(fl(g / d) * fl(x - p)); +0.0 where tri == -1 or d == 0"""
    x = np.asarray(x, np.float64); near = np.asarray(near, np.float64); dist = np.asarray(dist, np.float64); g = np.asarray(g, np.float64)
    live = (np.asarray(tri) >= 0) & (dist != 0.0)
    with np.errstate(all="ignore"):
        s = g / dist
        gx = s[:, None] * (x - near)
    return np.where(live[:, None], gx, 0.0)


def contributions(gx, w):
    """c[q, i, k] = -(w[q, i] * gx[q, k])"""
    with np.errstate(all="ignore"):
        return -(w[:, :, None] * gx[:, None, :])


def sort_keys(tri):
    """the sort's keys: tri + 1, 0 for tri = -1"""
    tri = np.asarray(tri, np.int64)
    return np.where(tri >= 0, tri + 1, 0).astype(np.uint32)


def sort_perm(tri):
    """the queries stably sorted by key (numpy's stable argsort)"""
    return np.argsort(sort_keys(tri), kind="stable")


def tree_sum(Y, m):
    """the fixed tree over axis 1 of Y (G, 32, ...) with m[g] live entries per group: y_j += y_{j+s} for j multiple of 2s, j + s < m"""
    Y = Y.copy()
    s = 1
    while s < FAN:
        for j in range(0, FAN, 2 * s):
            live = j + s < m
            Y[live, j] = Y[live, j] + Y[live, j + s]
        s *= 2
    return Y[:, 0]


def segment_sums(seg, vals):
    """R of every segment: seg (L,) non-decreasing segment ids, vals (L, ...) in segment order.  Returns (ids, sums) of the segments."""
    seg = np.asarray(seg); vals = np.asarray(vals, np.float64)
    if len(seg) == 0:
        return seg, vals
    while True:
        first = np.ones(len(seg), bool)
        first[1:] = seg[1:] != seg[:-1]
        start = np.flatnonzero(first)
        sid = np.cumsum(first) - 1
        j = np.arange(len(seg)) - start[sid]                     # offset in the segment
        if j.max() == 0:
            return seg, vals
        gfirst = (j % FAN) == 0
        gid = np.cumsum(gfirst) - 1
        G = int(gid[-1]) + 1
        Y = np.zeros((G, FAN) + vals.shape[1:])
        Y[gid, j % FAN] = vals
        m = np.bincount(gid, minlength=G)
        vals = tree_sum(Y, m)
        seg = seg[gfirst]


def grad_vertices(F, n_vertices, tri, gx, w):
    """the vertex gradient in the stated order: per vertex, +0.0 plus the segment sums of its incidences (t, i), ascending 3t + i"""
    F = np.asarray(F, np.int64)
    tri = np.asarray(tri)
    out = np.zeros((n_vertices, 3))
    perm = sort_perm(tri)
    keys = sort_keys(tri)[perm]
    live = keys > 0
    perm, keys = perm[live], keys[live]
    c = contributions(gx, w)[perm]                               # (L, 3 slots, 3)
    ids, R = segment_sums(keys.astype(np.int64), c)
    if len(ids) == 0:
        return out
    tri_ids = ids - 1
    has = np.zeros(len(F), bool); has[tri_ids] = True
    Rt = np.zeros((len(F), 3, 3)); Rt[tri_ids] = R
    flat = np.arange(3 * len(F))
    vert = F.reshape(-1)
    order = np.lexsort((flat, vert))                             # vertex-major, ascending 3t + i
    vert, flat = vert[order], flat[order]
    first = np.ones(len(vert), bool); first[1:] = vert[1:] != vert[:-1]
    start = np.flatnonzero(first)
    rank = np.arange(len(vert)) - start[np.cumsum(first) - 1]
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        sel = rank == r
        t, i = flat[sel] // 3, flat[sel] % 3
        use = has[t]
        v = vert[sel][use]
        out[v] = out[v] + Rt[t[use], i[use]]
    return out


def same_bits(a, b):
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))
