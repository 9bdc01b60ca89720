"""numpy restatement of the refit's contract (discregrid_b200/csrc/k8_refit.cu, DESIGN §3 "Refit"): every record the refit writes, from
the new vertices V, the triangles F and the build's leaf order, vectorised per tree level.  The maxima that skip NaN are np.fmax;
std::max / std::min with their tie and NaN rules are _smax / _smin; the pseudonormal angle is refit_acos on winding_ref.atan2."""
import numpy as np

import winding_ref as wr

DBL_MAX = np.finfo(np.float64).max


def _smax(a, b):                 # std::max(a, b): a unless a < b
    return np.where(a < b, b, a)


def _smin(a, b):                 # std::min(a, b): a unless b < a
    return np.where(b < a, b, a)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _unit(a):
    l = np.sqrt(_dot(a, a))
    return a / l[..., None]


def refit_acos(x):
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        return wr.atan2(np.sqrt((1.0 - x) * (1.0 + x)), x)


def _down(v):
    f = v.astype(np.float32)
    return np.where(f.astype(np.float64) > v, np.nextafter(f, np.float32(-np.inf)), f)


def _up(v):
    f = v.astype(np.float32)
    return np.where(f.astype(np.float64) < v, np.nextafter(f, np.float32(np.inf)), f)


def _first_extreme(x, init, lower):
    """std::min (lower) / std::max fold of x from `init`: NaN skipped, ties (-0 / +0) kept by the first element"""
    x = x[~np.isnan(x)]
    if len(x) == 0:
        return init
    v = x.min() if lower else x.max()
    if (lower and not v < init) or (not lower and not v > init):
        return init
    return x[np.argmax(x == v)]


def order_from_tree(kids):
    """leaf position -> triangle id, from dg_mesh_tree's kids (pre-order: leaves appear in leaf order)"""
    return kids[kids[:, 0] == -1, 1].astype(np.int64)


def preorder_splits(T):
    """the split position m of every node of dg_mesh_tree's pre-order numbering (-1 for a leaf)"""
    out, stack = [], [(0, T)]
    while stack:
        b, e = stack.pop()
        if e - b == 1:
            out.append(-1); continue
        m = (b + e) >> 1
        out.append(m)
        stack.append((m, e)); stack.append((b, m))
    return np.array(out, np.int64)


def _levels(T):
    """internal nodes by depth: lists of (b, e, parent m, side) arrays, root first"""
    levels, cur = [], [(0, T, -1, 0)] if T > 1 else []
    while cur:
        a = np.array(cur, np.int64)
        levels.append(a)
        nxt = []
        for b, e, _, _ in cur:
            m = (b + e) >> 1
            if m - b > 1:
                nxt.append((b, m, m, 0))
            if e - m > 1:
                nxt.append((m, e, m, 1))
        cur = nxt
    return levels


def _leaf_parent(T):
    parent = np.full(T, -1, np.int64); side = np.zeros(T, np.int64)
    for lv in _levels(T):
        for b, e, _, _ in lv:
            m = (b + e) >> 1
            if m - b == 1:
                parent[b] = m; side[b] = 0
            if e - m == 1:
                parent[m] = m; side[m] = 1
    return parent, side


class Refit:
    """all records of refit(V) for the mesh (F, order); attributes as the library lays them out (leaf order / split positions)"""

    def __init__(self, V, F, order, nodef_stride=5):
        V = np.ascontiguousarray(V, np.float64); F = np.asarray(F, np.int64); order = np.asarray(order, np.int64)
        T = len(order); self.T = T
        with np.errstate(all="ignore"):
            self._bounds(V)
            tv = V[F[order]]                                     # (T, 3, 3) vertices at each leaf position
            a, b, c = tv[:, 0], tv[:, 1], tv[:, 2]
            self._leaves(a, b, c, order)
            self._normals(V, F, order)
            self._tree(V, F, order, tv, nodef_stride)

    # ---- centre and half extent
    def _bounds(self, V):
        lo = np.array([_first_extreme(V[:, d], DBL_MAX, True) for d in range(3)])
        hi = np.array([_first_extreme(V[:, d], -DBL_MAX, False) for d in range(3)])
        c = 0.5 * (lo + hi)
        he = 0.0
        for d in range(3):
            he = float(_smax(he, _smax(hi[d] - c[d], c[d] - lo[d])))
        finite = bool(np.isfinite(V).all())
        if not finite or not np.isfinite(he):
            he = np.inf
            c = np.where(np.isfinite(c), c, 0.0)
        self.center, self.half_extent, self.finite = c, he, finite

    # ---- leaf records (bvh_records.h)
    def _leaves(self, a, b, c, order):
        T = self.T
        e0, e1 = b - a, c - a
        a00, a01, a11 = _dot(e0, e0), _dot(e0, e1), _dot(e1, e1)
        det = np.abs(a00 * a11 - a01 * a01)
        L = np.zeros((T, 16))
        L[:, 0:3], L[:, 3:6], L[:, 6:9] = a, e0, e1
        L[:, 9], L[:, 10], L[:, 11], L[:, 12], L[:, 13], L[:, 14] = a00, a01, a11, det, 1 / det, (a00 - 2 * a01) + a11
        Lb = L.view(np.uint64)
        Lb[:, 15] = order.astype(np.int64).astype(np.uint64) & np.uint64(0xffffffff)
        self.leaves = Lb
        ctr = self.center
        f = np.zeros((T, 16), np.float32)
        f[:, 0:3] = (a - ctr).astype(np.float32); f[:, 3:6] = e0.astype(np.float32); f[:, 6:9] = e1.astype(np.float32)
        e2 = e1 - e0
        n3 = np.stack([e0[:, 1] * e1[:, 2] - e0[:, 2] * e1[:, 1], e0[:, 2] * e1[:, 0] - e0[:, 0] * e1[:, 2], e0[:, 0] * e1[:, 1] - e0[:, 1] * e1[:, 0]], 1)
        f[:, 9], f[:, 10], f[:, 11] = a00.astype(np.float32), a01.astype(np.float32), a11.astype(np.float32)
        f[:, 12] = _dot(e2, e2).astype(np.float32)
        s = _smax(np.abs(n3[:, 0]), _smax(np.abs(n3[:, 1]), np.abs(n3[:, 2])))
        ok = (s > 0) & np.isfinite(s)
        ss = np.where(ok, s, 1.0)
        q = n3 / ss[:, None]
        ln = np.where(ok, s * np.sqrt((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]), 0.0)
        lpos = ln > 0
        f[:, 13:16] = np.where(lpos[:, None], (n3 / np.where(lpos, ln, 1.0)[:, None]).astype(np.float32), np.float32(0))
        self.leaves_f = f

    # ---- pseudonormals, per-leaf 7 x 3 blocks
    def _normals(self, V, F, order):
        T = len(F)
        a, b, c = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
        u, v = b - a, c - a
        x = np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1], -u[:, 0] * v[:, 2] + u[:, 2] * v[:, 0], u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], 1)
        pt = _unit(x)
        ang = np.stack([refit_acos(np.abs(_dot(_unit(b - a), _unit(c - a)))), refit_acos(np.abs(_dot(_unit(a - b), _unit(c - b)))),
                        refit_acos(np.abs(_dot(_unit(b - c), _unit(a - c))))], 1)
        acc = np.zeros((len(V), 3))
        terms = ang[:, :, None] * pt[:, None, :]                # (T, 3 slots, 3)
        for d in range(3):
            np.add.at(acc[:, d], F.reshape(-1), terms[:, :, d].reshape(-1))     # sequential, in (triangle, slot) order
        pv = _unit(acc)
        ea = np.stack([F[:, 0], F[:, 1], F[:, 0]], 1).reshape(-1); eb = np.stack([F[:, 1], F[:, 2], F[:, 2]], 1).reshape(-1)
        lo, hi = np.minimum(ea, eb), np.maximum(ea, eb)
        key = lo * (int(hi.max()) + 1) + hi
        idx = np.lexsort((np.arange(3 * T), key))                # by key, then (triangle, slot)
        ks = key[idx]
        start = np.r_[True, ks[1:] != ks[:-1]]
        gid = np.cumsum(start) - 1
        rank = np.arange(len(ks)) - np.flatnonzero(start)[gid]
        tri_sorted = idx // 3
        gsum = np.zeros((gid[-1] + 1, 3))
        for r in range(int(rank.max()) + 1):
            sel = rank == r
            if r == 0:
                gsum[gid[sel]] = pt[tri_sorted[sel]]
            else:
                gsum[gid[sel]] = gsum[gid[sel]] + pt[tri_sorted[sel]]
        pe = np.empty((3 * T, 3))
        pe[idx] = _unit(gsum)[gid]
        pe = pe.reshape(T, 3, 3)
        self.pn_tri, self.pn_edge, self.pn_vert = pt, pe, pv
        Fo = F[order]
        self.normals = np.concatenate([pv[Fo[:, 0]][:, None], pv[Fo[:, 1]][:, None], pv[Fo[:, 2]][:, None], pe[order], pt[order][:, None]], 1)

    # ---- sphere tree, child boxes, K5 clusters
    def _tree(self, V, F, order, tv, stride):
        T = self.T
        a, b, c = tv[:, 0], tv[:, 1], tv[:, 2]
        spheres = np.zeros((T, 8)); box = np.zeros((T, 12))
        clusters = np.zeros((T, 2, 16))
        # leaf sums (k8_leaf_sums)
        lS = (a + b) + c
        llo = _smin(_smin(_smin(np.full_like(a, DBL_MAX), a), b), c)
        lhi = _smax(_smax(_smax(np.full_like(a, -DBL_MAX), a), b), c)
        e0, e1 = b - a, c - a
        lN = 0.5 * np.stack([e0[:, 1] * e1[:, 2] - e0[:, 2] * e1[:, 1], e0[:, 2] * e1[:, 0] - e0[:, 0] * e1[:, 2], e0[:, 0] * e1[:, 1] - e0[:, 1] * e1[:, 0]], 1)
        lA = np.sqrt((lN[:, 0] * lN[:, 0] + lN[:, 1] * lN[:, 1]) + lN[:, 2] * lN[:, 2])
        lc = ((a + b) + c) / 3.0
        leaf = dict(S=lS, lo=llo, hi=lhi, A=lA, AC=lA[:, None] * lc, CS=lc, N=lN, p=lc, M=np.zeros((T, 9)), cnt=np.ones(T))
        node = {k: np.zeros_like(v) for k, v in leaf.items()}
        node["c"] = np.zeros((T, 3))
        # leaf spheres and leaf boxes in the parent's slots
        parent, side = _leaf_parent(T)
        sc = lc
        lr = _smax(_smax(np.sqrt(_dot(a - sc, a - sc)), np.sqrt(_dot(b - sc, b - sc))), np.sqrt(_dot(c - sc, c - sc)))
        lbox = np.concatenate([_smin(_smin(a, b), c), _smax(_smax(a, b), c)], 1)
        has = parent >= 0
        for s_ in (0, 1):
            sel = has & (side == s_)
            spheres[parent[sel], 4 * s_:4 * s_ + 3] = sc[sel]; spheres[parent[sel], 4 * s_ + 3] = lr[sel]
            box[parent[sel], 6 * s_:6 * s_ + 6] = lbox[sel]
        levels = _levels(T)

        def child(bb, ee):
            isleaf = (ee - bb) == 1
            mm = np.where(isleaf, bb, (bb + ee) >> 1)
            return {k: np.where(isleaf.reshape((-1,) + (1,) * (leaf[k].ndim - 1)), leaf[k][mm], node[k][mm]) for k in leaf}, isleaf

        for lv in reversed(levels):
            nb, ne = lv[:, 0], lv[:, 1]
            m = (nb + ne) >> 1
            L, Ll = child(nb, m); R, Rl = child(m, ne)
            S = L["S"] + R["S"]
            node["S"][m] = S
            node["c"][m] = S / (3.0 * (ne - nb))[:, None]
            node["lo"][m] = _smin(L["lo"], R["lo"]); node["hi"][m] = _smax(L["hi"], R["hi"])
            for s_, (X, Xl) in enumerate(((L, Ll), (R, Rl))):
                sel = ~Xl
                box[m[sel], 6 * s_:6 * s_ + 3] = X["lo"][sel]; box[m[sel], 6 * s_ + 3:6 * s_ + 6] = X["hi"][sel]
            A = L["A"] + R["A"]; cnt = L["cnt"] + R["cnt"]
            AC = L["AC"] + R["AC"]; CS = L["CS"] + R["CS"]; N = L["N"] + R["N"]
            p = np.where((A > 0.0)[:, None], AC / np.where(A > 0, A, 1.0)[:, None], CS / cnt[:, None])
            M = np.empty((len(m), 9))
            for j in range(3):
                for k in range(3):
                    M[:, 3 * j + k] = (L["M"][:, 3 * j + k] + (L["p"][:, j] - p[:, j]) * L["N"][:, k]) + \
                                      (R["M"][:, 3 * j + k] + (R["p"][:, j] - p[:, j]) * R["N"][:, k])
            for k_, v_ in (("A", A), ("cnt", cnt), ("AC", AC), ("CS", CS), ("N", N), ("p", p), ("M", M)):
                node[k_][m] = v_
        # radii: exact maxima over the node's vertices, NaN skipped
        r2s = np.zeros(T); r2k = np.zeros(T)
        for lv in levels:
            nb, ne = lv[:, 0], lv[:, 1]
            m = (nb + ne) >> 1
            n = ne - nb
            pos = np.repeat(nb, n) + (np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n))
            owner = np.repeat(m, n)
            vv = tv[pos]                                          # (P, 3, 3)
            dS = node["c"][owner][:, None, :] - vv
            dK = vv - node["p"][owner][:, None, :]
            qs = np.fmax.reduce(_dot(dS, dS), axis=1); qk = np.fmax.reduce(_dot(dK, dK), axis=1)
            starts = np.cumsum(n) - n
            r2s[m] = np.fmax(np.fmax.reduceat(qs, starts), 0.0)
            r2k[m] = np.fmax(np.fmax.reduceat(qk, starts), 0.0)
        for lv in levels:
            nb, ne, par, sd = lv[:, 0], lv[:, 1], lv[:, 2], lv[:, 3]
            m = (nb + ne) >> 1
            rec = np.concatenate([node["p"][m], node["N"][m], node["M"][m], np.sqrt(r2k[m])[:, None]], 1)
            for s_ in (0, 1):
                sel = (par >= 0) & (sd == s_)
                spheres[par[sel], 4 * s_:4 * s_ + 3] = node["c"][m[sel]]; spheres[par[sel], 4 * s_ + 3] = np.sqrt(r2s[m[sel]])
                clusters[par[sel], s_] = rec[sel]
            root = par < 0
            clusters[0, 0] = rec[root][0] if root.any() else clusters[0, 0]
        self.spheres, self.box, self.clusters = spheres, box, clusters
        self.wind_leaves = tv.reshape(T, 9)
        # fp32 node records
        ctr = self.center
        rec = np.zeros((T, 4 * stride), np.float32)
        rec[:, 0:3] = (spheres[:, 0:3] - ctr).astype(np.float32); rec[:, 3] = spheres[:, 3].astype(np.float32)
        rec[:, 4:7] = (spheres[:, 4:7] - ctr).astype(np.float32); rec[:, 7] = spheres[:, 7].astype(np.float32)
        for s_ in (0, 1):
            rec[:, 8 + 6 * s_:11 + 6 * s_] = _down(box[:, 6 * s_:6 * s_ + 3] - ctr)
            rec[:, 11 + 6 * s_:14 + 6 * s_] = _up(box[:, 6 * s_ + 3:6 * s_ + 6] - ctr)
        rec[0, 8:20] = 0
        self.nodes_f = rec

    def tree_spheres(self):
        """the spheres as dg_mesh_tree exports them ((2T - 1) x 8, pre-order, zeros at leaves)"""
        ms = preorder_splits(self.T)
        out = np.zeros((len(ms), 8))
        out[ms >= 0] = self.spheres[ms[ms >= 0]]
        return out
