"""numpy restatement of K11's contract (csrc/k11_field_grad.cu, DESIGN §3 "Interpolate VJP"): the gradient of
sum_q gphi[q] phi(x_q) + ggrad[q] . grad(x_q) with respect to a field's node values, in the stated summation order.  Written from the
contract: the rows N_j and D_jk are restated from the shape functions' structure (as tests/hessian_ref.py does), the segment sums are
K10's R (mesh_distance_grad_ref.segment_sums), and the node fold is built from the cell table."""
import numpy as np

from hessian_ref import CORNERS, X_EDGES, Y_EDGES, Z_EDGES
from mesh_distance_grad_ref import segment_sums

DBL_MAX = np.finfo(np.float64).max
UINT32_MAX = 0xFFFFFFFF
C64, E64 = 0.015625, 9.0 / 64.0


def locate(mn, mx, cell, inv, res, cmap, x):
    """K2's cell lookup: (valid, kept cell index, c0[n, 3], c1[n, 3]); the index clamped to n - 1 on each axis"""
    mn, mx, cell, inv = (np.asarray(a, np.float64) for a in (mn, mx, cell, inv))
    res = np.asarray(res, np.uint64)
    x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        valid = ((mn <= x) & (x <= mx)).all(axis=1)
        mi = np.zeros((len(x), 3), np.uint64)
        mi[valid] = ((x[valid] - mn) * inv).astype(np.uint64)
        mi = np.minimum(mi, res - 1)
        lin = res[1] * res[0] * mi[:, 2] + res[0] * mi[:, 1] + mi[:, 0]
        c = np.asarray(cmap, np.uint64)[lin] if cmap is not None else lin
        valid &= c != UINT32_MAX
        lo = mn + mi.astype(np.float64) * cell
        hi = lo + cell
        denom = hi - lo
        c0, c1 = 2.0 / denom, (hi + lo) / denom
    return valid, np.where(valid, c, 0).astype(np.int64), c0, c1


def rows(X, Y, Z):
    """N[n, 32] and the scaled derivative rows D[n, 32, 3] at xi = (X, Y, Z), in K2's operation order"""
    with np.errstate(all="ignore"):
        v = (X, Y, Z)
        sq = [a * a for a in v]
        L = [{-1: 1.0 - a, 1: 1.0 + a} for a in v]
        L3 = [{-1: 1.0 - 3.0 * a, 1: 1.0 + 3.0 * a} for a in v]
        x2, y2, z2 = sq
        facc = 1.0 / 64.0 * (9.0 * (x2 + y2 + z2) - 19.0)
        big = [9.0 * (3.0 * x2 + y2 + z2) - 19.0, 9.0 * (x2 + 3.0 * y2 + z2) - 19.0, 9.0 * (x2 + y2 + 3.0 * z2) - 19.0]   # A, B, C
        s18 = [18.0 * a for a in v]
        sA = [{-1: s18[a] - big[a], 1: s18[a] + big[a]} for a in range(3)]              # xmA / xpA ...
        one_m2 = [1.0 - q for q in sq]
        f = [9.0 / 64.0 * q for q in one_m2]
        fs = [{s: f[a] * L3[a][s] for s in (-1, 1)} for a in range(3)]                    # fxm / fxp ...
        t = [3.0 - 9.0 * q for q in sq]
        two = [2.0 * a for a in v]
        dP = [{-1: -t[a] - two[a], 1: t[a] - two[a]} for a in range(3)]                   # mX / pX ...
        P = [{s: one_m2[a] * L3[a][s] for s in (-1, 1)} for a in range(3)]               # Xm / Xp ...
        N, D = [], []
        for s in CORNERS:
            Lx, Ly, Lz = L[0][s[0]], L[1][s[1]], L[2][s[2]]
            N.append(facc * (Lx * Ly) * Lz)
            D.append([(sA[0][s[0]] * (Ly * Lz)) * C64, ((Lx * Lz) * sA[1][s[1]]) * C64, ((Lx * Ly) * sA[2][s[2]]) * C64])
        for a, edges in ((0, X_EDGES), (1, Y_EDGES), (2, Z_EDGES)):
            b, c = [k for k in range(3) if k != a]
            for s in edges:
                S = s[a]
                Lb, Lc = L[b][s[b]], L[c][s[c]]
                N.append(fs[a][S] * (Lb * Lc))
                d = [None] * 3
                d[a] = (dP[a][S] * (Lb * Lc)) * E64
                d[b] = ((P[a][S] if s[b] > 0 else -P[a][S]) * Lc) * E64
                d[c] = ((P[a][S] if s[c] > 0 else -P[a][S]) * Lb) * E64
                D.append(d)
        N = np.stack(N, axis=1)
        D = np.stack([np.stack(d, axis=1) for d in D], axis=1)
    return N, D


def contributions(N, D, c0, gphi, ggrad):
    """the contribution of each query to each slot, [n, 32]: the present terms gphi*N_j, (g0*c0x)*D_j0, (g1*c0y)*D_j1, (g2*c0z)*D_j2,
    the first one as is and the others added left to right"""
    with np.errstate(all="ignore"):
        t = None
        if gphi is not None:
            t = np.asarray(gphi, np.float64)[:, None] * N
        if ggrad is not None:
            a = np.asarray(ggrad, np.float64).reshape(-1, 3) * c0
            for k in range(3):
                term = a[:, k:k + 1] * D[:, :, k]
                t = term if t is None else t + term
    return t


def interpolate_vjp(mn, mx, cell, inv, res, nodes, cells, cmap, x, gphi=None, ggrad=None):
    """grad_nodes[n_nodes] in the contract's order.  cells: [n_cells_kept, 32] node ids; cmap: [nx*ny*nz] (UINT32_MAX = removed) or None"""
    nodes = np.asarray(nodes, np.float64)
    cells = np.asarray(cells, np.int64).reshape(-1, 32)
    x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
    out = np.zeros(len(nodes))
    valid, c, c0, c1 = locate(mn, mx, cell, inv, res, cmap, x)
    if len(cells):
        valid &= ~(nodes[cells] == DBL_MAX).any(axis=1)[c]
    key = np.where(valid, c + 1, 0)
    perm = np.argsort(key, kind="stable")
    perm = perm[key[perm] > 0]
    if len(perm) == 0:
        return out
    with np.errstate(all="ignore"):
        xi = c0[perm] * x[perm] - c1[perm]
    N, D = rows(xi[:, 0], xi[:, 1], xi[:, 2])
    t = contributions(N, D, c0[perm], None if gphi is None else np.asarray(gphi)[perm],
                      None if ggrad is None else np.asarray(ggrad).reshape(-1, 3)[perm])
    ids, R = segment_sums(key[perm], t)                             # R[k, j] of cell ids[k] - 1
    has = np.zeros(len(cells), bool); has[ids - 1] = True
    Rc = np.zeros((len(cells), 32)); Rc[ids - 1] = R
    flat = np.arange(32 * len(cells))
    node = cells.reshape(-1)
    order = np.lexsort((flat, node))                                 # node-major, ascending 32 * cell + j
    node, flat = node[order], flat[order]
    first = np.ones(len(node), bool); first[1:] = node[1:] != node[:-1]
    rank = np.arange(len(node)) - np.flatnonzero(first)[np.cumsum(first) - 1]
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        sel = rank == r
        cc, j = flat[sel] // 32, flat[sel] % 32
        use = has[cc]
        out[node[sel][use]] = out[node[sel][use]] + Rc[cc[use], j[use]]
    return out


def closed_form_cells(res, c):
    """the closed-form cell table (cell_node_id, csrc/dg_device.cuh) for the unreduced cells c of a grid of resolution res: [len(c), 32]
    node ids, int64.  Cell c is (i, j, k) with c = i + nx (j + ny k); slots 0-7 are the corners (di, dj, dk) = bits of the slot, slots 8-31
    the two inner nodes of each x, y and z edge"""
    nx, ny, nz = (int(r) for r in res)
    c = np.asarray(c, np.int64)
    k = c // (nx * ny); t = c - k * (nx * ny); j = t // nx; i = t - j * nx
    nv = (nx + 1) * (ny + 1) * (nz + 1)
    ne_x, ne_y = nx * (ny + 1) * (nz + 1), (nx + 1) * ny * (nz + 1)
    cols = []
    for jn in range(8):
        di, dj, dk = jn & 1, (jn >> 1) & 1, (jn >> 2) & 1
        cols.append((nx + 1) * (ny + 1) * (k + dk) + (nx + 1) * (j + dj) + i + di)
    for jn in range(8, 32):
        par, q = jn & 1, (jn - 8) >> 1
        grp, w = q >> 2, q & 3
        if grp == 0:                                                 # x edges at (j, k), (j, k + 1), (j + 1, k), (j + 1, k + 1)
            cols.append(nv + 2 * (nx * (ny + 1) * (k + (w & 1)) + nx * (j + (w >> 1)) + i) + par)
        elif grp == 1:                                               # y edges at (i, k), (i + 1, k), (i, k + 1), (i + 1, k + 1)
            cols.append(nv + 2 * ne_x + 2 * (ny * (nz + 1) * (i + (w & 1)) + ny * (k + (w >> 1)) + j) + par)
        else:                                                        # z edges at (i, j), (i, j + 1), (i + 1, j), (i + 1, j + 1)
            cols.append(nv + 2 * (ne_x + ne_y) + 2 * (nz * (nx + 1) * (j + (w & 1)) + nz * (i + (w >> 1)) + k) + par)
    return np.stack(cols, 1) if len(c) else np.zeros((0, 32), np.int64)


def _fold(out, node, flat, vals):
    """out[node] = ((out[node] + vals_1) + vals_2) + ... over each node's entries in ascending flat order"""
    order = np.lexsort((flat, node))
    node, vals = node[order], vals[order]
    first = np.ones(len(node), bool); first[1:] = node[1:] != node[:-1]
    rank = np.arange(len(node)) - np.flatnonzero(first)[np.cumsum(first) - 1]
    by_rank = np.argsort(rank, kind="stable")                       # step r adds every node's r-th entry: each node once per step
    bounds = np.concatenate([[0], np.cumsum(np.bincount(rank))]) if len(rank) else [0]
    for r in range(len(bounds) - 1):
        sel = by_rank[bounds[r]:bounds[r + 1]]
        out[node[sel]] = out[node[sel]] + vals[sel]


def interpolate_vjp_touched(mn, mx, cell, inv, res, nodes, cells, cmap, x, gphi=None, ggrad=None, chunk=1 << 17):
    """interpolate_vjp read from the rows of the cells that queries touch: cells is the [n_cells_kept, 32] table or a callable that returns
    the rows of an array of kept cell indices (closed_form_cells for a field made without a table); cmap None is the identity.  The node
    fold visits only the incidences of touched cells.  Skipping an empty segment gives the bits of adding +0.0 for it (the fold starts at
    +0.0 and a sum with a +0.0 operand is never -0.0), so this equals interpolate_vjp; it needs memory in the queries, not in the field."""
    rows_of = cells if callable(cells) else (lambda c, t=np.asarray(cells, np.int64).reshape(-1, 32): t[c])
    nodes = np.asarray(nodes, np.float64)
    x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
    out = np.zeros(len(nodes))
    valid, c, c0, c1 = locate(mn, mx, cell, inv, res, cmap, x)
    touched = np.unique(c[valid])
    if len(touched):
        has_max = (nodes[rows_of(touched)] == DBL_MAX).any(axis=1)
        valid &= ~has_max[np.minimum(np.searchsorted(touched, c), len(touched) - 1)]
    key = np.where(valid, c + 1, 0)
    perm = np.argsort(key, kind="stable")
    perm = perm[key[perm] > 0]
    if len(perm) == 0:
        return out
    gphi = None if gphi is None else np.asarray(gphi, np.float64)
    ggrad = None if ggrad is None else np.asarray(ggrad, np.float64).reshape(-1, 3)
    t = np.empty((len(perm), 32))
    for b in range(0, len(perm), chunk):
        p = perm[b:b + chunk]
        with np.errstate(all="ignore"):
            xi = c0[p] * x[p] - c1[p]
        N, D = rows(xi[:, 0], xi[:, 1], xi[:, 2])
        t[b:b + chunk] = contributions(N, D, c0[p], None if gphi is None else gphi[p], None if ggrad is None else ggrad[p])
    ids, R = segment_sums(key[perm], t)
    cc = ids.astype(np.int64) - 1
    node = rows_of(cc).astype(np.int64).reshape(-1)
    flat = (32 * cc[:, None] + np.arange(32)).reshape(-1)
    _fold(out, node, flat, R.reshape(-1))
    return out


def grid_vjp(grid, field_id, x, gphi=None, ggrad=None, nodes=None):
    """interpolate_vjp on a CubicLagrangeDiscreteGrid's field (its own node values unless `nodes` is given)"""
    d = grid._desc
    cmap = np.asarray(grid.m_cell_map[field_id], np.uint32)
    return interpolate_vjp(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.inv_cell_size[:], d.resolution[:],
                           grid.m_nodes[field_id] if nodes is None else nodes, grid.m_cells[field_id], cmap, x, gphi, ggrad)
