"""numpy restatement of K2's Hessian mode (interpolate_kernel<true, true>, discregrid_b200/csrc/k2_interp.cu, header comment; DESIGN.md
section 3), written from the contract alone in IEEE fp64 (numpy never fuses a*b+c, like the kernel built with -fmad=false).  Used by
tests/test_k2_hessian_emulated.py, tests/test_gpu_k2_hessian.py and the `hessian` mode of tools/k2_fuzz.py."""
import numpy as np

DBL_MAX = np.finfo(np.float64).max
UINT32_MAX = 0xFFFFFFFF

# the 32 nodes in the order of the value sum: corners (sx, sy, sz), then the x-, y- and z-edges, each given by its three signs (the edge's
# own axis carries the sign s of its 1/3 position)
CORNERS = [(-1, -1, -1), (1, -1, -1), (-1, 1, -1), (1, 1, -1), (-1, -1, 1), (1, -1, 1), (-1, 1, 1), (1, 1, 1)]
X_EDGES = [(-1, -1, -1), (1, -1, -1), (-1, -1, 1), (1, -1, 1), (-1, 1, -1), (1, 1, -1), (-1, 1, 1), (1, 1, 1)]
Y_EDGES = [(-1, -1, -1), (-1, 1, -1), (1, -1, -1), (1, 1, -1), (-1, -1, 1), (-1, 1, 1), (1, -1, 1), (1, 1, 1)]
Z_EDGES = [(-1, -1, -1), (-1, -1, 1), (-1, 1, -1), (-1, 1, 1), (1, -1, -1), (1, -1, 1), (1, 1, -1), (1, 1, 1)]
NODES = [("c", s) for s in CORNERS] + [(0, s) for s in X_EDGES] + [(1, s) for s in Y_EDGES] + [(2, s) for s in Z_EDGES]
PAIRS = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]


def _neg(s, v):
    """a sign applied as an exact negation, as the kernel does"""
    return v if s > 0 else -v


def restate_hessian(mn, mx, cell, inv, res, nodes, cells, cmap, x):
    """numpy restatement of K2's Hessian, vectorised over the queries x[n, 3], in the kernel's operation order: the cell lookup, the
    per-axis (c0, c1) table, xi, the shape functions' second derivatives and the 32-term sums.  cells: [n_cells_kept, 32] node ids,
    cmap: [nx*ny*nz] (UINT32_MAX = removed) or None for the identity.  Returns hess[n, 3, 3]."""
    mn, mx, cell, inv = (np.asarray(a, np.float64) for a in (mn, mx, cell, inv))
    res = np.asarray(res, np.uint64)
    x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
    n = len(x)
    with np.errstate(all="ignore"):
        valid = ((mn <= x) & (x <= mx)).all(axis=1)
        mi = np.zeros((n, 3), np.uint64)
        mi[valid] = ((x[valid] - mn) * inv).astype(np.uint64)
        mi = np.minimum(mi, res - 1)
        lin = res[1] * res[0] * mi[:, 2] + res[0] * mi[:, 1] + mi[:, 0]
        c = np.asarray(cmap, np.uint64)[lin] if cmap is not None else lin
        valid &= c != UINT32_MAX
        c = np.where(valid, c, 0)
        coeff = np.zeros((n, 32))
        if len(cells):
            coeff = np.asarray(nodes, np.float64)[np.asarray(cells, np.int64)[c.astype(np.int64)]]
        missing = (coeff == DBL_MAX).any(axis=1)
        lo = mn + mi.astype(np.float64) * cell
        hi = lo + cell
        denom = hi - lo
        c0, c1 = 2.0 / denom, (hi + lo) / denom
        xi = c0 * x - c1
        X, Y, Z = xi[:, 0], xi[:, 1], xi[:, 2]
        sq = [X * X, Y * Y, Z * Z]
        L = [{-1: 1.0 - v, 1: 1.0 + v} for v in (X, Y, Z)]                                  # _1mx / _1px ...
        L3 = [{-1: 1.0 - 3.0 * v, 1: 1.0 + 3.0 * v} for v in (X, Y, Z)]                     # _1m3x / _1p3x ...
        A = 9.0 * (3.0 * sq[0] + sq[1] + sq[2]) - 19.0
        B = 9.0 * (sq[0] + 3.0 * sq[1] + sq[2]) - 19.0
        Cc = 9.0 * (sq[0] + sq[1] + 3.0 * sq[2]) - 19.0
        e18 = [18.0 * X, 18.0 * Y, 18.0 * Z]
        sA = [{-1: e18[0] - A, 1: e18[0] + A}, {-1: e18[1] - B, 1: e18[1] + B}, {-1: e18[2] - Cc, 1: e18[2] + Cc}]   # xmA / xpA ...
        P, dP, ddP, d2c, t18 = [], [], [], [], []
        for a, v in enumerate((X, Y, Z)):
            om = 1.0 - sq[a]
            t3m9 = 3.0 - 9.0 * sq[a]
            t2 = 2.0 * v
            P.append({-1: om * L3[a][-1], 1: om * L3[a][1]})                                  # Xm / Xp
            dP.append({-1: -t3m9 - t2, 1: t3m9 - t2})                                          # mX / pX
            ddP.append({-1: -2.0 + e18[a], 1: -2.0 - e18[a]})                                   # P'' = -2 - 18 s X
            d2c.append({-1: 18.0 * L3[a][-1], 1: 18.0 * L3[a][1]})                              # 18 (1 -+ 3X)
            t18.append({-1: e18[a] * L[a][-1], 1: e18[a] * L[a][1]})                             # 18X (1 -+ X)

        def LL(a, sa, b, sb):
            return L[a][sa] * L[b][sb]
        h = {k: np.zeros(n) for k in PAIRS}
        corner, edge = 0.015625, 9.0 / 64.0
        for j, (kind, s) in enumerate(NODES):
            cj = coeff[:, j]

            def add(k, d2, scale):
                h[k] = h[k] + cj * (d2 * scale)
            if kind == "c":
                sx, sy, sz = s
                add((0, 0), d2c[0][sx] * LL(1, sy, 2, sz), corner)
                add((1, 1), d2c[1][sy] * LL(0, sx, 2, sz), corner)
                add((2, 2), d2c[2][sz] * LL(0, sx, 1, sy), corner)
                add((0, 1), (_neg(sy, sA[0][sx]) + _neg(sx, t18[1][sy])) * L[2][sz], corner)
                add((0, 2), (_neg(sz, sA[0][sx]) + _neg(sx, t18[2][sz])) * L[1][sy], corner)
                add((1, 2), (_neg(sz, sA[1][sy]) + _neg(sy, t18[2][sz])) * L[0][sx], corner)
                continue
            a = kind                                            # the edge's axis; b < c the other two
            b, cc = [k for k in range(3) if k != a]
            sa, sb, sc = s[a], s[b], s[cc]
            add((a, a), ddP[a][sa] * LL(b, sb, cc, sc), edge)
            add(tuple(sorted((a, b))), _neg(sb, dP[a][sa]) * L[cc][sc], edge)
            add(tuple(sorted((a, cc))), _neg(sc, dP[a][sa]) * L[b][sb], edge)
            add((b, cc), _neg(sb * sc, P[a][sa]), edge)
        hess = np.zeros((n, 3, 3))
        for (a, b), v in h.items():
            H = (v * c0[:, a]) * c0[:, b]
            hess[:, a, b] = H
            hess[:, b, a] = H
        hess[~valid | missing] = 0.0
    return hess


def symmetric_bits(hess):
    """hess[:, a, b] and hess[:, b, a] are the same bits for every a, b"""
    return all(np.array_equal(hess[:, a, b].view(np.uint64), hess[:, b, a].view(np.uint64)) for a in range(3) for b in range(3))
