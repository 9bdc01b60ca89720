"""numpy restatement of K13's contract (discregrid_b200/csrc/k13_isosurface_grad.cu, DESIGN §3 "Level-set gradients"): the gradient of K6's
vertex positions in a trainable field's node values, in the stated operation order, IEEE fp64 without FMA, so that the device and the CPU
emulation must equal these arrays bit for bit.  The lattice is isosurface_ref's, the lattice values at the endpoints come from the caller
(K2's value-only interpolate there) and the node sums are K11's (interpolate_vjp_ref.interpolate_vjp)."""
import numpy as np

import interpolate_vjp_ref
from isosurface_ref import MASK_OF_DIR

DBL_MAX = np.finfo(np.float64).max


def bad_edges(L, E):
    """how many edge ids are not edges of the lattice: lin(p) >= Np, or p + delta_d outside it on some axis"""
    E = np.asarray(E, np.uint64)
    lp = E // np.uint64(7)
    m = MASK_OF_DIR[(E % np.uint64(7)).astype(np.int64)]
    inside = lp < np.uint64(L.n_points)
    I, J, K = L.unlin(np.where(inside, lp, 0).astype(np.int64))
    ok = inside & (I + (m & 1) < L.np[0]) & (J + ((m >> 1) & 1) < L.np[1]) & (K + (m >> 2) < L.np[2])
    return int((~ok).sum())


def endpoints(L, E):
    """(x_p, x_q), each (n, 3): the lattice positions of the two ends of every edge (K6's lat_coord)"""
    E = np.asarray(E, np.int64)
    lp, dm = E // 7, MASK_OF_DIR[E % 7]
    ip = L.unlin(lp)
    xp = np.stack([L.coord(a, ip[a]) for a in range(3)], axis=1)
    xq = np.stack([L.coord(a, ip[a] + ((dm >> a) & 1)) for a in range(3)], axis=1)
    return xp, xq


def points(xp, xq):
    """the 2n queries of the node sums: query 2v = x_p of vertex v, 2v + 1 = x_q"""
    return np.stack([xp, xq], axis=1).reshape(-1, 3)


def vertex_grads(iso, fp, fq, xp, xq, gV):
    """(gphi_p, gphi_q, valid, t) per vertex from the endpoint values and the upstream gV (n, 3)"""
    fp, fq = np.asarray(fp, np.float64), np.asarray(fq, np.float64)
    gV = np.asarray(gV, np.float64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        delta = fq - fp
        t = (float(iso) - fp) / delta
        valid = (np.isfinite(fp) & (fp != DBL_MAX) & np.isfinite(fq) & (fq != DBL_MAX) & np.isfinite(delta) & (delta != 0.0) & np.isfinite(t))
        dx = xq - xp
        gt = (gV[:, 0] * dx[:, 0] + gV[:, 1] * dx[:, 1]) + gV[:, 2] * dx[:, 2]
        r = gt / delta
        gp = (t - 1.0) * r
        gq = -(t * r)
    return np.where(valid, gp, 0.0), np.where(valid, gq, 0.0), valid, t


def grad_nodes(mn, mx, cell, inv, res, nodes, cells, cmap, xp, xq, gp, gq, valid):
    """K11's node sums over the 2n endpoints, those of invalid vertices at +inf, with the upstream gphi alone"""
    x = points(np.where(valid[:, None], xp, np.inf), np.where(valid[:, None], xq, np.inf))
    g = np.stack([gp, gq], axis=1).reshape(-1)
    return interpolate_vjp_ref.interpolate_vjp(mn, mx, cell, inv, res, nodes, cells, cmap, x, g, None)
