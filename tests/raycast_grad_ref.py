"""numpy restatement of K12's contract (discregrid_b200/csrc/k12_raycast_grad.cu, DESIGN §3 "Ray-cast gradients"): the per-ray gradients
of the mesh cast (K9's hit) and of the level-set cast (K7's bracket) in the origins and directions, in the stated operation order, IEEE
fp64 without FMA, so that the device and the CPU emulation must equal these arrays bit for bit.  The vertex sums are K10's
(mesh_distance_grad_ref.grad_vertices) and the node sums K11's (interpolate_vjp_ref.interpolate_vjp)."""
import numpy as np

import interpolate_vjp_ref
import mesh_distance_grad_ref

DBL_MAX = np.finfo(np.float64).max
RAY_MISS = 0


def dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                     a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)


def _finite_nonzero(v):
    return np.isfinite(v) & (v != 0.0)


def mesh_ray_grads(V, F, d, t, tid, grad_t=None, grad_bary=None):
    """(g_o, g_d, valid) of the mesh cast; NULL upstreams are zeros"""
    V = np.asarray(V, np.float64); F = np.asarray(F, np.int64).reshape(-1, 3)
    d = np.ascontiguousarray(d, np.float64).reshape(-1, 3); t = np.asarray(t, np.float64); tid = np.asarray(tid, np.int64)
    n = len(d)
    gt = np.zeros(n) if grad_t is None else np.asarray(grad_t, np.float64)
    gb = np.zeros((n, 3)) if grad_bary is None else np.asarray(grad_bary, np.float64).reshape(-1, 3)
    T = F[np.where(tid >= 0, tid, 0)] if len(F) else np.zeros((n, 3), np.int64)
    v0, v1, v2 = V[T[:, 0]], V[T[:, 1]], V[T[:, 2]]
    with np.errstate(all="ignore"):
        nrm = cross(v1 - v0, v2 - v0)
        den, nn = dot(nrm, d), dot(nrm, nrm)
        valid = (tid >= 0) & _finite_nonzero(den) & _finite_nonzero(nn)
        w = (gb[:, 0:1] * (v2 - v1) + gb[:, 1:2] * (v0 - v2)) + gb[:, 2:3] * (v1 - v0)
        a = cross(nrm, w) / nn[:, None]
        s = (gt + dot(d, a)) / den
        go = a - s[:, None] * nrm
        gd = t[:, None] * go
    go = np.where(valid[:, None], go, 0.0)
    gd = np.where(valid[:, None], gd, 0.0)
    return go, gd, valid


def mesh_grad_vertices(F, n_vertices, tid, bary, go, valid):
    """K10's vertex sums of the contributions -(b_i * g_o) of the valid rays"""
    return mesh_distance_grad_ref.grad_vertices(F, n_vertices, np.where(valid, tid, -1), go, np.asarray(bary, np.float64).reshape(-1, 3))


def crossing_points(mn, mx, o, d, t_lo, status):
    """x_c = o + t_lo * d clamped to [mn, mx] as K7 clamps its samples; +inf for a miss"""
    mn, mx = np.asarray(mn, np.float64), np.asarray(mx, np.float64)
    o = np.ascontiguousarray(o, np.float64).reshape(-1, 3); d = np.ascontiguousarray(d, np.float64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        x = o + np.asarray(t_lo, np.float64)[:, None] * d
    x = np.where(x < mn, mn, np.where(x > mx, mx, x))
    return np.where((np.asarray(status) != RAY_MISS)[:, None], x, np.inf)


def field_ray_grads(d, t_lo, status, phi, grad, grad_t_lo=None, grad_t_hi=None):
    """(g_o, g_d, gphi, valid) of the level-set cast from K2's (phi, grad) at the crossing points"""
    d = np.ascontiguousarray(d, np.float64).reshape(-1, 3); t_lo = np.asarray(t_lo, np.float64)
    phi = np.asarray(phi, np.float64); grad = np.asarray(grad, np.float64).reshape(-1, 3)
    n = len(d)
    glo = np.zeros(n) if grad_t_lo is None else np.asarray(grad_t_lo, np.float64)
    ghi = np.zeros(n) if grad_t_hi is None else np.asarray(grad_t_hi, np.float64)
    with np.errstate(all="ignore"):
        den = dot(grad, d)
        valid = (np.asarray(status) != RAY_MISS) & np.isfinite(phi) & (phi != DBL_MAX) & _finite_nonzero(den)
        gphi = -(glo + ghi) / den
        go = gphi[:, None] * grad
        gd = t_lo[:, None] * go
    return (np.where(valid[:, None], go, 0.0), np.where(valid[:, None], gd, 0.0), np.where(valid, gphi, 0.0), valid)


def field_grad_nodes(mn, mx, cell, inv, res, nodes, cells, cmap, xc, gphi, valid):
    """K11's node sums over the crossing points of the valid rays with the upstream gphi"""
    x = np.where(np.asarray(valid)[:, None], xc, np.inf)
    return interpolate_vjp_ref.interpolate_vjp(mn, mx, cell, inv, res, nodes, cells, cmap, x, gphi, None)


same_bits = mesh_distance_grad_ref.same_bits
