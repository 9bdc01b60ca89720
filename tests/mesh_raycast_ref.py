"""Restatement of K9's contract (discregrid_b200/csrc/k9_mesh_raycast.cu) in numpy: the first hit of rays on a triangle mesh, by a
brute-force loop over every triangle.  The tests hold the kernel (emulated and on the device) to it bit for bit.

Contract, restated:
  Rays (o, d), one interval [t_min, t_max] (no NaN, t_min <= t_max).  A ray misses if o or d is not finite, or d = 0.
  kz = the axis of largest |d_a| (first on ties), kx = (kz + 1) % 3, ky = (kx + 1) % 3, swapped when d[kz] < 0;
  Sx = d[kx] / d[kz], Sy = d[ky] / d[kz], Sz = 1 / d[kz].
  Per vertex P of (v0, v1, v2) = V[F[id]] -> (A, B, C): p = P - o, Px = p[kx] - Sx p[kz], Py = p[ky] - Sy p[kz], Pz = Sz p[kz].
  U = Cx By - Cy Bx, V = Ax Cy - Ay Cx, W = Bx Ay - By Ax; det = (U + V) + W; T = (U Az + V Bz) + W Cz; t = T / det;
  zl / zh = min / max of (Az, Bz, Cz) folded left to right with (a < b ? a : b) / (a < b ? b : a); tol = max(|zl|, |zh|) * 2^-49.
  Accept iff the edge functions share a sign (positive form), det != 0, the sheared bounding box of (A, B, C) holds the origin
  (not all x > 0, not all x < 0, the same for y), zl - tol <= t <= zh + tol and t_min <= t <= t_max.
  Result: the lexicographic minimum of (t, id) over the accepted triangles (t compared as numbers, so -0.0 == +0.0 and the lower id wins);
  t has the winner's bits; barycentric = (U / det, V / det, W / det); status = ENTER (1) when det > 0, LEAVE (2) when det < 0.
  A miss: status MISS (0), t = +inf, id = -1, barycentric NaN.
"""
import numpy as np

MISS, ENTER, LEAVE = 0, 1, 2


def _sel(a, k):
    """a[i, k[i]] for an (n, 3) array a."""
    return np.take_along_axis(a, k[:, None], axis=1)[:, 0]


def _min(a, b):
    return np.where(a < b, a, b)


def _max(a, b):
    return np.where(a < b, b, a)


def raycast(V, F, origins, directions, t_min=0.0, t_max=np.inf, chunk=None):
    """(t, triangle_id, barycentric, status) of every ray on the mesh (V, F), by a loop over all triangles."""
    V = np.ascontiguousarray(V, dtype=np.float64).reshape(-1, 3)
    F = np.ascontiguousarray(F, dtype=np.int64).reshape(-1, 3)
    o = np.ascontiguousarray(origins, dtype=np.float64).reshape(-1, 3)
    d = np.ascontiguousarray(directions, dtype=np.float64).reshape(-1, 3)
    n = len(o)
    t_out = np.full(n, np.inf)
    id_out = np.full(n, -1, dtype=np.int32)
    bary = np.full((n, 3), np.nan)
    st = np.zeros(n, dtype=np.int32)
    tri = V[F]                                                     # (T, 3 vertices, 3)
    T = len(F)
    if chunk is None:
        chunk = max(1, min(4096, 2_000_000 // max(T, 1)))           # about 16 MB per (rays x triangles) array
    with np.errstate(all="ignore"):
        for b in range(0, n, chunk):
            oc, dc = o[b:b + chunk], d[b:b + chunk]
            m = len(oc)
            ok = np.all(np.abs(oc) <= np.finfo(np.float64).max, axis=1) & np.all(np.abs(dc) <= np.finfo(np.float64).max, axis=1) \
                & np.any(dc != 0.0, axis=1)
            ad = np.abs(dc)
            kz = np.zeros(m, dtype=np.int64)
            kz = np.where(ad[:, 1] > ad[:, 0], 1, kz)
            kz = np.where(ad[:, 2] > _sel(ad, kz), 2, kz)
            kx = (kz + 1) % 3
            ky = (kx + 1) % 3
            neg = _sel(dc, kz) < 0.0
            kx, ky = np.where(neg, ky, kx), np.where(neg, kx, ky)
            dz = _sel(dc, kz)
            Sx = _sel(dc, kx) / dz
            Sy = _sel(dc, ky) / dz
            Sz = 1.0 / dz
            ox, oy, oz = _sel(oc, kx), _sel(oc, ky), _sel(oc, kz)
            X, Y, Z = [], [], []
            for k in range(3):
                P = tri[:, k, :]                                     # (T, 3)
                px = P[:, kx].T - ox[:, None]                        # (m, T)
                py = P[:, ky].T - oy[:, None]
                pz = P[:, kz].T - oz[:, None]
                X.append(px - Sx[:, None] * pz)
                Y.append(py - Sy[:, None] * pz)
                Z.append(Sz[:, None] * pz)
            U = X[2] * Y[1] - Y[2] * X[1]
            Vv = X[0] * Y[2] - Y[0] * X[2]
            W = X[1] * Y[0] - Y[1] * X[0]
            acc = ((U >= 0) & (Vv >= 0) & (W >= 0)) | ((U <= 0) & (Vv <= 0) & (W <= 0))
            det = (U + Vv) + W
            acc &= det != 0.0
            acc &= ~((X[0] > 0) & (X[1] > 0) & (X[2] > 0)) & ~((X[0] < 0) & (X[1] < 0) & (X[2] < 0))
            acc &= ~((Y[0] > 0) & (Y[1] > 0) & (Y[2] > 0)) & ~((Y[0] < 0) & (Y[1] < 0) & (Y[2] < 0))
            TT = (U * Z[0] + Vv * Z[1]) + W * Z[2]
            t = TT / det
            zl = _min(_min(Z[0], Z[1]), Z[2])
            zh = _max(_max(Z[0], Z[1]), Z[2])
            tol = _max(np.abs(zl), np.abs(zh)) * 2.0 ** -49
            acc &= (zl - tol <= t) & (t <= zh + tol)
            acc &= (t_min <= t) & (t <= t_max)
            acc &= ok[:, None]
            # lexicographic minimum of (t, id): the smallest t, then the first (lowest) id among those equal to it
            tk = np.where(acc, t, np.inf)
            best = tk.min(axis=1) if T else np.full(m, np.inf)
            hit = acc.any(axis=1) if T else np.zeros(m, dtype=bool)
            win = np.argmax(acc & (tk == best[:, None]), axis=1) if T else np.zeros(m, dtype=np.int64)
            r = np.nonzero(hit)[0]
            w = win[r]
            t_out[b + r] = t[r, w]
            id_out[b + r] = w
            dd = det[r, w]
            bary[b + r, 0] = U[r, w] / dd
            bary[b + r, 1] = Vv[r, w] / dd
            bary[b + r, 2] = W[r, w] / dd
            st[b + r] = np.where(dd > 0, ENTER, LEAVE)
    return t_out, id_out, bary, st


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float64:
        return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))
    return np.array_equal(a, b)


# ---- meshes and rays shared by the emulated and the GPU tests ------------------------------------------------------------------------
def grid_mesh(n=6, tilt=True):
    """A coplanar n x n grid of squares split into triangles, in the plane z = 0 or tilted off every axis."""
    u, v = np.meshgrid(np.arange(n + 1, dtype=np.float64), np.arange(n + 1, dtype=np.float64), indexing="ij")
    P = np.stack([u.ravel(), v.ravel(), np.zeros(u.size)], axis=1) / n
    if tilt:
        c, s = np.cos(0.7), np.sin(0.7)
        R1 = np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
        c, s = np.cos(0.4), np.sin(0.4)
        R2 = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        P = P @ (R2 @ R1).T
    F = []
    for i in range(n):
        for j in range(n):
            a = i * (n + 1) + j
            F += [[a, a + n + 1, a + 1], [a + 1, a + n + 1, a + n + 2]]
    return P, np.array(F, dtype=np.uint32)


def random_rays(V, n, rng, spread=1.5):
    """Origins spread around the mesh's box, directions uniform on the sphere."""
    lo, hi = V.min(axis=0), V.max(axis=0)
    c, h = 0.5 * (lo + hi), 0.5 * (hi - lo) + 1e-300
    o = c + (rng.random((n, 3)) * 2 - 1) * h * spread
    d = rng.normal(size=(n, 3))
    return o, d


def aimed_rays(V, F, n, rng, spread=1.5):
    """Origins around the mesh aimed at random points of random triangles (so most rays hit)."""
    o, _ = random_rays(V, n, rng, spread)
    tri = V[F[rng.integers(0, len(F), n)]]
    w = rng.random((n, 3))
    w /= w.sum(axis=1, keepdims=True)
    target = (w[:, :, None] * tri).sum(axis=1)
    return o, target - o


def axis_rays(V, n, rng):
    """Directions along one or two axes (the other components exactly zero), both signs."""
    o, _ = random_rays(V, n, rng, 1.2)
    d = np.zeros((n, 3))
    ax = rng.integers(0, 3, n)
    d[np.arange(n), ax] = rng.choice([-1.0, 1.0], n) * (1 + rng.random(n))
    two = rng.random(n) < 0.4
    ax2 = (ax + 1 + rng.integers(0, 2, n)) % 3
    d[np.arange(n)[two], ax2[two]] = rng.normal(size=two.sum())
    return o, d


def in_plane_rays(V, F, n, rng):
    """Rays that lie (to rounding) in the plane of a random triangle: origin on the plane, direction along it."""
    tri = V[F[rng.integers(0, len(F), n)]].astype(np.float64)
    e0, e1 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    a, b = rng.normal(size=(n, 1)) * 2, rng.normal(size=(n, 1)) * 2
    o = tri[:, 0] + a * e0 + b * e1
    p, q = rng.normal(size=(n, 1)), rng.normal(size=(n, 1))
    return o, p * e0 + q * e1


def leak_rays(V, F, inside):
    """From the interior point `inside` to every vertex and to every edge midpoint."""
    E = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]).astype(np.int64)
    E = np.unique(np.sort(E, axis=1), axis=0)
    targets = np.concatenate([V, 0.5 * (V[E[:, 0]] + V[E[:, 1]])])
    o = np.broadcast_to(np.asarray(inside, np.float64), targets.shape).copy()
    return o, targets - o
