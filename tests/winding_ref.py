"""numpy restatement of K5's numerical contract (discregrid_b200/csrc/k5_winding.cu): the library's atan2, the exact triangle term, the
cluster records and the cut walk, written from the contract alone in IEEE fp64 (numpy and Python floats never fuse a*b+c).  Plus the small
meshes the winding tests share.  Used by tests/test_winding_emulated.py and tests/test_gpu_winding.py."""
import math
import os

import numpy as np

FOUR_PI = 12.566370614359172
PI, PI_LO = 3.1415926535897931160E+00, 1.2246467991473531772E-16
PI_2, PI_4, PI3_4 = 1.5707963267948965580E+00, 7.8539816339744827900E-01, 2.3561944901923448370E+00
AT = [3.33333333333329318027e-01, -1.99999999998764832476e-01, 1.42857142725034663711e-01, -1.11111104054623557880e-01,
      9.09088713343650656196e-02, -7.69187620504482999495e-02, 6.66107313738753120669e-02, -5.83357013379057348645e-02,
      4.97687799461593236017e-02, -3.65315727442169155270e-02, 1.62858201153657823623e-02]
ATAN_HI = [4.63647609000806093515e-01, 7.85398163397448278999e-01, 9.82793723247329054082e-01, 1.57079632679489655800e+00]
ATAN_LO = [2.26987774529616870924e-17, 3.06161699786838301793e-17, 1.39033110312309984516e-17, 6.12323399573676603587e-17]


def _atan_pos(t):
    t = np.asarray(t, np.float64)
    with np.errstate(all="ignore"):
        cases = [(t < 0.4375, None), ((t >= 0.4375) & (t < 0.6875), 0), ((t >= 0.6875) & (t < 1.1875), 1),
                 ((t >= 1.1875) & (t < 2.4375), 2), (t >= 2.4375, 3)]
        x = t.copy(); hi = np.zeros_like(t); lo = np.zeros_like(t)
        x = np.where(cases[1][0], (2.0 * t - 1.0) / (2.0 + t), x)
        x = np.where(cases[2][0], (t - 1.0) / (t + 1.0), x)
        x = np.where(cases[3][0], (t - 1.5) / (1.0 + 1.5 * t), x)
        x = np.where(cases[4][0], -1.0 / t, x)
        for mask, k in cases[1:]:
            hi = np.where(mask, ATAN_HI[k], hi); lo = np.where(mask, ATAN_LO[k], lo)
        z = x * x; w = z * z
        s1 = z * (AT[0] + w * (AT[2] + w * (AT[4] + w * (AT[6] + w * (AT[8] + w * AT[10])))))
        s2 = w * (AT[1] + w * (AT[3] + w * (AT[5] + w * (AT[7] + w * AT[9]))))
        r = np.where(cases[0][0], x - x * (s1 + s2), hi - ((x * (s1 + s2) - lo) - x))
        return np.where(t < 2.0 ** -29, t, r)


def atan2(y, x):
    """the library's atan2, elementwise"""
    y = np.asarray(y, np.float64); x = np.asarray(x, np.float64)
    y, x = np.broadcast_arrays(y, x)
    with np.errstate(all="ignore"):
        ax, ay = np.abs(x), np.abs(y)
        nx, ny = np.signbit(x), np.signbit(y)
        q = ay / ax
        z = np.where(nx & (q < 2.0 ** -60), 0.0, _atan_pos(np.where(np.isfinite(q), q, 0.0)))
        r = PI - (z - PI_LO)
        out = np.where(nx, np.where(ny, -r, r), np.where(ny, -z, z))
        # special cases, lowest priority first
        out = np.where(q > 2.0 ** 60, np.where(ny, -PI_2, PI_2), out)
        out = np.where(ay == np.inf, np.where(ny, -PI_2, PI_2), out)
        inf_x = np.where(ay == np.inf, np.where(nx, np.where(ny, -PI3_4, PI3_4), np.where(ny, -PI_4, PI_4)),
                         np.where(nx, np.where(ny, -PI, PI), np.where(ny, -0.0, 0.0)))
        out = np.where(ax == np.inf, inf_x, out)
        out = np.where(ax == 0.0, np.where(ny, -PI_2, PI_2), out)
        out = np.where(ay == 0.0, np.where(nx, np.where(ny, -PI, PI), y), out)
        out = np.where(np.isnan(x) | np.isnan(y), x + y, out)
    return out


def det_den(tris, p):
    """the two arguments of the exact term's atan2: tris (T, 9) [v0 v1 v2], p (n, 3) -> det (n, T), den (n, T)"""
    v = tris[None, :, :]
    px, py, pz = p[:, 0:1], p[:, 1:2], p[:, 2:3]
    with np.errstate(all="ignore"):
        ax, ay, az = v[..., 0] - px, v[..., 1] - py, v[..., 2] - pz
        bx, by, bz = v[..., 3] - px, v[..., 4] - py, v[..., 5] - pz
        cx, cy, cz = v[..., 6] - px, v[..., 7] - py, v[..., 8] - pz
        la = np.sqrt(ax * ax + ay * ay + az * az); lb = np.sqrt(bx * bx + by * by + bz * bz); lc = np.sqrt(cx * cx + cy * cy + cz * cz)
        kx, ky, kz = by * cz - bz * cy, bz * cx - bx * cz, bx * cy - by * cx
        det = ax * kx + ay * ky + az * kz
        ab = ax * bx + ay * by + az * bz; bc = bx * cx + by * cy + bz * cz; ca = cx * ax + cy * ay + cz * az
        den = la * lb * lc + ab * lc + bc * la + ca * lb
    return det, den


def solid_angles(tris, p):
    """exact terms: tris (T, 9) [v0 v1 v2], p (n, 3) -> (n, T)"""
    det, den = det_den(tris, p)
    return 2.0 * atan2(det, den)


def fold(terms):
    """left fold from 0.0 along the last axis (np.cumsum is sequential)"""
    t = np.concatenate([np.zeros(terms.shape[:-1] + (1,)), terms], axis=-1)
    return np.cumsum(t, axis=-1)[..., -1]


def exact_w(tris, p):
    return fold(solid_angles(tris, np.asarray(p, np.float64).reshape(-1, 3))) / FOUR_PI


class Records:
    """leaves (T, 9) and clusters[m] = (left, right), each a tuple (p, n, M, r), the root at clusters[0][0]; `order` is the leaf order"""

    def __init__(self, V, F, order):
        self.V, self.F, self.order = np.asarray(V, np.float64), np.asarray(F, np.int64), np.asarray(order, np.int64)
        T = len(self.order)
        self.leaves = self.V[self.F[self.order]].reshape(T, 9)
        self.clusters = [[None, None] for _ in range(T)]
        self._build(0, T, 0, 0)

    def _leaf(self, t):
        v0, v1, v2 = (self.V[self.F[t, k]].tolist() for k in range(3))
        e0 = [v1[d] - v0[d] for d in range(3)]; e1 = [v2[d] - v0[d] for d in range(3)]
        N = [0.5 * (e0[1] * e1[2] - e0[2] * e1[1]), 0.5 * (e0[2] * e1[0] - e0[0] * e1[2]), 0.5 * (e0[0] * e1[1] - e0[1] * e1[0])]
        A = math.sqrt(N[0] * N[0] + N[1] * N[1] + N[2] * N[2])
        c = [(v0[d] + v1[d] + v2[d]) / 3.0 for d in range(3)]
        return dict(A=A, AC=[A * c[d] for d in range(3)], CS=c, N=N, p=c, M=[0.0] * 9, cnt=1.0)

    def _build(self, b, e, idx, side):
        if e - b == 1:
            return self._leaf(self.order[b])
        m = (b + e) >> 1
        L = self._build(b, m, m, 0); R = self._build(m, e, m, 1)
        s = dict(A=L["A"] + R["A"], cnt=L["cnt"] + R["cnt"], AC=[L["AC"][d] + R["AC"][d] for d in range(3)],
                 CS=[L["CS"][d] + R["CS"][d] for d in range(3)], N=[L["N"][d] + R["N"][d] for d in range(3)])
        s["p"] = [s["AC"][d] / s["A"] if s["A"] > 0.0 else s["CS"][d] / s["cnt"] for d in range(3)]
        s["M"] = [(L["M"][3 * j + k] + (L["p"][j] - s["p"][j]) * L["N"][k]) + (R["M"][3 * j + k] + (R["p"][j] - s["p"][j]) * R["N"][k])
                  for j in range(3) for k in range(3)]
        vv = self.leaves[b:e].reshape(-1, 3)
        with np.errstate(all="ignore"):
            d = vv - np.array(s["p"])
            d2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
        # the max is the fold r2 = (r2 < d2) ? d2 : r2 from 0.0: a NaN d2 compares false and is skipped (np.fmax), where np.max would
        # return NaN.  Matters for meshes with non-finite vertices: p~ = +-inf gives r_c = inf, not 0
        r2 = float(np.fmax.reduce(d2, initial=0.0))
        self.clusters[idx][side] = (s["p"], s["N"], s["M"], math.sqrt(r2))
        return s

    def as_array(self):
        """(T, 2, 16) as the library stores them (zeros where there is no record)"""
        out = np.zeros((len(self.order), 2, 16))
        for m, pair in enumerate(self.clusters):
            for side, c in enumerate(pair):
                if c is not None:
                    out[m, side] = c[0] + c[1] + c[2] + [c[3]]
        return out

    def cut(self, x, beta):
        """the cut of the walk at point x: a list of ("leaf", pos) and ("far", term) in increasing leaf position"""
        px, py, pz = x
        T = len(self.order)
        out, stack = [], [(0, T, 0, 0)]
        while stack:
            b, e, idx, side = stack.pop()
            if e - b == 1:
                out.append(("leaf", b)); continue
            p, n, M, r = self.clusters[idx][side]
            rx, ry, rz = p[0] - px, p[1] - py, p[2] - pz
            r2 = rx * rx + ry * ry + rz * rz
            br = beta * r
            if r2 > br * br:
                r3 = r2 * math.sqrt(r2); r5 = r3 * r2
                dip = n[0] * rx + n[1] * ry + n[2] * rz
                tr = M[0] + M[4] + M[8]
                m0 = M[0] * rx + M[1] * ry + M[2] * rz; m1 = M[3] * rx + M[4] * ry + M[5] * rz; m2 = M[6] * rx + M[7] * ry + M[8] * rz
                rmr = rx * m0 + ry * m1 + rz * m2
                out.append(("far", (dip / r3 + tr / r3) - (3.0 * rmr) / r5))
            else:
                m = (b + e) >> 1
                stack.append((m, e, m, 1)); stack.append((b, m, m, 0))
        return out

    def w(self, pts, beta):
        pts = np.asarray(pts, np.float64).reshape(-1, 3)
        res = np.empty(len(pts))
        for i, x in enumerate(pts):
            c = self.cut(x.tolist(), beta)
            pos = [v for k, v in c if k == "leaf"]
            lt = iter(solid_angles(self.leaves[pos], x[None, :])[0].tolist()) if pos else iter(())
            S = 0.0
            for k, v in c:
                S = S + (next(lt) if k == "leaf" else v)
            res[i] = S / FOUR_PI
        return res


# ---------------------------------------------------------------------------------------------------------------- meshes
def read_obj(path):
    V, F = [], []
    with open(path) as f:
        for line in f:
            p = line.split()
            if not p:
                continue
            if p[0] == "v":
                V.append([float(t) for t in p[1:4]])
            elif p[0] == "f":
                F.append([int(t.split("/")[0]) - 1 for t in p[1:4]])
    return np.array(V, np.float64), np.array(F, np.uint32)


def cut_top(V, F, frac=0.15):
    """the open mesh of the tests: every triangle whose centroid lies in the top `frac` of the y-extent removed"""
    cy = V[F].mean(axis=1)[:, 1]
    lo, hi = V[:, 1].min(), V[:, 1].max()
    return V, np.ascontiguousarray(F[cy <= hi - frac * (hi - lo)])


def soup(seed=7):
    """a triangle soup: a closed octahedron, one face duplicated, a fin sharing an edge with three triangles, and a loose triangle"""
    V = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [0.3, 0.2, 1.6], [1.5, 1.5, 1.5],
                  [1.9, 1.4, 1.2], [1.3, 1.9, 1.1]], np.float64)
    F = [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5], [0, 2, 4], [0, 4, 6], [7, 8, 9]]
    return V, np.array(F, np.uint32)


def query_points(V, n, seed, near=0):
    """n uniform points in the 10 %-padded bounding box, plus `near` points within 1e-3 of the diagonal from a vertex"""
    rng = np.random.default_rng(seed)
    lo, hi = V.min(0), V.max(0)
    pad = 0.1 * (hi - lo)
    p = lo - pad + rng.random((n, 3)) * (hi - lo + 2 * pad)
    if near:
        diag = float(np.linalg.norm(hi - lo))
        q = V[rng.integers(0, len(V), near)] + (rng.random((near, 3)) - 0.5) * 2e-3 * diag
        p = np.concatenate([p, q])
    return p


def ref_resource(root, name):
    p = os.path.join(root, "oracle", "_ref", "resources", name)
    return p if os.path.exists(p) else None
