#!/usr/bin/env python
"""Parity fuzzer for K5 (generalized winding numbers, discregrid_b200/csrc/k5_winding.cu) against the numpy restatement of its contract
(tests/winding_ref.py), bit for bit, any NaN equal to any NaN.  K5 is pure fp64 without a filter, so its valid range is all of IEEE:
  trees     T = 1, 2, 3 and 2^k - 1, 2^k, 2^k + 1 for k <= 12 (a perfect tree, T = 2^k, is the one whose walk fills the stack to stack_depth
            entries: a stack one entry short overruns there), and happy_buddha.obj when it is staged
  ties      k1_fuzz.make_case's coplanar grids, cubes and octahedra with queries on faces, edges, vertices and symmetry planes (w exactly 1/2,
            1/4, 1/8), stacked sheets with duplicated triangles, slivers, random soups; and meshes with a subtree of zero-area triangles only
  scales    k1_fuzz.scale_cases at 10^-24 .. 10^17 and 10^+-150, 10^+-300, centred and offset: r2, |r|^5, det and den overflow or go subnormal
  nonfinite k1_fuzz.awkward_case meshes with NaN / inf vertices, and NaN, +-inf and huge query coordinates
  atan2     one-triangle meshes with queries that take every branch of k5_atan2 (in-plane det = +-0 with den > 0, < 0, = 0; vertices;
            extended edges; heights on the normal through the centroid that put |det/den| one ulp either side of 7/16, 11/16, 19/16, 39/16;
            |det/den| > 2^60 and < 2^-60 with den < 0)
at beta = 1, 2, 3.5 and inf, and at point counts around the warp and block sizes (every prefix gives the same bits).  With the `dg` backend
also the winding sign mode, against the reference's unsigned distance (k1_fuzz.reference) and the restatement's w: dg_mesh_distance,
dg_sample_sdf over whole lattices and over ranges whose ends are off multiples of 32 and 128, dg_add_function_sdf_band, and the
pseudonormal bits again after switching back.

usage: tools/k5_fuzz.py [rounds=40] [seed=0] [lib=build/bin/libk5emu.so]
  rounds  tie-rich meshes (k1_fuzz.make_case); the other families are fixed lists
  lib     a build of tests/emu/k5_emu.cpp (the K5 translation unit compiled for the CPU), or `dg`: the product library through its C-ABI
          (dg_mesh_create, dg_mesh_tree for the leaf order, dg_mesh_winding_number, dg_mesh_set_sign_mode ...), i.e. the CUDA kernels
The functions are shared with tests/test_winding_emulated.py and tests/test_gpu_winding_hessian_fuzz.py."""
import ctypes as C
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import k1_fuzz  # noqa: E402
import winding_ref as wr  # noqa: E402

dp, u32p, i32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
DBL_MAX = np.finfo(np.float64).max
K5_THREADS = 128                                   # csrc/k5_winding.h
COUNTS = (1, 31, 32, 33, K5_THREADS - 1, K5_THREADS, K5_THREADS + 1, 2 * K5_THREADS + 1)
BETAS = (1.0, 2.0, 3.5, math.inf)
DG_SIGN_PSEUDONORMAL, DG_SIGN_WINDING = 0, 1
same = k1_fuzz._same


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


class EmuK5:
    """a build of tests/emu/k5_emu.cpp: the K5 kernels and launchers run on the CPU"""

    def __init__(self, so):
        self.name = os.path.basename(so)
        lib = self.lib = C.CDLL(so)
        lib.emu_winding_create.restype = C.c_void_p
        lib.emu_winding_create.argtypes = [dp, C.c_uint64, u32p, C.c_uint64]
        lib.emu_winding_destroy.argtypes = [C.c_void_p]
        lib.emu_winding_records.argtypes = [C.c_void_p, i32p, dp, dp]
        lib.emu_winding_number.argtypes = [C.c_void_p, dp, C.c_uint64, C.c_double, dp]

    def mesh(self, V, F):
        h = self.lib.emu_winding_create(_p(V, dp), len(V), _p(F, u32p), len(F))
        assert h
        return (h, len(F))

    def destroy(self, m):
        self.lib.emu_winding_destroy(m[0])

    def order(self, m):
        o = np.empty(m[1], np.int32)
        self.lib.emu_winding_records(m[0], _p(o, i32p), None, None)
        return o.astype(np.int64)

    def w(self, m, x, beta):
        x = np.ascontiguousarray(x, np.float64)
        out = np.full(len(x), -7.0)
        assert self.lib.emu_winding_number(m[0], _p(x, dp), len(x), beta, _p(out, dp)) == 0
        return out


class DgK5(k1_fuzz.DgK1):
    """the product library through its C-ABI: the CUDA kernels on the current device"""

    def mesh(self, V, F):
        return (super().mesh(V, F), len(F))

    def destroy(self, m):
        super().destroy(m[0])

    def order(self, m):
        n = 2 * m[1] - 1
        kids = np.empty((n, 2), np.int32)
        self.capi.check(self.lib.dg_mesh_tree(m[0], None, _p(kids, i32p)))
        return kids[kids[:, 0] == -1, 1].astype(np.int64)            # the leaves in pre-order: leaf position -> triangle id

    def w(self, m, x, beta):
        x = np.ascontiguousarray(x, np.float64)
        out = np.full(len(x), -7.0)
        self.capi.check(self.lib.dg_mesh_winding_number(m[0], _p(x, dp), len(x), C.c_double(beta), _p(out, dp)))
        return out

    def set_mode(self, m, mode, beta):
        self.capi.check(self.lib.dg_mesh_set_sign_mode(m[0], mode, C.c_double(beta)))

    def sample_range(self, m, g, sign, l0, l1):
        out = np.full(l1 - l0, np.nan)
        self.capi.check(self.lib.dg_sample_sdf(m[0], C.byref(g), C.c_double(sign), l0, l1, _p(out, dp)))
        return out


def backend(lib):
    return DgK5() if lib == "dg" else EmuK5(lib)


# ---------------------------------------------------------------------------------------------------------------- expected values
class Expect:
    """the restatement's w for one mesh in the leaf order the backend reports"""

    def __init__(self, V, F, order):
        self.V, self.F, self.order = V, F, order
        self.leaves = np.ascontiguousarray(V[F[order]].reshape(-1, 9))
        self._rec = None

    def w(self, x, beta, chunk=1 << 14):
        x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
        if beta == math.inf:
            step = max(1, chunk * 64 // max(1, len(self.leaves)))
            return np.concatenate([wr.exact_w(self.leaves, x[i:i + step]) for i in range(0, len(x), step)] or [np.zeros(0)])
        if self._rec is None:
            self._rec = wr.Records(self.V, self.F, self.order)
        return self._rec.w(x, beta)


def check_w(be, m, ex, x, betas, label, counts=()):
    """w of the backend == the restatement's, for each beta; and every prefix count gives the first bits -> (points, mismatches, first)"""
    total = bad = 0
    first = None
    for beta in betas:
        got = be.w(m, x, beta)
        want = ex.w(x, beta)
        ok = same(got, want)
        total += len(x); bad += int((~ok).sum())
        if not ok.all() and first is None:
            i = int(np.nonzero(~ok)[0][0])
            first = f"MISMATCH {label} beta={beta} x={x[i].tolist()!r}: w {got[i]!r} vs {want[i]!r}"
        for c in counts:
            if c <= len(x):
                okc = same(be.w(m, x[:c], beta), got[:c])
                total += c; bad += int((~okc).sum())
                if not okc.all() and first is None:
                    first = f"MISMATCH {label} beta={beta} count {c}: first bad point {int(np.nonzero(~okc)[0][0])}"
    return total, bad, first


# ---------------------------------------------------------------------------------------------------------------- cases
def soup(rng, T, size=0.05):
    """T small random triangles in the unit cube"""
    c = rng.random((T, 1, 3))
    V = (c + size * rng.standard_normal((T, 3, 3))).reshape(-1, 3)
    return np.ascontiguousarray(V), np.arange(3 * T, dtype=np.uint32).reshape(T, 3)


TREE_SIZES = sorted({1, 2, 3} | {t for k in range(2, 13) for t in (2 ** k - 1, 2 ** k, 2 ** k + 1)})


def tree_cases(seed=0, sizes=TREE_SIZES):
    """(label, V, F, points) per tree size; the points: uniform in the padded box, near vertices"""
    rng = np.random.default_rng(seed)
    for T in sizes:
        V, F = soup(rng, T)
        yield f"tree T={T}", V, F, wr.query_points(V, 160, seed=T, near=40)


def zero_area_case(rng):
    """a cube plus 9 zero-area triangles (repeated / collinear vertices) far along x, so that after the builder's sorts they fill whole
    subtrees: clusters whose area sum A is 0 take the plain mean of the centroids"""
    V, F = k1_fuzz.cube()
    base = np.array([10.0, 0.3, 0.7])
    Z = []
    for i in range(9):                                           # dyadic coordinates: e0 x e1 is exactly 0 for the collinear ones too
        p = base + [0.5 * i, 0.125 * i, -0.0625 * i]
        d = rng.integers(-3, 4, 3).astype(np.float64) + [0.5, 0.0, 0.0]
        Z.append([p, p + d, p + 2.0 * d] if i % 3 else [p, p, p + d])
    VZ = np.array(Z, np.float64).reshape(-1, 3)
    V2 = np.concatenate([V, VZ])
    F2 = np.concatenate([F, len(V) + np.arange(len(VZ), dtype=np.uint32).reshape(-1, 3)])
    x = np.concatenate([k1_fuzz.queries(rng, V2, F2), VZ, VZ + 1e-3])
    return np.ascontiguousarray(V2), np.ascontiguousarray(F2, np.uint32), np.ascontiguousarray(x)


def has_zero_area_subtree(V, F, order):
    """some subtree of more than one triangle has area sum 0 (the cluster record's CS / cnt branch)"""
    e0 = V[F[order, 1]] - V[F[order, 0]]; e1 = V[F[order, 2]] - V[F[order, 0]]
    zero = ~np.cross(e0, e1).any(1)

    def walk(b, e):
        if e - b == 1:
            return False
        m = (b + e) >> 1
        return bool(zero[b:e].all()) or walk(b, m) or walk(m, e)
    return walk(0, len(order))


def tie_cases(rounds, seed=0):
    """(label, V, F, points, k) of k1_fuzz.make_case, and every 7th round a mesh with a zero-area subtree"""
    rng = np.random.default_rng(seed)
    for k in range(rounds):
        V, F, x = k1_fuzz.make_case(rng, k)
        yield f"case {k} (kind {k % 7}, {len(F)} tris)", V, F, x, k
        if k % 7 == 6:
            V, F, x = zero_area_case(rng)
            yield f"case {k} zero-area subtree", V, F, x, None


SCALE_EXPONENTS = k1_fuzz.SCALE_EXPONENTS + (-300, -150, 150, 300)


def scale_cases(seed=0, exponents=SCALE_EXPONENTS):
    rng = np.random.default_rng(seed + 1)
    for label, V, F in k1_fuzz.scale_cases(seed, exponents):
        with np.errstate(over="ignore", invalid="ignore"):
            x = k1_fuzz.queries(rng, V, F, flat=0.25)
        yield label, V, F, x


LOST = np.array([[np.nan, 0.0, 0.0], [0.0, np.nan, 0.0], [np.nan] * 3, [np.inf, 0.0, 0.0], [-np.inf, 1.0, 2.0], [0.0, 0.0, -np.inf],
                 [np.inf, -np.inf, np.inf], [1e300, 0.0, 0.0], [-1e308, 1e308, 0.0], [DBL_MAX, DBL_MAX, DBL_MAX], [1e160, 1e160, 1e160]])


def nonfinite_cases():
    """k1_fuzz.awkward_case meshes as they are (with NaN, infinite and huge queries), then with a NaN or an infinite vertex planted"""
    for i, (n_tri, scale, offset, degenerate) in enumerate(k1_fuzz.AWKWARD):
        V, F, x, lost = k1_fuzz.awkward_case(n_tri, scale, offset, degenerate)
        x = np.ascontiguousarray(np.concatenate([x, lost, LOST]))
        yield f"awkward {n_tri} x{scale:g}+{offset:g}", V, F, x
        for v in (np.nan, np.inf, -np.inf):
            V2 = V.copy()
            V2[(i + 1) % len(V2), i % 3] = v
            if n_tri >= 3:
                V2[-1] = [np.nan, np.inf, 0.0] if v != v else [v, 0.0, -v]
            yield f"awkward {n_tri} x{scale:g} vertex {v}", np.ascontiguousarray(V2), F, x


ATAN2_BOUNDS = (7 / 16, 11 / 16, 19 / 16, 39 / 16)


def _ratio(tri, p):
    det, den = wr.det_den(tri[None, :], p)
    with np.errstate(all="ignore"):
        return det[:, 0], den[:, 0], np.abs(det[:, 0] / den[:, 0])


def _bisect(f, lo, hi, steps=200):
    """the adjacent doubles lo < hi at which the boolean f changes (f(lo) != f(hi) on entry)"""
    flo = f(lo)
    for _ in range(steps):
        mid = 0.5 * (lo + hi)
        if mid <= lo or mid >= hi:
            break
        if f(mid) == flo:
            lo = mid
        else:
            hi = mid
    return lo, hi


def _one_ulp_points(tri, p, t, rng, k=12):
    """points within k ulps of p (per coordinate) at which |det/den| is the double just below t and t or the double just above"""
    steps = rng.integers(-k, k + 1, (20000, 3)).astype(np.float64)
    cand = p[None, :] + steps * np.spacing(np.abs(p))[None, :]
    q = _ratio(tri, cand)[2]
    out = [cand[q == np.nextafter(t, 0.0)][:2], cand[q == t][:1], cand[q == np.nextafter(t, 4.0)][:2]]
    return [c for c in out if len(c)]


def normal_heights(tri, seed=0):
    """points on the normal through the centroid: the bracketing heights (and two more ulps each way) around every |det/den| bound of the
    reduction, on both sides of the height h0 where den changes sign (den > 0 above it, den < 0 below); and next to each pair, points a
    few ulps off the normal at which |det/den| is exactly one ulp below the bound, the bound, and one ulp above"""
    rng = np.random.default_rng(seed)
    v = tri.reshape(3, 3)
    c = v.mean(0)
    n = np.cross(v[1] - v[0], v[2] - v[0]); n = n / np.linalg.norm(n)
    L = float(np.linalg.norm(v - c, axis=1).max())

    def pts(h):
        h = np.atleast_1d(np.asarray(h, np.float64))
        return c[None, :] + h[:, None] * n[None, :]

    def den_pos(h):
        return bool(_ratio(tri, pts(h))[1][0] > 0.0)
    h0lo, h0hi = _bisect(den_pos, 1e-9 * L, 1e3 * L)
    hs, exact = [h0lo, h0hi], []
    for t in ATAN2_BOUNDS:
        for lo, hi in ((h0hi, 1e6 * L), (1e-12 * L, h0lo)):
            a, b = _bisect(lambda h: bool(_ratio(tri, pts(h))[2][0] < t), lo, hi)
            hs += [a, b, np.nextafter(a, -np.inf), np.nextafter(np.nextafter(a, -np.inf), -np.inf), np.nextafter(b, np.inf),
                   np.nextafter(np.nextafter(b, np.inf), np.inf)]
            exact += _one_ulp_points(tri, pts(b)[0], t, rng)
    hs += [2.0 ** -40 * L, 2.0 ** -70 * L, 2.0 ** -200 * L, 5e-324, 1e6 * L, 1e150 * L]
    hs = np.array(hs, np.float64)
    return np.ascontiguousarray(np.concatenate([pts(hs), pts(-hs)] + exact))


def atan2_cases():
    """(label, V, F, points) of one-triangle meshes (w = 2 atan2(det, den) / 4 pi) whose points between them take every branch of k5_atan2;
    `atan2_coverage` checks that they do"""
    tri = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    F = np.array([[0, 1, 2]], np.uint32)
    g = np.linspace(-0.5, 1.5, 9)
    plane = np.stack(np.meshgrid(g, g, [0.0], indexing="ij"), -1).reshape(-1, 3)
    on_edges = np.array([[t, 0.0, 0.0] for t in (-1.0, -0.25, 0.5, 1.25, 3.0)] + [[0.0, t, 0.0] for t in (-2.0, 0.5, 2.0)] +
                        [[t, 1.0 - t, 0.0] for t in (-1.0, 0.25, 0.5, 2.0)])
    for z0 in (0.0, -0.0):
        for flip in (False, True):
            V = tri.copy(); V[:, 2] = z0
            if flip:
                V = V[[0, 2, 1]]
            p = np.concatenate([plane, on_edges, V])
            p = np.concatenate([p, p * [1.0, 1.0, -1.0]])            # z = -0.0 queries
            yield f"one triangle z={z0} flip={flip} in plane", np.ascontiguousarray(V), F, np.ascontiguousarray(p)
    rng = np.random.default_rng(5)
    for i in range(4):
        V = rng.standard_normal((3, 3)) * 10.0 ** (3 * i - 3)
        yield f"one triangle {i} normal heights", np.ascontiguousarray(V), F, normal_heights(V.reshape(9), seed=i)
    # centroid at the origin, so that the tiniest heights survive: |det/den| < 2^-60 and in [2^-60, 2^-29) with den < 0
    V = np.array([[1.0, 0.0, 0.0], [-0.5, 0.75, 0.0], [-0.5, -0.75, 0.0]])
    h = np.array([2.0 ** -30, 2.0 ** -45, 2.0 ** -62, 2.0 ** -70, 2.0 ** -200, 2.0 ** -1074])
    p = np.zeros((2 * len(h), 3)); p[:, 2] = np.concatenate([h, -h])
    yield "one triangle centred, tiny heights", V, F, p
    # |det/den| far beyond 2^60 with den of either sign, and den exactly 0: from the origin, a = (1, 0, 0), b = (-1, 2, -2), c = (e, 0, 1)
    # give |a| = 1, |b| = 3, |c| = 1, a.b = -1, b.c = -2 (e below half an ulp of 1 and 2), so den = ((3 - 1) - 2) + 3e = 3e exactly, det = 2
    for e in (2.0 ** -70, -2.0 ** -70, 2.0 ** -62, -2.0 ** -1000, 0.0, -0.0):
        for s in (1.0, 2.0 ** -500, 2.0 ** 500):
            for flip in (False, True):
                V = np.array([[1.0, 0.0, 0.0], [-1.0, 2.0, -2.0], [e, 0.0, 1.0]]) * s
                if flip:
                    V = V[[0, 2, 1]]
                yield f"one triangle den={3 * e:g} scale {s:g} flip={flip}", np.ascontiguousarray(V), F, np.zeros((1, 3))


def atan2_coverage(cases):
    """the branches of k5_atan2 the points of `cases` take -> set of names"""
    seen = set()
    for _, V, F, x in cases:
        det, den, q = _ratio(V.reshape(9), x)
        zd = det == 0.0
        neg = np.signbit(den)
        for name, m in (("det=+0,den>0", zd & ~np.signbit(det) & (den > 0)), ("det=-0,den>0", zd & np.signbit(det) & (den > 0)),
                        ("det=+0,den<0", zd & ~np.signbit(det) & (den < 0)), ("det=-0,den<0", zd & np.signbit(det) & (den < 0)),
                        ("det=0,den=0", zd & (den == 0.0)), ("den=0,det!=0", ~zd & (den == 0.0)),
                        ("q>2^60", ~zd & (q > 2.0 ** 60) & np.isfinite(q)), ("q<2^-60,den<0", ~zd & neg & (q < 2.0 ** -60)),
                        ("2^-60<=q<2^-29,den<0", neg & (q >= 2.0 ** -60) & (q < 2.0 ** -29)), ("q<2^-29,den>0", ~zd & ~neg & (q < 2.0 ** -29))):
            if m.any():
                seen.add(name)
        for t in ATAN2_BOUNDS:
            for side, m in (("den>0", ~neg & (den != 0)), ("den<0", neg & (den != 0))):
                below, above = q[m][q[m] < t], q[m][q[m] >= t]
                if len(below) and len(above) and below.max() == np.nextafter(t, 0) and above.min() <= np.nextafter(t, 4):
                    seen.add(f"{t}+-ulp,{side}")
    return seen


ATAN2_BRANCHES = {"det=+0,den>0", "det=-0,den>0", "det=+0,den<0", "det=-0,den<0", "det=0,den=0", "den=0,det!=0", "q>2^60", "q<2^-60,den<0",
                  "2^-60<=q<2^-29,den<0", "q<2^-29,den>0"}


# ---------------------------------------------------------------------------------------------------------------- runs
def run_cases(be, cases, betas=BETAS, counts=(), log=print, max_points=None):
    """w on every case -> (meshes, points checked, mismatches).  max_points: beta = 1, 2, 3.5 on the first max_points points only (the
    restatement walks them in Python); beta = inf on all"""
    meshes = total = bad = 0
    for label, V, F, x, *_ in cases:
        V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32); x = np.ascontiguousarray(x, np.float64)
        m = be.mesh(V, F)
        try:
            ex = Expect(V, F, be.order(m))
            fin = [b for b in betas if b != math.inf]
            xs = x if max_points is None else x[:max_points]
            for bs, pts in (([math.inf] if math.inf in betas else [], x), (fin, xs)):
                if bs:
                    n, b, msg = check_w(be, m, ex, pts, bs, label, counts)
                    total += n; bad += b
                    if msg: log(msg)
        finally:
            be.destroy(m)
        meshes += 1
    return meshes, total, bad


def run_large(be, n=1 << 20, seed=0, log=print):
    """one call with n points at beta = inf on a mesh of a few dozen triangles (an open torus strip): many blocks -> (points, mismatches)"""
    rng = np.random.default_rng(seed)
    V, F = soup(rng, 40, size=0.2)
    x = np.ascontiguousarray(wr.query_points(V, n, seed=seed + 1))
    x[rng.integers(0, n, 64)] = V[rng.integers(0, len(V), 64)]                        # exactly on vertices
    m = be.mesh(V, F)
    try:
        got = be.w(m, x, math.inf)
        want = Expect(V, F, be.order(m)).w(x, math.inf)
    finally:
        be.destroy(m)
    ok = same(got, want)
    if not ok.all():
        i = int(np.nonzero(~ok)[0][0])
        log(f"MISMATCH {n} points: point {i} x={x[i].tolist()!r}: w {got[i]!r} vs {want[i]!r}")
    return n, int((~ok).sum())


def off_ranges(n):
    """[l_begin, l_end) ranges whose ends are off multiples of 32 and 128"""
    out = [(0, n)]
    for a, b in ((1, 33), (31, 161), (97, 383), (127, 129), (255, 5 * 128 + 3)):
        if b <= n:
            out.append((a, b))
    if n > 300:
        out.append((n - 257, n - 1))
    return out


def check_sign(be, V, F, x, k, beta, sign, label):
    """the winding sign mode through the C-ABI (backend `dg`) -> (values checked, mismatches, first mismatch)"""
    ref = k1_fuzz.reference(V, F)
    m = be.mesh(V, F)
    total = bad = 0
    first = []

    def tally(ok, what):
        nonlocal total, bad
        total += ok.size; bad += int((~ok).sum())
        if not ok.all() and not first:
            first.append(f"MISMATCH {label} beta={beta} sign={sign} {what}: first at {int(np.nonzero(~ok.reshape(len(ok), -1).all(1))[0][0])}")
    try:
        ex = Expect(V, F, be.order(m))
        be.set_mode(m, DG_SIGN_WINDING, beta)
        # dg_mesh_distance, signed: the unsigned query's distance with the sign of w, its nearest point, entity and triangle
        du, nu, eu, tu = ref.distance(x, signed=False)
        w = ex.w(x, beta)
        d, nr, e, t = be.distance(m[0], x, 1)
        tally(same(d, np.where(w > 0.5, -du, du)) & same(nr, nu).all(1) & (e == eu) & (t == tu), "dg_mesh_distance")
        d, _, _, t = be.distance(m[0], LOST, 1, near=False)
        tally((d == DBL_MAX) & (t == -1), "dg_mesh_distance without an accepted triangle")
        # the node pass: whole lattice and ranges off the warp / block multiples; the band form
        mn, mx, res = k1_fuzz.case_lattice(k if k is not None else 0, V)
        g = be.grid(mn, mx, res)
        nn = k1_fuzz.num_nodes(res)
        xs = be.node_positions(g, nn)
        dn = ref.distance(xs, signed=False)[0]
        wn = np.where(ex.w(xs, beta) > 0.5, -dn, dn)
        want = wn if sign == 1.0 else sign * wn
        for l0, l1 in off_ranges(nn):
            tally(same(be.sample_range(m, g, sign, l0, l1), want[l0:l1]), f"dg_sample_sdf [{l0}, {l1})")
        band = 1.5 * float(np.max(be.cell_size(g)))
        tally(same(be.sample(m[0], g, sign, nn, band), k1_fuzz.band_expect(wn, sign, band)), "dg_add_function_sdf_band")
        # back to the pseudonormal mode: the reference's signed distances again
        be.set_mode(m, DG_SIGN_PSEUDONORMAL, 2.0)
        n, b, msg = k1_fuzz.check_points(be, m[0], ref, x, label + " pseudonormal again")
        total += n; bad += b
        if msg and not first:
            first.append(msg)
    finally:
        be.destroy(m)
    return total, bad, (first[0] if first else None)


def run_sign(be, rounds, seed=0, log=print):
    """the winding sign mode on the tie-rich meshes -> (meshes, values checked, mismatches)"""
    meshes = total = bad = 0
    for i, (label, V, F, x, k) in enumerate(tie_cases(rounds, seed)):
        beta, sign = BETAS[i % len(BETAS)], (1.0, -1.0)[(i // 2) % 2]
        n, b, msg = check_sign(be, V, F, x, k, beta, sign, label)
        meshes += 1; total += n; bad += b
        if msg: log(msg)
    return meshes, total, bad


def run(be, rounds, seed=0, log=print, large=None):
    """every family of cases through backend `be`; with the `dg` backend the sign mode too -> (meshes, points, mismatches)"""
    acc = [0, 0, 0]

    def add(r):
        for i in range(3):
            acc[i] += r[i]
    add(run_cases(be, tree_cases(seed), betas=(2.0, math.inf), counts=COUNTS, log=log, max_points=60))
    buddha = wr.ref_resource(ROOT, "happy_buddha.obj")
    if buddha:
        V, F = wr.read_obj(buddha)
        add(run_cases(be, [("happy_buddha", V, F, wr.query_points(V, 300, seed=seed, near=100))], betas=(math.inf, 2.0), log=log, max_points=100))
    add(run_cases(be, tie_cases(rounds, seed), log=log, max_points=400))
    add(run_cases(be, scale_cases(seed), betas=(2.0, math.inf), log=log, max_points=150))
    add(run_cases(be, nonfinite_cases(), betas=BETAS, counts=(33, 129), log=log))
    add(run_cases(be, atan2_cases(), betas=(2.0, math.inf), log=log))
    if large:
        n, b = run_large(be, large, seed, log)
        acc[0] += 1; acc[1] += n; acc[2] += b
    if isinstance(be, DgK5):
        add(run_sign(be, rounds, seed, log))
    return tuple(acc)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 40
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else os.path.join(ROOT, "build", "bin", "libk5emu.so")
    missing = ATAN2_BRANCHES - atan2_coverage(atan2_cases())
    if missing:
        print("atan2 cases miss branches:", sorted(missing))
        return 1
    meshes, total, bad = run(backend(lib), rounds, seed)
    print(f"{meshes} meshes, {total} points, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
