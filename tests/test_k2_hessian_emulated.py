"""K2's Hessian mode (interpolate_kernel<true, true>) compiled for the CPU by tests/emu, against a numpy restatement of its numerical contract
(k2_interp.cu, header comment; DESIGN.md section 3), against exact rational second derivatives of the shape functions, and on cubic
polynomials, which the 32-node element reproduces.  numpy float64 is IEEE arithmetic without FMA, like the kernel built with -fmad=false, so
the restatement is compared bit for bit.  tests/test_gpu_k2_hessian.py holds the device to the same restatement."""
import ctypes as C
import os
from fractions import Fraction

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal
from hessian_ref import DBL_MAX, NODES, UINT32_MAX, restate_hessian, symmetric_bits  # noqa: F401 (test_gpu_k2_hessian imports them here)
from test_oracle_golden import read_cdf

LIB = os.path.join(ROOT, "build", "bin", "libk2hemu.so")
_dp, _u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)
EPS = np.finfo(np.float64).eps


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def nan_bits_equal(a, b):
    """bit for bit, any NaN equal to any NaN (device fp64 units and x86 differ in the NaN they produce)"""
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and bool(((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))).all())


def restate_grid(g, field, x):
    """restate_hessian on a field of a read_cdf dictionary"""
    return restate_hessian(g["mn"], g["mx"], g["cell"], g["inv"], g["res"], g["nodes"][field], g["cells"][field], g["cmap"][field], x)


class Emu:
    def __init__(self):
        if not os.path.exists(LIB):
            pytest.skip(f"{LIB} not built (make cpp)")
        self.lib = C.CDLL(LIB)
        self.lib.emu_field_create.restype = C.c_void_p
        self.lib.emu_field_create.argtypes = [_dp, _u32p, _dp, _u32p, C.c_uint64, _u32p]
        self.lib.emu_field_destroy.argtypes = [C.c_void_p]
        self.lib.emu_interpolate.argtypes = [C.c_void_p, _dp, C.c_uint64, _dp, _dp]
        self.lib.emu_interpolate_hessian.argtypes = [C.c_void_p, _dp, C.c_uint64, _dp, _dp, _dp]

    def field(self, gd, res, nodes, cells, cmap):
        """cells None: the closed-form connectivity of addFunction (n_cells_kept = nx*ny*nz)"""
        keep = (np.ascontiguousarray(gd, np.float64), np.ascontiguousarray(res, np.uint32), np.ascontiguousarray(nodes, np.float64),
                None if cells is None else np.ascontiguousarray(cells, np.uint32), None if cmap is None else np.ascontiguousarray(cmap, np.uint32))
        n_kept = int(np.prod(keep[1].astype(np.uint64))) if cells is None else len(keep[3])
        h = self.lib.emu_field_create(_p(keep[0], _dp), _p(keep[1], _u32p), _p(keep[2], _dp), _p(keep[3], _u32p), n_kept, _p(keep[4], _u32p))
        assert h
        return h, keep

    def hessian(self, h, x):
        x = np.ascontiguousarray(x, np.float64)
        n = len(x)
        phi, grad, hess = np.full(n, np.nan), np.full((n, 3), np.nan), np.full((n, 3, 3), np.nan)
        assert self.lib.emu_interpolate_hessian(h, _p(x, _dp), n, _p(phi, _dp), _p(grad, _dp), _p(hess, _dp)) == 0
        return phi, grad, hess

    def gradient(self, h, x):
        x = np.ascontiguousarray(x, np.float64)
        phi, grad = np.full(len(x), np.nan), np.full((len(x), 3), np.nan)
        assert self.lib.emu_interpolate(h, _p(x, _dp), len(x), _p(phi, _dp), _p(grad, _dp)) == 0
        return phi, grad


@pytest.fixture(scope="module")
def emu():
    return Emu()


def check_mode(emu, h, x, want_hess, strict=True):
    """the Hessian mode's phi / grad are the gradient mode's bits, its hess the restatement's, exactly symmetric"""
    phi, grad, hess = emu.hessian(h, x)
    p2, g2 = emu.gradient(h, x)
    assert bits_equal(phi, p2) and bits_equal(grad, g2)
    assert symmetric_bits(hess)
    assert (bits_equal if strict else nan_bits_equal)(hess, want_hess)
    sentinel = phi == DBL_MAX
    assert not hess[sentinel].view(np.uint64).any()                     # +0.0 everywhere at DBL_MAX
    return phi, grad, hess


FIXTURES = [("box", "box.cdf", 0, False), ("box", "box.cdf", 0, True), ("red", "ref_sphere_reduced.cdm", 0, False),
            ("red", "ref_sphere_reduced.cdm", 1, False), ("nr", "ref_sphere_noreduction.cdm", 1, False)]


@pytest.mark.parametrize("tag,path,field,closed", FIXTURES)
def test_hessian_mode_matches_restatement_on_fixtures(emu, orc, tag, path, field, closed):
    """plain and reduced fields, explicit and closed-form connectivity, the committed query points (out-of-domain and removed cells
    included); and the same bits for any prefix of the queries (counts that are not a multiple of 32 or 128)"""
    q = np.load(os.path.join(GOLDEN, "ref_grid_queries.npz"))
    g = read_cdf(os.path.join(GOLDEN, path))
    gd, res = orc.grid_desc(g["mn"], g["mx"], g["res"], g["cell"], g["inv"])
    h, _keep = emu.field(gd, res, g["nodes"][field], None if closed else g["cells"][field], None if closed else g["cmap"][field])
    try:
        x = np.ascontiguousarray(q[tag + "_x"])
        want = restate_grid(g, field, x)
        phi, _grad, hess = check_mode(emu, h, x, want)
        assert (phi == DBL_MAX).any() and (phi != DBL_MAX).any() and np.abs(hess).max() > 0
        for m in (1, 31, 33, 77, 127, 129):
            assert bits_equal(emu.hessian(h, x[:m])[2], hess[:m])
    finally:
        emu.lib.emu_field_destroy(h)


def random_field(orc, rng, res, extremes):
    """a random anisotropic field with ~15% of its cells removed; `extremes` coefficients planted at random nodes"""
    mn = rng.uniform(-2, 0, 3)
    mx = mn + rng.uniform(0.3, 3.0, 3)
    gd, r = orc.grid_desc(mn, mx, res)
    n_nodes = orc.num_nodes(r)
    nodes = rng.standard_normal(n_nodes) * 10.0 ** rng.integers(-3, 4)
    for v in extremes:
        nodes[rng.integers(0, n_nodes, max(1, n_nodes // 200))] = v
    full = orc.build_cells(r)
    keep = rng.random(len(full)) < 0.85
    cmap = np.full(len(full), UINT32_MAX, np.uint32)
    cmap[keep] = np.arange(keep.sum(), dtype=np.uint32)
    return gd, r, nodes, full[keep], cmap


def field_queries(rng, gd, res, n):
    """random points in the domain grown by 10%, node positions (on cell faces and edges), and NaN / inf rows"""
    mn, mx = gd[0:3], gd[3:6]
    span = mx - mn
    x = mn - 0.1 * span + rng.random((n, 3)) * 1.2 * span
    cell = gd[6:9]
    faces = mn + rng.integers(0, np.asarray(res) + 1, (n // 4, 3)) * cell
    odd = np.array([[np.nan, mn[1], mn[2]], [np.inf, 0, 0], [mn[0], -np.inf, mn[2]], mx, mn])
    return np.ascontiguousarray(np.concatenate([x, np.minimum(faces, mx), odd]))


@pytest.mark.parametrize("seed,extremes", [(0, ()), (1, (DBL_MAX,)), (2, (1e308, -1e308)), (3, (np.inf, -np.inf)), (4, (np.nan,)),
                                           (5, (DBL_MAX, 1e308, -1e308, np.inf, -np.inf, np.nan, -DBL_MAX))])
def test_hessian_mode_matches_restatement_on_random_fields(emu, orc, seed, extremes):
    rng = np.random.default_rng(seed)
    res = rng.integers(2, 7, 3)
    gd, r, nodes, cells, cmap = random_field(orc, rng, res, extremes)
    h, _keep = emu.field(gd, r, nodes, cells, cmap)
    try:
        x = field_queries(rng, gd, res, 3001)
        want = restate_hessian(gd[0:3], gd[3:6], gd[6:9], gd[9:12], r, nodes, cells, cmap, x)
        _phi, _grad, hess = check_mode(emu, h, x, want, strict=not any(np.isnan(v) or np.isinf(v) for v in extremes))
        assert np.isfinite(hess).any()
        if any(np.isinf(v) for v in extremes):
            assert not np.isfinite(hess).all()                          # inf coefficients reach the Hessian, not masked as zeros
        for m in (5, 32, 100, 128, 1000):
            assert bits_equal(emu.hessian(h, x[:m])[2], hess[:m])
    finally:
        emu.lib.emu_field_destroy(h)


# ---------------------------------------------------------------------------------------------------- exact second derivatives
def _poly_mul(p, q):
    out = {}
    for ea, ca in p.items():
        for eb, cb in q.items():
            e = (ea[0] + eb[0], ea[1] + eb[1], ea[2] + eb[2])
            out[e] = out.get(e, 0) + ca * cb
    return out


def _poly_diff(p, axis):
    out = {}
    for e, c in p.items():
        if e[axis]:
            d = list(e); d[axis] -= 1
            out[tuple(d)] = out.get(tuple(d), 0) + c * e[axis]
    return out


def _lin(axis, a, b):
    """a + b * xi_axis"""
    e = [0, 0, 0]; e[axis] = 1
    return {(0, 0, 0): Fraction(a), tuple(e): Fraction(b)}


def shape_polynomial(j):
    """N_j as {exponents: Fraction}"""
    kind, s = NODES[j]
    if kind == "c":
        F = {(0, 0, 0): Fraction(-19), (2, 0, 0): Fraction(9), (0, 2, 0): Fraction(9), (0, 0, 2): Fraction(9)}
        p = _poly_mul(_poly_mul(_poly_mul(F, _lin(0, 1, s[0])), _lin(1, 1, s[1])), _lin(2, 1, s[2]))
        return {e: c / 64 for e, c in p.items()}
    a = kind
    e2 = [0, 0, 0]; e2[a] = 2
    p = _poly_mul({(0, 0, 0): Fraction(1), tuple(e2): Fraction(-1)}, _lin(a, 1, 3 * s[a]))
    for b in range(3):
        if b != a:
            p = _poly_mul(p, _lin(b, 1, s[b]))
    return {e: c * Fraction(9, 64) for e, c in p.items()}


def test_one_hot_fields_give_exact_second_derivatives(emu, orc):
    """one cell over [-1, 1]^3 (c0 = 1, c1 = 0: xi = x exactly); the field that is 1 on local node j and 0 elsewhere has the Hessian
    d2 N_j.  Compared with the exact rational value at the exact double xi: within a few ulps of the sum of the absolute terms"""
    gd, res = orc.grid_desc([-1.0] * 3, [1.0] * 3, [1, 1, 1])
    rng = np.random.default_rng(7)
    x = np.concatenate([rng.uniform(-1, 1, (40, 3)), [[0.0, 0.0, 0.0], [1.0, -1.0, 1.0], [1 / 3, -1 / 3, 0.5], [-1.0, 0.25, -0.75]]])
    cells = np.arange(32, dtype=np.uint32)[None, :]
    worst = 0.0
    for j in range(32):
        h, _keep = emu.field(gd, res, np.eye(32)[j], cells, np.zeros(1, np.uint32))
        try:
            hess = emu.hessian(h, x)[2]
        finally:
            emu.lib.emu_field_destroy(h)
        N = shape_polynomial(j)
        for a in range(3):
            for b in range(3):
                d2 = _poly_diff(_poly_diff(N, a), b)
                for i, p in enumerate(x):
                    xi = [Fraction(float(v)) for v in p]
                    terms = [c * xi[0] ** e[0] * xi[1] ** e[1] * xi[2] ** e[2] for e, c in d2.items()]
                    exact = sum(terms, Fraction(0))
                    scale = sum((abs(t) for t in terms), Fraction(0))
                    err = abs(Fraction(float(hess[i, a, b])) - exact)
                    assert err <= 8 * Fraction(EPS) * scale, (j, a, b, i, float(hess[i, a, b]), float(exact))
                    if scale:
                        worst = max(worst, float(err / scale) / EPS)
    assert worst <= 8


# ---------------------------------------------------------------------------------------------------- cubic polynomials are reproduced
CUBIC_EXPONENTS = [(a, b, c) for a in range(4) for b in range(4) for c in range(4) if a + b + c <= 3]


def random_cubic(rng):
    return {e: float(v) for e, v in zip(CUBIC_EXPONENTS, rng.uniform(-1, 1, len(CUBIC_EXPONENTS)))}


def eval_cubic(f, x):
    return sum(c * x[:, 0] ** e[0] * x[:, 1] ** e[1] * x[:, 2] ** e[2] for e, c in f.items())


def cubic_hessian(f, x):
    H = np.zeros((len(x), 3, 3))
    for a in range(3):
        for b in range(3):
            for e, c in f.items():
                d = list(e)
                k = c * d[a]; d[a] = max(d[a] - 1, 0)
                k *= d[b]; d[b] = max(d[b] - 1, 0)
                if k:
                    H[:, a, b] += k * x[:, 0] ** d[0] * x[:, 1] ** d[1] * x[:, 2] ** d[2]
    return H


CUBIC_GRIDS = [((-0.3, 0.1, -1.2), (0.9, 0.5, 1.0), (5, 3, 7)), ((0.0, 0.0, 0.0), (2.0, 0.25, 1.0), (4, 6, 3)),
               ((-1.5, -0.5, 0.2), (-0.2, 1.5, 0.4), (2, 9, 5))]


def cubic_reproduction_case(orc, k, seed=11):
    """(grid desc, res, node values, interior queries, the cubic f, the per-axis c0 = 2 / cell) of CUBIC_GRIDS[k]"""
    rng = np.random.default_rng(seed + k)
    mn, mx, res = CUBIC_GRIDS[k]
    gd, r = orc.grid_desc(mn, mx, res)
    f = random_cubic(rng)
    nodes = eval_cubic(f, orc.node_positions(gd, r, 0, orc.num_nodes(r)))
    mn, mx = np.array(mn), np.array(mx)
    x = mn + (0.02 + 0.96 * rng.random((2000, 3))) * (mx - mn)
    return gd, r, nodes, x, f, 2.0 / gd[6:9]


def check_cubic(hess, nodes, x, f, c0):
    tol = 1e-11 * np.abs(nodes).max() * c0[:, None] * c0[None, :]
    err = np.abs(hess - cubic_hessian(f, x))
    assert (err <= tol).all(), float((err / tol).max())


@pytest.mark.parametrize("k", range(len(CUBIC_GRIDS)))
def test_cubic_polynomials_are_reproduced(emu, orc, k):
    """a random complete cubic sampled at the node positions of an anisotropic grid: the Hessian equals the cubic's, entry by entry, to
    1e-11 max|f| c0_a c0_b"""
    gd, r, nodes, x, f, c0 = cubic_reproduction_case(orc, k)
    h, _keep = emu.field(gd, r, nodes, None, None)
    try:
        check_cubic(emu.hessian(h, x)[2], nodes, x, f, c0)
    finally:
        emu.lib.emu_field_destroy(h)
