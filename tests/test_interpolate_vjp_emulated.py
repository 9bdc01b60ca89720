"""K11 (discregrid_b200/csrc/k11_field_grad.cu) on the CPU: the product's kernels and C-ABI compiled into build/bin/libdgemu.so (tests/emu).
dg_interpolate_vjp on trainable fields must equal the numpy restatement of the contract (tests/interpolate_vjp_ref.py) bit for bit, and a
trainable field after dg_field_set_nodes must answer every query of the library with the bits of dg_field_create of the same values.  The
cases are shared with the device run (tests/test_gpu_interpolate_vjp.py), which passes the CUDA library instead."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT
import interpolate_vjp_ref as ref

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
DBL_MAX = np.finfo(np.float64).max
UINT32_MAX = 0xFFFFFFFF
DG_ERR_INVALID = -1
_dp, _u32p, _i32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def emu():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    from discregrid_b200._capi import SIGNATURES
    lib = C.CDLL(EMU)
    for name, (res, args) in SIGNATURES.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    return lib


def same_bits(a, b):
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def nan_same_bits(a, b):
    """bits equal, any NaN equal to any NaN"""
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


class Spec:
    """a field: grid descriptor, node values, cell table [n_cells_kept, 32], cell map"""

    def __init__(self, lib, mn, mx, res, nodes_fn=None, removed=None, seed=0):
        from discregrid_b200._capi import GridDesc
        self.lib = lib
        self.mn, self.mx = np.asarray(mn, np.float64), np.asarray(mx, np.float64)
        self.res = np.asarray(res, np.uint32)
        self.desc = GridDesc()
        assert lib.dg_grid_init(_p(self.mn, _dp), _p(self.mx, _dp), _p(self.res, _u32p), C.byref(self.desc)) == 0
        nn = C.c_uint64()
        assert lib.dg_grid_num_nodes(_p(self.res, _u32p), C.byref(nn)) == 0
        n_cells = int(np.prod(self.res.astype(np.int64)))
        cells = np.empty((n_cells, 32), np.uint32)
        assert lib.dg_build_cells(_p(self.res, _u32p), 0, n_cells, _p(cells, _u32p)) == 0
        cmap = np.arange(n_cells, dtype=np.uint32)
        if removed is not None:                                     # a reduced field: cells removed, the rest renumbered
            keep = np.ones(n_cells, bool); keep[removed] = False
            cmap = np.full(n_cells, UINT32_MAX, np.uint32); cmap[keep] = np.arange(keep.sum(), dtype=np.uint32)
            cells = cells[keep]
        self.cells, self.cmap = np.ascontiguousarray(cells), cmap
        rng = np.random.default_rng(seed)
        self.nodes = rng.standard_normal(nn.value) if nodes_fn is None else nodes_fn(rng, nn.value)

    def args(self, nodes=None):
        nodes = np.ascontiguousarray(self.nodes if nodes is None else nodes, np.float64)
        return (C.byref(self.desc), _p(nodes, _dp), len(nodes), _p(self.cells, _u32p), len(self.cells), _p(self.cmap, _u32p))

    def create(self, trainable=True, nodes=None):
        h = C.c_void_p()
        fn = self.lib.dg_field_create_trainable if trainable else self.lib.dg_field_create
        rc = fn(*self.args(nodes), C.byref(h))
        assert rc == 0, self.lib.dg_last_error()
        return h

    def restate(self, x, gphi, ggrad, nodes=None):
        d = self.desc
        return ref.interpolate_vjp(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.inv_cell_size[:], d.resolution[:],
                                   self.nodes if nodes is None else nodes, self.cells, self.cmap, x, gphi, ggrad)

    def points(self, rng, n):
        return self.mn + rng.random((n, 3)) * (self.mx - self.mn)


def vjp(lib, h, n_nodes, x, gphi, ggrad):
    x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
    out = np.full(n_nodes, np.nan)
    gp = None if gphi is None else np.ascontiguousarray(gphi, np.float64)
    gg = None if ggrad is None else np.ascontiguousarray(ggrad, np.float64)
    rc = lib.dg_interpolate_vjp(h, _p(x, _dp), len(x), _p(gp, _dp), _p(gg, _dp), _p(out, _dp))
    assert rc == 0, lib.dg_last_error()
    return out


def _dbl_max_nodes(rng, n):
    v = rng.standard_normal(n)
    v[rng.choice(n, 3, replace=False)] = DBL_MAX
    return v


def field_specs(lib):
    """the field families: dense 1x1x1, anisotropic 3x4x5, 16^3, a reduced field with removed cells, DBL_MAX coefficients"""
    return {
        "dense_1": Spec(lib, [0.0, 0.0, 0.0], [1.0, 1.0, 1.0], [1, 1, 1], seed=1),
        "aniso_3x4x5": Spec(lib, [-1.0, 0.0, 2.0], [2.0, 1.5, 3.0], [3, 4, 5], seed=2),
        "dense_16": Spec(lib, [-0.7, -0.3, -0.5], [0.9, 1.1, 0.6], [16, 16, 16], seed=3),
        "reduced": Spec(lib, [0.0, -1.0, 0.5], [1.2, 0.4, 1.5], [6, 5, 4], removed=[0, 3, 7, 11, 12, 13, 40, 77, 119], seed=4),
        "dbl_max": Spec(lib, [-1.0, -1.0, -1.0], [1.0, 1.0, 1.0], [4, 3, 5], nodes_fn=_dbl_max_nodes, seed=5),
    }


def special_points(spec, rng):
    """faces, corners and the domain's max faces (the clamp), outside, NaN, and the centres of removed cells"""
    mn, mx, res = spec.mn, spec.mx, spec.res.astype(np.int64)
    cell = (mx - mn) / res
    P = [mn, mx, np.array([mx[0], mn[1], mx[2]]), np.array([mn[0], mx[1], mn[2]])]
    for k in range(3):                                             # points on the max faces and on inner faces
        for _ in range(4):
            p = spec.points(rng, 1)[0]; p[k] = mx[k]; P.append(p)
            p = spec.points(rng, 1)[0]; p[k] = mn[k] + cell[k] * rng.integers(0, res[k] + 1); P.append(p)
    corner = mn + cell * rng.integers(0, res + 1, size=(8, 3))
    P += list(corner)
    P += [mn - 1e-9, mx + np.array([0.0, 1e-12, 0.0]), np.array([np.nan, mn[1], mn[2]]), np.array([mn[0], np.inf, mn[2]])]
    removed = np.flatnonzero(spec.cmap == UINT32_MAX)
    for c in removed[:4]:
        i, j, k = c % res[0], (c // res[0]) % res[1], c // (res[0] * res[1])
        P.append(mn + (np.array([i, j, k]) + 0.5) * cell)
    return np.array(P)


UPSTREAMS = ["phi", "grad", "both"]


def upstreams(rng, n, which, special=False):
    def vals(shape):
        v = rng.standard_normal(shape)
        if special:
            pool = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2e-308, np.inf, -np.inf, np.nan, 1e308, -1e308])
            mask = rng.random(shape) < 0.3
            v[mask] = rng.choice(pool, size=int(mask.sum()))
        return v
    gphi = vals(n) if which in ("phi", "both") else None
    ggrad = vals((n, 3)) if which in ("grad", "both") else None
    return gphi, ggrad


def check_case(lib, spec, h, x, gphi, ggrad):
    got = vjp(lib, h, len(spec.nodes), x, gphi, ggrad)
    want = spec.restate(x, gphi, ggrad)
    assert nan_same_bits(got, want), (np.flatnonzero(~((got == want) | (np.isnan(got) & np.isnan(want))))[:10], len(x))
    return got


def run_families(lib, n_random=300):
    """every field family x query family x upstream: bit for bit against the restatement"""
    rng = np.random.default_rng(11)
    for name, spec in field_specs(lib).items():
        h = spec.create()
        try:
            for which in UPSTREAMS:
                for n in (0, 1, 31, 32, 33, n_random):
                    x = spec.points(rng, n)
                    check_case(lib, spec, h, x, *upstreams(rng, n, which))
                x = special_points(spec, rng)
                check_case(lib, spec, h, x, *upstreams(rng, len(x), which))
                check_case(lib, spec, h, x, *upstreams(rng, len(x), which, special=True))
        finally:
            lib.dg_field_destroy(h)


def run_one_cell(lib, sizes=(32 * 32 + 1, 3000)):
    """one cell with 32^2 + 1 queries (three levels of the tree), and every query in one cell, beside a few others"""
    spec = Spec(lib, [-1.0, 0.0, 2.0], [2.0, 1.5, 3.0], [3, 4, 5], seed=7)
    rng = np.random.default_rng(12)
    h = spec.create()
    try:
        cell = (spec.mx - spec.mn) / spec.res
        lo = spec.mn + cell * np.array([1, 2, 3])
        for n in sizes:
            x = lo + rng.random((n, 3)) * cell
            others = spec.points(rng, 40)
            xm = np.concatenate([others[:20], x, others[20:]])
            for which in UPSTREAMS:
                check_case(lib, spec, h, x, *upstreams(rng, n, which))
                check_case(lib, spec, h, xm, *upstreams(rng, len(xm), which, special=True))
    finally:
        lib.dg_field_destroy(h)


def run_signed_zero(lib):
    """an untouched node gets +0.0, and so does a node whose every contribution is -0.0: the fold starts at +0.0"""
    spec = field_specs(lib)["reduced"]
    h = spec.create()
    try:
        rng = np.random.default_rng(13)
        x = spec.points(rng, 64)
        got = vjp(lib, h, len(spec.nodes), x, np.full(64, -0.0), None)
        assert same_bits(got, spec.restate(x, np.full(64, -0.0), None))
        assert not np.signbit(got).any() and (got == 0).all()
        got = vjp(lib, h, len(spec.nodes), x[:1], rng.standard_normal(1), rng.standard_normal((1, 3)))
        untouched = np.ones(len(spec.nodes), bool)
        untouched[np.unique(spec.cells)] = False                   # nodes no kept cell references
        assert untouched.any() and (got[untouched].view(np.uint64) == 0).all()
    finally:
        lib.dg_field_destroy(h)


def run_set_nodes_parity(lib):
    """after set_nodes, a trainable field answers interpolate (value, gradient, Hessian), the isosurface, the raycast and the density map
    with the bits of dg_field_create of the same values; the VJP sees the new DBL_MAX coefficients"""
    rng = np.random.default_rng(14)
    for name in ("aniso_3x4x5", "reduced", "dbl_max"):
        spec = field_specs(lib)[name]
        h = spec.create(nodes=rng.standard_normal(len(spec.nodes)))          # made with other values, then set
        new = spec.nodes.copy()
        if name == "dbl_max":
            new[np.flatnonzero(new == DBL_MAX)[:1]] = 0.25                    # one DBL_MAX lifted, the others kept
        assert lib.dg_field_set_nodes(h, _p(new, _dp), len(new)) == 0, lib.dg_last_error()
        plain = spec.create(trainable=False, nodes=new)
        try:
            x = np.concatenate([spec.points(rng, 200), special_points(spec, rng)])
            n = len(x)
            o = np.repeat(spec.mn[None] - 0.1, 50, axis=0) + rng.random((50, 3)) * 0.05
            dirs = rng.standard_normal((50, 3))
            outs = []
            for f in (h, plain):
                phi, grad, hess = np.empty(n), np.empty((n, 3)), np.empty((n, 3, 3))
                assert lib.dg_interpolate_hessian_batch(f, _p(x, _dp), n, _p(phi, _dp), _p(grad, _dp), _p(hess, _dp)) == 0
                phi2, grad2 = np.empty(n), np.empty((n, 3))
                assert lib.dg_interpolate_batch(f, _p(x, _dp), n, _p(phi2, _dp), _p(grad2, _dp)) == 0
                d = np.empty(400)
                assert lib.dg_density_map(f, 0.3, 1000.0, 0, 0, 400, _p(d, _dp)) == 0
                t_lo, t_hi, st = np.empty(50), np.empty(50), np.empty(50, np.int32)
                assert lib.dg_field_raycast(f, _p(o, _dp), _p(dirs, _dp), 50, 0.1, 0.0, np.inf, _p(t_lo, _dp), _p(t_hi, _dp), _p(st, _i32p)) == 0
                s = C.c_void_p()
                assert lib.dg_isosurface_create(f, 0.1, 2, C.byref(s), None) == 0, lib.dg_last_error()
                nv, nt = C.c_uint64(), C.c_uint64()
                lib.dg_isosurface_sizes(s, C.byref(nv), C.byref(nt))
                V, T = np.empty((nv.value, 3)), np.empty((nt.value, 3), np.uint32)
                lib.dg_isosurface_copy(s, _p(V, _dp), _p(T, _u32p))
                lib.dg_isosurface_destroy(s)
                outs.append((phi, grad, hess, phi2, grad2, d, t_lo, t_hi, st.astype(np.float64), V, T.astype(np.float64)))
            for a, b in zip(*outs):
                assert nan_same_bits(a, b), name
            gphi, ggrad = upstreams(rng, n, "both")
            got = vjp(lib, h, len(new), x, gphi, ggrad)
            assert nan_same_bits(got, spec.restate(x, gphi, ggrad, nodes=new))
        finally:
            lib.dg_field_destroy(h)
            lib.dg_field_destroy(plain)


def run_refusals(lib):
    """refused before anything is written, with a message: a field not made by the trainable creator, a wrong node count, no upstream,
    n >= 2^32 - 1, and 32 n_cells_kept >= 2^32"""
    spec = field_specs(lib)["aniso_3x4x5"]
    plain = spec.create(trainable=False)
    h = spec.create()
    try:
        nn = len(spec.nodes)
        x = np.zeros((1, 3)); g = np.ones(1); out = np.full(nn, 7.0)
        assert lib.dg_interpolate_vjp(plain, _p(x, _dp), 1, _p(g, _dp), None, _p(out, _dp)) == DG_ERR_INVALID
        assert b"dg_field_create_trainable" in lib.dg_last_error()
        assert lib.dg_field_set_nodes(plain, _p(spec.nodes, _dp), nn) == DG_ERR_INVALID
        assert b"dg_field_create_trainable" in lib.dg_last_error()
        assert lib.dg_field_set_nodes(h, _p(spec.nodes, _dp), nn - 1) == DG_ERR_INVALID
        assert lib.dg_interpolate_vjp(h, _p(x, _dp), 1, None, None, _p(out, _dp)) == DG_ERR_INVALID
        assert lib.dg_interpolate_vjp(h, _p(x, _dp), (1 << 32) - 1, _p(g, _dp), None, _p(out, _dp)) == DG_ERR_INVALID
        assert b"2^32" in lib.dg_last_error()
        assert (out == 7.0).all()
        out0 = np.full(nn, 7.0)                                     # n = 0 overwrites with zeros
        assert lib.dg_interpolate_vjp(h, None, 0, _p(g, _dp), None, _p(out0, _dp)) == 0
        assert same_bits(out0, np.zeros(nn))
    finally:
        lib.dg_field_destroy(plain)
        lib.dg_field_destroy(h)
    from discregrid_b200._capi import GridDesc
    big, res = GridDesc(), np.array([512, 512, 512], np.uint32)     # 2^27 cells: 32 * n_cells_kept = 2^32
    assert lib.dg_grid_init(_p(np.zeros(3), _dp), _p(np.ones(3), _dp), _p(res, _u32p), C.byref(big)) == 0
    hb = C.c_void_p()
    assert lib.dg_field_create_trainable(C.byref(big), None, 0, None, 1 << 27, None, C.byref(hb)) == DG_ERR_INVALID
    assert b"2^32" in lib.dg_last_error() and not hb.value
    spec = field_specs(lib)["aniso_3x4x5"]                         # the shared checks name the entry point that was called
    args = list(spec.args())
    args[1] = None
    assert lib.dg_field_create_trainable(*args, C.byref(hb)) == DG_ERR_INVALID
    assert lib.dg_last_error().startswith(b"dg_field_create_trainable: nodes is NULL")
    assert lib.dg_field_create(*args, C.byref(hb)) == DG_ERR_INVALID
    assert lib.dg_last_error().startswith(b"dg_field_create: nodes is NULL")


def test_vjp_families_equal_restatement(emu):
    run_families(emu)


def test_vjp_one_cell_three_levels(emu):
    run_one_cell(emu)


def test_vjp_signed_zero(emu):
    run_signed_zero(emu)


def test_set_nodes_parity_with_dg_field_create(emu):
    run_set_nodes_parity(emu)


def test_vjp_refusals(emu):
    run_refusals(emu)


def test_restatement_is_the_transpose_of_interpolate(emu):
    """the restatement itself: its rows are dg_shape_functions' N and dN, and the VJP of gphi is sum_q gphi_q phi_q up to rounding"""
    rng = np.random.default_rng(15)
    xi = rng.uniform(-1.0, 1.0, (50, 3))
    xi[:4] = [[-1, -1, -1], [1, 1, 1], [1 / 3, -1 / 3, 0], [0, 0, 0]]
    N, dN = np.empty((50, 32)), np.empty((50, 32, 3))
    assert emu.dg_shape_functions(_p(xi, _dp), 50, _p(N, _dp), _p(dN, _dp)) == 0
    rN, rD = ref.rows(xi[:, 0], xi[:, 1], xi[:, 2])
    assert same_bits(rN, N) and same_bits(rD, dN)
    spec = field_specs(emu)["dense_16"]
    h = spec.create()
    try:
        x = spec.points(rng, 500); g = rng.standard_normal(500)
        phi = np.empty(500)
        assert emu.dg_interpolate_batch(h, _p(x, _dp), 500, _p(phi, _dp), None) == 0
        got = vjp(emu, h, len(spec.nodes), x, g, None)
        assert abs(got @ spec.nodes - g @ phi) <= 1e-10 * (np.abs(g) @ np.abs(phi) + 1)
    finally:
        emu.dg_field_destroy(h)
