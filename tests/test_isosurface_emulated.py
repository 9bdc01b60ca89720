"""Level sets by marching tetrahedra (K6, discregrid_b200/csrc/k6_isosurface.cu) on the CPU: the product's kernels and C-ABI compiled into
build/bin/libdgemu.so (tests/emu).  dg_isosurface_create must equal the numpy restatement of the contract (tests/isosurface_ref.py) bit for
bit -- vertices as uint64 views, triangles exactly -- on the lattice values the library's own host interpolate gives.  The GPU runs are
tests/test_gpu_isosurface.py."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from test_oracle_golden import read_cdf, read_obj
import isosurface_ref as ir

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
DBL_MAX = np.finfo(np.float64).max
DG_ERR_INVALID = -1
UINT32_MAX = 0xFFFFFFFF
_dp, _u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)


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


class Field:
    """a dg_field of the emulated library and its grid descriptor"""

    def __init__(self, emu, desc, handle):
        self.emu, self.desc, self.h = emu, desc, handle

    def __del__(self):
        self.emu.dg_field_destroy(self.h)

    def lattice(self, s):
        d = self.desc
        return ir.Lattice(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.resolution[:], s)

    def interpolate(self, x):
        x = np.ascontiguousarray(x, np.float64)
        phi = np.empty(len(x))
        assert self.emu.dg_interpolate_batch(self.h, _p(x, _dp), len(x), _p(phi, _dp), None) == 0
        return phi

    def values(self, L):
        return self.interpolate(L.points())

    def extract(self, iso, s):
        """dg_isosurface_create + copy -> (V, T, timings)"""
        r = C.c_void_p()
        tm = np.full(5, -1.0)
        rc = self.emu.dg_isosurface_create(self.h, iso, s, C.byref(r), _p(tm, _dp))
        assert rc == 0, self.emu.dg_last_error()
        nv, nt = C.c_uint64(), C.c_uint64()
        assert self.emu.dg_isosurface_sizes(r, C.byref(nv), C.byref(nt)) == 0
        V, T = np.empty((nv.value, 3)), np.empty((nt.value, 3), np.uint32)
        assert self.emu.dg_isosurface_copy(r, _p(V, _dp), _p(T, _u32p)) == 0
        assert self.emu.dg_isosurface_destroy(r) == 0
        return V, T, tm


def grid_desc(mn, mx, res):
    from discregrid_b200.grid import grid_desc as gd
    return gd(np.asarray(mn, np.float64), np.asarray(mx, np.float64), res)


def dense_field(emu, mn, mx, res, fn):
    d = grid_desc(mn, mx, res)
    n = C.c_uint64()
    assert emu.dg_grid_num_nodes(d.resolution, C.byref(n)) == 0
    x = np.empty((n.value, 3))
    assert emu.dg_node_positions(C.byref(d), 0, n.value, _p(x, _dp)) == 0
    nodes = np.ascontiguousarray(fn(x), np.float64)
    h = C.c_void_p()
    n_cells = int(np.prod(np.array(res, np.int64)))
    assert emu.dg_field_create(C.byref(d), _p(nodes, _dp), len(nodes), None, n_cells, None, C.byref(h)) == 0, emu.dg_last_error()
    return Field(emu, d, h)


def sphere_sdf(x, c=(0.03, -0.02, 0.01), r=0.6):
    return np.linalg.norm(x - np.asarray(c), axis=1) - r


def torus_sdf(x, R=0.6, r=0.25):
    q = np.hypot(x[:, 0], x[:, 1]) - R
    return np.hypot(q, x[:, 2]) - r


def make_field(emu, name):
    if name == "sphere":
        return dense_field(emu, [-1, -1, -1], [1, 1, 1], (9, 9, 9), sphere_sdf)
    if name == "torus":
        return dense_field(emu, [-1, -1, -0.5], [1, 1, 0.5], (12, 12, 6), torus_sdf)
    if name == "box_cdf":
        g = read_cdf(os.path.join(GOLDEN, "box.cdf"))
        d = grid_desc(g["mn"], g["mx"], tuple(int(r) for r in g["res"]))
        nodes, cells, cmap = g["nodes"][0], np.ascontiguousarray(g["cells"][0]), np.ascontiguousarray(g["cmap"][0])
        h = C.c_void_p()
        assert emu.dg_field_create(C.byref(d), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), C.byref(h)) == 0
        return Field(emu, d, h)
    if name == "box_band":                                                  # reduced narrow band of 2 cell diagonals (K1 + K4)
        V, F = read_obj(os.path.join(GOLDEN, "box.obj"))
        V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
        m = C.c_void_p()
        assert emu.dg_mesh_create(_p(V, _dp), len(V), _p(F, _u32p), len(F), C.byref(m)) == 0
        mn, mx = np.empty(3), np.empty(3)
        assert emu.dg_generate_sdf_domain(_p(V, _dp), len(V), _p(mn, _dp), _p(mx, _dp)) == 0
        d = grid_desc(mn, mx, (8, 8, 8))
        band = 2.0 * float(np.linalg.norm(np.array(d.cell_size[:])))
        r = C.c_void_p()
        assert emu.dg_reduced_band_create(m, C.byref(d), 1.0, band, 0, C.byref(r), None) == 0, emu.dg_last_error()
        h = C.c_void_p()
        assert emu.dg_field_create_reduced(r, C.byref(h)) == 0
        emu.dg_reduced_band_destroy(r)
        emu.dg_mesh_destroy(m)
        return Field(emu, d, h)
    raise KeyError(name)


def same_bits(a, b):
    """bit for bit; NaN counts as equal to NaN (the device's default NaN has another payload than the host's)"""
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64)))


def check_against_restatement(f, iso, s):
    V, T, tm = f.extract(iso, s)
    L = f.lattice(s)
    Vr, Tr = ir.extract(L, f.values(L), iso)
    assert same_bits(V, Vr), (V.shape, Vr.shape)
    assert T.dtype == np.uint32 and np.array_equal(T, Tr), (T.shape, Tr.shape)
    assert (tm >= 0).all()
    return V, T


@pytest.mark.parametrize("s", [1, 2, 3])
@pytest.mark.parametrize("name", ["box_cdf", "sphere", "torus", "box_band"])
def test_equals_restatement(emu, name, s):
    f = make_field(emu, name)
    diag = float(np.linalg.norm(np.array(f.desc.cell_size[:])))
    n = []
    for iso in (0.0, 0.5 * diag, -0.5 * diag):
        V, T = check_against_restatement(f, iso, s)
        n.append(len(T))
    assert n[0] > 0


@pytest.mark.parametrize("name,chi", [("sphere", 2), ("torus", 0)])
@pytest.mark.parametrize("s", [1, 2])
def test_closed_oriented_and_no_unreferenced_vertices(emu, name, chi, s):
    f = make_field(emu, name)
    V, T = check_against_restatement(f, 0.0, s)
    closed, oriented = ir.edge_use(T)
    assert closed and oriented
    assert np.array_equal(np.unique(T), np.arange(len(V)))
    assert ir.euler_characteristic(V, T) == chi
    assert ir.signed_volume(V, T) > 0
    # outward: the normals point along the SDF's gradient at the triangle centroids
    n = ir.normals(V, T)
    c = V[T.astype(np.int64)].mean(axis=1)
    g = (sphere_sdf if name == "sphere" else torus_sdf)
    eps = 1e-6
    grad = np.stack([(g(c + eps * e) - g(c - eps * e)) / (2 * eps) for e in np.eye(3)], axis=1)
    nd = np.linalg.norm(n, axis=1) > 1e-12
    assert (np.einsum("ij,ij->i", n[nd], grad[nd]) > 0).all()


def test_iso_hit_exactly_by_lattice_values(emu):
    f = make_field(emu, "sphere")
    L = f.lattice(2)
    vals = f.values(L)
    near = np.nonzero(np.abs(vals) < 0.1)[0]
    iso = float(vals[near[len(near) // 2]])
    assert (vals == iso).sum() >= 1
    V, T = check_against_restatement(f, iso, 2)
    closed, oriented = ir.edge_use(T)                      # still closed by vertex ids: coincident vertices are not welded
    assert closed and oriented
    tri = V[T.astype(np.int64)]
    area = np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    assert (area == 0).any()                               # zero-area triangles at the point where f == iso are kept


def test_all_sentinel_field_and_iso_outside_the_values_give_nothing(emu):
    f = dense_field(emu, [0, 0, 0], [1, 2, 3], (3, 4, 5), lambda x: np.full(len(x), DBL_MAX))
    for s in (1, 3):
        V, T, _ = f.extract(0.0, s)
        assert V.shape == (0, 3) and T.shape == (0, 3)
    g = make_field(emu, "sphere")
    for iso in (5.0, -5.0):
        V, T, _ = g.extract(iso, 2)
        assert len(V) == 0 and len(T) == 0


def test_no_kept_cell_gives_nothing(emu):
    d = grid_desc([0, 0, 0], [1, 1, 1], (4, 4, 4))
    cells = np.zeros((1, 32), np.uint32)
    cmap = np.full(64, UINT32_MAX, np.uint32)
    h = C.c_void_p()
    assert emu.dg_field_create(C.byref(d), None, 0, _p(cells, _u32p), 0, _p(cmap, _u32p), C.byref(h)) == 0, emu.dg_last_error()
    V, T, _ = Field(emu, d, h).extract(0.0, 2)
    assert len(V) == 0 and len(T) == 0


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_non_finite_and_huge_coefficients(emu, seed):
    rng = np.random.default_rng(seed)
    special = np.array([np.nan, np.inf, -np.inf, DBL_MAX, -DBL_MAX, 1.7e308, -1.7e308, 1e308, -1e308, 0.0, -0.0])

    def fn(x):
        v = rng.standard_normal(len(x))
        k = rng.random(len(x)) < 0.15
        v[k] = rng.choice(special, k.sum())
        return v
    f = dense_field(emu, [-1, -2, 0], [1, 1, 0.5], (5, 4, 3), fn)
    for s in (1, 2):
        for iso in (0.0, 0.25, -1e308, 1.6e308):
            check_against_restatement(f, iso, s)


def test_refusals(emu):
    f = make_field(emu, "sphere")
    r = C.c_void_p()
    for iso in (np.nan, np.inf, -np.inf):
        assert emu.dg_isosurface_create(f.h, iso, 1, C.byref(r), None) == DG_ERR_INVALID and not r.value
        assert b"iso" in emu.dg_last_error()
    for s in (0, 17):
        assert emu.dg_isosurface_create(f.h, 0.0, s, C.byref(r), None) == DG_ERR_INVALID and not r.value
        assert b"subdivisions" in emu.dg_last_error()
    assert emu.dg_isosurface_create(None, 0.0, 1, C.byref(r), None) == DG_ERR_INVALID
    assert emu.dg_isosurface_create(f.h, 0.0, 1, None, None) == DG_ERR_INVALID
    # a lattice of 2^31 points or more: 82^3 cells at s = 16 give 1313^3 = 2,263,571,297 points (a field with no kept cell: nothing to pack)
    d = grid_desc([0, 0, 0], [1, 1, 1], (82, 82, 82))
    cells = np.zeros((1, 32), np.uint32)
    cmap = np.full(82 ** 3, UINT32_MAX, np.uint32)
    h = C.c_void_p()
    assert emu.dg_field_create(C.byref(d), None, 0, _p(cells, _u32p), 0, _p(cmap, _u32p), C.byref(h)) == 0
    big = Field(emu, d, h)
    assert emu.dg_isosurface_create(big.h, 0.0, 16, C.byref(r), None) == DG_ERR_INVALID and not r.value
    assert b"2^31" in emu.dg_last_error()
    # NULL outputs where the count is not zero; sizes with NULL arguments
    assert emu.dg_isosurface_create(f.h, 0.0, 1, C.byref(r), None) == 0
    V = np.empty((1 << 16, 3)); T = np.empty((1 << 16, 3), np.uint32)
    assert emu.dg_isosurface_copy(r, None, _p(T, _u32p)) == DG_ERR_INVALID
    assert emu.dg_isosurface_copy(r, _p(V, _dp), None) == DG_ERR_INVALID
    assert emu.dg_isosurface_copy_device(r, None, _p(T, _u32p), None) == DG_ERR_INVALID
    assert emu.dg_isosurface_copy_device(r, _p(V, _dp), None, None) == DG_ERR_INVALID
    n = C.c_uint64()
    assert emu.dg_isosurface_sizes(r, None, C.byref(n)) == DG_ERR_INVALID
    assert emu.dg_isosurface_sizes(None, C.byref(n), C.byref(n)) == DG_ERR_INVALID
    assert emu.dg_isosurface_copy(None, _p(V, _dp), _p(T, _u32p)) == DG_ERR_INVALID
    assert emu.dg_isosurface_destroy(r) == 0
    assert emu.dg_isosurface_destroy(None) == 0
    # an empty result may be copied with NULL outputs
    assert emu.dg_isosurface_create(f.h, 5.0, 1, C.byref(r), None) == 0
    assert emu.dg_isosurface_copy(r, None, None) == 0 and emu.dg_isosurface_copy_device(r, None, None, None) == 0
    emu.dg_isosurface_destroy(r)


def test_s1_lattice_is_the_vertex_nodes(emu):
    """for s = 1 the lattice positions are the bits of the grid's vertex nodes wherever those lie inside the domain"""
    f = make_field(emu, "box_cdf")
    L = f.lattice(1)
    x = np.empty((L.n_points, 3))
    assert emu.dg_node_positions(C.byref(f.desc), 0, L.n_points, _p(x, _dp)) == 0
    inside = (x <= np.array(f.desc.domain_max[:])).all(axis=1)
    assert inside.sum() > 0
    assert np.array_equal(L.points()[inside].view(np.uint64), x[inside].view(np.uint64))
