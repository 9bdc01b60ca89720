"""GenerateDensityMap with reduction in one call (dg_reduced_density_map_create: K3 + reduceField(0, p0) + reduceField(1, p1)) on the CPU: the
product's kernels and C-ABI compiled into build/bin/libdgemu.so (tests/emu).  The whole entry point must equal the two-step route --
dg_field_create + dg_density_map, dg_build_cells + identity map, then dg_reduce_field on each field with every pass on the host and keep flags
evaluated in numpy with the tool's expressions -- bit for bit, and rebuild the reference tool's own .cdm files.  The GPU runs are
tests/test_gpu_density_reduced.py."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal
from test_oracle_golden import read_cdf

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
CASES = json.load(open(os.path.join(GOLDEN, "ref_density_cases.json")))
DBL_MAX = np.finfo(np.float64).max
REFERENCE_SORT, HOST_PASSES = 1, 2
DG_ERR_INVALID = -1
_dp, _u32p, _u8p, _vp = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), C.c_void_p

# every fixture: (SDF file, h, rho0, reference .cdm); the sphere's is the one tests/test_gpu_reference_tools.py pins GenerateDensityMap to
FIXTURES = {"sphere": ("ref_sphere.cdf", 0.15, 1000.0, "ref_sphere_reduced.cdm")}
FIXTURES.update({k: (c["sdf"], float.fromhex(c["h_hex"]), c["rho0"], c["file"]) for k, c in CASES.items()})


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


def desc_of(g):
    from discregrid_b200.grid import grid_desc
    return grid_desc(g["mn"], g["mx"], g["res"], g["cell"], g["inv"])


def cell_diag(d):
    c = d.cell_size
    return np.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2])


def n_grid_cells(d):
    return int(np.prod(np.array(d.resolution[:], np.uint64)))


def call_new(emu, d, nodes, cells, cmap, h, rho0, flags=0):
    """dg_reduced_density_map_create -> status, or ((nodes, cells, cmap) of field 0, of field 1, timings)"""
    nodes = np.ascontiguousarray(nodes, np.float64); cells = np.ascontiguousarray(cells, np.uint32); cmap = np.ascontiguousarray(cmap, np.uint32)
    r0, r1 = _vp(), _vp()
    tm = np.full(13, -1.0)
    rc = emu.dg_reduced_density_map_create(C.byref(d), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), h, rho0, flags,
                                           C.byref(r0), C.byref(r1), _p(tm, _dp))
    if rc != 0:
        assert not r0.value and not r1.value
        return rc
    out = []
    for r in (r0, r1):
        nn, nc = C.c_uint64(), C.c_uint64()
        assert emu.dg_reduced_band_sizes(r, C.byref(nn), C.byref(nc)) == 0
        f = (np.empty(nn.value), np.empty((nc.value, 32), np.uint32), np.empty(n_grid_cells(d), np.uint32))
        assert emu.dg_reduced_band_copy(r, _p(f[0], _dp), _p(f[1], _u32p), _p(f[2], _u32p)) == 0
        assert emu.dg_reduced_band_destroy(r) == 0
        out.append(f)
    return out[0], out[1], tm


def reduce_host(emu, d, nodes, cells, keep, flags):
    nodes = np.ascontiguousarray(nodes, np.float64).copy(); cells = np.ascontiguousarray(cells, np.uint32).copy()
    keep = np.ascontiguousarray(keep, np.uint8)
    cmap = np.empty(n_grid_cells(d), np.uint32)
    n_out, c_out, tm = C.c_uint64(), C.c_uint64(), np.zeros(5)
    assert emu.dg_reduce_field(C.byref(d), _p(nodes, _dp), len(nodes), _p(keep, _u8p), _p(cells, _u32p), len(cells), _p(cmap, _u32p),
                               flags | HOST_PASSES, C.byref(n_out), C.byref(c_out), _p(tm, _dp)) == 0, emu.dg_last_error()
    return (nodes[:n_out.value].copy(), cells[:c_out.value].copy(), cmap), tm[4]


def density_dense(emu, d, nodes, cells, cmap, h, rho0):
    """addFunction(DensityMapFunction) with the predicate on: dg_field_create + dg_density_map(no_reduction = 0)"""
    nodes = np.ascontiguousarray(nodes, np.float64); cells = np.ascontiguousarray(cells, np.uint32); cmap = np.ascontiguousarray(cmap, np.uint32)
    f = _vp()
    assert emu.dg_field_create(C.byref(d), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), C.byref(f)) == 0
    dens = np.empty(len(nodes))
    assert emu.dg_density_map(f, h, rho0, 0, 0, len(nodes), _p(dens, _dp)) == 0
    emu.dg_field_destroy(f)
    return dens


def call_old(emu, d, nodes, cells, cmap, h, rho0, flags=0):
    """the two-step route: density field, closed-form cells (dg_build_cells) + identity map, then dg_reduce_field (host passes) on each
    field with the tool's predicates and != DBL_MAX (:1073), evaluated in numpy with the tool's expressions"""
    dens = density_dense(emu, d, nodes, cells, cmap, h, rho0)
    diag = cell_diag(d)
    with np.errstate(invalid="ignore", over="ignore"):
        keep0 = (-6.0 * h < nodes + diag) & (nodes - diag < 2.0 * h) & (nodes != DBL_MAX)
        keep1 = (0.0 <= dens) & (dens <= 3.0 * rho0) & (dens != DBL_MAX)
    f0, tie0 = reduce_host(emu, d, nodes, cells, keep0, flags)
    res = np.array(d.resolution[:], np.uint32)
    cells1 = np.empty((n_grid_cells(d), 32), np.uint32)
    assert emu.dg_build_cells(_p(res, _u32p), 0, len(cells1), _p(cells1, _u32p)) == 0
    f1, tie1 = reduce_host(emu, d, dens, cells1, keep1, flags)
    return f0, f1, (tie0, tie1)


def same_field(a, b):
    return bits_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def check_against_old(emu, d, nodes, cells, cmap, h, rho0, flags):
    got = call_new(emu, d, nodes, cells, cmap, h, rho0, flags)
    assert not isinstance(got, int), emu.dg_last_error()
    want = call_old(emu, d, nodes, cells, cmap, h, rho0, flags)
    assert same_field(got[0], want[0]) and same_field(got[1], want[1])
    tm = got[2]
    assert (tm[10], tm[11]) == want[2]
    assert (tm[:10] >= 0).all() and tm[12] >= tm[:10].sum() - 1e-6
    return got


def write_cdm(path, g, f0, f1):
    """the reference's save() of a two-field grid (cubic_lagrange_discrete_grid.cpp:678-719)"""
    with open(path, "wb") as fh:
        fh.write(struct.pack("<6d", *g["mn"], *g["mx"])); fh.write(struct.pack("<3I", *[int(r) for r in g["res"]]))
        fh.write(struct.pack("<3d", *g["cell"])); fh.write(struct.pack("<3d", *g["inv"]))
        fh.write(struct.pack("<QQ", int(np.prod(g["res"].astype(np.uint64))), 2))
        for k in range(3):
            fh.write(struct.pack("<Q", 2))
            for f in (f0, f1):
                fh.write(struct.pack("<Q", len(f[k]))); fh.write(np.ascontiguousarray(f[k]).tobytes())


def cdm_equal(a, b):
    """.cdm files a and b byte for byte, except that a NaN node value may carry another NaN's payload (the -DBL_MAX fixture holds NaNs, and
    which payload an operation on two NaNs returns is left to the hardware by IEEE 754).  Every other byte must match."""
    ra, rb = open(a, "rb").read(), open(b, "rb").read()
    if ra == rb:
        return True
    if len(ra) != len(rb):
        return False
    ga, gb = read_cdf(a), read_cdf(b)
    if not all(np.array_equal(ga[k], gb[k]) for k in ("res", "n_cells", "n_fields")) or \
            not all(bits_equal(ga[k], gb[k]) for k in ("mn", "mx", "cell", "inv")):
        return False
    for f in range(len(ga["nodes"])):
        na, nb = ga["nodes"][f], gb["nodes"][f]
        both_nan = np.isnan(na) & np.isnan(nb) if len(na) == len(nb) else None
        if both_nan is None or not np.array_equal(na.view(np.uint64)[~both_nan], nb.view(np.uint64)[~both_nan]):
            return False
        if not (np.array_equal(ga["cells"][f], gb["cells"][f]) and np.array_equal(ga["cmap"][f], gb["cmap"][f])):
            return False
    return True


def load_sdf(name):
    g = read_cdf(os.path.join(GOLDEN, name))
    return g, desc_of(g), g["nodes"][0], g["cells"][0], g["cmap"][0]


@pytest.mark.parametrize("flags", [0, REFERENCE_SORT])
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_fixtures_equal_two_step_route_and_reference_tool(emu, tmp_path, name, flags):
    """the sphere and the four reference-tool fixtures (bunny, dragon inverted, the dense band field with DBL_MAX nodes, the anisotropic
    grid whose survivors share Z-curve keys): the same two fields as the two-step route, written byte-identical to the tool's .cdm"""
    src, h, rho0, ref = FIXTURES[name]
    g, d, nodes, cells, cmap = load_sdf(src)
    f0, f1, tm = check_against_old(emu, d, nodes, cells, cmap, h, rho0, flags)
    if name == "aniso":
        assert tm[10] == 1.0
    out = str(tmp_path / "out.cdm")
    write_cdm(out, g, f0, f1)
    assert open(out, "rb").read() == open(os.path.join(GOLDEN, ref), "rb").read()


# ------------------------------------------------------------------------------------------------ hand-made SDF arrays
def box_grid(res=(2, 2, 2), cell=(3.0, 4.0, 12.0)):
    """a grid whose cells measure 3 x 4 x 12: cell_diag = 13 exactly"""
    from discregrid_b200.grid import grid_desc
    mx = [c * r for c, r in zip(cell, res)]
    d = grid_desc([0.0, 0.0, 0.0], mx, res)
    assert cell_diag(d) == 13.0
    return d


def dense_layout(emu, d):
    nn = C.c_uint64()
    assert emu.dg_grid_num_nodes(d.resolution, C.byref(nn)) == 0
    nc = n_grid_cells(d)
    res = np.array(d.resolution[:], np.uint32)
    cells = np.empty((nc, 32), np.uint32)
    assert emu.dg_build_cells(_p(res, _u32p), 0, nc, _p(cells, _u32p)) == 0
    return nn.value, cells, np.arange(nc, dtype=np.uint32)


def positions(emu, d, n):
    x = np.empty((n, 3))
    assert emu.dg_node_positions(C.byref(d), 0, n, _p(x, _dp)) == 0
    return x


@pytest.mark.parametrize("flags", [0, REFERENCE_SORT])
def test_sdf_predicate_edges(emu, flags):
    """h = 1, cell_diag = 13: v + 13 == -6h at v = -19 and v - 13 == 2h at v = 15 (both rejected: strict <), a nextafter step either side,
    and -0.0.  Every other node holds 1e6 (rejected), so the cells of the middle vertex survive exactly when its value is kept."""
    d = box_grid()
    n, cells, cmap = dense_layout(emu, d)
    mid = 13                                                                 # vertex (1, 1, 1): a node of all eight cells
    cases = [(-19.0, False), (np.nextafter(-19.0, np.inf), True), (np.nextafter(-19.0, -np.inf), False),
             (15.0, False), (np.nextafter(15.0, -np.inf), True), (np.nextafter(15.0, np.inf), False), (-0.0, True), (0.0, True)]
    for v, kept in cases:
        nodes = np.full(n, 1e6)
        nodes[mid] = v
        f0, f1, _ = check_against_old(emu, d, nodes, cells, cmap, 1.0, 1000.0, flags)
        assert (len(f0[1]) == 8) == kept and (len(f0[1]) == 0) == (not kept), v
        if kept:
            assert bits_equal(f0[0][np.nonzero(f0[0] != 1e6)[0]], np.array([v])), v   # -0.0 survives as -0.0


@pytest.mark.parametrize("flags", [0, REFERENCE_SORT])
def test_density_predicate_edges(emu, flags):
    """the density field's bounds: 0.0 (nodes beyond 2h get +0.0, kept by 0 <= v) and v == 3 rho0 (rho0 = +inf: every integrated node is
    +inf == 3 rho0 and kept, a node whose integral is 0 gets NaN and is not); a negative rho0 keeps nothing"""
    d = box_grid((3, 2, 2))
    n, cells, cmap = dense_layout(emu, d)
    x = positions(emu, d, n)
    nodes = x[:, 2] - 12.0 + 0.25 * x[:, 0]                                  # a plane: the interpolation is exact
    for h, rho0 in ((2.0, np.inf), (13.0, np.inf), (2.0, -1.0), (2.0, 1000.0)):
        dens = density_dense(emu, d, nodes, cells, cmap, h, rho0)
        f0, f1, _ = check_against_old(emu, d, nodes, cells, cmap, h, rho0, flags)
        with np.errstate(invalid="ignore"):
            keep1 = (0.0 <= dens) & (dens <= 3.0 * rho0) & (dens != DBL_MAX)
        assert len(f1[1]) == int(keep1[cells].any(axis=1).sum())              # the cells with a kept node survive, with all their nodes
        if rho0 == np.inf:
            assert (dens == np.inf).any() and (dens == 0.0).any() == (h == 2.0) and (f1[0] == np.inf).any()
        if rho0 == -1.0:                                                     # 0 <= v && v <= -3 holds nowhere
            assert (dens < 0).any() and len(f1[0]) == 0
        else:
            assert len(f1[1]) > 0


def test_all_dbl_max_sdf_gives_empty_fields(emu):
    d = box_grid((3, 2, 2))
    n, cells, cmap = dense_layout(emu, d)
    for flags in (0, REFERENCE_SORT):
        f0, f1, tm = check_against_old(emu, d, np.full(n, DBL_MAX), cells, cmap, 1.0, 1000.0, flags)
        for f in (f0, f1):
            assert len(f[0]) == 0 and len(f[1]) == 0 and (f[2] == 0xFFFFFFFF).all()


def test_h_that_keeps_every_cell(emu):
    """h wider than the domain: p0 holds everywhere, every quadrature point lies outside the domain (density 0, kept by p1)"""
    g, d, nodes, cells, cmap = load_sdf("ref_sphere.cdf")
    for flags in (0, REFERENCE_SORT):
        f0, f1, _ = check_against_old(emu, d, nodes, cells, cmap, 1e3, 1000.0, flags)
        for f in (f0, f1):
            assert len(f[1]) == len(cmap) and np.array_equal(f[2], np.arange(len(cmap), dtype=np.uint32)) and len(f[0]) == len(nodes)


def test_fewer_rows_than_grid_cells(emu):
    """n_cells < nx*ny*nz: the SDF field keeps its first rows, the rest of its cell map is 0xffffffff; the reduced SDF cell map holds i at
    every i >= n_cells (the reference's resize + iota)"""
    g, d, nodes, cells, cmap = load_sdf("ref_sphere.cdf")
    k = 700
    cmap = cmap.copy(); cmap[k:] = 0xFFFFFFFF
    for flags in (0, REFERENCE_SORT):
        f0, _, _ = check_against_old(emu, d, nodes, cells[:k], cmap, 0.15, 1000.0, flags)
        assert np.array_equal(f0[2][k:], np.arange(k, len(cmap), dtype=np.uint32))


def test_refusals(emu):
    """a reduced SDF field, a row naming a node >= n_nodes, a bad cell map entry, h <= 0 or NaN, unknown flags, NULL arguments and a grid of
    2^31 nodes or more are refused with DG_ERR_INVALID, as the two-step route refuses them"""
    g, d, nodes, cells, cmap = load_sdf("ref_sphere.cdf")
    red = read_cdf(os.path.join(GOLDEN, "ref_sphere_reduced.cdm"))
    assert call_new(emu, d, red["nodes"][0], red["cells"][0], red["cmap"][0], 0.15, 1000.0) == DG_ERR_INVALID
    assert b"already reduced" in emu.dg_last_error()
    bad = cells.copy(); bad[417, 5] = len(nodes)
    assert call_new(emu, d, nodes, bad, cmap, 0.15, 1000.0) == DG_ERR_INVALID
    assert b"node id >= n_nodes" in emu.dg_last_error()
    f = _vp()
    assert emu.dg_field_create(C.byref(d), _p(nodes, _dp), len(nodes), _p(bad, _u32p), len(bad), _p(cmap, _u32p), C.byref(f)) == DG_ERR_INVALID
    badmap = cmap.copy(); badmap[3] = len(cells)
    assert call_new(emu, d, nodes, cells, badmap, 0.15, 1000.0) == DG_ERR_INVALID
    for h in (0.0, -0.15, float("nan"), -float("inf")):
        assert call_new(emu, d, nodes, cells, cmap, h, 1000.0) == DG_ERR_INVALID, h
    for flags in (HOST_PASSES, 4, 0x80000000):
        assert call_new(emu, d, nodes, cells, cmap, 0.15, 1000.0, flags) == DG_ERR_INVALID
    assert call_new(emu, d, nodes, np.concatenate([cells, cells[:1]]), cmap, 0.15, 1000.0) == DG_ERR_INVALID    # more rows than cells
    r0, r1 = _vp(), _vp()
    assert emu.dg_reduced_density_map_create(C.byref(d), None, len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), 0.15, 1000.0, 0,
                                             C.byref(r0), C.byref(r1), None) == DG_ERR_INVALID
    assert emu.dg_reduced_density_map_create(C.byref(d), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), 0.15, 1000.0, 0,
                                             None, C.byref(r1), None) == DG_ERR_INVALID
    big = desc_of(g)
    for k in range(3):                                                       # 700^3: 2,408,356,301 nodes, in [2^31, 2^32)
        big.resolution[k] = 700; big.cell_size[k] = 1.0 / 700; big.inv_cell_size[k] = 700.0
    assert emu.dg_reduced_density_map_create(C.byref(big), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), 0.15, 1000.0,
                                             0, C.byref(r0), C.byref(r1), None) == DG_ERR_INVALID
    assert b"grid too large" in emu.dg_last_error() and not r0.value and not r1.value
