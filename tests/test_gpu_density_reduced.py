"""GenerateDensityMap with reduction in one GPU call -- dg_reduced_density_map_create, CubicLagrangeDiscreteGrid.addReducedDensityMap (Python
and C++) and GenerateDensityMap -- against the reference tool's own .cdm fixtures (tests/golden/make_density_golden.py) and against the
two-step route it replaces (dg_density_map, then dg_reduce_field on each field with the tool's predicates).  Bar: bit-exact."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, ref_resource
from test_density_reduced_emulated import FIXTURES, REFERENCE_SORT, call_new, cdm_equal, cell_diag, density_dense, n_grid_cells, same_field, write_cdm
from test_oracle_golden import read_cdf

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
BIN = os.path.join(ROOT, "build", "bin")
GENERATE_SDF = os.path.join(BIN, "GenerateSDF")
GENERATE_DENSITY_MAP = os.path.join(BIN, "GenerateDensityMap")
H_CELL_DIAGONALS = 1.0                 # h of the full-size runs, in cell diagonals of the SDF's grid


def lib():
    from discregrid_b200 import _capi as capi
    return capi.lib


def reduce_gpu(d, nodes, cells, keep, flags):
    """dg_reduce_field with its default passes (index passes on the GPU)"""
    from discregrid_b200 import _capi as capi
    nodes = np.ascontiguousarray(nodes, np.float64).copy(); cells = np.ascontiguousarray(cells, np.uint32).copy()
    keep = np.ascontiguousarray(keep, np.uint8)
    cmap = np.empty(n_grid_cells(d), np.uint32)
    n_out, c_out, tm = C.c_uint64(), C.c_uint64(), np.zeros(5)
    capi.check(capi.lib.dg_reduce_field(C.byref(d), capi.ptr(nodes, capi.F64P), len(nodes), keep.ctypes.data_as(C.POINTER(C.c_uint8)),
                                        capi.ptr(cells, capi.U32P), len(cells), capi.ptr(cmap, capi.U32P), flags, C.byref(n_out), C.byref(c_out),
                                        capi.ptr(tm, capi.F64P)))
    return (nodes[:n_out.value].copy(), cells[:c_out.value].copy(), cmap), tm[4]


def capi_old(d, nodes, cells, cmap, h, rho0, flags=0):
    """the two-step route on the GPU: dg_density_map, dg_build_cells + identity map, dg_reduce_field on each field"""
    from discregrid_b200 import _capi as capi
    dens = density_dense(capi.lib, d, nodes, cells, cmap, h, rho0)
    diag = cell_diag(d)
    keep0 = (-6.0 * h < nodes + diag) & (nodes - diag < 2.0 * h) & (nodes != DBL_MAX)
    keep1 = (0.0 <= dens) & (dens <= 3.0 * rho0) & (dens != DBL_MAX)
    f0, tie0 = reduce_gpu(d, nodes, cells, keep0, flags)
    del nodes, keep0
    res = np.array(d.resolution[:], np.uint32)
    cells1 = np.empty((n_grid_cells(d), 32), np.uint32)
    capi.check(capi.lib.dg_build_cells(capi.ptr(res, capi.U32P), 0, len(cells1), capi.ptr(cells1, capi.U32P)))
    f1, tie1 = reduce_gpu(d, dens, cells1, keep1, flags)
    return f0, f1, (tie0, tie1)


def capi_new(d, nodes, cells, cmap, h, rho0, flags=0):
    got = call_new(lib(), d, nodes, cells, cmap, h, rho0, flags)
    assert not isinstance(got, int), lib().dg_last_error()
    return got


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_fixtures_capi_python_and_generate_density_map(dg, tmp_path, name):
    """the sphere and the four reference-tool fixtures: the C-ABI (both sorts) equals the two-step route and writes the tool's .cdm byte for
    byte; so do the Python method and GenerateDensityMap"""
    src, h, rho0, ref = FIXTURES[name]
    path = os.path.join(GOLDEN, src)
    want = os.path.join(GOLDEN, ref)
    g = read_cdf(path)
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    d = sdf._desc
    nodes, cells, cmap = sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0]
    for flags in (0, REFERENCE_SORT):
        f0, f1, tm = capi_new(d, nodes, cells, cmap, h, rho0, flags)
        old = capi_old(d, nodes, cells, cmap, h, rho0, flags)
        assert same_field(f0, old[0]) and same_field(f1, old[1]) and (tm[10], tm[11]) == old[2], (name, flags)
        out = str(tmp_path / f"capi{flags}.cdm")
        write_cdm(out, g, f0, f1)
        assert cdm_equal(out, want)
    assert sdf.addReducedDensityMap(dg.DensityMapFunction(0, h, rho0)) == 1 and sdf.nFields() == 2
    out = str(tmp_path / "py.cdm")
    sdf.save(out)
    assert cdm_equal(out, want)
    out = str(tmp_path / "cli.cdm")
    r = subprocess.run([GENERATE_DENSITY_MAP, "-s", repr(h), "-r", repr(rho0), "-o", out, path], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert cdm_equal(out, want)


def test_python_method_rules(dg):
    """other argument types and no_reduction are refused with TypeError; what the C-ABI refuses raises DiscregridError; nothing changes"""
    from discregrid_b200 import DiscregridError
    sdf = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_sphere.cdf"))
    with pytest.raises(TypeError):
        sdf.addReducedDensityMap(lambda x: 0.0)
    with pytest.raises(TypeError):
        sdf.addReducedDensityMap(dg.DensityMapFunction(0, 0.15, 1000.0, no_reduction=True))
    with pytest.raises(DiscregridError):
        sdf.addReducedDensityMap(dg.DensityMapFunction(0, -0.15, 1000.0))
    assert sdf.nFields() == 1 and len(sdf.m_nodes[0]) == sdf.nNodes()


def generate_sdf(tmp_path, name, invert, res):
    mesh = ref_resource(name)
    if mesh is None:
        pytest.skip(f"{name} not staged (make -C oracle ref)")
    out = str(tmp_path / f"{name}_{res}.cdf")
    r = subprocess.run([GENERATE_SDF, "-r", f"{res} {res} {res}", "-o", out] + (["-i"] if invert else []) + [mesh], capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


def h_for(d):
    return H_CELL_DIAGONALS * float(cell_diag(d))


@pytest.mark.parametrize("name,invert,res", [("bunny.obj", False, 128), ("dragon.obj", True, 128), ("bunny.obj", False, 256), ("dragon.obj", True, 256)])
def test_full_size_equals_two_step_route(dg, tmp_path, name, invert, res):
    """SDFs made by GenerateSDF on the GPU, h = one cell diagonal: both reduced fields equal the two-step route bit for bit"""
    path = generate_sdf(tmp_path, name, invert, res)
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    d = sdf._desc
    h = h_for(d)
    new = capi_new(d, sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0], h, 1000.0)
    old = capi_old(d, sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0], h, 1000.0)
    assert 0 < len(new[0][0]) < sdf.nNodes() and 0 < len(new[1][0])
    assert same_field(new[0], old[0]) and same_field(new[1], old[1]) and (new[2][10], new[2][11]) == old[2]


def test_full_size_256_generate_density_map_memory(dg, tmp_path):
    """GenerateDensityMap on a 256^3 bunny SDF: the output equals the C-ABI's fields, and the tool's peak RSS stays below the loaded SDF
    (nodes, cells, cell map) + both reduced fields + the host sort's arrays (a 64-bit key, a 16-byte key/position pair and a 32-bit rank per
    survivor of the larger field) + a 2 GiB margin for the process itself (CUDA context, libraries, streams)"""
    path = generate_sdf(tmp_path, "bunny.obj", False, 256)
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    d = sdf._desc
    h = h_for(d)
    n, nc = sdf.nNodes(), sdf.nCells()
    f0, f1, _ = capi_new(d, sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0], h, 1000.0)
    del sdf
    out = str(tmp_path / "bunny256.cdm")
    probe = ("import resource, subprocess, sys; r = subprocess.run(sys.argv[1:], capture_output=True); "
             "print(r.returncode, resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss)")
    r = subprocess.run([sys.executable, "-c", probe, GENERATE_DENSITY_MAP, "-s", repr(h), "-r", "1000.0", "-o", out, path],
                       capture_output=True, text=True, timeout=1200)
    rc, peak_kib = (int(v) for v in r.stdout.split())
    assert rc == 0, r.stderr
    loaded = 8 * n + 128 * nc + 4 * nc
    outputs = sum(8 * len(f[0]) + 128 * len(f[1]) + 4 * len(f[2]) for f in (f0, f1))
    sort = (8 + 16 + 4) * max(len(f0[0]), len(f1[0]))
    assert peak_kib * 1024 < loaded + outputs + sort + (2 << 30), (peak_kib, loaded, outputs, sort)
    got = dg.CubicLagrangeDiscreteGrid(out)
    assert got.nFields() == 2
    for k, f in enumerate((f0, f1)):
        assert bits_equal(got.m_nodes[k], f[0]) and np.array_equal(got.m_cells[k], f[1]) and np.array_equal(got.m_cell_map[k], f[2])
