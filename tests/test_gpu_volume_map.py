"""The volume map on the GPU -- dg_volume_map[_device], dg_reduced_volume_map_create, CubicLagrangeDiscreteGrid.addFunction /
addReducedVolumeMap (Python, and the C++ facade through GenerateVolumeMap) -- against orc_volume_map (tests/cpp/volume_oracle.cpp), the
reference-side generator's .cdm fixtures (tests/golden/make_volume_golden.py) and the two-step route it replaces (dg_volume_map, then
dg_reduce_field on each field).  Bar: bit-exact."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal
from test_density_reduced_emulated import REFERENCE_SORT, cdm_equal, cell_diag, load_sdf, n_grid_cells, same_field
from test_gpu_density_reduced import generate_sdf, reduce_gpu
from test_volume_map_emulated import CASES, SDFS, Field, call_new, oracle, orcv, volume_dense  # noqa: F401 (orcv)

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
BIN = os.path.join(ROOT, "build", "bin")
GENERATE_VOLUME_MAP = os.path.join(BIN, "GenerateVolumeMap")
REF_GENERATOR = os.path.join(ROOT, "oracle", "_ref", "bin", "RefGenerateVolumeMap")


def lib():
    from discregrid_b200 import _capi as capi
    return capi.lib


def capi_old(d, nodes, cells, cmap, h, scale, flags=0):
    """the two-step route on the GPU: dg_volume_map, dg_build_cells + identity map, dg_reduce_field on each field"""
    from discregrid_b200 import _capi as capi
    vol = volume_dense(capi.lib, d, nodes, cells, cmap, h, scale)
    diag = cell_diag(d)
    with np.errstate(invalid="ignore", over="ignore"):
        keep0 = (-6.0 * h < nodes + diag) & (nodes - diag < 2.0 * h) & (nodes != DBL_MAX)
        keep1 = (0.0 <= vol) & (vol != DBL_MAX)
    f0, tie0 = reduce_gpu(d, nodes, cells, keep0, flags)
    res = np.array(d.resolution[:], np.uint32)
    cells1 = np.empty((n_grid_cells(d), 32), np.uint32)
    capi.check(capi.lib.dg_build_cells(capi.ptr(res, capi.U32P), 0, len(cells1), capi.ptr(cells1, capi.U32P)))
    f1, tie1 = reduce_gpu(d, vol, cells1, keep1, flags)
    return f0, f1, (tie0, tie1)


def capi_new(d, nodes, cells, cmap, h, scale, flags=0):
    got = call_new(lib(), d, nodes, cells, cmap, h, scale, flags)
    assert not isinstance(got, int), lib().dg_last_error()
    return got


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_capi_python_and_generate_volume_map(dg, tmp_path, name):
    """each fixture of the reference-side generator: the C-ABI (both sorts) equals the two-step route; the Python methods, GenerateVolumeMap
    (the C++ facade's addFunction / addReducedVolumeMap) and the reference-side generator, when built, write the fixture's .cdm byte for byte"""
    c = CASES[name]
    h, scale, dense = float.fromhex(c["h_hex"]), c["scale"], c["no_reduction"]
    path = os.path.join(GOLDEN, c["sdf"])
    want = os.path.join(GOLDEN, c["file"])
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    d = sdf._desc
    nodes, cells, cmap = sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0]
    if not dense:
        for flags in (0, REFERENCE_SORT):
            f0, f1, tm = capi_new(d, nodes, cells, cmap, h, scale, flags)
            old = capi_old(d, nodes, cells, cmap, h, scale, flags)
            assert same_field(f0, old[0]) and same_field(f1, old[1]) and (tm[10], tm[11]) == old[2], flags
        fid = sdf.addReducedVolumeMap(dg.VolumeMapFunction(0, h, scale))
    else:
        fid = sdf.addFunction(dg.VolumeMapFunction(0, h, scale, no_reduction=True))
    assert fid == 1 and sdf.nFields() == 2
    out = str(tmp_path / "py.cdm")
    sdf.save(out)
    assert cdm_equal(out, want)
    tools = [GENERATE_VOLUME_MAP] + ([REF_GENERATOR] if os.path.exists(REF_GENERATOR) else [])
    for tool in tools:
        out = str(tmp_path / (os.path.basename(tool) + ".cdm"))
        cmd = [tool, "-s", repr(h), "--scale", repr(scale), "-o", out] + (["--no-reduction"] if dense else []) + [path]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        assert cdm_equal(out, want), tool


@pytest.mark.parametrize("h_cells", [0.3, 1.0, 2.5])
@pytest.mark.parametrize("no_reduction", [False, True])
@pytest.mark.parametrize("src", SDFS)
def test_device_equals_oracle(dg, orcv, src, no_reduction, h_cells):
    """dense and reduced SDFs, with and without the predicate, h from below a cell diagonal to several: the device equals the oracle"""
    g, d, nodes, cells, cmap = load_sdf(src)
    h = h_cells * float(cell_diag(d))
    got = volume_dense(lib(), d, nodes, cells, cmap, h, 0.8, no_reduction)
    assert bits_equal(got, oracle(orcv, d, nodes, cells, cmap, h, 0.8, no_reduction))


def test_non_finite_coefficients(dg, orcv):
    g, d, nodes, cells, cmap = load_sdf("ref_sphere.cdf")
    nodes = nodes.copy()
    idx = np.random.default_rng(7).choice(len(nodes), 40, replace=False)
    nodes[idx[:10]] = np.nan; nodes[idx[10:20]] = np.inf; nodes[idx[20:30]] = -np.inf; nodes[idx[30:]] = -DBL_MAX
    h = float(cell_diag(d))
    for no_reduction in (False, True):
        got = volume_dense(lib(), d, nodes, cells, cmap, h, 0.8, no_reduction)
        assert bits_equal(got, oracle(orcv, d, nodes, cells, cmap, h, 0.8, no_reduction))


def test_tensor_device_route_same_bits_as_host_route(dg):
    """dg_volume_map_device into a CUDA tensor, on torch's current stream and on a side stream, gives the host route's bits"""
    import torch
    from discregrid_b200 import _capi as capi
    import ctypes as C
    g, d, nodes, cells, cmap = load_sdf("ref_bunny_12.cdf")
    h = float(cell_diag(d))
    f = Field(lib(), d, nodes, cells, cmap)
    try:
        want = f.volume(h, 0.8, False)
        for stream in (torch.cuda.current_stream(), torch.cuda.Stream()):
            out = torch.full((f.n_grid,), -1.0, dtype=torch.float64, device="cuda")
            torch.cuda.current_stream().synchronize()
            capi.check(capi.lib.dg_volume_map_device(f.h, h, 0.8, 0, 0, f.n_grid, C.c_void_p(out.data_ptr()), C.c_void_p(stream.cuda_stream)))
            stream.synchronize()
            assert bits_equal(out.cpu().numpy(), want)
        part = torch.empty(100, dtype=torch.float64, device="cuda")
        capi.check(capi.lib.dg_volume_map_device(f.h, h, 0.8, 0, 50, 150, C.c_void_p(part.data_ptr()), None))
        torch.cuda.synchronize()
        assert bits_equal(part.cpu().numpy(), want[50:150])
    finally:
        f.close()


def test_python_method_rules(dg):
    """other argument types and no_reduction are refused with TypeError; what the C-ABI refuses raises DiscregridError; nothing changes"""
    from discregrid_b200 import DiscregridError
    sdf = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_sphere.cdf"))
    with pytest.raises(TypeError):
        sdf.addReducedVolumeMap(dg.DensityMapFunction(0, 0.15, 1000.0))
    with pytest.raises(TypeError):
        sdf.addReducedVolumeMap(dg.VolumeMapFunction(0, 0.15, no_reduction=True))
    for h, s in ((-0.15, 0.8), (float("inf"), 0.8), (0.15, float("nan"))):
        with pytest.raises(DiscregridError):
            sdf.addReducedVolumeMap(dg.VolumeMapFunction(0, h, s))
        with pytest.raises(DiscregridError):
            sdf.addFunction(dg.VolumeMapFunction(0, h, s))
    assert sdf.nFields() == 1 and len(sdf.m_nodes[0]) == sdf.nNodes()


@pytest.mark.parametrize("res", [128, 256])
def test_full_size_bunny(dg, orcv, tmp_path, res):
    """a bunny SDF made by GenerateSDF on the GPU, h = one cell diagonal: the one-call route equals the two-step route, the Python method
    equals both, and strided ranges of the dense volume field equal the oracle"""
    path = generate_sdf(tmp_path, "bunny.obj", False, res)
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    d = sdf._desc
    h = float(cell_diag(d))
    nodes, cells, cmap = sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0]
    new = capi_new(d, nodes, cells, cmap, h, 0.8)
    old = capi_old(d, nodes, cells, cmap, h, 0.8)
    assert 0 < len(new[0][0]) < sdf.nNodes() and 0 < len(new[1][0]) < sdf.nNodes()
    assert same_field(new[0], old[0]) and same_field(new[1], old[1])
    f = Field(lib(), d, nodes, cells, cmap)
    try:
        vol = f.volume(h, 0.8, False)
    finally:
        f.close()
    inside = vol[(vol != DBL_MAX) & (vol > 0)]
    assert len(inside) > 1000 and inside.max() <= 0.8 * 4.2991 * h ** 3
    n = len(vol)
    for l0 in np.linspace(0, n - 2000, 6).astype(np.int64):
        want = oracle(orcv, d, nodes, cells, cmap, h, 0.8, False, int(l0), int(l0) + 2000)
        assert bits_equal(vol[l0:l0 + 2000], want), l0
    assert sdf.addReducedVolumeMap(dg.VolumeMapFunction(0, h, 0.8)) == 1
    assert same_field((sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0]), new[0])
    assert same_field((sdf.m_nodes[1], sdf.m_cells[1], sdf.m_cell_map[1]), new[1])
