"""Narrow-band K1 on the GPU: addFunction(func, pred) with pred(x) = |md.signed_distance(x).distance| <= band -- the classifier kernels and
the band form of the node loop (k1_sdf.cu) through the C-ABI, the Python mirror (MeshDistanceBand), the C++ facade and GenerateSDF --band,
against the reference's own classes (oracle/_ref, through tests/golden/make_band_golden.py) and the committed fixtures.  Bar: bit-exact."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, ref_resource

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
CASES = json.load(open(os.path.join(GOLDEN, "ref_band_cases.json")))
REF_GRID_SO = os.path.join(ROOT, "oracle", "_ref", "libdiscregrid_ref.so")


def load_mesh(dg, name):
    if name.startswith("golden/"):
        return dg.TriangleMesh(os.path.join(ROOT, "tests", name))
    p = ref_resource(name)
    if p is None:
        pytest.skip(f"{name} not staged (make -C oracle ref)")
    return dg.TriangleMesh(p)


def ref_band_field(mesh, mn, mx, res, invert, band, reduce, path):
    """the reference's own band field -- addFunction(func, pred) [+ reduceField(always true)] -- saved to `path` (tests/golden/make_band_golden.py)"""
    if not os.path.exists(REF_GRID_SO):
        pytest.skip("oracle/_ref/libdiscregrid_ref.so not built")
    import sys
    sys.path.insert(0, GOLDEN)
    from make_band_golden import reference_band_grid
    g = reference_band_grid(np.ascontiguousarray(mesh.vertices, np.float64), np.ascontiguousarray(mesh.faces, np.uint32), mn, mx, res, invert, band, reduce)
    g.save(path)
    g.close()


@pytest.mark.parametrize("name,invert,res", [("bunny.obj", False, (24, 24, 24)), ("dragon.obj", True, (20, 20, 20)), ("happy_buddha.obj", False, (14, 14, 14))])
def test_band_reference_meshes_vs_oracle_add_function(dg, tmp_path, name, invert, res):
    """bunny, dragon (inverted) and happy_buddha (not watertight) at several band widths -- 0, half a cell, 2 cell diagonals, wider than the
    domain: Python mirror addFunction(MeshSignedDistance, pred=MeshDistanceBand) == the reference's own addFunction(func, pred), every bit"""
    mesh = load_mesh(dg, name)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    cell = (mx - mn) / np.array(res, float)
    for w in (0.0, 0.5 * float(cell.min()), 2.0 * float(np.sqrt((cell * cell).sum())), 10.0 * float((mx - mn).max())):
        sdf = dg.CubicLagrangeDiscreteGrid(mn, mx, list(res))
        sdf.addFunction(dg.MeshSignedDistance(md, invert=invert), False, dg.MeshDistanceBand(md, w))
        path = str(tmp_path / "ref.cdf")
        ref_band_field(mesh, mn, mx, res, invert, w, False, path)
        ref = dg.CubicLagrangeDiscreteGrid(path)
        assert bits_equal(sdf.m_nodes[0], ref.m_nodes[0]), (name, w)
        assert np.array_equal(sdf.m_cells[0], ref.m_cells[0]) and np.array_equal(sdf.m_cell_map[0], ref.m_cell_map[0])


@pytest.mark.parametrize("name", sorted(CASES))
def test_generate_sdf_band_writes_the_fixture_files(dg, tmp_path, name):
    """GenerateSDF --band W (reduced) and --band W --no-reduction: the .cdf is byte-identical to the reference's fixture"""
    case = CASES[name]
    exe = os.path.join(ROOT, "build", "bin", "GenerateSDF")
    src = os.path.join(ROOT, "tests", case["mesh"]) if case["mesh"].startswith("golden/") else ref_resource(case["mesh"])
    if src is None:
        pytest.skip(f"{case['mesh']} not staged")
    out = str(tmp_path / "out.cdf")
    (a, b) = case["domain"]
    cmd = [exe, "-r", " ".join(str(r) for r in case["res"]), "-d", " ".join(repr(float(v)) for v in a + b), "-o", out, "--band", case["band_hex"]]
    cmd += ["-i"] if case["invert"] else []
    cmd += [] if case["reduce"] else ["--no-reduction"]
    r = subprocess.run(cmd + [src], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert open(out, "rb").read() == open(os.path.join(GOLDEN, case["file"]), "rb").read()
    r = subprocess.run([exe, "--band", "0.1", "--gpus", "2", src], capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "--band" in r.stderr


def test_reduced_band_field_interpolates_like_the_reference(dg, tmp_path):
    """Python mirror: addFunction(band) + reduceField(always true) == the reference's reduced band field (bunny fixture), and interpolating
    it (value + gradient, DBL_MAX in removed cells) gives the reference class's values bit for bit"""
    from oracle_api import RefGrid, have_ref_grid
    case = CASES["bunny_20"]
    mesh = load_mesh(dg, case["mesh"])
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = (np.array(v) for v in case["domain"])
    sdf = dg.CubicLagrangeDiscreteGrid(mn, mx, case["res"])
    sdf.addFunction(dg.MeshSignedDistance(md), False, dg.MeshDistanceBand(md, float.fromhex(case["band_hex"])))
    sdf.reduceField(0, lambda x, v: np.ones(len(v), bool))
    path = str(tmp_path / "bunny_band.cdf")
    sdf.save(path)
    assert open(path, "rb").read() == open(os.path.join(GOLDEN, case["file"]), "rb").read()
    if not have_ref_grid():
        pytest.skip("oracle/_ref/libdiscregrid_ref.so not built")
    ref = RefGrid(os.path.join(GOLDEN, case["file"]))
    rng = np.random.default_rng(5)
    x = mn + rng.random((20000, 3)) * (mx - mn)
    phi, grad = sdf.interpolate(0, x, gradient=True)
    rphi, rgrad = ref.interpolate(0, x, grad=True)
    assert bits_equal(phi, rphi) and bits_equal(grad, rgrad)
    assert (phi == DBL_MAX).any() and (phi != DBL_MAX).any()


def test_band_predicate_rules(dg):
    """MeshDistanceBand is a plain predicate too; a band over another mesh distance object, a negative / NaN band and any other predicate
    are refused"""
    mesh = load_mesh(dg, "golden/sphere.obj")
    md, md2 = dg.TriangleMeshDistance(mesh), dg.TriangleMeshDistance(mesh)
    x = np.array([[0.0, 0.0, 0.0], [5.0, 5.0, 5.0]])
    p = dg.MeshDistanceBand(md, 1.0)
    assert list(p(x)) == list(np.abs(md.signed_distance(x).distance) <= 1.0)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    sdf = dg.CubicLagrangeDiscreteGrid(mn, mx, [6, 6, 6])
    with pytest.raises(TypeError):
        sdf.addFunction(dg.MeshSignedDistance(md), False, dg.MeshDistanceBand(md2, 1.0))
    with pytest.raises(TypeError):
        sdf.addFunction(dg.MeshSignedDistance(md), False, lambda x: True)
    for bad in (-1.0, float("nan")):
        with pytest.raises(ValueError):
            dg.MeshDistanceBand(md, bad)
    from discregrid_b200 import _capi as capi
    out = np.empty(sdf.nNodes())
    assert capi.lib.dg_add_function_sdf_band(md.handle, C.byref(sdf._desc), 1.0, -0.5, capi.ptr(out, capi.F64P), None, None, None) == capi.DG_ERR_INVALID


@pytest.mark.parametrize("name,invert", [("bunny.obj", False), ("dragon.obj", True), ("happy_buddha.obj", False)])
def test_band_full_size_device_form_matches_full_node_loop(dg, name, invert):
    """256^3: dg_sample_sdf_band_device == dg_sample_sdf_device on every in-band node (bit for bit) and DBL_MAX exactly where |full| > w,
    for w = 2 cell diagonals and w = 0.5 cell; the device form honours sub-ranges (a sentinel buffer stays untouched outside)"""
    torch = pytest.importorskip("torch")
    from discregrid_b200 import _capi as capi
    mesh = load_mesh(dg, name)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    desc = dg.grid_desc(mn, mx, [256, 256, 256])
    n = C.c_uint64(); capi.check(capi.lib.dg_grid_num_nodes(desc.resolution, C.byref(n))); n = n.value
    sign = -1.0 if invert else 1.0
    dev = torch.device("cuda", 0)
    full = torch.empty(n, dtype=torch.float64, device=dev)
    band = torch.empty(n, dtype=torch.float64, device=dev)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    capi.check(capi.lib.dg_sample_sdf_device(md.handle, C.byref(desc), sign, 0, n, C.c_void_p(full.data_ptr()), s))
    cell = np.array(desc.cell_size[:])
    for w in (2.0 * float(np.sqrt((cell * cell).sum())), 0.5 * float(cell.min())):
        band.fill_(float("nan"))
        capi.check(capi.lib.dg_sample_sdf_band_device(md.handle, C.byref(desc), sign, w, 0, n, C.c_void_p(band.data_ptr()), s))
        torch.cuda.synchronize()
        inb = full.abs() <= w
        assert 0 < int(inb.sum()) < n
        assert torch.equal(band[inb].view(torch.int64), full[inb].view(torch.int64))
        assert bool((band[~inb] == DBL_MAX).all())
    a, b = n // 3 + 17, 2 * n // 3 - 5
    band.fill_(7.25)
    capi.check(capi.lib.dg_sample_sdf_band_device(md.handle, C.byref(desc), sign, w, a, b, C.c_void_p(band[a:].data_ptr()), s))
    torch.cuda.synchronize()
    inb = full[a:b].abs() <= w
    assert torch.equal(band[a:b][inb].view(torch.int64), full[a:b][inb].view(torch.int64)) and bool((band[a:b][~inb] == DBL_MAX).all())
    assert bool((band[:a] == 7.25).all()) and bool((band[b:] == 7.25).all())
