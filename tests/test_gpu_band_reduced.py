"""The reduced narrow band in one GPU call -- dg_reduced_band_create, CubicLagrangeDiscreteGrid.addReducedBandField (Python and C++) and
GenerateSDF --band -- against the two-step route it replaces (addFunction with the band predicate, then reduceField with an always-true
predicate), against the committed reference fixtures and, where oracle/_ref is built, against the reference's own classes.  Bar: bit-exact."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, ref_resource

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
CASES = json.load(open(os.path.join(GOLDEN, "ref_band_cases.json")))
REF_GRID_SO = os.path.join(ROOT, "oracle", "_ref", "libdiscregrid_ref.so")
GENERATE_SDF = os.path.join(ROOT, "build", "bin", "GenerateSDF")


def load_mesh(dg, name):
    if name.startswith("golden/"):
        return dg.TriangleMesh(os.path.join(ROOT, "tests", name))
    p = ref_resource(name)
    if p is None:
        pytest.skip(f"{name} not staged (make -C oracle ref)")
    return dg.TriangleMesh(p)


def capi_new(md, desc, sign, band, flags=0):
    """dg_reduced_band_create + sizes + copy: (nodes, cells, cell_map, timings_ms)"""
    from discregrid_b200 import _capi as capi
    h = C.c_void_p()
    tm = np.zeros(7)
    capi.check(capi.lib.dg_reduced_band_create(md.handle, C.byref(desc), sign, band, flags, C.byref(h), capi.ptr(tm, capi.F64P)))
    try:
        nn, nc = C.c_uint64(), C.c_uint64()
        capi.check(capi.lib.dg_reduced_band_sizes(h, C.byref(nn), C.byref(nc)))
        nodes = np.empty(nn.value); cells = np.empty((nc.value, 32), np.uint32)
        cmap = np.empty(int(np.prod(np.array(desc.resolution[:], np.uint64))), np.uint32)
        capi.check(capi.lib.dg_reduced_band_copy(h, capi.ptr(nodes, capi.F64P), capi.ptr(cells, capi.U32P), capi.ptr(cmap, capi.U32P)))
    finally:
        capi.lib.dg_reduced_band_destroy(h)
    return nodes, cells, cmap, tm


def capi_old(md, desc, sign, band, flags=0):
    """dg_add_function_sdf_band, keep = always true and != DBL_MAX (:1073), dg_reduce_field (default: index passes on the GPU)"""
    from discregrid_b200 import _capi as capi
    nn = C.c_uint64(); capi.check(capi.lib.dg_grid_num_nodes(desc.resolution, C.byref(nn)))
    nc = int(np.prod(np.array(desc.resolution[:], np.uint64)))
    nodes = np.empty(nn.value); cells = np.empty((nc, 32), np.uint32); cmap = np.empty(nc, np.uint32)
    capi.check(capi.lib.dg_add_function_sdf_band(md.handle, C.byref(desc), sign, band, capi.ptr(nodes, capi.F64P), capi.ptr(cells, capi.U32P),
                                                 capi.ptr(cmap, capi.U32P), None))
    keep = np.ascontiguousarray(nodes != DBL_MAX, np.uint8)
    n_out, c_out = C.c_uint64(), C.c_uint64()
    tm = np.zeros(5)
    capi.check(capi.lib.dg_reduce_field(C.byref(desc), capi.ptr(nodes, capi.F64P), len(nodes), keep.ctypes.data_as(C.POINTER(C.c_uint8)),
                                        capi.ptr(cells, capi.U32P), nc, capi.ptr(cmap, capi.U32P), flags, C.byref(n_out), C.byref(c_out),
                                        capi.ptr(tm, capi.F64P)))
    return nodes[:n_out.value].copy(), cells[:c_out.value].copy(), cmap, tm


def same(a, b):
    return bits_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def python_old(dg, md, mn, mx, res, invert, w):
    sdf = dg.CubicLagrangeDiscreteGrid(mn, mx, list(res))
    sdf.addFunction(dg.MeshSignedDistance(md, invert=invert), False, dg.MeshDistanceBand(md, w))
    sdf.reduceField(0, lambda x, v: np.ones(len(v), bool))
    return sdf


def python_new(dg, md, mn, mx, res, invert, w):
    sdf = dg.CubicLagrangeDiscreteGrid(mn, mx, list(res))
    assert sdf.addReducedBandField(dg.MeshSignedDistance(md, invert=invert), dg.MeshDistanceBand(md, w)) == 0
    return sdf


def fields(sdf):
    return sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0]


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_python_capi_and_generate_sdf(dg, tmp_path, name):
    """the four band fixtures: the C-ABI (both sorts) equals the two-step route; the Python method equals the Python two-step route and, for
    the reduced fixtures, is saved byte-identical to them; GenerateSDF --band writes the reduced fixtures byte for byte"""
    case = CASES[name]
    mesh = load_mesh(dg, case["mesh"])
    md = dg.TriangleMeshDistance(mesh)
    g_mn, g_mx = (np.array(v) for v in case["domain"])
    sign, band = (-1.0 if case["invert"] else 1.0), float.fromhex(case["band_hex"])
    desc = dg.grid_desc(g_mn, g_mx, case["res"])
    for flags in (0, 1):
        assert same(capi_new(md, desc, sign, band, flags), capi_old(md, desc, sign, band, flags)), (name, flags)
    new = python_new(dg, md, g_mn, g_mx, case["res"], case["invert"], band)
    assert same(fields(new), fields(python_old(dg, md, g_mn, g_mx, case["res"], case["invert"], band)))
    if case["reduce"]:
        path = str(tmp_path / "py.cdf")
        new.save(path)
        assert open(path, "rb").read() == open(os.path.join(GOLDEN, case["file"]), "rb").read()
        out = str(tmp_path / "cli.cdf")
        src = os.path.join(ROOT, "tests", case["mesh"]) if case["mesh"].startswith("golden/") else ref_resource(case["mesh"])
        cmd = [GENERATE_SDF, "-r", " ".join(str(r) for r in case["res"]), "-d", " ".join(repr(float(v)) for v in case["domain"][0] + case["domain"][1]),
               "-o", out, "--band", case["band_hex"]] + (["-i"] if case["invert"] else []) + [src]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        assert open(out, "rb").read() == open(os.path.join(GOLDEN, case["file"]), "rb").read()


@pytest.mark.parametrize("name,invert,res", [("bunny.obj", False, (24, 24, 24)), ("dragon.obj", True, (20, 20, 20)), ("happy_buddha.obj", False, (14, 14, 14))])
def test_reference_meshes_equal_two_step_route_and_reference(dg, tmp_path, name, invert, res):
    """bunny, dragon (inverted) and happy_buddha at 4 widths -- 0, half a cell, 2 cell diagonals, wider than the domain: addReducedBandField
    == addFunction(band) + reduceField(always true), and == the reference's own addFunction(func, pred) + reduceField where it is built"""
    mesh = load_mesh(dg, name)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    cell = (mx - mn) / np.array(res, float)
    for w in (0.0, 0.5 * float(cell.min()), 2.0 * float(np.sqrt((cell * cell).sum())), 10.0 * float((mx - mn).max())):
        new = python_new(dg, md, mn, mx, res, invert, w)
        assert same(fields(new), fields(python_old(dg, md, mn, mx, res, invert, w))), (name, w)
        if os.path.exists(REF_GRID_SO):
            sys.path.insert(0, GOLDEN)
            from make_band_golden import reference_band_grid
            ref = reference_band_grid(np.ascontiguousarray(mesh.vertices, np.float64), np.ascontiguousarray(mesh.faces, np.uint32), mn, mx, res,
                                      invert, w, True)
            path = str(tmp_path / "ref.cdf")
            ref.save(path); ref.close()
            mine = str(tmp_path / "new.cdf")
            new.save(mine)
            assert open(mine, "rb").read() == open(path, "rb").read(), (name, w)


@pytest.mark.parametrize("name,invert", [("bunny.obj", False), ("dragon.obj", True), ("happy_buddha.obj", False)])
def test_full_size_256_equals_two_step_route(dg, name, invert):
    """256^3 at w = 2 cell diagonals and 0.5 cell: dg_reduced_band_create == dg_add_function_sdf_band + dg_reduce_field (GPU passes)"""
    mesh = load_mesh(dg, name)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    desc = dg.grid_desc(mn, mx, [256, 256, 256])
    cell = np.array(desc.cell_size[:])
    sign = -1.0 if invert else 1.0
    for w in (2.0 * float(np.sqrt((cell * cell).sum())), 0.5 * float(cell.min())):
        new = capi_new(md, desc, sign, w)
        old = capi_old(md, desc, sign, w)
        assert 0 < len(new[0]) and same(new, old), (name, w)
        assert new[3][5] == old[3][4]


def closed_form_cells(torch, res, c):
    """cell_node_id (dg_device.cuh) for the cells c (int64 tensor): (len(c), 32) node ids of the unreduced grid"""
    nx, ny, nz = (int(r) for r in res)
    k = c // (nx * ny); t = c - k * (nx * ny); j = t // nx; i = t - j * nx
    nv = (nx + 1) * (ny + 1) * (nz + 1)
    ne_x, ne_y = nx * (ny + 1) * (nz + 1), (nx + 1) * ny * (nz + 1)
    cols = []
    for jn in range(8):
        di, dj, dk = jn & 1, (jn >> 1) & 1, (jn >> 2) & 1
        cols.append((nx + 1) * (ny + 1) * (k + dk) + (nx + 1) * (j + dj) + i + di)
    for jn in range(8, 32):
        par, q = jn & 1, (jn - 8) >> 1
        grp, w = q >> 2, q & 3
        if grp == 0:
            cols.append(nv + 2 * (nx * (ny + 1) * (k + (w & 1)) + nx * (j + (w >> 1)) + i) + par)
        elif grp == 1:
            cols.append(nv + 2 * ne_x + 2 * (ny * (nz + 1) * (i + (w & 1)) + ny * (k + (w >> 1)) + j) + par)
        else:
            cols.append(nv + 2 * (ne_x + ne_y) + 2 * (nz * (nx + 1) * (j + (w & 1)) + nz * (i + (w >> 1)) + k) + par)
    return torch.stack(cols, 1)


def test_full_size_512_bunny_against_the_dense_band_and_generate_sdf_memory(dg, tmp_path):
    """512^3 bunny, w = 2 cell diagonals: every kept cell sees, through its renumbered row, the dense band coefficients of its closed-form
    nodes (dg_sample_sdf_band_device); the node ids form a permutation of [0, m); GenerateSDF --band peaks below its output arrays + 2 GiB"""
    torch = pytest.importorskip("torch")
    from discregrid_b200 import _capi as capi
    mesh = load_mesh(dg, "bunny.obj")
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    res = (512, 512, 512)
    desc = dg.grid_desc(mn, mx, list(res))
    cell = np.array(desc.cell_size[:])
    w = 2.0 * float(np.sqrt((cell * cell).sum()))
    nodes, cells, cmap, tm = capi_new(md, desc, 1.0, w)
    m = len(nodes)
    assert 0 < m and 0 < len(cells) < len(cmap)
    dev = torch.device("cuda", 0)
    g_cells = torch.from_numpy(cells.view(np.int32)).to(dev).long()
    seen = torch.zeros(m, dtype=torch.bool, device=dev)
    assert int(g_cells.min()) >= 0 and int(g_cells.max()) < m
    seen[g_cells.flatten()] = True
    assert bool(seen.all())                                                      # every id of [0, m) is used: a permutation of the survivors
    nn = C.c_uint64(); capi.check(capi.lib.dg_grid_num_nodes(desc.resolution, C.byref(nn)))
    dense = torch.empty(nn.value, dtype=torch.float64, device=dev)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    capi.check(capi.lib.dg_sample_sdf_band_device(md.handle, C.byref(desc), 1.0, w, 0, nn.value, C.c_void_p(dense.data_ptr()), s))
    torch.cuda.synchronize()
    g_nodes = torch.from_numpy(nodes).to(dev)
    g_map = torch.from_numpy(cmap.view(np.int32)).to(dev).long()
    kept = torch.nonzero(g_map != -1).flatten()
    assert len(kept) == len(cells) and torch.equal(g_map[kept], torch.arange(len(cells), device=dev))
    assert np.array_equal(closed_form_cells(torch, (7, 5, 3), torch.arange(105, device=dev)).cpu().numpy(), build_cells(capi, (7, 5, 3)))
    for a in range(0, len(kept), 1 << 22):
        c = kept[a:a + (1 << 22)]
        want = dense[closed_form_cells(torch, res, c)]
        got = g_nodes[g_cells[g_map[c]]]
        assert torch.equal(got.view(torch.int64), want.view(torch.int64))
    del dense, g_cells, g_nodes, g_map, kept, seen
    torch.cuda.empty_cache()
    out = str(tmp_path / "bunny512.cdf")
    probe = ("import resource, subprocess, sys; r = subprocess.run(sys.argv[1:], capture_output=True); "
             "print(r.returncode, resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss)")
    r = subprocess.run([sys.executable, "-c", probe, GENERATE_SDF, "-r", "512 512 512", "-o", out, "--band", repr(w), ref_resource("bunny.obj")],
                       capture_output=True, text=True, timeout=1200)
    rc, peak_kib = (int(v) for v in r.stdout.split())
    assert rc == 0, r.stderr
    arrays = 8 * m + 128 * len(cells) + 4 * len(cmap)
    assert os.path.getsize(out) >= arrays
    assert peak_kib * 1024 < arrays + (2 << 30), (peak_kib, arrays)
    got = dg.CubicLagrangeDiscreteGrid(out)
    assert bits_equal(got.m_nodes[0], nodes) and np.array_equal(got.m_cells[0], cells) and np.array_equal(got.m_cell_map[0], cmap)


def build_cells(capi, res):
    r = np.array(res, np.uint32)
    n = int(np.prod(r.astype(np.uint64)))
    out = np.empty((n, 32), np.uint32)
    capi.check(capi.lib.dg_build_cells(capi.ptr(r, capi.U32P), 0, n, capi.ptr(out, capi.U32P)))
    return out


def test_reduced_band_rules(dg):
    """a band over another mesh distance object and other argument types are refused; a negative band is refused by the C-ABI"""
    mesh = load_mesh(dg, "golden/sphere.obj")
    md, md2 = dg.TriangleMeshDistance(mesh), dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    sdf = dg.CubicLagrangeDiscreteGrid(mn, mx, [6, 6, 6])
    with pytest.raises(TypeError):
        sdf.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md2, 1.0))
    with pytest.raises(TypeError):
        sdf.addReducedBandField(dg.MeshSignedDistance(md), lambda x: True)
    from discregrid_b200 import _capi as capi
    h = C.c_void_p()
    assert capi.lib.dg_reduced_band_create(md.handle, C.byref(sdf._desc), 1.0, -0.5, 0, C.byref(h), None) == capi.DG_ERR_INVALID
    assert sdf.nFields() == 0
