"""Queries that stay on the GPU -- TriangleMeshDistance.signed_distance / unsigned_distance and CubicLagrangeDiscreteGrid.interpolate on CUDA
tensors (with autograd), dg_field_create_reduced, and the grid classes (Python and C++) that make a reduced field's first interpolation
field from the handle its reduced call kept.  Every result is compared bit for bit (uint64 views) with the host route, which the existing
suites hold to the reference's own fixtures."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, ref_resource

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
DEVICE_QUERY_CHECK = os.path.join(ROOT, "build", "bin", "device_query_check")
BAND_CASES = json.load(open(os.path.join(GOLDEN, "ref_band_cases.json")))
DENSITY_CASES = json.load(open(os.path.join(GOLDEN, "ref_density_cases.json")))
BOX_BAND = BAND_CASES["box_edge"]
BUNNY_DENSITY = DENSITY_CASES["bunny_12"]


def capi():
    from discregrid_b200 import _capi
    return _capi


def device():
    """where the test's tensors live: CUDA, or the CPU under the emulated library (whose device memory is host memory)"""
    return "cpu" if capi().EMULATED else "cuda"


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(device())


def host(t):
    return t.detach().cpu().numpy()


def late_tensor(a):
    """a on the device, written on a side stream behind ~0.1 s of GPU work (the host does not wait): returns (tensor, stream).  A query that
    is not ordered after the side stream reads zeros."""
    import torch
    if capi().EMULATED:
        return to_dev(a), None
    s = torch.cuda.Stream()
    value = to_dev(a)
    out = torch.zeros_like(value)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)
        out.copy_(value)
    return out, s


def stream_ctx(s):
    import contextlib
    if s is None:
        return contextlib.nullcontext()
    import torch
    return torch.cuda.stream(s)


def same_result(got, want):
    return (bits_equal(host(got.distance), want.distance) and bits_equal(host(got.nearest_point), want.nearest_point)
            and np.array_equal(host(got.nearest_entity), want.nearest_entity) and np.array_equal(host(got.triangle_id), want.triangle_id))


def odd_rows():
    return np.array([[np.nan, 0.0, 0.0], [np.inf, 0.0, 0.0], [-np.inf, 1.0, 2.0], [0.0, np.nan, np.inf], [1e300, -1e300, 0.0]])


# ------------------------------------------------------------------------------------------------ 1. mesh distance on CUDA tensors
def mesh_fixtures(dg):
    t = np.load(os.path.join(GOLDEN, "ref_torus_queries.npz"))
    s = np.load(os.path.join(GOLDEN, "ref_sphere_surface.npz"))
    a = s["sphere_args"]
    return [(dg.bumpy_torus(48, 48, 1.0, 0.4, 0.05, 7, 5), t["x"]), (dg.uv_sphere(int(a[0]), int(a[1]), a[2], tuple(a[3:6])), s["x"])]


@pytest.mark.parametrize("which", [0, 1])
def test_mesh_distance_tensors_equal_host(dg, which):
    """the committed query fixtures plus NaN / inf rows, produced on a side stream just before the call: all four Result fields, signed and
    unsigned, equal the host route; the Result is made of device tensors of the documented dtypes"""
    import torch
    mesh, x = mesh_fixtures(dg)[which]
    md = dg.TriangleMeshDistance(mesh)
    x = np.concatenate([x, odd_rows()])
    for signed in (True, False):
        want = md.signed_distance(x) if signed else md.unsigned_distance(x)
        xt, s = late_tensor(x)
        with stream_ctx(s):
            got = md.signed_distance(xt) if signed else md.unsigned_distance(xt)
            got = type(got)(*(t.clone() for t in got))     # ordered on the same stream
        if not capi().EMULATED:
            torch.cuda.synchronize()
        assert got.distance.device.type == device() and got.distance.dtype == torch.float64 and got.nearest_point.shape == (len(x), 3)
        assert got.nearest_entity.dtype == torch.int32 and got.triangle_id.dtype == torch.int32
        assert same_result(got, want), signed


def test_mesh_distance_tensor_shapes_and_refusals(dg, torus_small):
    import torch
    md = dg.TriangleMeshDistance(torus_small)
    x = np.load(os.path.join(GOLDEN, "ref_torus_queries.npz"))["x"][:64]
    got = md.signed_distance(to_dev(np.empty((0, 3))))
    assert got.distance.shape == (0,) and got.nearest_point.shape == (0, 3)
    assert same_result(md.signed_distance(to_dev(x[5])), md.signed_distance(x[5]))
    assert md.signed_distance(to_dev(x[5])).distance.shape == (1,)
    wide = to_dev(np.ascontiguousarray(np.concatenate([x, x], axis=1)))        # a non-contiguous (n, 3) view
    assert not wide[:, 1:4].is_contiguous()
    assert same_result(md.unsigned_distance(wide[:, 1:4]), md.unsigned_distance(np.concatenate([x, x], axis=1)[:, 1:4]))
    with pytest.raises(TypeError, match="float64"):
        md.signed_distance(to_dev(x).float())
    with pytest.raises(ValueError):
        md.signed_distance(to_dev(x[:, :2].copy()))
    # numpy and CPU tensors keep the host route on the CUDA build
    if not capi().EMULATED:
        r = md.signed_distance(torch.from_numpy(x))
        assert isinstance(r.distance, np.ndarray) and bits_equal(r.distance, md.signed_distance(x).distance)


# ------------------------------------------------------------------------------------------------ 2. interpolate on CUDA tensors
INTERP_FIELDS = [("ref_bunny_12.cdf", 0), ("ref_aniso_reduced.cdf", 0), ("ref_density_bunny_12.cdm", 0), ("ref_density_bunny_12.cdm", 1),
                 ("box.cdf", 0), ("ref_sphere_reduced.cdm", 1)]


def query_points(g, n=3000, seed=0):
    """random points in the domain grown by 10% (some outside it), the committed query points, and NaN / inf rows"""
    rng = np.random.default_rng(seed)
    mn, mx = g.domain()
    span = mx - mn
    x = mn - 0.1 * span + rng.random((n, 3)) * 1.2 * span
    q = np.load(os.path.join(GOLDEN, "ref_grid_queries.npz"))
    return np.concatenate([x, q["box_x"], q["red_x"], odd_rows()])


@pytest.mark.parametrize("path,field", INTERP_FIELDS)
def test_interpolate_tensors_equal_host(dg, path, field):
    """value-only and with gradient, on the stream the input was produced on: the bits of the host interpolate, including DBL_MAX with a zero
    gradient outside the domain and in removed cells"""
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, path))
    x = query_points(g)
    phi_h, grad_h = g.interpolate(field, x, gradient=True)
    assert (phi_h == DBL_MAX).any() and (phi_h != DBL_MAX).any()
    assert not grad_h[phi_h == DBL_MAX].any()
    xt, s = late_tensor(x)
    with stream_ctx(s):
        phi, grad = g.interpolate(field, xt, gradient=True)
        phi, grad = phi.clone(), grad.clone()
        phi_only = g.interpolate(field, xt).clone()
    if not capi().EMULATED:
        torch.cuda.synchronize()
    assert phi.device.type == device() and phi.dtype == torch.float64 and grad.shape == (len(x), 3)
    assert bits_equal(host(phi), phi_h) and bits_equal(host(grad), grad_h)
    assert bits_equal(host(phi_only), g.interpolate(field, x))


def test_interpolate_single_point_and_default_field(dg):
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_bunny_12.cdf"))
    x = query_points(g, 10)
    assert bits_equal(host(g.interpolate(to_dev(x[3]))), g.interpolate(x[3]))
    assert g.interpolate(0, to_dev(np.empty((0, 3)))).shape == (0,)
    with pytest.raises(TypeError, match="float64"):
        g.interpolate(0, to_dev(x).float())


# ------------------------------------------------------------------------------------------------ 3. autograd
def test_autograd_backward_is_grad_out_times_k2_gradient(dg):
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_density_bunny_12.cdm"))
    x = query_points(g)
    rng = np.random.default_rng(1)
    gout = to_dev(rng.standard_normal(len(x)))
    _, grad = g.interpolate(0, to_dev(x), gradient=True)
    for gradient in (False, True):
        xt = to_dev(x).requires_grad_(True)
        out = g.interpolate(0, xt, gradient=gradient)
        phi = out[0] if gradient else out
        assert phi.grad_fn is not None
        if gradient:
            assert not out[1].requires_grad and bits_equal(host(out[1]), host(grad))
        phi.backward(gout)
        assert bits_equal(host(xt.grad), host(gout[:, None] * grad))
    with torch.no_grad():
        assert g.interpolate(0, to_dev(x).requires_grad_(True)).grad_fn is None


def test_autograd_is_first_order_only(dg):
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_bunny_12.cdf"))
    xt = to_dev(query_points(g, 200)).requires_grad_(True)
    phi = g.interpolate(0, xt)
    (gx,) = torch.autograd.grad(phi, xt, torch.ones_like(phi), create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()


# ------------------------------------------------------------------------------------------------ 4. dg_field_create_reduced
def n_grid_cells(d):
    return int(np.prod(np.array(d.resolution[:], np.uint64)))


def handle_arrays(h, d):
    """dg_reduced_band_copy of a handle that stays alive"""
    from discregrid_b200.grid import _copy_reduced
    return _copy_reduced(h, n_grid_cells(d), keep=True)


def field_from_arrays(d, f):
    h = C.c_void_p()
    capi().check(capi().lib.dg_field_create(C.byref(d), capi().ptr(f[0], capi().F64P), len(f[0]), capi().ptr(f[1], capi().U32P), len(f[1]),
                                            capi().ptr(f[2], capi().U32P), C.byref(h)))
    return h


def field_from_handle(r):
    h = C.c_void_p()
    capi().check(capi().lib.dg_field_create_reduced(r, C.byref(h)))
    return h


def field_info(h):
    a = (C.c_uint64 * 4)()
    capi().check(capi().lib.dg_field_info(h, a))
    return list(a)


def interp(f, x):
    phi, grad = np.empty(len(x)), np.empty((len(x), 3))
    x = np.ascontiguousarray(x)
    capi().check(capi().lib.dg_interpolate_batch(f, capi().ptr(x, capi().F64P), len(x), capi().ptr(phi, capi().F64P), capi().ptr(grad, capi().F64P)))
    return phi, grad


def probe_points(dg, d, seed=2):
    """random points, grid node positions and points on cell faces (one coordinate exactly on a cell boundary)"""
    from discregrid_b200.grid import CubicLagrangeDiscreteGrid
    g = CubicLagrangeDiscreteGrid(d.domain_min[:], d.domain_max[:], d.resolution[:])
    rng = np.random.default_rng(seed)
    mn, mx = np.array(d.domain_min[:]), np.array(d.domain_max[:])
    cs, res = np.array(d.cell_size[:]), np.array(d.resolution[:])
    rand = mn + rng.random((2000, 3)) * (mx - mn)
    nodes = g.nodePositions()[rng.integers(0, g.nNodes(), 2000)]
    face = mn + rng.random((3000, 3)) * (mx - mn)
    for i in range(len(face)):
        k = i % 3
        face[i, k] = mn[k] + rng.integers(0, res[k] + 1) * cs[k]
    return np.concatenate([rand, nodes, face])


def band_handle(dg, d):
    md = dg.TriangleMeshDistance(dg.TriangleMesh(os.path.join(ROOT, "tests", BOX_BAND["mesh"])))
    r = C.c_void_p()
    capi().check(capi().lib.dg_reduced_band_create(md.handle, C.byref(d), 1.0, float.fromhex(BOX_BAND["band_hex"]), 0, C.byref(r), None))
    return r


def density_handles(dg):
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, BUNNY_DENSITY["sdf"]))
    r = (C.c_void_p(), C.c_void_p())
    cp = capi()
    capi().check(cp.lib.dg_reduced_density_map_create(C.byref(g._desc), cp.ptr(g.m_nodes[0], cp.F64P), len(g.m_nodes[0]), cp.ptr(g.m_cells[0], cp.U32P),
                                                      len(g.m_cells[0]), cp.ptr(g.m_cell_map[0], cp.U32P), float.fromhex(BUNNY_DENSITY["h_hex"]),
                                                      BUNNY_DENSITY["rho0"], 0, C.byref(r[0]), C.byref(r[1]), None))
    return g._desc, r


def function_handle(dg, name):
    from discregrid_b200.grid import _DeviceCallbacks
    from test_gpu_device_function import CASES, new_grid, types_of
    case = CASES[name]
    g = new_grid(dg, case)
    f, s, q = types_of(dg, case)
    cb = _DeviceCallbacks(func=f, sample=s, node=q)
    r = C.c_void_p()
    cb.check(capi().lib.dg_reduced_function_create(C.byref(g._desc), cb.func, None, cb.sample, None, cb.node, None, 0, 0, C.byref(r), None))
    return g._desc, r


def reduce_field_handle(dg, name, pred=None):
    from discregrid_b200.grid import _DeviceCallbacks
    from test_gpu_device_function import CASES, new_grid, types_of
    case = CASES[name]
    g = new_grid(dg, case)
    f, s, q = types_of(dg, case)
    g.addFunction(f, False, s)
    cb = _DeviceCallbacks(node=pred or q)
    cp = capi()
    r = C.c_void_p()
    cb.check(cp.lib.dg_reduce_field_device(C.byref(g._desc), cp.ptr(g.m_nodes[0], cp.F64P), len(g.m_nodes[0]), cp.ptr(g.m_cells[0], cp.U32P),
                                           len(g.m_cells[0]), cb.node, None, 0, 0, C.byref(r), None))
    return g._desc, r


def all_handles(dg):
    from discregrid_b200.grid import grid_desc
    d = grid_desc(*BOX_BAND["domain"], BOX_BAND["res"])
    out = [("band", d, band_handle(dg, d))]
    dd, (r0, r1) = density_handles(dg)
    out += [("density_sdf", dd, r0), ("density", dd, r1)]
    out.append(("function",) + function_handle(dg, "aniso_reduced"))
    out.append(("reduce_field",) + reduce_field_handle(dg, "box_reduced"))
    return out


def test_field_create_reduced_equals_field_create_of_the_copy(dg):
    """handles of all four creators: the field made from the handle interpolates like dg_field_create of the copied arrays (random points,
    node positions, cell faces), has the same dg_field_info, and keeps working after the handle is destroyed"""
    removed = 0
    for name, d, r in all_handles(dg):
        arrays = handle_arrays(r, d)
        assert 0 < len(arrays[1]) <= n_grid_cells(d), name
        a, b = field_from_arrays(d, arrays), field_from_handle(r)
        try:
            assert field_info(a) == field_info(b), name
            capi().check(capi().lib.dg_reduced_band_destroy(r))
            x = probe_points(dg, d)
            pa, ga = interp(a, x)
            pb, gb = interp(b, x)
            assert bits_equal(pa, pb) and bits_equal(ga, gb), name
            assert (pa != DBL_MAX).any(), name
            if len(arrays[1]) < n_grid_cells(d):
                removed += 1
                assert (pa == DBL_MAX).any(), name
        finally:
            capi().lib.dg_field_destroy(a); capi().lib.dg_field_destroy(b)
    assert removed >= 3


def test_field_create_reduced_without_kept_cells(dg):
    import torch
    d, r = reduce_field_handle(dg, "box_reduced", dg.DeviceNodePredicate(lambda x, v: torch.zeros(len(x), dtype=torch.bool, device=x.device)))
    try:
        assert len(handle_arrays(r, d)[1]) == 0
        f = field_from_handle(r)
    finally:
        capi().lib.dg_reduced_band_destroy(r)
    try:
        phi, grad = interp(f, probe_points(dg, d))
        assert (phi == DBL_MAX).all() and not grad.any()
        assert field_info(f)[:2] == [0, 0]
    finally:
        capi().lib.dg_field_destroy(f)


def test_field_create_reduced_refuses_a_handle_of_another_device(dg):
    if dg.device_count() < 2:
        pytest.skip("needs two GPUs")
    from discregrid_b200.grid import grid_desc
    d = grid_desc(*BOX_BAND["domain"], BOX_BAND["res"])
    capi().check(capi().lib.dg_set_device(0))
    r = band_handle(dg, d)
    try:
        capi().check(capi().lib.dg_set_device(1))
        h = C.c_void_p()
        assert capi().lib.dg_field_create_reduced(r, C.byref(h)) == capi().DG_ERR_INVALID and not h.value
    finally:
        capi().lib.dg_set_device(0)
        capi().lib.dg_reduced_band_destroy(r)


# ------------------------------------------------------------------------------------------------ 5. the grid class keeps the handle
def reduced_grids(dg):
    """(grid, field ids) after each reduced grid call"""
    from test_gpu_device_function import CASES, new_grid, types_of
    md = dg.TriangleMeshDistance(dg.TriangleMesh(os.path.join(ROOT, "tests", BOX_BAND["mesh"])))
    band = dg.CubicLagrangeDiscreteGrid(*BOX_BAND["domain"], BOX_BAND["res"])
    band.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, float.fromhex(BOX_BAND["band_hex"])))
    case = CASES["aniso_reduced"]
    fn = new_grid(dg, case)
    fn.addReducedFunction(*types_of(dg, case))
    case = CASES["box_reduced"]
    rf = new_grid(dg, case)
    f, s, q = types_of(dg, case)
    rf.addFunction(f, False, s)
    rf.reduceField(0, q)
    dens = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, BUNNY_DENSITY["sdf"]))
    dens.addReducedDensityMap(dg.DensityMapFunction(0, float.fromhex(BUNNY_DENSITY["h_hex"]), BUNNY_DENSITY["rho0"]))
    return [("band", band, [0]), ("function", fn, [0]), ("reduce_field", rf, [0]), ("density", dens, [0, 1])], md


def test_grid_first_interpolate_uses_the_kept_handle(dg, monkeypatch, tmp_path):
    """after each reduced call the first interpolate makes no dg_field_create call, and returns what a grid loaded from the saved file returns"""
    grids, _md = reduced_grids(dg)
    lib = capi().lib

    def refuse(*_a):
        raise AssertionError("dg_field_create called")
    got = {}
    with monkeypatch.context() as m:
        m.setattr(lib, "dg_field_create", refuse)
        for name, g, ids in grids:
            x = probe_points(dg, g._desc)
            for k in ids:
                assert k in g._reduced
                got[name, k] = g.interpolate(k, x, gradient=True) + (host(g.interpolate(k, to_dev(x))),)
                assert k not in g._reduced and k in g._fields
    for name, g, ids in grids:
        path = str(tmp_path / f"{name}.cdf")
        g.save(path)
        fresh = dg.CubicLagrangeDiscreteGrid(path)
        x = probe_points(dg, g._desc)
        for k in ids:
            phi, grad = fresh.interpolate(k, x, gradient=True)
            assert bits_equal(got[name, k][0], phi) and bits_equal(got[name, k][1], grad) and bits_equal(got[name, k][2], phi), (name, k)


def test_grid_invalidation_releases_kept_handles(dg):
    """a call that invalidates the device fields (here load; addFunction and reduceField do the same) releases the kept handles too"""
    grids, _md = reduced_grids(dg)
    for name, g, ids in grids:
        assert sorted(g._reduced) == ids, name
        g.load(os.path.join(GOLDEN, "box.cdf"))
        assert not g._reduced and not g._fields, name


# ------------------------------------------------------------------------------------------------ 6. queries inside device callbacks
def test_interpolate_inside_a_device_function_equals_the_host_route(dg):
    """addReducedFunction(DeviceFunction(lambda x, k: src.interpolate(0, x) - r), ..., DeviceNodePredicate) equals nodePositions -> host
    interpolate -> addSampledFunction -> reduceField with the same predicate"""
    src = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_bunny_12.cdf"))
    mn, mx = src.domain()
    r, vmax = 0.03125, 0.25
    src.interpolate(0, mn[None, :])                   # the device field exists before the call
    one = dg.CubicLagrangeDiscreteGrid(mn, mx, (17, 13, 15))
    one.addReducedFunction(dg.DeviceFunction(lambda x, k: src.interpolate(0, x) - r), None, dg.DeviceNodePredicate(lambda x, v: v <= vmax))
    two = dg.CubicLagrangeDiscreteGrid(mn, mx, (17, 13, 15))
    two.addSampledFunction(src.interpolate(0, two.nodePositions()) - r)
    two.reduceField(0, lambda x, v: v <= vmax)
    assert 0 < len(one.m_nodes[0]) < one.nNodes()
    assert bits_equal(one.m_nodes[0], two.m_nodes[0]) and np.array_equal(one.m_cells[0], two.m_cells[0])
    assert np.array_equal(one.m_cell_map[0], two.m_cell_map[0])


def check_distance_callback(dg, mesh, res):
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    a = dg.CubicLagrangeDiscreteGrid(mn, mx, (res, res, res))
    a.addFunction(dg.MeshSignedDistance(md))
    b = dg.CubicLagrangeDiscreteGrid(mn, mx, (res, res, res))
    b.addFunction(dg.DeviceFunction(lambda x, k: md.signed_distance(x).distance))
    assert bits_equal(a.m_nodes[0], b.m_nodes[0]) and np.array_equal(a.m_cells[0], b.m_cells[0])


def test_signed_distance_inside_a_device_function_box(dg):
    check_distance_callback(dg, dg.TriangleMesh(os.path.join(GOLDEN, "box.obj")), 12)


def test_full_size_signed_distance_inside_a_device_function_box_128(dg):
    check_distance_callback(dg, dg.TriangleMesh(os.path.join(GOLDEN, "box.obj")), 128)


def test_full_size_signed_distance_inside_a_device_function_bunny_128(dg):
    path = ref_resource("bunny.obj")
    if path is None:
        pytest.skip("bunny.obj not staged (make -C oracle ref)")
    check_distance_callback(dg, dg.TriangleMesh(path), 128)


# ------------------------------------------------------------------------------------------------ 7. the C++ facade
def test_cpp_reduced_fields_interpolate_without_upload(dg, tmp_path):
    """device_query_check: the facade's addReducedBandField and addReducedDensityMap, then interpolate, with a dg_field_create that refuses;
    its phi and gradients equal the Python class's"""
    md = dg.TriangleMeshDistance(dg.TriangleMesh(os.path.join(ROOT, "tests", BOX_BAND["mesh"])))
    band = float.fromhex(BOX_BAND["band_hex"])
    h, rho0 = float.fromhex(BUNNY_DENSITY["h_hex"]), BUNNY_DENSITY["rho0"]
    mn, mx = BOX_BAND["domain"]
    res = BOX_BAND["res"][0]
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, (res, res, res))
    g.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, band))
    dens = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, BUNNY_DENSITY["sdf"]))
    dens.addReducedDensityMap(dg.DensityMapFunction(0, h, rho0))
    x = np.concatenate([probe_points(dg, g._desc), probe_points(dg, dens._desc)])
    pts = str(tmp_path / "points.f64")
    x.tofile(pts)
    out = str(tmp_path / "q")
    args = [DEVICE_QUERY_CHECK, out, os.path.join(ROOT, "tests", BOX_BAND["mesh"])] + [float.hex(float(v)) for v in (*mn, *mx)]
    args += [str(res), float.hex(band), os.path.join(GOLDEN, BUNNY_DENSITY["sdf"]), float.hex(h), float.hex(rho0), pts]
    r = subprocess.run(args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    for suffix, grid, k in (("band", g, 0), ("sdf", dens, 0), ("density", dens, 1)):
        raw = np.fromfile(f"{out}_{suffix}.f64")
        phi, grad = grid.interpolate(k, x, gradient=True)
        assert bits_equal(raw[:len(x)], phi) and bits_equal(raw[len(x):].reshape(-1, 3), grad), suffix
