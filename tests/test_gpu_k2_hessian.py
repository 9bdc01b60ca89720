"""K2's Hessian mode on the device: dg_interpolate_hessian_batch[_device], CubicLagrangeDiscreteGrid.interpolate(..., hessian=True) with its
second-order autograd, and the C++ facade's batched Hessian overload.  The Hessian is held bit for bit to the numpy restatement of the
contract in tests/test_k2_hessian_emulated.py; phi and grad to the gradient mode (dg_interpolate_batch_device)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, ref_resource
from test_gpu_device_queries import INTERP_FIELDS, device, host, query_points, to_dev
from test_k2_hessian_emulated import CUBIC_GRIDS, check_cubic, nan_bits_equal, random_cubic, restate_hessian, symmetric_bits

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
HESSIAN_CHECK = os.path.join(ROOT, "build", "bin", "hessian_check")


def capi():
    from discregrid_b200 import _capi
    return _capi


def restate(g, field, x):
    d = g._desc
    return restate_hessian(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.inv_cell_size[:], d.resolution[:], g.m_nodes[field],
                           g.m_cells[field], g.m_cell_map[field], x)


def sync():
    if not capi().EMULATED:
        import torch
        torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 1. bits
@pytest.mark.parametrize("path,field", INTERP_FIELDS)
def test_device_hessian_equals_restatement(dg, path, field):
    """plain, anisotropic reduced and density fields, with points outside the domain, in removed cells and NaN / inf rows: hess has the
    restatement's bits and is exactly symmetric; phi and grad have the gradient mode's bits; the host entry point returns the same"""
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, path))
    x = query_points(g)
    xt = to_dev(x)
    phi, grad, hess = g.interpolate(field, xt, hessian=True)
    phi_g, grad_g = g.interpolate(field, xt, gradient=True)
    sync()
    assert phi.device.type == device() and hess.dtype == torch.float64 and hess.shape == (len(x), 3, 3)
    assert bits_equal(host(phi), host(phi_g)) and bits_equal(host(grad), host(grad_g))
    want = restate(g, field, x)
    assert bits_equal(host(hess), want) and symmetric_bits(host(hess))
    sentinel = host(phi) == DBL_MAX
    assert sentinel.any() and not host(hess)[sentinel].view(np.uint64).any() and np.abs(want).max() > 0
    hp, hg, hh = g.interpolate(field, x, hessian=True)
    assert isinstance(hh, np.ndarray) and hh.shape == (len(x), 3, 3)
    assert bits_equal(hp, host(phi)) and bits_equal(hg, host(grad)) and bits_equal(hh, want)


def test_host_entry_point_pinned_pageable_and_several_chunks(dg):
    """1.2 M points (three chunks of the host pipeline): pageable and page-locked buffers give the device route's bits"""
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_density_bunny_12.cdm"))
    rng = np.random.default_rng(3)
    mn, mx = g.domain()
    x = mn - 0.05 * (mx - mn) + rng.random((1_200_000, 3)) * 1.1 * (mx - mn)
    d = g.interpolate(1, to_dev(x), hessian=True)
    sync()
    want = [host(t) for t in d]
    got = g.interpolate(1, x, hessian=True)
    assert all(bits_equal(a, b) for a, b in zip(got, want))
    if capi().EMULATED:
        return
    cp = capi()
    xp = torch.from_numpy(x).pin_memory()
    out = [torch.empty(s, dtype=torch.float64).pin_memory() for s in ((len(x),), (len(x), 3), (len(x), 3, 3))]
    ptrs = [C.cast(C.c_void_p(t.data_ptr()), cp.F64P) for t in [xp] + out]
    cp.check(cp.lib.dg_interpolate_hessian_batch(g._device_field(1), ptrs[0], len(x), *ptrs[1:]))
    assert all(bits_equal(t.numpy(), w) for t, w in zip(out, want))


def test_cubic_from_a_device_function_is_reproduced(dg):
    """a random complete cubic sampled by a torch DeviceFunction on anisotropic grids: the device Hessian equals the cubic's to
    1e-11 max|f| c0_a c0_b, and has the restatement's bits"""
    for k, (mn, mx, res) in enumerate(CUBIC_GRIDS):
        rng = np.random.default_rng(11 + k)
        f = random_cubic(rng)

        def fn(x, _keep, f=f):
            return sum(c * x[:, 0] ** e[0] * x[:, 1] ** e[1] * x[:, 2] ** e[2] for e, c in f.items())
        g = dg.CubicLagrangeDiscreteGrid(mn, mx, res)
        g.addFunction(dg.DeviceFunction(fn))
        mnv, mxv = np.array(mn), np.array(mx)
        x = mnv + (0.02 + 0.96 * rng.random((2000, 3))) * (mxv - mnv)
        hess = host(g.interpolate(0, to_dev(x), hessian=True)[2])
        check_cubic(hess, g.m_nodes[0], x, f, 2.0 / g.cellSize())
        assert bits_equal(hess, restate(g, 0, x))


# ------------------------------------------------------------------------------------------------ 2. autograd
def interior_points(g, n, seed, margin=1e-3):
    """points at least `margin` cell widths from every cell face"""
    rng = np.random.default_rng(seed)
    res, cell = np.array(g.resolution(), np.int64), g.cellSize()
    ijk = rng.integers(0, res, (n, 3))
    return g.domain()[0] + (ijk + margin + (1 - 2 * margin) * rng.random((n, 3))) * cell


def test_functional_hessian_equals_kernel_hessian(dg):
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_bunny_12.cdf"))
    x = to_dev(interior_points(g, 12, 0))
    H = host(g.interpolate(0, x, hessian=True)[2])
    full = host(torch.autograd.functional.hessian(lambda xx: g.interpolate(0, xx, hessian=True)[0].sum(), x))
    assert full.shape == (12, 3, 12, 3)
    for i in range(12):
        assert bits_equal(full[i, :, i, :], H[i]), i
        off = np.delete(full[i], i, axis=1)
        assert (off == 0).all()


def test_double_backward_is_einsum_of_the_hessian(dg):
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_density_bunny_12.cdm"))
    x = query_points(g, 500)
    rng = np.random.default_rng(4)
    v, w = to_dev(rng.standard_normal((len(x), 3))), to_dev(rng.standard_normal(len(x)))
    _, grad, H = g.interpolate(0, to_dev(x), hessian=True)
    xt = to_dev(x).requires_grad_(True)
    phi, gout, hess = g.interpolate(0, xt, hessian=True)
    assert phi.grad_fn is not None and bits_equal(host(gout), host(grad)) and bits_equal(host(hess), host(H))
    (gx,) = torch.autograd.grad(phi, xt, w, create_graph=True)
    assert bits_equal(host(gx), host(w[:, None] * grad))
    (gx * v).sum().backward()
    assert bits_equal(host(xt.grad), host(torch.einsum("na,nab->nb", w[:, None] * v, H)))
    # the returned grad: its vector-Jacobian product
    xt.grad = None
    phi, gout, _ = g.interpolate(0, xt, hessian=True)
    (gx,) = torch.autograd.grad(gout, xt, v)
    assert bits_equal(host(gx), host(torch.einsum("na,nab->nb", v, H)))


def test_gradcheck_and_gradgradcheck_away_from_cell_faces(dg):
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_bunny_12.cdf"))
    x = to_dev(interior_points(g, 16, 5)).requires_grad_(True)
    assert torch.autograd.gradgradcheck(lambda xx: g.interpolate(0, xx, hessian=True)[0], (x,))
    assert torch.autograd.gradcheck(lambda xx: g.interpolate(0, xx, hessian=True)[:2], (x,))


def test_third_derivative_raises_and_no_grad(dg):
    import torch
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_bunny_12.cdf"))
    x = to_dev(interior_points(g, 50, 6))
    xt = x.clone().requires_grad_(True)
    phi = g.interpolate(0, xt, hessian=True)[0]
    (gx,) = torch.autograd.grad(phi.sum(), xt, create_graph=True)
    (hx,) = torch.autograd.grad(gx.sum(), xt, create_graph=True)
    with pytest.raises(RuntimeError):
        hx.sum().backward()
    _, gout, hess = g.interpolate(0, xt, hessian=True)
    (gg,) = torch.autograd.grad(gout.sum(), xt, create_graph=True)
    with pytest.raises(RuntimeError):
        gg.sum().backward()
    with pytest.raises(RuntimeError):
        hess.sum().backward()
    with torch.no_grad():
        assert all(t.grad_fn is None for t in g.interpolate(0, xt, hessian=True))
    assert all(t.grad_fn is None for t in g.interpolate(0, x, hessian=True))


# ------------------------------------------------------------------------------------------------ 3. refusals
def test_refusals(dg):
    import torch
    cp = capi()
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "ref_bunny_12.cdf"))
    f = g._device_field(0)
    n = 10
    x = np.ascontiguousarray(query_points(g, n)[:n])
    bufs = [np.empty(n), np.empty((n, 3)), np.empty((n, 3, 3))]
    for k in range(3):
        args = [cp.ptr(b, cp.F64P) if i != k else None for i, b in enumerate(bufs)]
        assert cp.lib.dg_interpolate_hessian_batch(f, cp.ptr(x, cp.F64P), n, *args) == cp.DG_ERR_INVALID
    assert cp.lib.dg_interpolate_hessian_batch(None, cp.ptr(x, cp.F64P), n, *[cp.ptr(b, cp.F64P) for b in bufs]) == cp.DG_ERR_INVALID
    assert cp.lib.dg_interpolate_hessian_batch(f, None, 0, None, None, None) == cp.DG_OK
    xt = to_dev(x)
    tb = [torch.empty(s, dtype=torch.float64, device=xt.device) for s in ((n,), (n, 3), (n, 3, 3))]
    for k in range(4):
        args = [t.data_ptr() if i != k else None for i, t in enumerate([xt] + tb)]
        assert cp.lib.dg_interpolate_hessian_batch_device(f, args[0], n, *args[1:], None) == cp.DG_ERR_INVALID
    assert cp.lib.dg_interpolate_hessian_batch_device(f, None, 0, None, None, None, None) == cp.DG_OK
    with pytest.raises(TypeError, match="float64"):
        g.interpolate(0, xt.float(), hessian=True)
    with pytest.raises(ValueError):
        g.interpolate(0, xt[:, :2].contiguous(), hessian=True)
    empty = g.interpolate(0, to_dev(np.empty((0, 3))), hessian=True)
    assert [tuple(t.shape) for t in empty] == [(0,), (0, 3), (0, 3, 3)]
    if not capi().EMULATED and dg.device_count() >= 2:
        with pytest.raises(ValueError):
            g.interpolate(0, xt.to("cuda:1"), hessian=True)


# ------------------------------------------------------------------------------------------------ 4. full size
def test_full_size_hessian_mode_phi_grad_equal_gradient_mode_bunny_128(dg):
    """10 M uniform queries on the 128^3 bunny SDF: the Hessian mode's phi and grad are the gradient mode's, bit for bit"""
    import torch
    path = ref_resource("bunny.obj")
    if path is None:
        pytest.skip("bunny.obj not staged (make -C oracle ref)")
    mesh = dg.TriangleMesh(path)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
    g.addFunction(dg.MeshSignedDistance(md))
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.from_numpy(mn).cuda() + torch.rand((10_000_000, 3), dtype=torch.float64, device="cuda", generator=gen) * torch.from_numpy(mx - mn).cuda()
    phi, grad, hess = g.interpolate(0, x, hessian=True)
    phi_g, grad_g = g.interpolate(0, x, gradient=True)
    assert torch.equal(phi.view(torch.int64), phi_g.view(torch.int64)) and torch.equal(grad.view(torch.int64), grad_g.view(torch.int64))
    assert torch.equal(hess.view(torch.int64), hess.transpose(1, 2).contiguous().view(torch.int64))
    k = torch.randint(0, len(x), (20000,), device="cuda", generator=gen)
    xs = host(x[k])
    assert bits_equal(host(hess[k]), restate(g, 0, xs))


# ------------------------------------------------------------------------------------------------ 5. the C++ facade
@pytest.mark.parametrize("path,field", [("ref_bunny_12.cdf", 0), ("ref_density_bunny_12.cdm", 1)])
def test_cpp_facade_hessian_overload(dg, tmp_path, path, field):
    g = dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, path))
    x = query_points(g)
    pts, out = str(tmp_path / "points.f64"), str(tmp_path / "out.f64")
    np.ascontiguousarray(x).tofile(pts)
    r = subprocess.run([HESSIAN_CHECK, os.path.join(GOLDEN, path), str(field), pts, out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(out)
    n = len(x)
    phi, grad, hess = g.interpolate(field, x, hessian=True)
    assert bits_equal(raw[:n], phi) and bits_equal(raw[n:4 * n].reshape(-1, 3), grad) and bits_equal(raw[4 * n:].reshape(-1, 3, 3), hess)
    assert nan_bits_equal(hess, restate(g, field, x))
