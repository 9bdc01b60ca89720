"""K11 on the device: dg_interpolate_vjp[_device] on trainable fields, bit for bit against the numpy restatement of the contract
(tests/interpolate_vjp_ref.py) on the families of tests/test_interpolate_vjp_emulated.py, and CubicLagrangeDiscreteGrid.interpolate(...,
coefficients=c): its autograd in c and x, its refusals, and a small fit of a field by gradient descent."""
import ctypes as C

import numpy as np
import pytest

import interpolate_vjp_ref as ref
from test_interpolate_vjp_emulated import (field_specs, nan_same_bits, run_families, run_one_cell, run_refusals, run_set_nodes_parity,
                                           run_signed_zero, same_bits, upstreams)

pytestmark = pytest.mark.gpu


def capi():
    from discregrid_b200 import _capi
    return _capi


def dev():
    import torch
    return torch.device("cpu") if capi().EMULATED else torch.device("cuda", 0)


def sync():
    if not capi().EMULATED:
        import torch
        torch.cuda.synchronize()


def test_vjp_families_on_device():
    run_families(capi().lib, n_random=20000)


def test_vjp_one_cell_on_device():
    run_one_cell(capi().lib, sizes=(32 * 32 + 1, 3000, 32 ** 3 + 1))


def test_vjp_signed_zero_on_device():
    run_signed_zero(capi().lib)


def test_set_nodes_parity_on_device():
    run_set_nodes_parity(capi().lib)


def test_vjp_refusals_on_device():
    run_refusals(capi().lib)


def _torch_vjp(lib, h, n_nodes, x, gphi, ggrad, stream=None):
    import torch
    out = torch.full((n_nodes,), float("nan"), dtype=torch.float64, device=x.device)
    rc = lib.dg_interpolate_vjp_device(h, x.data_ptr(), len(x), None if gphi is None else gphi.data_ptr(),
                                       None if ggrad is None else ggrad.data_ptr(), out.data_ptr(), stream)
    assert rc == 0, lib.dg_last_error()
    return out


def test_device_form_equals_host_form_repeated_and_on_a_side_stream():
    """the device form gives the host form's bits, on the same stream again and on another stream; set_nodes_device likewise"""
    import torch
    lib = capi().lib
    rng = np.random.default_rng(21)
    for name, spec in field_specs(lib).items():
        h = spec.create()
        try:
            n = 2000 if capi().EMULATED else 200000
            x = np.concatenate([spec.points(rng, n), spec.points(rng, 10)[:, :1].repeat(3, 1)])
            gphi, ggrad = upstreams(rng, len(x), "both", special=True)
            want = spec.restate(x, gphi, ggrad)
            host = np.empty(len(spec.nodes))
            assert lib.dg_interpolate_vjp(h, x.ctypes.data_as(C.POINTER(C.c_double)), len(x), gphi.ctypes.data_as(C.POINTER(C.c_double)),
                                          ggrad.ctypes.data_as(C.POINTER(C.c_double)), host.ctypes.data_as(C.POINTER(C.c_double))) == 0
            assert nan_same_bits(host, want), name
            xt, gp, gg = (torch.tensor(a, device=dev()) for a in (x, gphi, ggrad))
            st = None if capi().EMULATED else torch.cuda.current_stream().cuda_stream
            runs = [_torch_vjp(lib, h, len(spec.nodes), xt, gp, gg, st) for _ in range(2)]
            if not capi().EMULATED:
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    runs.append(_torch_vjp(lib, h, len(spec.nodes), xt, gp, gg, side.cuda_stream))
                torch.cuda.current_stream().wait_stream(side)
                nodes_t = torch.tensor(spec.nodes, device=dev())
                assert lib.dg_field_set_nodes_device(h, nodes_t.data_ptr(), len(spec.nodes), st) == 0
                runs.append(_torch_vjp(lib, h, len(spec.nodes), xt, gp, gg, st))
            sync()
            for r in runs:
                assert nan_same_bits(r.cpu().numpy(), want), name
        finally:
            lib.dg_field_destroy(h)


def _grid(dg, res=(6, 5, 4), seed=0):
    g = dg.CubicLagrangeDiscreteGrid([-1.0, 0.0, 2.0], [2.0, 1.5, 3.0], list(res))
    rng = np.random.default_rng(seed)
    fid = g.addSampledFunction(rng.standard_normal(g.nNodes()))
    return g, fid, rng


def _points(rng, n):
    import torch
    return torch.tensor(np.array([-1.0, 0.0, 2.0]) + rng.random((n, 3)) * np.array([3.0, 1.5, 1.0]), device=dev())


def test_interpolate_coefficients_forward_and_backward_bits(dg):
    """phi and grad with coefficients=c have the bits of interpolate on a field whose nodes are c; c.grad has the restatement's bits"""
    import torch
    g, fid, rng = _grid(dg)
    c = torch.tensor(rng.standard_normal(g.nNodes()), device=dev(), requires_grad=True)
    x = _points(rng, 3000)
    phi, grad = g.interpolate(fid, x, gradient=True, coefficients=c)
    g2, fid2, _ = _grid(dg)
    g2.setNodes(fid2, c.detach())
    p2, gr2 = g2.interpolate(fid2, x.cpu().numpy(), gradient=True)
    assert same_bits(phi.detach().cpu().numpy(), p2) and same_bits(grad.detach().cpu().numpy(), gr2)
    gp, gg = torch.tensor(rng.standard_normal(3000), device=dev()), torch.tensor(rng.standard_normal((3000, 3)), device=dev())
    ((phi * gp).sum() + (grad * gg).sum()).backward()
    want = ref.grid_vjp(g, fid, x.cpu().numpy(), gp.cpu().numpy(), gg.cpu().numpy(), nodes=c.detach().cpu().numpy())
    assert same_bits(c.grad.cpu().numpy(), want)
    c.grad = None
    g.interpolate(fid, x, coefficients=c).mul(gp).sum().backward()
    assert same_bits(c.grad.cpu().numpy(), ref.grid_vjp(g, fid, x.cpu().numpy(), gp.cpu().numpy(), None, nodes=c.detach().cpu().numpy()))


def test_gradcheck_in_c_and_jointly_in_x_and_c(dg):
    import torch
    g, fid, rng = _grid(dg, res=(2, 2, 3))
    c = torch.tensor(rng.standard_normal(g.nNodes()), device=dev(), requires_grad=True)
    x = _points(rng, 12)
    assert torch.autograd.gradcheck(lambda cc: g.interpolate(fid, x, coefficients=cc), (c,))
    assert torch.autograd.gradcheck(lambda cc: g.interpolate(fid, x, gradient=True, coefficients=cc), (c,))
    xr = x.clone().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda xx, cc: g.interpolate(fid, xx, gradient=True, coefficients=cc), (xr, c))


def test_backward_after_an_interleaved_call_with_other_coefficients(dg):
    """the VJP's validity depends on the values (DBL_MAX): a backward after a forward with other coefficients repacks the saved ones"""
    import torch
    g, fid, rng = _grid(dg)
    c1 = torch.tensor(rng.standard_normal(g.nNodes()), device=dev(), requires_grad=True)
    c2 = torch.tensor(np.full(g.nNodes(), np.finfo(np.float64).max), device=dev())    # every cell a sentinel
    x = _points(rng, 500)
    phi = g.interpolate(fid, x, coefficients=c1)
    assert (g.interpolate(fid, x, coefficients=c2) == np.finfo(np.float64).max).all()
    phi.sum().backward()
    want = ref.grid_vjp(g, fid, x.cpu().numpy(), np.ones(500), None, nodes=c1.detach().cpu().numpy())
    assert same_bits(c1.grad.cpu().numpy(), want) and (want != 0).any()


def test_backward_after_set_nodes_or_after_the_grid_is_gone(dg):
    """the graph keeps the trainable field its forward used: a backward after setNodes dropped it from the grid, or after the grid itself was
    collected, gives the restatement's bits for the forward's coefficients"""
    import gc
    import torch
    for drop in ("setNodes", "grid"):
        g, fid, rng = _grid(dg)
        c = torch.tensor(rng.standard_normal(g.nNodes()), device=dev(), requires_grad=True)
        x = _points(rng, 700)
        phi, grad = g.interpolate(fid, x, gradient=True, coefficients=c)
        gp, gg = torch.tensor(rng.standard_normal(700), device=dev()), torch.tensor(rng.standard_normal((700, 3)), device=dev())
        want = ref.grid_vjp(g, fid, x.cpu().numpy(), gp.cpu().numpy(), gg.cpu().numpy(), nodes=c.detach().cpu().numpy())
        if drop == "setNodes":
            g.setNodes(fid, np.zeros(g.nNodes()))
            assert (g.interpolate(fid, x, coefficients=torch.zeros_like(c)) == 0).all()     # a new trainable field for the grid
        else:
            del g
            gc.collect()
        ((phi * gp).sum() + (grad * gg).sum()).backward()
        sync()
        assert same_bits(c.grad.cpu().numpy(), want), drop


def test_double_backward_and_refusals(dg):
    import torch
    g, fid, rng = _grid(dg)
    nn = g.nNodes()
    c = torch.tensor(rng.standard_normal(nn), device=dev(), requires_grad=True)
    x = _points(rng, 20).requires_grad_(True)
    phi = g.interpolate(fid, x, coefficients=c)
    (gc,) = torch.autograd.grad(phi.sum(), c, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gc.sum(), c)
    with pytest.raises(ValueError):
        g.interpolate(fid, x, coefficients=c[:-1])
    with pytest.raises(TypeError):
        g.interpolate(fid, x, coefficients=c.float())
    with pytest.raises(ValueError):
        g.interpolate(fid, x, hessian=True, coefficients=c)
    with pytest.raises(TypeError):
        g.interpolate(fid, x.detach().cpu().numpy(), coefficients=c)
    if not capi().EMULATED:
        with pytest.raises(ValueError):
            g.interpolate(fid, x, coefficients=c.detach().cpu())
    with pytest.raises(ValueError):
        g.setNodes(fid, np.zeros(nn + 1))


def test_set_nodes_keeps_a_trained_field(dg, tmp_path):
    """setNodes copies the values into m_nodes: save() writes them and every other method sees them"""
    import torch
    g, fid, rng = _grid(dg)
    c = torch.tensor(rng.standard_normal(g.nNodes()), device=dev())
    x = _points(rng, 100)
    before = g.interpolate(fid, x, coefficients=c)
    g.setNodes(fid, c)
    assert same_bits(g.interpolate(fid, x).cpu().numpy(), before.cpu().numpy())
    g.save(str(tmp_path / "trained.cdf"))
    g3 = dg.CubicLagrangeDiscreteGrid(str(tmp_path / "trained.cdf"))
    assert same_bits(g3.m_nodes[fid], c.cpu().numpy())


def test_fit_sphere_sdf_with_adam_on_device(dg):
    """Adam on a 32^3 field against sphere SDF samples plus an eikonal term lowers the loss by at least 100x"""
    import torch
    g = dg.CubicLagrangeDiscreteGrid([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0], [32] * 3)
    fid = g.addSampledFunction(np.zeros(g.nNodes()))
    torch.manual_seed(0)
    x = torch.rand((100000, 3), dtype=torch.float64, device=dev()) * 1.8 - 0.9
    sdf = x.norm(dim=1) - 0.5
    c = torch.zeros(g.nNodes(), dtype=torch.float64, device=dev(), requires_grad=True)
    opt = torch.optim.Adam([c], lr=0.0125)              # a fifth of a cell: a node step moves grad by about 2 lr / cell
    losses = []
    for _ in range(500):
        phi, grad = g.interpolate(fid, x, gradient=True, coefficients=c)
        loss = ((phi - sdf) ** 2).mean() + 0.1 * ((grad.norm(dim=1) - 1.0) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] * 100 <= losses[0], (losses[0], losses[-1], min(losses))


def test_cpp_facade_set_nodes_and_vjp_on_device(dg, tmp_path):
    """the C++ facade's setNodesDevice and interpolate_vjp (tests/cpp/field_grad_check.cpp) give the Python route's node gradient"""
    import os
    import subprocess
    import torch
    from conftest import ROOT
    exe = os.path.join(ROOT, "build", "bin", "field_grad_check")
    if not os.path.exists(exe):
        pytest.skip("build/bin/field_grad_check not built (make cpp)")
    g, fid, rng = _grid(dg)
    path = str(tmp_path / "g.cdf")
    g.save(path)
    n = 5000
    x = np.array([-1.0, 0.0, 2.0]) + rng.random((n, 3)) * np.array([3.0, 1.5, 1.0])
    gp, gg, v = rng.standard_normal(n), rng.standard_normal((n, 3)), rng.standard_normal(g.nNodes())
    files = []
    for name, a in (("x", x), ("gp", gp), ("gg", gg), ("v", v)):
        files.append(str(tmp_path / f"{name}.f64")); a.astype(np.float64).tofile(files[-1])
    out = str(tmp_path / "out.f64")
    r = subprocess.run([exe, path, *files, out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    c = torch.tensor(v, device=dev(), requires_grad=True)
    phi, grad = g.interpolate(fid, torch.tensor(x, device=dev()), gradient=True, coefficients=c)
    ((phi * torch.tensor(gp, device=dev())).sum() + (grad * torch.tensor(gg, device=dev())).sum()).backward()
    assert same_bits(np.fromfile(out, np.float64), c.grad.cpu().numpy())
