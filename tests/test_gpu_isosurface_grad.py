"""K13 on the device: dg_isosurface_vjp[_device] bit for bit against the numpy restatement of the contract (tests/isosurface_grad_ref.py) on
the families of tests/test_isosurface_grad_emulated.py, and the autograd of CubicLagrangeDiscreteGrid.isosurface(coefficients=): the forward's
bits, gradcheck, backward after setNodes and after the grid is dropped, double backward, streams, the chain through a mesh distance, an
Adam fit, the bunny and the C++ facade."""
import gc
import os

import numpy as np
import pytest

from conftest import ROOT, ref_resource
from test_isosurface_grad_emulated import (run_clamp, run_exact_values, run_families, run_huge_values, run_large_lattice_refusal, run_refusals,
                                           run_special_upstreams_and_sizes, same_bits)

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


def T(a, grad=False):
    import torch
    return torch.tensor(np.asarray(a, np.float64), device=dev(), requires_grad=grad)


def N(t):
    return t.detach().cpu().numpy()


def test_families_on_device():
    run_families(capi().lib)


def test_exact_huge_and_clamp_on_device():
    lib = capi().lib
    run_exact_values(lib)
    run_huge_values(lib)
    run_clamp(lib)


def test_specials_and_sizes_on_device():
    run_special_upstreams_and_sizes(capi().lib)


def test_refusals_on_device():
    run_refusals(capi().lib)


def test_large_lattice_refused_on_device():
    run_large_lattice_refusal(capi().lib)


def sphere_grid(dg, res=8, r=0.55, c=(0.03, -0.02, 0.01)):
    g = dg.CubicLagrangeDiscreteGrid([-1.0] * 3, [1.0] * 3, [res] * 3)
    X = np.asarray(g.nodePositions(), np.float64).reshape(-1, 3)
    v = np.sqrt(((X - np.asarray(c)) ** 2).sum(1)) - r
    return g, g.addSampledFunction(v), v


def host_vjp(g, fid, iso, s, E, gV):
    """dg_isosurface_vjp (host form) on the grid's trainable field, which holds m_nodes"""
    c = capi()
    E = np.ascontiguousarray(E, np.uint64); gV = np.ascontiguousarray(gV, np.float64)
    out = np.empty(len(g.m_nodes[fid]))
    c.check(c.lib.dg_isosurface_vjp(g._trainable_field(fid).handle, iso, s, len(E), c.ptr(E, c.U64P), c.ptr(gV, c.F64P), c.ptr(out, c.F64P)))
    return out


def test_coefficients_forward_bits_and_gradient(dg):
    """isosurface(coefficients=c) gives the bits of isosurface() on a field whose m_nodes are c, with edge ids; its backward equals the host
    form of the VJP; without device=True it raises"""
    rng = np.random.default_rng(1)
    g, fid, v = sphere_grid(dg, 8)
    cn = v + 0.02 * rng.standard_normal(len(v))
    g2, fid2, _ = sphere_grid(dg, 8)
    g2.setNodes(fid2, cn)
    for s in (1, 2):
        c = T(cn, True)
        V, Tr, E = g.isosurface(fid, 0.05, s, device=True, coefficients=c, edges=True)
        assert V.requires_grad and not Tr.requires_grad and not E.requires_grad and E.dtype.is_signed and E.dtype.itemsize == 8
        Vh, Th, Eh = g2.isosurface(fid2, 0.05, s, edges=True)
        assert Eh.dtype == np.uint64
        assert same_bits(N(V), Vh) and np.array_equal(N(Tr), Th.astype(np.int32)) and np.array_equal(N(E).view(np.uint64), Eh)
        Vd, Td = g2.isosurface(fid2, 0.05, s, device=True)
        assert same_bits(N(Vd), Vh)
        gV = rng.standard_normal(Vh.shape)
        (V * T(gV)).sum().backward()
        sync()
        assert same_bits(N(c.grad), host_vjp(g2, fid2, 0.05, s, Eh, gV))
    with pytest.raises(ValueError):
        g.isosurface(fid, 0.0, 1, coefficients=T(cn))
    with pytest.raises(ValueError):
        g.isosurface(fid, 0.0, 1, device=True, coefficients=T(cn[:-1]))
    with pytest.raises(TypeError):
        g.isosurface(fid, 0.0, 1, device=True, coefficients=T(cn).float())


def _far_iso(g, fid, s, iso=0.0):
    """an iso at least 1e-3 away from every lattice value, so that small changes of c keep the topology"""
    from isosurface_ref import Lattice, lattice_values
    vals = lattice_values(g, fid, Lattice.of_grid(g, s))
    while np.abs(vals - iso).min() < 1e-3:
        iso += 1.3e-3
    return iso


def test_gradcheck_sphere(dg):
    """torch.autograd.gradcheck in c (the nodes with the largest gradient) on an 8^3 sphere field at s = 1 and 2"""
    import torch
    g, fid, v = sphere_grid(dg, 8)
    for s in (1, 2):
        iso = _far_iso(g, fid, s)
        c = T(v, True)
        V = g.isosurface(fid, iso, s, device=True, coefficients=c)[0]
        V.sum().backward()
        idx = np.argsort(-np.abs(N(c.grad)))[:6]
        cb = c.detach()

        def f(sub):
            full = cb.clone(); full[idx] = sub
            return g.isosurface(fid, iso, s, device=True, coefficients=full)[0]
        assert torch.autograd.gradcheck(f, (T(N(cb)[idx], True),), eps=1e-7, atol=1e-5, rtol=1e-4, fast_mode=True)


def test_backward_after_set_nodes_and_after_the_grid_is_dropped(dg):
    rng = np.random.default_rng(2)
    g, fid, v = sphere_grid(dg, 8)
    gref, fref, _ = sphere_grid(dg, 8)
    E_all = []
    for drop in (False, True):
        c = T(v + 0.01 * rng.standard_normal(len(v)), True)
        V, _, E = g.isosurface(fid, 0.0, 2, device=True, coefficients=c, edges=True)
        gV = rng.standard_normal(tuple(V.shape))
        if drop:
            del g
            gc.collect()
        else:
            g.setNodes(fid, v * 2.0)
        (V * T(gV)).sum().backward()
        sync()
        gref.setNodes(fref, N(c))
        assert same_bits(N(c.grad), host_vjp(gref, fref, 0.0, 2, N(E).view(np.uint64), gV)), f"drop={drop}"
        E_all.append(len(E))
    assert min(E_all) > 0


def test_double_backward_raises(dg):
    import torch
    g, fid, v = sphere_grid(dg, 6)
    c = T(v, True)
    V = g.isosurface(fid, 0.0, 1, device=True, coefficients=c)[0]
    (gc_,) = torch.autograd.grad(V.sum(), c, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gc_.sum(), c)


def test_tensor_route_on_two_streams(dg):
    """the same bits on torch's default stream and on a side stream, twice"""
    import torch
    rng = np.random.default_rng(3)
    g, fid, v = sphere_grid(dg, 32)
    cn = v + 0.01 * rng.standard_normal(len(v))
    runs = []
    for k in range(4):
        stream = torch.cuda.Stream() if k % 2 else torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            c = T(cn, True)
            V, _, E = g.isosurface(fid, 0.0, 2, device=True, coefficients=c, edges=True)
            gV = torch.sin(V.detach() * 7.0)
            (V * gV).sum().backward()
        torch.cuda.synchronize()
        runs.append((N(V), N(c.grad)))
    for r in runs[1:]:
        assert same_bits(r[0], runs[0][0]) and same_bits(r[1], runs[0][1])


def test_chain_through_the_mesh_distance(dg):
    """V from isosurface(coefficients=c), then a fixed target mesh's signed_distance(V), then loss.backward(): c.grad is K13's VJP of K10's
    point gradient, bit for bit"""
    import torch
    g, fid, v = sphere_grid(dg, 12, r=0.5)
    tg, tf, _ = sphere_grid(dg, 12, r=0.62)
    Vt, Tt = tg.isosurface(tf, 0.0, 1)
    target = dg.TriangleMeshDistance(Vt, Tt)
    c = T(v, True)
    V, _, E = g.isosurface(fid, 0.0, 1, device=True, coefficients=c, edges=True)
    loss = (target.signed_distance(V).distance ** 2).sum()
    loss.backward()
    sync()
    V2 = V.detach().clone().requires_grad_(True)
    (target.signed_distance(V2).distance ** 2).sum().backward()
    sync()
    g2, fid2, _ = sphere_grid(dg, 12, r=0.5)
    assert same_bits(N(c.grad), host_vjp(g2, fid2, 0.0, 1, N(E).view(np.uint64), N(V2.grad)))
    assert np.abs(N(c.grad)).max() > 0


def test_tensor_adam_fit_of_a_sphere(dg):
    """Adam on a 32^3 sphere SDF of radius 0.45 towards a sphere mesh of radius 0.6: the mean squared distance of the extracted vertices to
    the target falls below a tenth of its start within 60 steps"""
    import torch
    g, fid, v = sphere_grid(dg, 32, r=0.45)
    tg, tf, _ = sphere_grid(dg, 16, r=0.6)
    Vt, Tt = tg.isosurface(tf, 0.0, 1)
    target = dg.TriangleMeshDistance(Vt, Tt)
    c = T(v, True)
    opt = torch.optim.Adam([c], lr=2e-3)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        V = g.isosurface(fid, 0.0, 1, device=True, coefficients=c)[0]
        loss = (target.signed_distance(V).distance ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.1 * losses[0], losses[::10]


def test_bunny_256_same_bits_on_two_runs(dg):
    """the bunny's 256^3 SDF as a trainable field: extraction and VJP at s = 1 and 2 give the same bits on two runs"""
    p = ref_resource("bunny.obj")
    if p is None:
        pytest.skip("bunny.obj not staged (make -C oracle ref)")
    from winding_ref import read_obj
    V0, F0 = read_obj(p)
    md = dg.TriangleMeshDistance(V0, F0)
    mn, mx = dg.generate_sdf_domain(V0)
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, (256, 256, 256))
    fid = g.addFunction(dg.MeshSignedDistance(md))
    for s in (1, 2):
        runs = []
        for _ in range(2):
            c = T(g.m_nodes[fid], True)
            V, _, E = g.isosurface(fid, 0.0, s, device=True, coefficients=c, edges=True)
            (V * 0.5 + V * V).sum().backward()
            sync()
            runs.append((N(V), N(E), N(c.grad)))
        assert len(runs[0][1]) > 100000
        for a, b in zip(runs[0], runs[1]):
            assert np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64)), f"s={s}"
        assert np.isfinite(runs[0][2]).all()


def test_cpp_facade_isosurface_vjp_on_device(dg, tmp_path):
    """CubicLagrangeDiscreteGrid::isosurface with edge ids and isosurface_vjp (tests/cpp/isosurface_grad_check.cpp) give the Python route's
    vertices, edge ids and node gradient"""
    import subprocess
    exe = os.path.join(ROOT, "build", "bin", "isosurface_grad_check")
    if not os.path.exists(exe):
        pytest.skip("build/bin/isosurface_grad_check not built (make cpp)")
    g, fid, v = sphere_grid(dg, 10)
    gpath = str(tmp_path / "g.cdf")
    g.save(gpath)
    Vh, _, Eh = g.isosurface(fid, 0.01, 2, edges=True)
    gV = np.random.default_rng(4).standard_normal(Vh.shape)
    gpath_v = str(tmp_path / "gv.f64"); gV.tofile(gpath_v)
    out = str(tmp_path / "out.f64")
    r = subprocess.run([exe, gpath, "0.01", "2", gpath_v, out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(out, np.float64)
    c = T(v, True)
    V, _, E = g.isosurface(fid, 0.01, 2, device=True, coefficients=c, edges=True)
    (V * T(gV)).sum().backward()
    sync()
    want = np.concatenate([Vh.reshape(-1), Eh.astype(np.float64), N(c.grad)])
    assert same_bits(got, want)
