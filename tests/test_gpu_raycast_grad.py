"""K12 on the device: dg_mesh_raycast_vjp[_device] and dg_field_raycast_vjp[_device] bit for bit against the numpy restatement of the
contract (tests/raycast_grad_ref.py) on the families of tests/test_raycast_grad_emulated.py, and the autograd of
TriangleMeshDistance.raycast and CubicLagrangeDiscreteGrid.raycast: gradcheck, the saved positions, double backward, the host route
against the tensor route, streams, and large calls."""
import os

import numpy as np
import pytest

from conftest import ROOT, GOLDEN, ref_resource
import raycast_grad_ref as ref
from test_raycast_grad_emulated import (field_rays, mesh_rays, run_field_edge_cases, run_field_families, run_field_refusals,
                                        run_mesh_edge_cases, run_mesh_families, run_mesh_refusals, same_bits, torus_sdf)

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


def test_mesh_families_on_device():
    run_mesh_families(capi().lib, n=300 if capi().EMULATED else 20000)


def test_mesh_edge_cases_on_device():
    run_mesh_edge_cases(capi().lib)


def test_mesh_refusals_on_device():
    run_mesh_refusals(capi().lib)


def test_field_families_on_device():
    run_field_families(capi().lib, n=100 if capi().EMULATED else 20000)


def test_field_edge_cases_on_device():
    run_field_edge_cases(capi().lib)


def test_field_refusals_on_device():
    run_field_refusals(capi().lib)


def _torus(dg, nu=12, nv=8):
    m = dg.bumpy_torus(nu, nv)
    return m.vertices, m.faces


def _clean_rays(md, V, rng, n, margin=0.1):
    """camera rays whose hits lie away from every edge (finite differences stay on one triangle)"""
    o, d, _ = mesh_rays(V, None, rng, 8 * n)["camera"]
    t, tid, b, _ = md.raycast(o, d)
    ok = np.flatnonzero((tid >= 0) & (np.nan_to_num(b, nan=0.0).min(1) > margin))[:n]
    assert len(ok) >= n // 2
    return o[ok], d[ok]


def test_mesh_autograd_bits_and_saved_positions(dg):
    """the tensor route's gradients are the restatement's; a refit between forward and backward changes nothing, with V given or not"""
    import torch
    V, F = _torus(dg, 24, 16)
    md = dg.TriangleMeshDistance(V, F)
    rng = np.random.default_rng(1)
    o, d, _ = mesh_rays(V, F, rng, 400)["camera"]
    gt, gb = rng.standard_normal(len(o)), rng.standard_normal((len(o), 3))
    ot, dt_, Vt = T(o, True), T(d, True), T(V, True)
    t, tid, bary, st = md.raycast(ot, dt_, vertices=Vt)
    assert not tid.requires_grad and not st.requires_grad
    md.refit(V + 0.3)                                            # the backward reads the saved V, not the mesh's records
    ((t * T(gt)).nan_to_num(0.0, 0.0, 0.0).sum() + (bary * T(gb)).nan_to_num(0.0, 0.0, 0.0).sum()).backward()
    sync()
    go, gd, valid = ref.mesh_ray_grads(V, F, d, N(t), N(tid), np.where(N(tid) >= 0, gt, 0.0), np.where(N(tid)[:, None] >= 0, gb, 0.0))
    gv = ref.mesh_grad_vertices(F, len(V), N(tid), N(bary), go, valid)
    assert same_bits(N(ot.grad), go) and same_bits(N(dt_.grad), gd) and same_bits(N(Vt.grad), gv)
    # no V: the positions of the last construct / refit, uploaded at the backward
    md2 = dg.TriangleMeshDistance(V, F)
    ot2 = T(o, True)
    t2, tid2, b2, _ = md2.raycast(ot2, T(d))
    md2.refit(V * 1.5)
    ((t2 * T(gt)).nan_to_num(0.0, 0.0, 0.0).sum() + (b2 * T(gb)).nan_to_num(0.0, 0.0, 0.0).sum()).backward()
    sync()
    assert same_bits(N(ot2.grad), go)


def test_mesh_gradcheck_torus(dg):
    import torch
    V, F = _torus(dg)
    md = dg.TriangleMeshDistance(V, F)
    o, d = _clean_rays(md, V, np.random.default_rng(2), 6)
    ot, dt_, Vt = T(o, True), T(d, True), T(V, True)
    fn = lambda a, b, c: tuple(x for x in md.raycast(a, b, vertices=c) if x.dtype == torch.float64)
    assert torch.autograd.gradcheck(fn, (ot, dt_, Vt), eps=1e-6, atol=1e-5, rtol=1e-4)


def test_mesh_gradcheck_bunny(dg):
    import torch
    p = ref_resource("bunny.obj")
    if p is None:
        pytest.skip("bunny.obj not staged (make -C oracle ref)")
    from winding_ref import read_obj
    V, F = read_obj(p)
    md = dg.TriangleMeshDistance(V, F)
    o, d = _clean_rays(md, V, np.random.default_rng(3), 4, margin=0.15)
    fn = lambda a, b: tuple(x for x in md.raycast(a, b) if x.dtype == torch.float64)
    assert torch.autograd.gradcheck(fn, (T(o, True), T(d, True)), eps=1e-7, atol=1e-5, rtol=1e-4)
    # in V: a subset of the vertices of the hit triangles
    _, tid, _, _ = md.raycast(o, d)
    idx = np.unique(np.asarray(F, np.int64)[tid].reshape(-1))
    Vt = T(V)
    def fv(sub):
        full = Vt.clone(); full[idx] = sub
        return tuple(x for x in md.raycast(T(o), T(d), vertices=full) if x.dtype == torch.float64)
    assert torch.autograd.gradcheck(fv, (T(np.asarray(V)[idx], True),), eps=1e-7, atol=1e-5, rtol=1e-4)


def _sdf_grid(dg, res=(12, 12, 6)):
    g = dg.CubicLagrangeDiscreteGrid([-1.0, -1.0, -0.5], [1.0, 1.0, 0.5], list(res))
    X = np.asarray(g.nodePositions(), np.float64).reshape(-1, 3)
    fid = g.addSampledFunction(torus_sdf(X))
    return g, fid, torus_sdf(X)


def test_field_autograd_bits_and_gradcheck(dg):
    """t_lo and t_hi of the trainable route: gradients equal the restatement; gradcheck in o, d and a subset of c"""
    import torch
    g, fid, nodes = _sdf_grid(dg)
    rng = np.random.default_rng(4)
    o, d, _ = field_rays(rng, 300)["camera"]
    c = T(nodes + 0.01 * rng.standard_normal(len(nodes)), True)
    ot, dt_ = T(o, True), T(d, True)
    t_lo, t_hi, st = g.raycast(fid, ot, dt_, coefficients=c)
    assert not st.requires_grad
    glo, ghi = rng.standard_normal(len(o)), rng.standard_normal(len(o))
    hit = N(st) != 0
    ((t_lo * T(np.where(hit, glo, 0.0))).sum() + (t_hi * T(np.where(hit, ghi, 0.0))).sum()).backward()
    sync()
    g2, fid2, _ = _sdf_grid(dg)
    g2.setNodes(fid2, N(c))
    xc = ref.crossing_points(g._desc.domain_min[:], g._desc.domain_max[:], o, d, N(t_lo), N(st))
    phi, grad = g2.interpolate(fid2, xc, gradient=True)
    go, gd, gphi, valid = ref.field_ray_grads(d, N(t_lo), N(st), phi, grad, np.where(hit, glo, 0.0), np.where(hit, ghi, 0.0))
    dd = g._desc
    gn = ref.field_grad_nodes(dd.domain_min[:], dd.domain_max[:], dd.cell_size[:], dd.inv_cell_size[:], dd.resolution[:], N(c),
                              g.m_cells[fid], np.asarray(g.m_cell_map[fid], np.uint32), xc, gphi, valid)
    assert same_bits(N(ot.grad), go) and same_bits(N(dt_.grad), gd) and same_bits(N(c.grad), gn)
    # the dense field without coefficients=: origins and directions only
    ot3 = T(o, True)
    t3, _, _ = g2.raycast(fid2, ot3, T(d))
    (t3 * T(np.where(hit, glo, 0.0))).nan_to_num(0.0, 0.0, 0.0).sum().backward()
    sync()
    go3, _, _, _ = ref.field_ray_grads(d, N(t3), N(st), phi, grad, np.where(hit, glo, 0.0), None)
    assert same_bits(N(ot3.grad), go3)
    # gradcheck at crossings away from cell faces
    frac = ((np.where(np.isfinite(xc), xc, 0.0) - np.asarray(dd.domain_min[:])) * np.asarray(dd.inv_cell_size[:])) % 1.0
    sel = np.flatnonzero(hit & (frac.min(1) > 0.15) & (frac.max(1) < 0.85))[:4]
    assert len(sel) >= 2
    fo = lambda a, b: g.raycast(fid, a, b, coefficients=c.detach())[0]
    assert torch.autograd.gradcheck(fo, (T(o[sel], True), T(d[sel], True)), eps=1e-7, atol=1e-5, rtol=1e-4)
    idx = np.argsort(-np.abs(N(c.grad)))[:6]
    cb = c.detach()
    def fc(sub):
        full = cb.clone(); full[idx] = sub
        return g.raycast(fid, T(o[sel]), T(d[sel]), coefficients=full)[0]
    assert torch.autograd.gradcheck(fc, (T(N(cb)[idx], True),), eps=1e-7, atol=1e-5, rtol=1e-4)


def test_double_backward_raises_and_vertex_count_refused(dg):
    import torch
    V, F = _torus(dg)
    md = dg.TriangleMeshDistance(V, F)
    o, d = _clean_rays(md, V, np.random.default_rng(5), 4)
    ot = T(o, True)
    t = md.raycast(ot, T(d))[0]
    (go,) = torch.autograd.grad(t.sum(), ot, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(go.sum(), ot)
    with pytest.raises(ValueError):
        md.raycast(ot, T(d), vertices=T(np.asarray(V)[:-1], True))
    g, fid, nodes = _sdf_grid(dg)
    c = T(nodes, True)
    t_lo = g.raycast(fid, T(o, True), T(d), coefficients=c)[0]
    (gc,) = torch.autograd.grad(t_lo.nan_to_num(0.0, 0.0, 0.0).sum(), c, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(gc.sum(), c)
    with pytest.raises(ValueError):
        g.raycast(fid, T(o), T(d), coefficients=c[:-1])
    with pytest.raises(TypeError):
        g.raycast(fid, o, d, coefficients=c)


def test_tensor_route_equals_host_route_on_two_streams_and_again(dg):
    import torch
    lib = capi().lib
    V, F = _torus(dg, 60, 40)
    md = dg.TriangleMeshDistance(V, F)
    rng = np.random.default_rng(6)
    o, d, _ = mesh_rays(V, F, rng, 200000)["camera"]
    t, tid, b, _ = md.raycast(o, d)
    gt, gb = rng.standard_normal(len(o)), rng.standard_normal((len(o), 3))
    Vh = np.ascontiguousarray(V, np.float64)
    host = [np.empty((len(o), 3)), np.empty((len(o), 3)), np.empty((len(Vh), 3))]
    c = capi()
    c.check(lib.dg_mesh_raycast_vjp(md.handle, len(o), c.ptr(d, c.F64P), c.ptr(t, c.F64P), c.ptr(tid, c.I32P), c.ptr(b, c.F64P),
                                    c.ptr(Vh, c.F64P), c.ptr(gt, c.F64P), c.ptr(gb, c.F64P), *(c.ptr(a, c.F64P) for a in host)))
    runs = []
    for s in range(3):
        stream = torch.cuda.Stream() if s == 2 else torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            ot, dt_, Vt = T(o, True), T(d, True), T(V, True)
            tt, _, bb, _ = md.raycast(ot, dt_, vertices=Vt)
            ((tt * T(gt)).nan_to_num(0.0, 0.0, 0.0).sum() + (bb * T(gb)).nan_to_num(0.0, 0.0, 0.0).sum()).backward()
        torch.cuda.synchronize()
        runs.append((N(ot.grad), N(dt_.grad), N(Vt.grad)))
    for r in runs:
        for a, w in zip(r, host):
            assert same_bits(a, np.where(np.isnan(w), 0.0, w))
    g, fid, nodes = _sdf_grid(dg, (48, 48, 24))
    o, d, _ = field_rays(rng, 200000)["camera"]
    tl, th, st = g.raycast(fid, o, d)
    glo = rng.standard_normal(len(o))
    hg = [np.empty((len(o), 3)), np.empty((len(o), 3))]
    c.check(lib.dg_field_raycast_vjp(g._device_field(fid), len(o), c.ptr(o, c.F64P), c.ptr(d, c.F64P), c.ptr(tl, c.F64P), c.ptr(st, c.I32P),
                                     c.ptr(glo, c.F64P), None, *(c.ptr(a, c.F64P) for a in hg), None))
    for s in range(3):
        stream = torch.cuda.Stream() if s == 2 else torch.cuda.current_stream()
        with torch.cuda.stream(stream):
            ot, dt_ = T(o, True), T(d, True)
            t_lo = g.raycast(fid, ot, dt_)[0]
            (t_lo * T(np.where(st != 0, glo, 0.0))).nan_to_num(0.0, 0.0, 0.0).sum().backward()
        torch.cuda.synchronize()
        assert same_bits(N(ot.grad), hg[0]) and same_bits(N(dt_.grad), hg[1])


def test_large_bunny_calls(dg):
    """10^6 rays through each cast's backward on the bunny (mesh, and its 128^3 trainable SDF)"""
    import torch
    p = ref_resource("bunny.obj")
    if p is None:
        pytest.skip("bunny.obj not staged (make -C oracle ref)")
    from winding_ref import read_obj
    V, F = read_obj(p)
    md = dg.TriangleMeshDistance(V, F)
    rng = np.random.default_rng(8)
    o, d, _ = mesh_rays(V, F, rng, 1000000)["camera"]
    ot, Vt = T(o, True), T(V, True)
    t, tid, b, _ = md.raycast(ot, T(d), vertices=Vt)
    t.nan_to_num(0.0, 0.0, 0.0).sum().backward()
    sync()
    hit = N(tid) >= 0
    assert hit.sum() > 100000 and np.isfinite(N(ot.grad)).all() and np.isfinite(N(Vt.grad)).all()
    s = N(Vt.grad).sum(0) + N(ot.grad).sum(0)                  # translation invariance, summed over all rays
    assert np.abs(s).max() <= 1e-6 * np.abs(N(ot.grad)).sum()
    mn, mx = dg.generate_sdf_domain(V)
    grid = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
    fid = grid.addFunction(dg.MeshSignedDistance(md))
    c = T(grid.m_nodes[fid], True)
    ot = T(o, True)
    t_lo, _, st = grid.raycast(fid, ot, T(d), coefficients=c)
    t_lo.nan_to_num(0.0, 0.0, 0.0).sum().backward()
    sync()
    assert (N(st) != 0).sum() > 100000 and np.isfinite(N(c.grad)).all() and np.isfinite(N(ot.grad)).all()


def test_cpp_facade_raycast_vjp_on_device(dg, tmp_path):
    """TriangleMeshDistance::raycast_vjp and CubicLagrangeDiscreteGrid::raycast_vjp (tests/cpp/raycast_grad_check.cpp) give the Python
    route's gradients"""
    import subprocess
    import torch
    exe = os.path.join(ROOT, "build", "bin", "raycast_grad_check")
    if not os.path.exists(exe):
        pytest.skip("build/bin/raycast_grad_check not built (make cpp)")
    from discregrid_b200.mesh import TriangleMesh
    mesh_path = os.path.join(GOLDEN, "sphere.obj")
    m = TriangleMesh(mesh_path)
    V, F = np.ascontiguousarray(m.vertices, np.float64), m.faces
    md = dg.TriangleMeshDistance(V, F)
    g, fid, nodes = _sdf_grid(dg)
    gpath = str(tmp_path / "g.cdf")
    g.save(gpath)
    rng = np.random.default_rng(9)
    n = 3000
    o = np.tile([0.13, -0.07, 2.5], (n, 1)); d = (rng.random((n, 3)) - 0.5) * np.array([1.6, 1.6, 0.0]) - np.array([0.0, 0.0, 2.5])
    gt, gb, v = rng.standard_normal(n), rng.standard_normal((n, 3)), nodes + 0.01 * rng.standard_normal(len(nodes))
    files = []
    for name, a in (("V", V), ("v", v), ("o", o), ("d", d), ("gt", gt), ("gb", gb)):
        files.append(str(tmp_path / f"{name}.f64")); np.ascontiguousarray(a, np.float64).tofile(files[-1])
    out = str(tmp_path / "out.f64")
    r = subprocess.run([exe, mesh_path, files[0], gpath, *files[1:], out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(out, np.float64)
    ot, dt_, Vt = T(o, True), T(d, True), T(V, True)
    t, tid, b, _ = md.raycast(ot, dt_, 0.0, 1e300, vertices=Vt)
    hit = N(tid) >= 0
    ((t * T(np.where(hit, gt, 0.0))).nan_to_num(0.0, 0.0, 0.0).sum() + (b * T(np.where(hit[:, None], gb, 0.0))).nan_to_num(0.0, 0.0, 0.0).sum()).backward()
    c = T(v, True)
    of, df = T(o, True), T(d, True)
    t_lo, _, st = g.raycast(fid, of, df, 0.0, 0.0, 1e300, coefficients=c)
    (t_lo * T(np.where(N(st) != 0, gt, 0.0))).nan_to_num(0.0, 0.0, 0.0).sum().backward()
    sync()
    want = np.concatenate([N(a).reshape(-1) for a in (ot.grad, dt_.grad, Vt.grad, of.grad, df.grad, c.grad)])
    assert same_bits(got, want)
