"""Differentiable mesh distances on the device (K10, discregrid_b200/csrc/k10_distance_grad.cu, radix_sort.cu and K1's
mesh_distance_bary_kernel): TriangleMeshDistance.nearest against signed_distance / unsigned_distance and the weights, grad_points and
grad_vertices against the numpy restatement (tests/mesh_distance_grad_ref.py) bit for bit on box, sphere and torus in both sign modes; the
same bits on two streams and on a repeated call; the CUDA-tensor route against the host route; torch.autograd.gradcheck in the points and in
the vertices on the torus and bunny.obj; the gradient after a refit between forward and backward; a double backward raising; bunny.obj with
10^6 points; and the refusals."""

import numpy as np
import pytest

from test_gpu_isosurface import mesh_of
import mesh_distance_grad_ref as gr
import winding_ref as wr

pytestmark = pytest.mark.gpu


def capi():
    from discregrid_b200 import _capi
    return _capi


def mesh(dg, name):
    if name == "sphere":
        m = dg.uv_sphere(24, 48, 0.8)
        return np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)
    if name == "open_torus":
        V, F = mesh_of(dg, "torus")
        return wr.cut_top(V, F)
    return mesh_of(dg, name)


def queries(V, n, seed):
    """random points around the mesh, some on its vertices (d == 0), some NaN (no triangle)"""
    rng = np.random.default_rng(seed)
    lo, hi = V.min(0), V.max(0)
    x = 0.5 * (lo + hi) + rng.uniform(-1, 1, (n, 3)) * 0.7 * (hi - lo)
    k = max(1, n // 16)
    x[:k] = V[rng.integers(0, len(V), k)]
    x[k:2 * k:3] = np.nan
    return np.ascontiguousarray(x[rng.permutation(n)])


def vjp_host(md, x, r, g, points=True, vertices=True):
    c = capi()
    n = len(x)
    gp = np.full((n, 3), 7.0) if points else None
    gv = np.full((md.n_vertices, 3), 7.0) if vertices else None
    rc = c.lib.dg_mesh_distance_vjp(md.handle, n, c.ptr(x, c.F64P), c.ptr(r.distance, c.F64P), c.ptr(r.nearest_point, c.F64P),
                                    c.ptr(r.triangle_id, c.I32P), c.ptr(r.barycentric, c.F64P), c.ptr(g, c.F64P), c.ptr(gp, c.F64P),
                                    c.ptr(gv, c.F64P))
    return rc, gp, gv


def restated(V, F, x, r, g):
    s, t, ent = gr.leaf_params(V, F, r.triangle_id, x)
    w = gr.weights(s, t)
    gx = gr.grad_points(x, r.distance, r.nearest_point, r.triangle_id, g)
    return w, gx, gr.grad_vertices(F, len(V), r.triangle_id, gx, w), ent


def bits(a, b, what):
    assert gr.same_bits(a, b), f"{what}: {np.count_nonzero(np.asarray(a).view(np.uint64) != np.asarray(b).view(np.uint64))} values differ"


@pytest.mark.parametrize("name,mode,signed", [("box", "pseudonormal", True), ("sphere", "pseudonormal", True), ("torus", "pseudonormal", True),
                                              ("torus", "pseudonormal", False), ("open_torus", "winding", True)])
def test_equals_restatement(dg, name, mode, signed):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F).set_sign_mode(mode)
    for n in (2000, 1001):
        x = queries(V, n, n)
        r = md.nearest(x, signed)
        want = md.signed_distance(x) if signed else md.unsigned_distance(x)
        for k in range(4):
            assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)), f"{name}: field {k}"
        assert (r.triangle_id == -1).any() and (r.distance == 0).any()
        g = np.random.default_rng(n).standard_normal(n)
        w, gx, gv, ent = restated(V, F, x, r, g)
        bits(r.barycentric, w, f"{name}: barycentric")
        hit = r.triangle_id >= 0
        assert np.array_equal(ent[hit], r.nearest_entity[hit])
        rc, gp_c, gv_c = vjp_host(md, x, r, g)
        assert rc == 0, capi().lib.dg_last_error()
        bits(gp_c, gx, f"{name}: grad_points")
        bits(gv_c, gv, f"{name}: grad_vertices")
        rc, gp2, gv2 = vjp_host(md, x, r, g)                      # a repeated call
        bits(gp2, gp_c, "repeat"); bits(gv2, gv_c, "repeat")


def test_long_segment_and_zero_queries(dg):
    """every query on one triangle of the box (a segment of 40 000 queries), and n = 0"""
    V, F = mesh(dg, "box")
    md = dg.TriangleMeshDistance(V, F)
    rng = np.random.default_rng(3)
    a, b, c = V[F[5, 0]], V[F[5, 1]], V[F[5, 2]]
    u = rng.random((40000, 2))
    u = np.where(u.sum(1, keepdims=True) > 1, 1 - u, u) * 0.98 + 0.005
    nrm = np.cross(b - a, c - a)
    x = np.ascontiguousarray(a + u[:, :1] * (b - a) + u[:, 1:] * (c - a) + rng.uniform(0.01, 0.2, (40000, 1)) * nrm / np.linalg.norm(nrm))
    r = md.nearest(x)
    assert (r.triangle_id == 5).all()
    g = rng.standard_normal(len(x))
    _, gx, gv, _ = restated(V, F, x, r, g)
    rc, gp_c, gv_c = vjp_host(md, x, r, g)
    assert rc == 0
    bits(gp_c, gx, "grad_points"); bits(gv_c, gv, "grad_vertices")
    e = np.empty((0, 3))
    r0 = md.nearest(e)
    rc, gp0, gv0 = vjp_host(md, e, r0, np.empty(0))
    assert rc == 0 and gp0.shape == (0, 3) and gr.same_bits(gv0, np.zeros_like(gv0))


def test_refusals(dg):
    c = capi()
    V, F = mesh(dg, "box")
    md = dg.TriangleMeshDistance(V, F)
    x = queries(V, 100, 4)
    r = md.nearest(x)
    g = np.ones(len(x))
    for bad in (12, 10 ** 6, -2):
        tri = r.triangle_id.copy(); tri[50] = bad
        rc, gp, gv = vjp_host(md, x, r._replace(triangle_id=tri), g)
        assert rc == c.DG_ERR_INVALID and "triangle ids outside" in c.lib.dg_last_error().decode()
        assert (gp == 7.0).all() and (gv == 7.0).all(), "nothing is written before a refusal"
    gv = np.empty((len(V), 3))
    assert c.lib.dg_mesh_distance_vjp(None, len(x), c.ptr(x, c.F64P), c.ptr(r.distance, c.F64P), c.ptr(r.nearest_point, c.F64P),
                                      c.ptr(r.triangle_id, c.I32P), c.ptr(r.barycentric, c.F64P), c.ptr(g, c.F64P), None,
                                      c.ptr(gv, c.F64P)) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_distance_bary(None, c.ptr(x, c.F64P), len(x), 1, None, None, None, None, None) == c.DG_ERR_INVALID
    assert c.lib.dg_last_error().decode().startswith("dg_mesh_distance_bary:")
    if dg.device_count() > 1:                                     # a mesh on another device
        dg._capi.check(c.lib.dg_set_device(1))
        try:
            md1 = dg.TriangleMeshDistance(V, F)
        finally:
            dg._capi.check(c.lib.dg_set_device(0))
        rc, _, _ = vjp_host(md1, x, r, g)
        assert rc == c.DG_ERR_INVALID and "device" in c.lib.dg_last_error().decode()


# ------------------------------------------------------------------------------------------------ CUDA tensors and autograd
def test_tensor_route_equals_host_route_on_two_streams(dg):
    import torch
    V, F = mesh(dg, "torus")
    md = dg.TriangleMeshDistance(V, F)
    x = queries(V, 5000, 5)
    r = md.nearest(x)
    xt = torch.from_numpy(x).cuda()
    rt = md.nearest(xt)
    for k in range(5):
        assert np.array_equal(np.asarray(rt[k].cpu()).view(np.uint8), np.asarray(r[k]).view(np.uint8)), f"field {k}"
    g = np.random.default_rng(6).standard_normal(len(x))
    _, gp_h, gv_h = vjp_host(md, x, r, g)
    gt = torch.from_numpy(g).cuda()

    def device_vjp():
        gp = torch.empty((len(x), 3), dtype=torch.float64, device="cuda")
        gv = torch.empty((md.n_vertices, 3), dtype=torch.float64, device="cuda")
        capi().check(capi().lib.dg_mesh_distance_vjp_device(md.handle, len(x), xt.data_ptr(), rt.distance.data_ptr(), rt.nearest_point.data_ptr(),
                                                            rt.triangle_id.data_ptr(), rt.barycentric.data_ptr(), gt.data_ptr(), gp.data_ptr(),
                                                            gv.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return gp.cpu().numpy(), gv.cpu().numpy()
    for _ in range(2):
        gp, gv = device_vjp()
        bits(gp, gp_h, "grad_points, device form"); bits(gv, gv_h, "grad_vertices, device form")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gp, gv = device_vjp()
    bits(gp, gp_h, "grad_points, side stream"); bits(gv, gv_h, "grad_vertices, side stream")
    # autograd gives the same bits (vertices=V refits the mesh to its own vertices first: compare with the host route after that refit)
    xg = xt.clone().requires_grad_(True)
    Vt = torch.from_numpy(V).cuda().requires_grad_(True)
    d = md.signed_distance(xg, vertices=Vt).distance
    d.backward(gt)
    r2 = md.nearest(x)
    assert gr.same_bits(d.detach().cpu().numpy(), r2.distance)
    _, gp_h2, gv_h2 = vjp_host(md, x, r2, g)
    bits(xg.grad.cpu().numpy(), gp_h2, "autograd grad in x")
    bits(Vt.grad.cpu().numpy(), gv_h2, "autograd grad in V")


def generic_points(md, V, n, seed, eps=1e-5):
    """points near the surface whose nearest triangle and entity stay the same under +-eps in every axis and which lie in a face region"""
    rng = np.random.default_rng(seed)
    lo, hi = V.min(0), V.max(0)
    x = 0.5 * (lo + hi) + rng.uniform(-1, 1, (40 * n, 3)) * 0.6 * (hi - lo)
    r = md.signed_distance(x)
    ok = (r.nearest_entity == 6) & (np.abs(r.distance) > 1e-3)
    for k in range(3):
        for sgn in (-1, 1):
            y = x.copy(); y[:, k] += sgn * 100 * eps
            ry = md.signed_distance(y)
            ok &= (ry.triangle_id == r.triangle_id) & (ry.nearest_entity == r.nearest_entity)
    x = x[ok][:n]
    assert len(x) == n
    return np.ascontiguousarray(x)


def _gradcheck(dg, name):
    import torch
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    x = generic_points(md, V, 12, 7)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda p: md.signed_distance(p).distance, (xt,), eps=1e-6, atol=1e-7, rtol=1e-5)
    assert torch.autograd.gradcheck(lambda p: md.unsigned_distance(p).distance, (xt,), eps=1e-6, atol=1e-7, rtol=1e-5)
    # in V: the vertices of the nearest triangles move, the rest stay
    tri = md.signed_distance(x).triangle_id
    idx = torch.from_numpy(np.unique(F[tri].reshape(-1)).astype(np.int64)).cuda()
    V0 = torch.from_numpy(V).cuda()
    sub = V0[idx].clone().requires_grad_(True)
    xd = xt.detach()

    def f(s):
        Vs = V0.index_put((idx,), s)
        return md.signed_distance(xd, vertices=Vs).distance
    assert torch.autograd.gradcheck(f, (sub,), eps=1e-6, atol=1e-7, rtol=1e-5)


def test_tensor_gradcheck_torus(dg):
    _gradcheck(dg, "torus")


def test_tensor_gradcheck_bunny(dg):
    _gradcheck(dg, "bunny")


def test_tensor_refit_between_forward_and_backward(dg):
    import torch
    V, F = mesh(dg, "torus")
    md = dg.TriangleMeshDistance(V, F)
    x = torch.from_numpy(queries(V, 3000, 8)).cuda()
    g = torch.from_numpy(np.random.default_rng(9).standard_normal(3000)).cuda()
    grads = []
    for refit_again in (False, True):
        xg = x.clone().requires_grad_(True)
        Vt = torch.from_numpy(V).cuda().requires_grad_(True)
        d = md.signed_distance(xg, vertices=Vt).distance
        if refit_again:
            md.refit(torch.from_numpy(V * 1.1 + 0.05).cuda())
        d.backward(g)
        grads.append((xg.grad.cpu().numpy(), Vt.grad.cpu().numpy()))
    bits(grads[1][0], grads[0][0], "grad in x after a refit")
    bits(grads[1][1], grads[0][1], "grad in V after a refit")


def test_tensor_double_backward_raises(dg):
    import torch
    V, F = mesh(dg, "torus")
    md = dg.TriangleMeshDistance(V, F)
    x = torch.from_numpy(queries(V, 64, 10)).cuda().requires_grad_(True)
    d = md.signed_distance(x).distance
    (gx,) = torch.autograd.grad(d.sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()
    with pytest.raises((TypeError, ValueError)):
        md.signed_distance(x, vertices=torch.from_numpy(V).cuda().float())
    with pytest.raises(TypeError):
        md.signed_distance(x, vertices=V)


def test_large_bunny_tensor(dg):
    """10^6 points around bunny.obj through autograd in x and V, against the restatement"""
    import torch
    V, F = mesh(dg, "bunny")
    md = dg.TriangleMeshDistance(V, F)
    x = queries(V, 10 ** 6, 11)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    Vt = torch.from_numpy(V).cuda().requires_grad_(True)
    g = np.random.default_rng(12).standard_normal(len(x))
    r = md.signed_distance(xt, vertices=Vt)
    r.distance.backward(torch.from_numpy(g).cuda())
    rn = md.nearest(x)
    assert gr.same_bits(r.distance.detach().cpu().numpy(), rn.distance)
    w, gx, gv, _ = restated(V, F, x, rn, g)
    bits(rn.barycentric, w, "barycentric")
    bits(xt.grad.cpu().numpy(), gx, "grad in x")
    bits(Vt.grad.cpu().numpy(), gv, "grad in V")
