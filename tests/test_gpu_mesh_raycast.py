"""Ray casts on a mesh on the device (K9, discregrid_b200/csrc/k9_mesh_raycast.cu): TriangleMeshDistance.raycast against the brute-force
numpy restatement of the contract (tests/mesh_raycast_ref.py) bit for bit on box, sphere, torus, bunny.obj and dragon.obj, and after a refit
(before and after the first cast); no leaks through vertices and edges; status against K5's winding number; the hit point against the
barycentric weights and against dg_mesh_distance; K7's hits on bunny SDFs against K9's along the same rays; the CUDA-tensor route (also from
a side stream) and 10 M rays in one call; the C++ facade; and the refusals."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, ref_resource
from test_gpu_isosurface import diag, mesh_of, sdf_grid
import mesh_raycast_ref as mr
import winding_ref as wr

pytestmark = pytest.mark.gpu

CHECK = os.path.join(ROOT, "build", "bin", "mesh_raycast_check")
INF = float("inf")


def capi():
    from discregrid_b200 import _capi
    return _capi


def mesh(dg, name):
    if name == "sphere":
        m = dg.uv_sphere(24, 48, 0.8)
        return np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)
    return mesh_of(dg, name)


def mixed(V, F, n, seed):
    rng = np.random.default_rng(seed)
    parts = [mr.random_rays(V, n, rng), mr.aimed_rays(V, F, n, rng), mr.axis_rays(V, n // 4, rng), mr.in_plane_rays(V, F, n // 4, rng)]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def same(got, want, what):
    for g, w, nm in zip(got, want, ("t", "triangle_id", "barycentric", "status")):
        g, w = np.asarray(g), np.asarray(w)
        ok = mr.same_bits(g, w) if g.dtype == np.float64 else np.array_equal(g, w)
        if not ok:
            gb = g.view(np.uint64).reshape(len(g), -1) if g.dtype == np.float64 else g.reshape(len(g), -1)
            wb = w.view(np.uint64).reshape(len(w), -1) if w.dtype == np.float64 else w.reshape(len(w), -1)
            bad = np.flatnonzero((gb != wb).any(axis=1))
            raise AssertionError(f"{what}: {nm} differs on {len(bad)} rays, first {bad[0]}: {g[bad[0]]!r} vs {w[bad[0]]!r}")


@pytest.mark.parametrize("name", ["box", "sphere", "torus"])
@pytest.mark.parametrize("mode", ["pseudonormal", "winding"])
def test_equals_restatement(dg, name, mode):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F).set_sign_mode(mode)
    O, D = mixed(V, F, 1500, 1)
    for lo, hi in ((0.0, INF), (0.0, 1.0), (-INF, INF), (-0.5, 2.0)):
        same(md.raycast(O, D, lo, hi), mr.raycast(V, F, O, D, lo, hi), f"{name} on [{lo}, {hi}]")


@pytest.mark.parametrize("name", ["bunny", "dragon"])
def test_bunny_and_dragon_equal_restatement(dg, name):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    O, D = mixed(V, F, 1000, 2)
    got = md.raycast(O, D)
    same(got, mr.raycast(V, F, O, D), name)
    assert (got[3] != mr.MISS).mean() > 0.4


def test_refit_before_and_after_the_first_cast(dg):
    from test_gpu_refit import twist
    V, F = mesh(dg, "torus")
    V1 = np.ascontiguousarray(twist(V, 0.8))
    O, D = mixed(V1, F, 1500, 3)
    want = mr.raycast(V1, F, O, D)
    a = dg.TriangleMeshDistance(V, F).refit(V1)              # refit first: the vertex records are built by the refit's kernels
    same(a.raycast(O, D), want, "refit before the first cast")
    b = dg.TriangleMeshDistance(V, F)
    same(b.raycast(O, D), mr.raycast(V, F, O, D), "before the refit")
    b.refit(V1)                                               # the existing records are refit in place
    same(b.raycast(O, D), want, "refit after the first cast")
    b.refit(V)
    same(b.raycast(O, D), mr.raycast(V, F, O, D), "refit back")


INSIDE = {"box": lambda V: 0.5 * (V.min(0) + V.max(0)), "sphere": lambda V: np.array([0.01, -0.02, 0.03]),
          "torus": lambda V: np.array([1.0, 0.0, 0.0])}


@pytest.mark.parametrize("name", ["box", "sphere", "torus"])
def test_no_leaks(dg, name):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    O, D = mr.leak_rays(V, F, INSIDE[name](V))
    got = md.raycast(O, D)
    same(got, mr.raycast(V, F, O, D), name + " leak rays")
    assert np.all(got[3] != mr.MISS), f"{int(np.sum(got[3] == mr.MISS))} of {len(O)} rays leak"


@pytest.mark.parametrize("name", ["box", "sphere", "torus"])
def test_status_follows_the_winding_number(dg, name):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    rng = np.random.default_rng(4)
    size = float(np.abs(V.max(0) - V.min(0)).max())
    O, D = mr.random_rays(V, 6000, rng, 1.3)
    far = np.abs(md.unsigned_distance(O).distance) > 0.02 * size
    O, D = O[far], D[far]
    w = md.winding_number(O, float("inf"))
    t, tid, b, st = md.raycast(O, D)
    inside = w > 0.5
    assert inside.sum() > 100 and (~inside).sum() > 100
    assert np.all(st[inside] == mr.LEAVE)
    assert np.all(st[~inside] != mr.LEAVE)
    assert (st[~inside] == mr.ENTER).sum() > 100


@pytest.mark.parametrize("name", ["torus", "bunny"])
def test_hit_points_are_consistent(dg, name):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    rng = np.random.default_rng(5)                     # rays in general position (a ray in a triangle's plane has no well-defined hit point)
    parts = [mr.random_rays(V, 3000, rng), mr.aimed_rays(V, F, 3000, rng)]
    O, D = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    t, tid, b, st = md.raycast(O, D)
    h = st != mr.MISS
    x = O[h] + t[h, None] * D[h]
    y = (b[h, :, None] * V[F[tid[h]].astype(np.int64)]).sum(axis=1)
    size = float(np.abs(V).max())
    rel = float(np.abs(x - y).max()) / size
    dist = float(np.abs(md.unsigned_distance(x).distance).max()) / size
    print(f"{name}: {int(h.sum())} hits; max |o + t d - sum b_i v_i| = {rel:.2e}, max mesh distance = {dist:.2e} (relative to max |v|)")
    # K1's distance is the square root of a squared distance formed with cancellation: on the surface it is ~sqrt(eps) * size, not 0
    assert rel < 1e-12 and dist < 1e-7


@pytest.mark.parametrize("res", [128, 256])
def test_bunny_k7_hits_agree_with_the_mesh(dg, res):
    g, md, V, F = sdf_grid(dg, "bunny", (res, res, res))
    rng = np.random.default_rng(6)
    mn, mx = g.domain()
    ext = mx - mn
    O = mn + rng.random((20000, 3)) * ext
    D = rng.standard_normal((20000, 3))
    out = np.abs(md.signed_distance(O).distance) > 2 * diag(g)
    outside = md.winding_number(O, float("inf")) < 0.5
    O, D = O[out & outside], D[out & outside]
    lo, hi, s7 = g.raycast(0, O, D)
    t, tid, b, s9 = md.raycast(O, D)
    both = (s7 == mr.ENTER) & (s9 == mr.ENTER)
    gap = np.linalg.norm((lo[both] - t[both])[:, None] * D[both], axis=1) / diag(g)
    near = np.abs(md.unsigned_distance(O[both] + lo[both, None] * D[both]).distance) / diag(g)
    print(f"bunny {res}^3: {int(both.sum())} rays hit both; K7 - K9 along the ray: median {np.median(gap):.4f}, 99th percentile "
          f"{np.percentile(gap, 99):.4f}, max {gap.max():.4f} cell diagonals; K7 hit to mesh: max {near.max():.4f} cell diagonals; "
          f"K9 only {int(((s9 == mr.ENTER) & (s7 != mr.ENTER)).sum())}, K7 only {int(((s7 == mr.ENTER) & (s9 != mr.ENTER)).sum())}")
    assert both.sum() > 2000
    assert near.max() < 0.5 and np.percentile(gap, 99) < 0.5


def test_tensor_route_same_bits_including_a_side_stream(dg):
    import torch
    V, F = mesh(dg, "torus")
    md = dg.TriangleMeshDistance(V, F)
    O, D = mixed(V, F, 5000, 7)
    want = md.raycast(O, D, -1.0, 3.0)
    Ot, Dt = torch.tensor(O, device="cuda"), torch.tensor(D, device="cuda")
    got = md.raycast(Ot, Dt, -1.0, 3.0)
    assert got[0].is_cuda and got[1].dtype == torch.int32 and got[2].shape == (len(O), 3)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        O2 = Ot * 1.0                                                # made on the side stream: the cast must see it
        side = md.raycast(O2, Dt, -1.0, 3.0)
    s.synchronize()
    for r in (got, side):
        same(tuple(x.cpu().numpy() for x in r), want, "tensor route")
    with pytest.raises(TypeError):
        md.raycast(Ot.float(), Dt)


def test_large_ten_million_rays(dg):
    import torch
    V, F = mesh(dg, "torus")
    md = dg.TriangleMeshDistance(V, F)
    n = 10_000_000
    gen = torch.Generator(device="cuda").manual_seed(0)
    O = torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=gen) * 3.0 - 1.5
    D = torch.randn((n, 3), dtype=torch.float64, device="cuda", generator=gen)
    t, tid, b, st = md.raycast(O, D)
    sample = torch.randint(0, n, (2000,), device="cuda", generator=gen)
    Os, Ds = O[sample].cpu().numpy(), D[sample].cpu().numpy()
    same((t[sample].cpu().numpy(), tid[sample].cpu().numpy(), b[sample].cpu().numpy(), st[sample].cpu().numpy()), mr.raycast(V, F, Os, Ds),
         "10 M rays, sample")
    print(f"10 M rays: {int((st == mr.ENTER).sum())} enter, {int((st == mr.LEAVE).sum())} leave")


def test_facade_equals_python(dg, tmp_path):
    if not os.path.exists(CHECK):
        pytest.skip("build/bin/mesh_raycast_check not built (make cpp)")
    V, F = mesh(dg, "torus")
    obj = tmp_path / "torus.obj"
    with open(obj, "w") as f:
        for v in V:
            f.write("v %.17g %.17g %.17g\n" % tuple(v))
        for tr in F:
            f.write("f %d %d %d\n" % tuple(tr + 1))
    O, D = mixed(V, F, 1000, 8)
    np.hstack([O, D]).tofile(tmp_path / "rays.f64")
    md = dg.TriangleMeshDistance(V, F)
    n = len(O)
    for t0, t1 in ((0.0, INF), (-1.0, 2.0)):
        out = tmp_path / "out.bin"
        r = subprocess.run([CHECK, str(obj), str(tmp_path / "rays.f64"), repr(t0), repr(t1), str(out)], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        raw = out.read_bytes()
        t = np.frombuffer(raw[:8 * n], np.float64)
        b = np.frombuffer(raw[8 * n:32 * n], np.float64).reshape(n, 3)
        tid = np.frombuffer(raw[32 * n:36 * n], np.int32)
        st = np.frombuffer(raw[36 * n:], np.int32)
        same((t, tid, b, st), md.raycast(O, D, t0, t1), f"facade on [{t0}, {t1}]")


def test_invalid_arguments(dg):
    import ctypes as C
    c = capi()
    V, F = mesh(dg, "box")
    md = dg.TriangleMeshDistance(V, F)
    O = np.zeros((4, 3)); D = np.ones((4, 3))
    t = np.full(4, 7.0); tid = np.full(4, 7, np.int32); b = np.full((4, 3), 7.0); st = np.full(4, 7, np.int32)
    P = lambda a, ty=c.F64P: c.ptr(a, ty)
    args = lambda: [P(O), P(D), 4]
    outs = lambda: [P(t), P(tid, c.I32P), P(b), P(st, c.I32P)]
    assert c.lib.dg_mesh_raycast(None, *args(), 0.0, 1.0, *outs()) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast(md.handle, *args(), float("nan"), 1.0, *outs()) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast(md.handle, *args(), 0.0, float("nan"), *outs()) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast(md.handle, *args(), 1.0, 0.0, *outs()) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast(md.handle, None, P(D), 4, 0.0, 1.0, *outs()) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast(md.handle, *args(), 0.0, 1.0, None, P(tid, c.I32P), P(b), P(st, c.I32P)) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast(md.handle, *args(), 0.0, 1.0, P(t), None, P(b), P(st, c.I32P)) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast(md.handle, *args(), 0.0, 1.0, P(t), P(tid, c.I32P), P(b), None) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast_device(None, None, None, 0, 0.0, 1.0, None, None, None, None, None) == c.DG_ERR_INVALID
    assert c.lib.dg_mesh_raycast_device(md.handle, None, None, 0, 1.0, 0.0, None, None, None, None, None) == c.DG_ERR_INVALID
    assert np.all(t == 7.0) and np.all(tid == 7) and np.all(b == 7.0) and np.all(st == 7)      # nothing written
    assert c.lib.dg_mesh_raycast(md.handle, None, None, 0, 0.0, 1.0, None, None, None, None) == c.DG_OK
    assert c.lib.dg_mesh_raycast(md.handle, *args(), 0.0, 1.0, P(t), P(tid, c.I32P), None, P(st, c.I32P)) == c.DG_OK   # barycentric optional
    with pytest.raises(ValueError):
        md.raycast(O, D[:3])
