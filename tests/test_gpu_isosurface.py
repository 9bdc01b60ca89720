"""Level sets on the device (K6, discregrid_b200/csrc/k6_isosurface.cu): CubicLagrangeDiscreteGrid.isosurface against the numpy restatement
of the contract (tests/isosurface_ref.py) bit for bit, on numpy arrays and CUDA tensors; closedness and orientation on SDFs of closed meshes;
dense == reduced band; the winding sign mode repairing an open mesh; the round trip through TriangleMeshDistance; the C++ facade through
DiscreteFieldToMesh; and a lattice large enough for several chunks of the values pass."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, ref_resource
import isosurface_ref as ir
import winding_ref as wr

pytestmark = pytest.mark.gpu

GENERATE_SDF = os.path.join(ROOT, "build", "bin", "GenerateSDF")
FIELD_TO_MESH = os.path.join(ROOT, "build", "bin", "DiscreteFieldToMesh")


def capi():
    from discregrid_b200 import _capi
    return _capi


def same_bits(a, b):
    """bit for bit; NaN counts as equal to NaN (the device's default NaN has another payload than the host's)"""
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64)))


def diag(g):
    return float(np.linalg.norm(g.cellSize()))


def sphere_sdf(x, c=(0.03, -0.02, 0.01), r=0.6):
    return np.linalg.norm(x - np.asarray(c), axis=1) - r


def analytic(dg, res, fn, mn=(-1, -1, -1), mx=(1, 1, 1)):
    g = dg.CubicLagrangeDiscreteGrid(np.array(mn, np.float64), np.array(mx, np.float64), res)
    g.addSampledFunction(fn(g.nodePositions()))
    return g


def mesh_of(dg, name):
    if name == "box":
        return wr.read_obj(os.path.join(GOLDEN, "box.obj"))
    if name == "torus":
        m = dg.bumpy_torus(48, 48, 1.0, 0.4, 0.05, 7, 5)
        return np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)
    if name == "sphere_mesh":
        m = dg.uv_sphere(24, 48, 0.8)
        return np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)
    base = name[5:] if name.startswith("open_") else name
    p = ref_resource(base + ".obj")
    if p is None:
        pytest.skip(f"{base}.obj not staged (make -C oracle ref)")
    V, F = wr.read_obj(p)
    return wr.cut_top(V, F) if name.startswith("open_") else (V, F)


def sdf_grid(dg, name, res, band=None, winding=False):
    V, F = mesh_of(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    if winding:
        md.set_sign_mode("winding")
    mn, mx = dg.generate_sdf_domain(V)
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, res)
    if band is None:
        g.addFunction(dg.MeshSignedDistance(md))
    else:
        g.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, band))
    return g, md, V, F


def field(dg, name):
    if name == "box_cdf":
        return dg.CubicLagrangeDiscreteGrid(os.path.join(GOLDEN, "box.cdf"))
    if name == "sphere":
        return analytic(dg, (9, 9, 9), sphere_sdf)
    if name == "torus":
        return sdf_grid(dg, "torus", (16, 16, 8))[0]
    if name == "torus_band":                                               # reduced narrow band of 2 cell diagonals
        V, _ = mesh_of(dg, "torus")
        mn, mx = dg.generate_sdf_domain(V)
        return sdf_grid(dg, "torus", (16, 16, 8), band=2.0 * float(np.linalg.norm((mx - mn) / np.array([16, 16, 8]))))[0]
    if name in ("bunny64", "bunny128"):
        r = int(name[5:])
        return sdf_grid(dg, "bunny", (r, r, r))[0]
    raise KeyError(name)


def restated(g, iso, s, field_id=0):
    L = ir.Lattice.of_grid(g, s)
    return ir.extract(L, ir.lattice_values(g, field_id, L), iso)


@pytest.mark.parametrize("name", ["box_cdf", "sphere", "torus", "torus_band"])
def test_equals_restatement(dg, name):
    g = field(dg, name)
    h = diag(g)
    for s in (1, 2, 3):
        for iso in (0.0, 0.5 * h, -0.5 * h):
            V, T = g.isosurface(0, iso, s)
            Vr, Tr = restated(g, iso, s)
            assert same_bits(V, Vr) and np.array_equal(T, Tr), (name, s, iso, V.shape, Vr.shape)
            assert (g.last_isosurface_ms >= 0).all()


@pytest.mark.parametrize("name", ["bunny64", "bunny128"])
def test_bunny_equals_restatement(dg, name):
    g = field(dg, name)
    for s in (1, 2):
        V, T = g.isosurface(0, 0.0, s)
        Vr, Tr = restated(g, 0.0, s)
        assert same_bits(V, Vr) and np.array_equal(T, Tr)
        print(f"{name} s={s}: {len(V)} vertices, {len(T)} triangles, stages (ms) {np.round(g.last_isosurface_ms, 2).tolist()}")


def test_special_fields_equal_restatement(dg):
    g = dg.CubicLagrangeDiscreteGrid(np.array([-1.0, -2.0, 0.0]), np.array([1.0, 1.0, 0.5]), (5, 4, 3))
    rng = np.random.default_rng(3)
    n = g.nNodes()
    v = rng.standard_normal(n)
    k = rng.random(n) < 0.15
    v[k] = rng.choice(np.array([np.nan, np.inf, -np.inf, ir.DBL_MAX, -ir.DBL_MAX, 1.7e308, -1.7e308, 1e308, -1e308, 0.0, -0.0]), k.sum())
    g.addSampledFunction(v)
    g.addSampledFunction(np.full(n, ir.DBL_MAX))
    for s in (1, 2, 3):
        for iso in (0.0, 0.25, -1e308, 1.6e308):
            V, T = g.isosurface(0, iso, s)
            Vr, Tr = restated(g, iso, s)
            assert same_bits(V, Vr) and np.array_equal(T, Tr)
        V, T = g.isosurface(1, 0.0, s)
        assert V.shape == (0, 3) and T.shape == (0, 3)
    with pytest.raises(capi().DiscregridError):
        g.isosurface(0, float("nan"))
    with pytest.raises(capi().DiscregridError):
        g.isosurface(0, 0.0, 17)


def test_tensor_route_same_bits(dg):
    import torch
    g = field(dg, "torus_band")
    V, T = g.isosurface(0, 0.0, 2)
    Vd, Td = g.isosurface(0, 0.0, 2, device=True)
    if not capi().EMULATED:
        assert Vd.is_cuda and Td.is_cuda
    assert Vd.dtype == torch.float64 and Td.dtype == torch.int32 and Td.shape == T.shape
    assert np.array_equal(Vd.cpu().numpy().view(np.uint64), V.view(np.uint64))
    assert np.array_equal(Td.cpu().numpy().astype(np.uint32), T)


def gradient_share(g, V, T):
    n = ir.normals(V, T)
    c = V[T.astype(np.int64)].mean(axis=1)
    _, grad = g.interpolate(0, c, gradient=True)
    nd = np.linalg.norm(n, axis=1) > 0
    return float((np.einsum("ij,ij->i", n[nd], grad[nd]) > 0).mean()), int(nd.sum())


@pytest.mark.parametrize("name,chi", [("sphere", 2), ("torus", 0), ("bunny", None)])
def test_closed_and_oriented(dg, name, chi):
    if name == "sphere":
        g = analytic(dg, (24, 24, 24), sphere_sdf)
    elif name == "torus":
        g = sdf_grid(dg, "torus", (48, 48, 24))[0]
    else:
        g = sdf_grid(dg, "bunny", (64, 64, 64))[0]
    for s in (1, 2):
        V, T = g.isosurface(0, 0.0, s)
        closed, oriented = ir.edge_use(T)
        assert closed and oriented, (name, s)
        assert np.array_equal(np.unique(T), np.arange(len(V)))
        if chi is not None:
            assert ir.euler_characteristic(V, T) == chi
        assert ir.signed_volume(V, T) > 0
        share, m = gradient_share(g, V, T)
        print(f"{name} s={s}: dot(normal, grad phi) > 0 on {share:.6f} of {m} non-degenerate triangles")
        if name == "sphere":
            assert share == 1.0


@pytest.mark.parametrize("name,res", [("torus", (32, 32, 16)), ("bunny", (64, 64, 64))])
def test_dense_equals_reduced_band(dg, name, res):
    g, md, V, F = sdf_grid(dg, name, res)
    band = 3.0 * diag(g)
    g.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, band))
    for s in (1, 2):
        Vd, Td = g.isosurface(0, 0.0, s)
        Vb, Tb = g.isosurface(1, 0.0, s)
        assert np.array_equal(Vd.view(np.uint64), Vb.view(np.uint64)) and np.array_equal(Td, Tb), (name, s)


def test_winding_mode_closes_the_open_bunny(dg):
    gw, _, V, F = sdf_grid(dg, "open_bunny", (64, 64, 64), winding=True)
    Vw, Tw = gw.isosurface(0, 0.0, 1)
    closed, oriented = ir.edge_use(Tw)
    assert closed and oriented
    assert ir.signed_volume(Vw, Tw) > 0
    gp = sdf_grid(dg, "open_bunny", (64, 64, 64))[0]
    Vp, Tp = gp.isosurface(0, 0.0, 1)
    print(f"open bunny: winding mode {len(Tw)} triangles, closed; pseudonormal mode {len(Tp)} triangles, edge-use counts "
          f"{dict(enumerate(ir.edge_use_counts(Tp).tolist()))}")


@pytest.mark.parametrize("name", ["sphere_mesh", "bunny"])
def test_round_trip_through_mesh_distance(dg, name):
    g, md, V0, F0 = sdf_grid(dg, name, (64, 64, 64))
    L = ir.Lattice.of_grid(g, 1)
    assert not (ir.lattice_values(g, 0, L) == 0.0).any()
    V, T = g.isosurface(0, 0.0, 1)
    md2 = dg.TriangleMeshDistance(V, T)
    rng = np.random.default_rng(7)
    mn, mx = g.domain()
    x = mn + rng.random((200000, 3)) * (mx - mn)
    phi = g.interpolate(0, x)
    far = np.abs(phi) > 2.0 * diag(g)
    x, phi = x[far][:20000], phi[far][:20000]
    assert len(x) == 20000
    d2 = md2.signed_distance(x).distance
    assert (np.sign(d2) == np.sign(phi)).all()
    err = float(np.abs(md.unsigned_distance(V).distance).max())
    print(f"{name} 64^3: {len(V)} vertices within {err:.3e} of the input mesh ({err / diag(g):.4f} cell diagonals)")
    assert err < 0.5 * diag(g)


def test_tool_equals_python(dg, tmp_path):
    cdf = tmp_path / "torus.cdf"
    obj_in = tmp_path / "torus.obj"
    m = dg.bumpy_torus(48, 48, 1.0, 0.4, 0.05, 7, 5)
    m.exportOBJ(str(obj_in))
    subprocess.run([GENERATE_SDF, "-r", "24 24 12", "-o", str(cdf), str(obj_in)], check=True, capture_output=True)
    g = dg.CubicLagrangeDiscreteGrid(str(cdf))
    h = diag(g)
    for s, iso in ((1, 0.0), (2, 0.25 * h), (3, -0.25 * h)):
        out = tmp_path / f"level_{s}.obj"
        subprocess.run([FIELD_TO_MESH, "-s", str(s), "-i", repr(iso), "-o", str(out), str(cdf)], check=True, capture_output=True)
        back = dg.TriangleMesh(str(out))
        V, T = g.isosurface(0, iso, s)
        assert np.array_equal(np.asarray(back.vertices, np.float64).view(np.uint64), V.view(np.uint64))
        assert np.array_equal(np.asarray(back.faces, np.uint32), T)


def test_large_lattice_runs_several_value_chunks(dg):
    g = analytic(dg, (130, 130, 130), sphere_sdf)           # s = 2: 261^3 = 17,779,581 lattice points > 2^24
    V, T = g.isosurface(0, 0.0, 2)
    Vr, Tr = restated(g, 0.0, 2)
    assert same_bits(V, Vr) and np.array_equal(T, Tr)
    closed, oriented = ir.edge_use(T)
    assert closed and oriented
