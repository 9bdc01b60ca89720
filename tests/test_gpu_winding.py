"""The winding sign mode on the device (K5, discregrid_b200/csrc/k5_winding.cu): winding numbers against the numpy restatement of the contract
(tests/winding_ref.py) bit for bit, on numpy arrays and CUDA tensors; watertight meshes, where the winding mode must reproduce the
pseudonormal mode's fields bit for bit at every node with a nonzero distance; open and non-manifold meshes, where it must follow w; the
reduced band; the C++ facade and GenerateSDF --sign winding."""
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, ref_resource
import winding_ref as wr

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
GENERATE_SDF = os.path.join(ROOT, "build", "bin", "GenerateSDF")
WINDING_CHECK = os.path.join(ROOT, "build", "bin", "winding_check")


def capi():
    from discregrid_b200 import _capi
    return _capi


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to("cpu" if capi().EMULATED else "cuda")


def torus_small(dg):
    m = dg.bumpy_torus(48, 48, 1.0, 0.4, 0.05, 7, 5)
    return np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)


def mesh(dg, name):
    if name == "box":
        return wr.read_obj(os.path.join(GOLDEN, "box.obj"))
    if name == "torus":
        return torus_small(dg)
    if name == "open_torus":
        return wr.cut_top(*torus_small(dg))
    if name == "soup":
        return wr.soup()
    base = name[5:] if name.startswith("open_") else name
    base = base[:-6] if base.endswith("_small") else base
    p = ref_resource(base + ".obj")
    if p is None:
        pytest.skip(f"{base}.obj not staged (make -C oracle ref)")
    V, F = wr.read_obj(p)
    if name.startswith("open_"):
        V, F = wr.cut_top(V, F)
    if name.endswith("_small"):
        F = np.ascontiguousarray(F[:3000])
    return V, F


def leaf_order(md):
    """leaf position -> triangle id: the leaves of dg_mesh_tree in pre-order"""
    _, kids = md.tree()
    return kids[kids[:, 0] == -1, 1].astype(np.int64)


SMALL = ["box", "torus", "open_torus", "soup", "open_bunny_small"]


@pytest.mark.parametrize("name", SMALL)
def test_device_w_matches_restatement(dg, name):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    order = leaf_order(md)
    rec = wr.Records(V, F, order)
    p = wr.query_points(V, 200, seed=21, near=40)
    w_inf = md.winding_number(p, math.inf)
    assert bits_equal(w_inf, wr.exact_w(rec.leaves, p))
    w2 = md.winding_number(p, 2.0)
    assert bits_equal(w2, rec.w(p, 2.0))
    assert bits_equal(md.winding_number(p), w2)                              # default beta = 2
    try:
        import torch  # noqa: F401
    except ImportError:
        return
    for beta in (2.0, math.inf):
        t = md.winding_number(to_dev(p), beta)
        assert bits_equal(t.cpu().numpy(), md.winding_number(p, beta))
    single = md.winding_number(to_dev(p[0]), 2.0)
    assert bits_equal(single.cpu().numpy(), w2[:1])


def test_refusals(dg):
    V, F = mesh(dg, "box")
    md = dg.TriangleMeshDistance(V, F)
    for beta in (math.nan, 0.5, -1.0):
        with pytest.raises(capi().DiscregridError):
            md.winding_number(np.zeros((1, 3)), beta)
        with pytest.raises(capi().DiscregridError):
            md.set_sign_mode("winding", beta)
    with pytest.raises(ValueError):
        md.set_sign_mode("angle")
    assert md.sign_mode == "pseudonormal"
    md.set_sign_mode("winding", math.inf)
    assert md.sign_mode == "winding"
    import ctypes as C
    grp = C.c_void_p()
    assert capi().lib.dg_mesh_group_create(md.handle, 1, None, C.byref(grp)) == capi().DG_ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------- watertight meshes
def fields(dg, V, F, res, mode, sign):
    """dense, band (2 cell diagonals) and reduced-band fields of one mesh in one sign mode (with `sign` = -1: inverted)"""
    md = dg.TriangleMeshDistance(V, F).set_sign_mode(mode)
    mn, mx = dg.generate_sdf_domain(V)
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, list(res))
    band = 2.0 * float(np.linalg.norm(g.m_cell_size))
    inv = sign < 0
    g.addFunction(dg.MeshSignedDistance(md, invert=inv))
    g.addFunction(dg.MeshSignedDistance(md, invert=inv), False, dg.MeshDistanceBand(md, band))
    r = dg.CubicLagrangeDiscreteGrid(mn, mx, list(res))
    r.addReducedBandField(dg.MeshSignedDistance(md, invert=inv), dg.MeshDistanceBand(md, band))
    return g.m_nodes[0], g.m_nodes[1], (r.m_nodes[0], r.m_cells[0], r.m_cell_map[0])


def check_watertight(dg, name, res, sign=1.0):
    V, F = mesh(dg, name)
    dense_p, band_p, red_p = fields(dg, V, F, res, "pseudonormal", sign)
    dense_w, band_w, red_w = fields(dg, V, F, res, "winding", sign)
    for a, b in ((dense_p, dense_w), (band_p, band_w), (red_p[0], red_w[0])):
        nz = a != 0.0
        bad = np.flatnonzero(a.view(np.uint64)[nz] != b.view(np.uint64)[nz])
        assert len(bad) == 0, f"{name} {res}: {len(bad)} nodes differ, first values {a[nz][bad[:5]]} vs {b[nz][bad[:5]]}"
        assert bits_equal(np.abs(a), np.abs(b))
    assert np.array_equal(red_p[1], red_w[1]) and np.array_equal(red_p[2], red_w[2])


@pytest.mark.parametrize("name", ["box", "torus"])
def test_watertight_fields_equal_pseudonormal_small(dg, name):
    check_watertight(dg, name, (12, 12, 10))
    check_watertight(dg, name, (9, 11, 7), sign=-1.0)


@pytest.mark.parametrize("name,res", [(n, r) for n in ("box", "torus", "bunny", "dragon") for r in (64, 128)])
def test_watertight_fields_equal_pseudonormal_full_size(dg, name, res):
    check_watertight(dg, name, (res, res, res))


# ---------------------------------------------------------------------------------------------------------------- open and non-manifold meshes
def check_open(dg, name, n_points, res):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F)
    mn, mx = dg.generate_sdf_domain(V)
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, [res] * 3)
    x = g.nodePositions()
    p = np.concatenate([wr.query_points(V, n_points, seed=31), x])
    w_inf, w2 = md.winding_number(p, math.inf), md.winding_number(p, 2.0)
    err = float(np.max(np.abs(w2 - w_inf)))
    assert err <= 0.1, err
    md.set_sign_mode("winding")
    g.addFunction(dg.MeshSignedDistance(md))
    node_w = w_inf[n_points:]
    clear = np.abs(node_w - 0.5) > 0.15
    assert np.array_equal((g.m_nodes[0] < 0)[clear], (node_w > 0.5)[clear])
    d = md.signed_distance(p[:n_points]).distance
    clear_p = np.abs(w_inf[:n_points] - 0.5) > 0.15
    assert np.array_equal((d < 0)[clear_p], (w_inf[:n_points] > 0.5)[clear_p])
    return err


def test_open_mesh_small(dg):
    check_open(dg, "open_torus", 2000, 12)


@pytest.mark.parametrize("name", ["open_bunny", "happy_buddha"])
def test_open_meshes_full_size(dg, name):
    err = check_open(dg, name, 20000, 32)
    print(f"{name}: max |w(beta=2) - w(inf)| = {err:.4g}")


@pytest.mark.parametrize("name", ["open_torus", "open_bunny_small"])
def test_reduced_band_equals_two_step(dg, name):
    V, F = mesh(dg, name)
    md = dg.TriangleMeshDistance(V, F).set_sign_mode("winding")
    mn, mx = dg.generate_sdf_domain(V)
    res = [14, 12, 13]
    a = dg.CubicLagrangeDiscreteGrid(mn, mx, res)
    band = 2.0 * float(np.linalg.norm(a.m_cell_size))
    a.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, band))
    b = dg.CubicLagrangeDiscreteGrid(mn, mx, res)
    b.addFunction(dg.MeshSignedDistance(md), False, dg.MeshDistanceBand(md, band))
    b.reduceField(0, lambda x, v: np.ones(len(v), bool))
    assert bits_equal(a.m_nodes[0], b.m_nodes[0])
    assert np.array_equal(a.m_cells[0], b.m_cells[0]) and np.array_equal(a.m_cell_map[0], b.m_cell_map[0])


# ---------------------------------------------------------------------------------------------------------------- tools
def test_cpp_generate_sdf_winding_box_is_box_cdf(tmp_path):
    out = tmp_path / "box.cdf"
    subprocess.run([GENERATE_SDF, "--sign", "winding", "-r", "5 5 5", "-o", str(out), os.path.join(GOLDEN, "box.obj")], check=True,
                   capture_output=True)
    assert out.read_bytes() == open(os.path.join(GOLDEN, "box.cdf"), "rb").read()
    r = subprocess.run([GENERATE_SDF, "--sign", "winding", "--gpus", "2", "-o", str(tmp_path / "x.cdf"), os.path.join(GOLDEN, "box.obj")],
                       capture_output=True, text=True)
    assert r.returncode != 0 and "one GPU" in r.stderr


def write_obj(path, V, F):
    with open(path, "w") as f:
        for v in V:
            f.write("v %.17g %.17g %.17g\n" % tuple(v))
        for t in F:
            f.write("f %d %d %d\n" % tuple(int(i) + 1 for i in t))


def test_cpp_generate_sdf_winding_open_bunny(dg, tmp_path):
    V, F = mesh(dg, "open_bunny")
    obj = tmp_path / "open_bunny.obj"
    write_obj(obj, V, F)
    out = tmp_path / "open_bunny.cdf"
    subprocess.run([GENERATE_SDF, "--sign", "winding", "-r", "24 24 24", "-o", str(out), str(obj)], check=True, capture_output=True)
    g = dg.CubicLagrangeDiscreteGrid(str(out))
    V2, F2 = wr.read_obj(str(obj))
    md = dg.TriangleMeshDistance(V2, F2)
    w = md.winding_number(g.nodePositions(), 2.0)
    vals = g.m_nodes[0]
    assert np.array_equal(vals < 0, w > 0.5)
    md.set_sign_mode("winding")
    py = dg.CubicLagrangeDiscreteGrid(g.m_domain[0], g.m_domain[1], [24, 24, 24])
    py.addFunction(dg.MeshSignedDistance(md))
    assert bits_equal(py.m_nodes[0], vals)


def test_cpp_facade_winding_check(dg, tmp_path):
    V, F = mesh(dg, "open_torus")
    obj = tmp_path / "open_torus.obj"
    write_obj(obj, V, F)
    V2, F2 = wr.read_obj(str(obj))
    p = wr.query_points(V2, 500, seed=41)
    p.tofile(tmp_path / "p.f64")
    subprocess.run([WINDING_CHECK, str(obj), str(tmp_path / "p.f64"), "2", str(tmp_path / "o.f64")], check=True, capture_output=True)
    o = np.fromfile(tmp_path / "o.f64")
    md = dg.TriangleMeshDistance(V2, F2).set_sign_mode("winding")
    assert bits_equal(o[:500], md.winding_number(p, 2.0))
    assert bits_equal(o[500:], md.signed_distance(p).distance)
