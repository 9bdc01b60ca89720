"""The refit on the device (K8, discregrid_b200/csrc/k8_refit.cu): the records the C-ABI exposes (sphere tree, pseudonormals) against the numpy
restatement of the contract (tests/refit_ref.py) bit for bit; winding numbers after a refit against tests/winding_ref.py; a refit mesh against
a fresh dg_mesh_create of the same vertices; the host and CUDA-tensor routes; the memory dg_mesh_info reports."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, bits_equal, ref_resource
import refit_ref as rr
import winding_ref as wr

pytestmark = pytest.mark.gpu

DBL_MAX = np.finfo(np.float64).max
ORCTREE = os.path.join(ROOT, "build", "bin", "liborctree.so")
REFIT_CHECK = os.path.join(ROOT, "build", "bin", "refit_check")
_dp, _i32p, _u32p = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)


class TreeOracle:
    """the reference's query rule (the CPU oracle) over the tree and pseudonormals a mesh exports (tests/cpp/oracle_from_tree.cpp)"""

    def __init__(self, md, V, F):
        if not os.path.exists(ORCTREE):
            pytest.skip("build/bin/liborctree.so not built (make cpp)")
        self.lib = C.CDLL(ORCTREE)
        self.V, self.F = np.ascontiguousarray(V, np.float64), np.ascontiguousarray(F, np.uint32)
        sph, kids = md.tree()
        tri, edge, vert = md.pseudonormals()
        f = self.lib.orc_mesh_create_from_tree
        f.restype = C.c_void_p
        f.argtypes = [_dp, C.c_uint64, _u32p, C.c_uint64, _dp, _i32p, _dp, _dp, _dp]
        self._keep = [np.ascontiguousarray(a) for a in (sph, kids, tri, edge, vert)]
        self.h = f(self.V.ctypes.data_as(_dp), len(self.V), self.F.ctypes.data_as(_u32p), len(self.F), *[
            a.ctypes.data_as(_i32p if a.dtype == np.int32 else _dp) for a in self._keep])
        self.lib.orc_mesh_destroy.argtypes = [C.c_void_p]
        self.lib.orc_mesh_distance.argtypes = [C.c_void_p, _dp, C.c_uint64, C.c_int, _dp, _dp, _i32p, _i32p]

    def distance(self, x, signed=True):
        x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
        n = len(x)
        d = np.empty(n); q = np.empty((n, 3)); e = np.empty(n, np.int32); t = np.empty(n, np.int32)
        self.lib.orc_mesh_distance(self.h, x.ctypes.data_as(_dp), n, int(signed), d.ctypes.data_as(_dp), q.ctypes.data_as(_dp),
                                   e.ctypes.data_as(_i32p), t.ctypes.data_as(_i32p))
        return d, q, e, t

    def close(self):
        self.lib.orc_mesh_destroy(self.h)


def capi():
    from discregrid_b200 import _capi
    return _capi


def twist(V, angle):
    lo, hi = V[:, 1].min(), V[:, 1].max()
    t = angle * (V[:, 1] - lo) / (hi - lo)
    c, s = np.cos(t), np.sin(t)
    return np.stack([c * V[:, 0] + s * V[:, 2], V[:, 1], -s * V[:, 0] + c * V[:, 2]], 1)


def torus(dg, amp=0.05):
    m = dg.bumpy_torus(48, 40, 1.0, 0.4, amp, 7, 5)
    return np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)


def resource(name):
    p = ref_resource(name)
    if p is None or not os.path.exists(p):
        pytest.skip(f"{name} not staged (make -C oracle ref)")
    return wr.read_obj(p)


def check_records(md, V, F):
    sph, kids = md.tree()
    order = rr.order_from_tree(kids)
    want = rr.Refit(V, F, order)
    assert bits_equal(sph, want.tree_spheres()), "sphere tree"
    tri, edge, vert = md.pseudonormals()
    assert bits_equal(tri, want.pn_tri), "triangle pseudonormals"
    assert bits_equal(edge, want.pn_edge), "edge pseudonormals"
    used = np.zeros(len(V), bool); used[F.reshape(-1)] = True
    assert bits_equal(vert[used], want.pn_vert[used]), "vertex pseudonormals"
    assert np.isnan(vert[~used]).all()


@pytest.mark.parametrize("name", ["torus", "bunny", "large_dragon", "large_happy_buddha"])
def test_records_equal_the_restatement(dg, name):
    if name == "torus":
        V, F = torus(dg)
    else:
        V, F = resource({"bunny": "bunny.obj", "large_dragon": "dragon.obj", "large_happy_buddha": "happy_buddha.obj"}[name])
    md = dg.TriangleMeshDistance(V, F)
    for a in (0.5, 1.5):
        V1 = twist(V, a)
        md.refit(V1)
        check_records(md, V1, F)


def test_winding_after_refit_equals_the_restatement(dg):
    """open (cut_top) bunny: w and the winding sign mode follow V', whether or not the winding records existed before the refit"""
    V, F = wr.cut_top(*resource("bunny.obj"))
    V1 = twist(V, 0.8) * 1.1
    x = wr.query_points(V1, 150, seed=3, near=50)
    want = wr.Records(V1, F, rr.order_from_tree(dg.TriangleMeshDistance(V, F).tree()[1])).w(x, 2.0)
    for used_before in (False, True):
        md = dg.TriangleMeshDistance(V, F)
        if used_before:
            md.winding_number(x[:4])
        md.refit(V1)
        assert bits_equal(md.winding_number(x, 2.0), want)
        md.set_sign_mode("winding")
        d = md.signed_distance(x).distance
        u = md.unsigned_distance(x).distance
        assert bits_equal(d, np.where(want > 0.5, -u, u))


@pytest.mark.parametrize("name,angle", [("bunny", 0.5), ("bunny", 1.5), ("large_dragon", 0.5)])
def test_queries_equal_the_reference_rule_over_the_refit_tree(dg, orc, name, angle):
    """dg_mesh_distance (signed and unsigned: distance, nearest point, entity, triangle), dg_sample_sdf at 128^3 (strided sample), the band
    and dg_reduced_band_create after a refit, against the reference's rule run over the exported refit tree and pseudonormals, bit for bit"""
    V, F = resource("bunny.obj" if name == "bunny" else "dragon.obj")
    V1 = twist(V, angle)
    md = dg.TriangleMeshDistance(V, F).refit(V1)
    ref = TreeOracle(md, V1, F)
    try:
        x = wr.query_points(V1, 50000, seed=5, near=50000)
        for signed in (True, False):
            got = md.signed_distance(x) if signed else md.unsigned_distance(x)
            want = ref.distance(x, signed)
            for f in range(4):
                assert bits_equal(got[f], want[f]), (signed, f)
        mn, mx = dg.generate_sdf_domain(V1)
        gd, res = orc.grid_desc(mn, mx, (128, 128, 128))
        ids = np.arange(0, orc.num_nodes(res), 53, dtype=np.uint64)
        xn = orc.node_positions_at(gd, res, ids)
        dn = ref.distance(xn, True)[0]
        grid = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
        grid.addFunction(dg.MeshSignedDistance(md))
        assert bits_equal(grid.m_nodes[0][ids.astype(np.int64)], dn)
        cell = (mx - mn) / 128.0
        w = 2.0 * float(np.sqrt((cell * cell).sum()))
        band = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
        band.addFunction(dg.MeshSignedDistance(md), False, dg.MeshDistanceBand(md, w))
        assert bits_equal(band.m_nodes[0][ids.astype(np.int64)], np.where(np.abs(dn) <= w, dn, DBL_MAX))
        red = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
        assert red.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, w)) == 0
        band.reduceField(0, lambda p, v: np.ones(len(v), bool))
        assert bits_equal(red.m_nodes[0], band.m_nodes[0])
        assert np.array_equal(red.m_cells[0], band.m_cells[0]) and np.array_equal(red.m_cell_map[0], band.m_cell_map[0])
    finally:
        ref.close()


@pytest.mark.parametrize("amp,angle", [(0.05, 0.3), (0.15, 1.2)])
def test_refit_mesh_against_a_fresh_build(dg, amp, angle):
    V, F = torus(dg)
    V1 = twist(torus(dg, amp)[0], angle)
    md = dg.TriangleMeshDistance(V, F).refit(V1)
    fresh = dg.TriangleMeshDistance(V1, F)
    mn, mx = V1.min(0) - 0.1, V1.max(0) + 0.1
    ext = float(np.abs(V1).max())
    rng = np.random.default_rng(1)
    x = np.concatenate([mn + rng.random((60000, 3)) * (mx - mn), V1[rng.integers(0, len(V1), 40000)] + rng.normal(0, 1e-3, (40000, 3))])
    a, b = md.signed_distance(x).distance, fresh.signed_distance(x).distance
    tol = 4 * np.spacing(np.abs(b)) + 1e-13 * ext
    assert (np.abs(np.abs(a) - np.abs(b)) <= tol).all()
    far = np.abs(b) > 1e-9 * ext
    assert (np.sign(a[far]) == np.sign(b[far])).all()
    # the grid path (K1's node loop) on the refit mesh, every node of a 128^3 grid
    grid = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
    grid.addFunction(dg.MeshSignedDistance(md))
    g2 = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
    g2.addFunction(dg.MeshSignedDistance(fresh))
    ga, gb = grid.m_nodes[0], g2.m_nodes[0]
    assert (np.abs(np.abs(ga) - np.abs(gb)) <= 4 * np.spacing(np.abs(gb)) + 1e-13 * ext).all()
    far = np.abs(gb) > 1e-9 * ext
    assert (np.sign(ga[far]) == np.sign(gb[far])).all()


def test_refit_is_idempotent_and_forgets_earlier_positions(dg):
    V, F = torus(dg)
    a = dg.TriangleMeshDistance(V, F).refit(twist(V, 1.0)).refit(twist(V, 0.2))
    b = dg.TriangleMeshDistance(V, F).refit(twist(V, 0.2))
    x = wr.query_points(V, 5000, seed=2, near=2000)
    ra, rb = a.signed_distance(x), b.signed_distance(x)
    for f in range(4):
        assert bits_equal(ra[f], rb[f])
    assert bits_equal(a.tree()[0], b.tree()[0])


def test_memory_grows_by_the_stated_amount(dg):
    V, F = torus(dg)
    md = dg.TriangleMeshDistance(V, F)
    before = md.info()["device_bytes"]
    md.refit(twist(V, 0.1))
    nV, T = len(V), len(F)
    n1 = (nV + 63) // 64
    entries = n1 + max((n1 + 63) // 64, 1)
    want = (24 * nV                     # positions
            + 12 * T + 12 * T + 4 * T   # F by triangle, F by leaf position, leaf order
            + 4 * (nV + 1) + 12 * T     # incidence CSR
            + 16 * (T - 1)              # internal nodes by depth
            + 392 * T + 56 * entries + 40
            + 24 * T + 24 * T + 24 * nV + 72 * T)    # pseudonormal scratch
    assert md.info()["device_bytes"] - before == want
    md.refit(twist(V, 0.2))
    assert md.info()["device_bytes"] - before == want          # kept, not grown


def test_tensor_route_equals_host_route(dg):
    import torch
    V, F = torus(dg)
    V1 = twist(V, 0.7)
    a = dg.TriangleMeshDistance(V, F).refit(V1)
    dev = "cpu" if capi().EMULATED else "cuda"
    b = dg.TriangleMeshDistance(V, F).refit(torch.from_numpy(V1).to(dev))
    c = dg.TriangleMeshDistance(V, F)
    if not capi().EMULATED:
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            t = torch.from_numpy(V1).to(dev, non_blocking=False) * 1.0       # produced on the side stream, read there
            c.refit(t)
        torch.cuda.synchronize()
    else:
        c.refit(V1)
    for m in (b, c):
        assert bits_equal(m.tree()[0], a.tree()[0])
        for k in range(3):
            assert bits_equal(m.pseudonormals()[k], a.pseudonormals()[k])
    x = wr.query_points(V1, 3000, seed=4, near=1000)
    for f in range(4):
        assert bits_equal(b.signed_distance(x)[f], a.signed_distance(x)[f])


def test_refusals_through_python(dg):
    V, F = torus(dg)
    md = dg.TriangleMeshDistance(V, F)
    with pytest.raises(Exception):
        md.refit(V[:-1])
    with pytest.raises(ValueError):
        md.refit(V.reshape(-1))


def test_pseudonormals_of_a_null_mesh_are_refused(dg):
    from discregrid_b200 import _capi as capi
    a = np.empty(9)
    assert capi.lib.dg_mesh_pseudonormals(None, capi.ptr(a, capi.F64P), capi.ptr(a, capi.F64P), capi.ptr(a, capi.F64P)) == capi.DG_ERR_INVALID


def test_device_form_refuses_host_memory(dg):
    if capi().EMULATED:
        pytest.skip("the emulated library has no device memory")
    V, F = torus(dg)
    md = dg.TriangleMeshDistance(V, F)
    V1 = np.ascontiguousarray(twist(V, 0.3))
    assert capi().lib.dg_mesh_refit_device(md.handle, V1.ctypes.data, len(V1), None) == capi().DG_ERR_INVALID
    x = wr.query_points(V, 1000, seed=6)
    assert bits_equal(md.signed_distance(x).distance, dg.TriangleMeshDistance(V, F).signed_distance(x).distance)   # not failed, unchanged
    md.refit(V1)


def test_facade_refit_equals_python(dg, tmp_path):
    if not os.path.exists(REFIT_CHECK):
        pytest.skip("build/bin/refit_check not built (make cpp)")
    V, F = torus(dg)
    obj = tmp_path / "torus.obj"
    with open(obj, "w") as f:
        for v in V:
            f.write("v %.17g %.17g %.17g\n" % tuple(v))
        for t in F:
            f.write("f %d %d %d\n" % tuple(t + 1))
    V1 = np.ascontiguousarray(twist(V, 0.6))
    x = wr.query_points(V1, 2000, seed=8, near=1000)
    V1.tofile(tmp_path / "v.f64"); x.tofile(tmp_path / "x.f64")
    r = subprocess.run([REFIT_CHECK, str(obj), str(tmp_path / "v.f64"), str(tmp_path / "x.f64"), str(tmp_path / "out.f64")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(tmp_path / "out.f64")
    assert bits_equal(got, dg.TriangleMeshDistance(V, F).refit(V1).signed_distance(x).distance)
