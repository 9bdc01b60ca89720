"""K9 (ray casts on a mesh, discregrid_b200/csrc/k9_mesh_raycast.cu) on the CPU: the product's translation unit compiled through tests/emu
(build/bin/libk9emu.so, and libk9emu_nocull.so with culling compiled out) against the brute-force numpy restatement of its contract in
tests/mesh_raycast_ref.py, bit for bit on t, triangle_id, barycentric and status."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT, GOLDEN
import mesh_raycast_ref as mr

LIBS = {"cull": os.path.join(ROOT, "build", "bin", "libk9emu.so"), "nocull": os.path.join(ROOT, "build", "bin", "libk9emu_nocull.so")}
DP, U32P, I32P, VP = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.c_void_p


def _load(path):
    if not os.path.exists(path):
        pytest.skip(f"{os.path.relpath(path, ROOT)} not built (make cpp)")
    lib = C.CDLL(path)
    lib.emu_k9_create.restype = VP
    lib.emu_k9_create.argtypes = [DP, C.c_uint64, U32P, C.c_uint64]
    lib.emu_k9_destroy.argtypes = [VP]
    lib.emu_k9_raycast.argtypes = [VP, DP, DP, C.c_uint64, C.c_double, C.c_double, DP, I32P, DP, I32P]
    lib.emu_k9_counters.argtypes = [C.POINTER(C.c_ulonglong)]
    return lib


@pytest.fixture(scope="module")
def libs():
    out = {k: _load(p) for k, p in LIBS.items()}
    assert out["cull"].emu_k9_cull() == 1 and out["nocull"].emu_k9_cull() == 0
    return out


def P(a, t=DP):
    return a.ctypes.data_as(t)


def emu_cast(lib, V, F, o, d, t_min=0.0, t_max=np.inf):
    V = np.ascontiguousarray(V, np.float64)
    F = np.ascontiguousarray(F, np.uint32)
    o = np.ascontiguousarray(o, np.float64)
    d = np.ascontiguousarray(d, np.float64)
    h = lib.emu_k9_create(P(V), len(V), P(F, U32P), len(F))
    assert h
    try:
        n = len(o)
        t, tid, b, st = np.empty(n), np.empty(n, np.int32), np.empty((n, 3)), np.empty(n, np.int32)
        assert lib.emu_k9_raycast(h, P(o), P(d), n, t_min, t_max, P(t), P(tid, I32P), P(b), P(st, I32P)) == 0
    finally:
        lib.emu_k9_destroy(h)
    return t, tid, b, st


def assert_same(got, want, what):
    names = ("t", "triangle_id", "barycentric", "status")
    for g, w, nm in zip(got, want, names):
        g, w = np.asarray(g), np.asarray(w)
        if g.dtype == np.float64:
            gb, wb = g.view(np.uint64).reshape(len(g), -1), w.view(np.uint64).reshape(len(w), -1)
            bad = np.flatnonzero((gb != wb).any(axis=1))
        else:
            bad = np.flatnonzero(g != w)
        assert len(bad) == 0, f"{what}: {nm} differs on {len(bad)} of {len(g)} rays, first ray {bad[0]}: {g[bad[0]]!r} vs {w[bad[0]]!r}"


def check(libs, V, F, o, d, what, t_min=0.0, t_max=np.inf):
    """both emulated builds equal the restatement bit for bit; returns the result"""
    want = mr.raycast(V, F, o, d, t_min, t_max)
    for k, lib in libs.items():
        assert_same(emu_cast(lib, V, F, o, d, t_min, t_max), want, f"{what} ({k})")
    return want


def box_mesh():
    from discregrid_b200.mesh import TriangleMesh
    m = TriangleMesh(os.path.join(GOLDEN, "box.obj"))
    return m.vertices, m.faces


def sphere_mesh():
    from discregrid_b200.mesh import uv_sphere
    m = uv_sphere(12, 24)
    return m.vertices, m.faces


def torus_mesh():
    from discregrid_b200.mesh import bumpy_torus
    m = bumpy_torus(24, 20)
    return m.vertices, m.faces


CLOSED = {"box": (box_mesh, lambda V: 0.5 * (V.min(0) + V.max(0))), "sphere": (sphere_mesh, lambda V: np.array([0.01, -0.02, 0.03])),
          "torus": (torus_mesh, lambda V: np.array([1.0, 0.0, 0.0]))}


def mixed_rays(V, F, rng, n=400):
    parts = [mr.random_rays(V, n, rng), mr.aimed_rays(V, F, n, rng), mr.axis_rays(V, n // 2, rng), mr.in_plane_rays(V, F, n // 2, rng)]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


@pytest.mark.parametrize("name", ["box", "sphere", "torus"])
def test_closed_meshes_match_the_restatement(libs, name):
    V, F = CLOSED[name][0]()
    rng = np.random.default_rng(7)
    o, d = mixed_rays(V, F, rng)
    t, tid, b, st = check(libs, V, F, o, d, name)
    assert (st != mr.MISS).mean() > 0.3
    # segments: the same rays on [0, 1], and infinite bounds with a negative t_min
    check(libs, V, F, o, d, name + " segments", 0.0, 1.0)
    check(libs, V, F, o, d, name + " all of the line", -np.inf, np.inf)
    check(libs, V, F, o, d, name + " negative t_min", -0.5, 3.0)


@pytest.mark.parametrize("name", ["box", "sphere", "torus"])
def test_hits_exactly_at_the_bounds(libs, name):
    V, F = CLOSED[name][0]()
    rng = np.random.default_rng(11)
    o, d = mr.aimed_rays(V, F, 200, rng)
    t, tid, b, st = mr.raycast(V, F, o, d)
    h = np.flatnonzero(st != mr.MISS)
    for i in h[:12]:
        for lo, hi in ((t[i], np.inf), (0.0, t[i]), (t[i], t[i])):
            w = check(libs, V, F, o[i:i + 1], d[i:i + 1], f"{name} ray {i} on [{lo!r}, {hi!r}]", lo, hi)
            assert w[1][0] == tid[i] and w[0][0] == t[i]


def test_status_is_pinned_by_the_box(libs):
    V, F = box_mesh()
    c = 0.5 * (V.min(0) + V.max(0))
    ext = V.max(0) - V.min(0)
    dirs = np.array([[1, 0.1, 0.2], [-1, 0.2, -0.1], [0.1, 1, 0.3], [0.2, -1, 0.1], [0.3, 0.1, 1], [-0.1, 0.2, -1]], np.float64)
    o_out = c - 2.0 * dirs * ext                                   # outside, aimed at the centre: enters
    t, tid, b, st = check(libs, V, F, o_out, dirs, "box from outside")
    assert np.all(st == mr.ENTER)
    t, tid, b, st = check(libs, V, F, np.tile(c, (6, 1)), dirs, "box from inside")
    assert np.all(st == mr.LEAVE)
    # the hit point agrees with the barycentric combination of the winner's vertices
    x = c + t[:, None] * dirs
    y = (b[:, :, None] * V[F[tid].astype(np.int64)]).sum(axis=1)
    assert np.allclose(x, y, rtol=0, atol=1e-12 * np.abs(V).max())


@pytest.mark.parametrize("name", ["box", "sphere", "torus"])
def test_no_leaks_through_vertices_and_edges(libs, name):
    V, F = CLOSED[name][0]()
    o, d = mr.leak_rays(V, F, CLOSED[name][1](V))
    t, tid, b, st = check(libs, V, F, o, d, name + " leaks")
    assert np.all(st != mr.MISS), f"{np.sum(st == mr.MISS)} rays leak"
    # status: a ray that ends in a vertex hits every triangle of its fan at the same t; the lowest id wins, whichever way it faces


def test_single_triangle(libs):
    V = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0]])
    F = np.array([[0, 1, 2]], np.uint32)
    rng = np.random.default_rng(3)
    o, d = mixed_rays(V, F, rng, 200)
    o = np.concatenate([o, [[0.25, 0.25, 1.0], [0.25, 0.25, -1.0], [0.0, 0.0, 1.0], [0.5, 0.5, 1.0]]])
    d = np.concatenate([d, [[0, 0, -1.0], [0, 0, 1.0], [0, 0, -1.0], [0, 0, -1.0]]])
    t, tid, b, st = check(libs, V, F, o, d, "single triangle")
    assert t[-4] == 1.0 and st[-4] == mr.ENTER and st[-3] == mr.LEAVE        # normal +z: a ray going down crosses it from outside
    assert st[-2] != mr.MISS and st[-1] != mr.MISS                              # a vertex and an edge


def test_duplicated_triangles_the_lower_id_wins(libs):
    V, F = sphere_mesh()
    T = len(F)
    F2 = np.concatenate([F, F[::-1], F[:, [1, 2, 0]]])                          # each triangle three times (the third copy rotated)
    rng = np.random.default_rng(5)
    o, d = mr.aimed_rays(V, F2, 400, rng)
    t, tid, b, st = check(libs, V, F2, o, d, "duplicates")
    h = st != mr.MISS
    assert h.mean() > 0.5
    # the second copy is computed exactly as the first, so it never wins; the rotated copy may round t differently
    assert not np.any((tid >= T) & (tid < 2 * T))


@pytest.mark.parametrize("tilt", [False, True])
def test_coplanar_grid_edges_and_vertices(libs, tilt):
    V, F = mr.grid_mesh(6, tilt)
    n = np.cross(V[F[0, 1]] - V[F[0, 0]], V[F[0, 2]] - V[F[0, 0]])
    rng = np.random.default_rng(9)
    E = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]).astype(np.int64)
    s = rng.random((len(E), 1))
    targets = np.concatenate([V, V[E[:, 0]] + s * (V[E[:, 1]] - V[E[:, 0]]), 0.5 * (V[E[:, 0]] + V[E[:, 1]])])
    o = targets + n * (0.5 + rng.random((len(targets), 1))) + rng.normal(size=targets.shape) * 0.05
    d = targets - o
    t, tid, b, st = check(libs, V, F, o, d, "grid: rays through vertices and edges")
    inner = np.all((targets > V.min(0) + 1e-9) & (targets < V.max(0) - 1e-9), axis=1) if not tilt else None
    if inner is not None:
        assert np.all(st[inner] != mr.MISS)
    o2, d2 = mr.in_plane_rays(V, F, 600, rng)
    check(libs, V, F, o2, d2, "grid: rays in its plane")


def test_degenerate_and_non_finite_meshes(libs):
    V, F = sphere_mesh()
    V = V.copy()
    # zero-area triangles: collapsed (two equal vertices) and collinear
    Vz = np.concatenate([V, [[0.0, 0, 0], [0.5, 0.5, 0.5], [1.0, 1.0, 1.0]]])
    nV = len(V)
    Fz = np.concatenate([F, [[nV, nV + 1, nV + 2], [0, 0, 1], [2, 2, 2]]]).astype(np.uint32)
    rng = np.random.default_rng(13)
    o, d = mixed_rays(Vz, Fz, rng, 300)
    o = np.concatenate([o, [[0.5, 0.5, 0.5 - 1.0]], [[-1.0, -1.0, -1.0]]])
    d = np.concatenate([d, [[0.0, 0.0, 1.0]], [[1.0, 1.0, 1.0]]])
    check(libs, Vz, Fz, o, d, "zero-area triangles")
    # a NaN vertex: the tree's boxes mean nothing, culling is off and the result is still the restatement's
    Vn = V.copy()
    Vn[5] = np.nan
    o, d = mixed_rays(Vn, F, rng, 300)
    check(libs, Vn, F, o, d, "NaN vertex")
    Vi = V.copy()
    Vi[7, 1] = np.inf
    check(libs, Vi, F, o, d, "inf vertex")


def test_special_rays(libs):
    V, F = torus_mesh()
    inf, nan = np.inf, np.nan
    o = np.array([[0, 0, 2.0], [nan, 0, 2], [0, inf, 2], [1, 0, 2], [1, 0, 2], [1, 0, 2], [1, 0, 2], [1e300, 0, 0], [1, 0, 1e-300]])
    d = np.array([[0, 0, 0.0], [0, 0, -1], [0, 0, -1], [nan, 0, -1], [0, -inf, -1], [0, 0, -1e-310], [0, 0, -1e300], [-1, 0, 0], [0, 0, -1]])
    t, tid, b, st = check(libs, V, F, o, d, "special rays")
    assert np.all(st[:5] == mr.MISS) and np.all(tid[:5] == -1) and np.all(np.isinf(t[:5]))
    assert np.all(np.isnan(b[:5]))
    assert st[6] != mr.MISS and st[8] == mr.LEAVE                                # huge direction; origin inside the tube


def test_rays_touching_box_faces(libs):
    V, F = box_mesh()
    lo, hi = V.min(0), V.max(0)
    rng = np.random.default_rng(17)
    n = 300
    o = lo + rng.random((n, 3)) * (hi - lo)
    ax = rng.integers(0, 3, n)
    o[np.arange(n), ax] = np.where(rng.random(n) < 0.5, lo[ax], hi[ax])          # on a face plane
    d = rng.normal(size=(n, 3))
    d[np.arange(n), ax] = 0.0                                                   # along it
    o -= 3 * d
    check(libs, V, F, o, d, "rays along the box faces")
    o2 = np.where(rng.random((n, 3)) < 0.5, lo, hi) - 2 * np.ones(3)           # aimed exactly at corners
    check(libs, V, F, o2, np.where(rng.random((n, 3)) < 0.5, lo, hi) - o2, "rays at the box corners")


@pytest.mark.parametrize("scale", [1e-20, 1e-8, 1.0, 1e6, 1e15])
def test_mesh_scales(libs, scale):
    V, F = torus_mesh()
    rng = np.random.default_rng(19)
    o, d = mixed_rays(V, F, rng, 200)
    shift = np.array([0.3, -0.2, 0.1])
    check(libs, (V + shift) * scale, F, (o + shift) * scale, d * scale, f"scale {scale:g}")
    check(libs, (V + shift) * scale, F, (o + shift) * scale, d, f"scale {scale:g}, unit directions")


def test_culling_visits_few_boxes(libs):
    """Culling is not only exact but effective: on a torus of 9,600 triangles a hitting ray tests few of them."""
    from discregrid_b200.mesh import bumpy_torus
    m = bumpy_torus(80, 60)
    V, F = m.vertices, m.faces
    rng = np.random.default_rng(23)
    o, d = mr.aimed_rays(V, F, 200, rng)
    lib = libs["cull"]
    lib.emu_k9_counters_reset()
    emu_cast(lib, V, F, o, d)
    c = (C.c_ulonglong * 3)()
    lib.emu_k9_counters(c)
    assert c[2] == 200
    assert c[1] / 200 < 0.02 * len(F), f"{c[1] / 200:.0f} triangles tested per ray"
