"""K10 (differentiable mesh distances, discregrid_b200/csrc/k10_distance_grad.cu and radix_sort.cu, with K1's mesh_distance_bary_kernel) on
the CPU: the product's translation units compiled through tests/emu -- the whole C-ABI in build/bin/libdgemu.so and the sort and VJP passes
alone in build/bin/libk10emu.so -- against the numpy restatement of the contract in tests/mesh_distance_grad_ref.py, bit for bit: the forward
against dg_mesh_distance, the weights, the sort permutation against numpy's stable argsort, grad_points and grad_vertices."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT, GOLDEN
from test_isosurface_emulated import emu  # noqa: F401 (fixture: build/bin/libdgemu.so with the C-ABI's signatures)
import mesh_distance_grad_ref as gr
import winding_ref as wr

K10EMU = os.path.join(ROOT, "build", "bin", "libk10emu.so")
DP, U32P, I32P = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
DG_ERR_INVALID = -1


@pytest.fixture(scope="module")
def k10():
    if not os.path.exists(K10EMU):
        pytest.skip("build/bin/libk10emu.so not built (make cpp)")
    lib = C.CDLL(K10EMU)
    lib.emu_k10_sort.argtypes = [U32P, U32P, C.c_uint64, C.c_int, U32P, U32P]
    lib.emu_k10_vjp.argtypes = [C.c_uint64, DP, DP, DP, I32P, DP, DP, U32P, C.c_uint64, C.c_uint64, DP, DP]
    return lib


def P(a, t=DP):
    return None if a is None else a.ctypes.data_as(t)


def mesh(name):
    if name == "box":
        return wr.read_obj(os.path.join(GOLDEN, "box.obj"))
    import discregrid_b200 as dg
    if name == "sphere":
        m = dg.uv_sphere(12, 24, 0.8)
    else:
        m = dg.bumpy_torus(24, 16, 1.0, 0.4, 0.05, 7, 5)
    V, F = np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)
    return (wr.cut_top(V, F) if name == "open_torus" else (V, F))


def queries(V, F, n, seed):
    """random points around the mesh, some on its vertices (d == 0), some NaN (no triangle)"""
    rng = np.random.default_rng(seed)
    lo, hi = V.min(0), V.max(0)
    c, h = 0.5 * (lo + hi), 0.7 * (hi - lo)
    x = c + rng.uniform(-1, 1, (n, 3)) * h
    k = max(1, n // 16)
    x[:k] = V[rng.integers(0, len(V), k)]
    x[k:2 * k:3] = np.nan
    return np.ascontiguousarray(x[rng.permutation(n)])


class Mesh:
    def __init__(self, lib, V, F, mode="pseudonormal"):
        self.lib, self.V, self.F = lib, np.ascontiguousarray(V, np.float64), np.ascontiguousarray(F, np.uint32)
        self.h = C.c_void_p()
        assert lib.dg_mesh_create(P(self.V), len(self.V), P(self.F, U32P), len(self.F), C.byref(self.h)) == 0, lib.dg_last_error()
        if mode == "winding":
            assert lib.dg_mesh_set_sign_mode(self.h, 1, 2.0) == 0

    def __del__(self):
        self.lib.dg_mesh_destroy(self.h)

    def distance(self, x, signed):
        n = len(x)
        out = np.empty(n), np.empty((n, 3)), np.empty(n, np.int32), np.empty(n, np.int32)
        assert self.lib.dg_mesh_distance(self.h, P(x), n, int(signed), P(out[0]), P(out[1]), P(out[2], I32P), P(out[3], I32P)) == 0
        return out

    def nearest(self, x, signed):
        n = len(x)
        out = np.empty(n), np.empty((n, 3)), np.empty(n, np.int32), np.empty(n, np.int32), np.empty((n, 3))
        assert self.lib.dg_mesh_distance_bary(self.h, P(x), n, int(signed), P(out[0]), P(out[1]), P(out[2], I32P), P(out[3], I32P),
                                              P(out[4])) == 0, self.lib.dg_last_error()
        return out

    def vjp(self, x, r, g, points=True, vertices=True):
        n = len(x)
        gp = np.full((n, 3), 7.0) if points else None
        gv = np.full((len(self.V), 3), 7.0) if vertices else None
        rc = self.lib.dg_mesh_distance_vjp(self.h, n, P(x), P(r[0]), P(r[1]), P(r[3], I32P), P(r[4]), P(g), P(gp), P(gv))
        return rc, gp, gv


def restated(V, F, x, r, g):
    """(weights, grad_points, grad_vertices) of the restatement for the forward outputs r"""
    s, t, ent = gr.leaf_params(V, F, r[3], x)
    w = gr.weights(s, t)
    gx = gr.grad_points(x, r[0], r[1], r[3], g)
    return w, gx, gr.grad_vertices(F, len(V), r[3], gx, w), ent, gr.nearest_point(V, F, r[3], s, t)


def assert_bits(got, want, what):
    assert gr.same_bits(got, want), f"{what}: {np.count_nonzero(np.asarray(got).view(np.uint64) != np.asarray(want).view(np.uint64))} values differ"


def run_k10(k10, V, F, x, r, g):
    n = len(x)
    gp, gv = np.full((n, 3), 7.0), np.full((len(V), 3), 7.0)
    F = np.ascontiguousarray(F, np.uint32)
    assert k10.emu_k10_vjp(n, P(x), P(r[0]), P(r[1]), P(r[3], I32P), P(r[4]), P(g), P(F, U32P), len(F), len(V), P(gp), P(gv)) == 0
    return gp, gv


@pytest.mark.parametrize("name,mode,signed", [("box", "pseudonormal", True), ("sphere", "pseudonormal", True), ("torus", "pseudonormal", True),
                                              ("torus", "pseudonormal", False), ("open_torus", "winding", True)])
def test_forward_and_gradients_equal_restatement(emu, k10, name, mode, signed):
    V, F = mesh(name)
    m = Mesh(emu, V, F, mode)
    x = queries(V, F, 333, 1)                                    # not a multiple of 32
    want = m.distance(x, signed)
    r = m.nearest(x, signed)
    for k, nm in enumerate(("distance", "nearest_point", "nearest_entity", "triangle_id")):
        assert np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)), f"{name}: {nm} differs from dg_mesh_distance"
    assert (r[3] == -1).any() and (r[0] == 0).any() and (r[3] >= 0).sum() > 250
    if mode == "winding":
        assert (r[0] < 0).any() and (r[0] > 0).any()
    g = np.random.default_rng(2).standard_normal(len(x))
    w, gx, gv, ent, p = restated(V, F, x, r, g)
    assert_bits(r[4], w, f"{name}: barycentric")
    hit = r[3] >= 0
    assert np.array_equal(ent[hit], r[2][hit]), f"{name}: restated entity"
    assert_bits(p, np.where((r[3] >= 0)[:, None], r[1], np.nan), f"{name}: nearest point from the weights")
    rc, gp_c, gv_c = m.vjp(x, r, g)
    assert rc == 0, emu.dg_last_error()
    assert_bits(gp_c, gx, f"{name}: grad_points")
    assert_bits(gv_c, gv, f"{name}: grad_vertices")
    gp_k, gv_k = run_k10(k10, V, F, x, r, g)
    assert_bits(gp_k, gx, f"{name}: grad_points (libk10emu)")
    assert_bits(gv_k, gv, f"{name}: grad_vertices (libk10emu)")
    assert np.abs(gv).sum() > 0


def test_outputs_are_optional(emu):
    V, F = mesh("box")
    m = Mesh(emu, V, F)
    x = queries(V, F, 70, 3)
    r = m.nearest(x, True)
    g = np.linspace(-1, 1, len(x))
    w, gx, gv, _, _ = restated(V, F, x, r, g)
    rc, gp_only, none = m.vjp(x, r, g, vertices=False)
    assert rc == 0 and none is None
    assert_bits(gp_only, gx, "grad_points alone")
    rc, none, gv_only = m.vjp(x, r, g, points=False)
    assert rc == 0 and none is None
    assert_bits(gv_only, gv, "grad_vertices alone")
    n = len(x)
    bary = np.empty((n, 3))
    assert emu.dg_mesh_distance_bary(m.h, P(x), n, 1, None, None, None, None, P(bary)) == 0
    assert_bits(bary, r[4], "weights alone")


def test_every_query_on_one_triangle(emu, k10):
    """one segment of 2500 queries: three levels of the tree"""
    V, F = mesh("box")
    rng = np.random.default_rng(4)
    a, b, c = V[F[5, 0]], V[F[5, 1]], V[F[5, 2]]
    u = rng.random((2500, 2))
    u = np.where(u.sum(1, keepdims=True) > 1, 1 - u, u) * 0.98 + 0.005
    nrm = np.cross(b - a, c - a)
    x = a + u[:, :1] * (b - a) + u[:, 1:] * (c - a) + rng.uniform(0.01, 0.2, (2500, 1)) * nrm / np.linalg.norm(nrm)
    x = np.ascontiguousarray(x)
    m = Mesh(emu, V, F)
    r = m.nearest(x, True)
    assert (r[3] == 5).all()
    g = rng.standard_normal(len(x))
    w, gx, gv, _, _ = restated(V, F, x, r, g)
    rc, gp_c, gv_c = m.vjp(x, r, g)
    assert rc == 0
    assert_bits(gp_c, gx, "grad_points")
    assert_bits(gv_c, gv, "grad_vertices")
    assert_bits(run_k10(k10, V, F, x, r, g)[1], gv, "grad_vertices (libk10emu)")
    # the tree is not the left-to-right sum: the restatement is what pins the bits
    c = gr.contributions(gx, w)[:, 0, 0]
    assert gv[F[5, 0], 0] == gr.segment_sums(np.zeros(len(c), np.int64), c)[1][0]


def test_zero_queries(emu, k10):
    V, F = mesh("box")
    m = Mesh(emu, V, F)
    x = np.empty((0, 3))
    r = m.nearest(x, True)
    rc, gp, gv = m.vjp(x, r, np.empty(0))
    assert rc == 0 and gp.shape == (0, 3)
    assert gr.same_bits(gv, np.zeros_like(gv))
    e = np.empty(0)
    assert emu.dg_mesh_distance_vjp(m.h, 0, None, None, None, None, None, None, None, P(np.full((len(V), 3), 7.0))) == 0
    assert run_k10(k10, V, F, x, r, e)[1].sum() == 0


@pytest.mark.parametrize("key_bits", [1, 4, 8, 9, 16, 17, 24, 25, 32])
def test_sort_is_numpys_stable_argsort(k10, key_bits):
    rng = np.random.default_rng(key_bits)
    for n in (1, 31, 1000, 5003):
        hi = 1 << key_bits
        pool = rng.integers(0, hi, max(2, n // 3), dtype=np.uint64)          # every bit in use, and duplicates
        keys = pool[rng.integers(0, len(pool), n)].astype(np.uint32)
        keys[::7] = hi - 1
        ko, vo = np.empty(n, np.uint32), np.empty(n, np.uint32)
        assert k10.emu_k10_sort(P(keys, U32P), None, n, key_bits, P(ko, U32P), P(vo, U32P)) == 0
        perm = np.argsort(keys, kind="stable")
        assert np.array_equal(vo, perm), f"{key_bits} bits, n = {n}: permutation"
        assert np.array_equal(ko, keys[perm])
        vals = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
        assert k10.emu_k10_sort(P(keys, U32P), P(vals, U32P), n, key_bits, P(ko, U32P), P(vo, U32P)) == 0
        assert np.array_equal(vo, vals[perm])
    assert k10.emu_k10_sort_passes(key_bits) == max(1, -(-key_bits // 8))


def test_three_digit_passes(k10):
    """70 000 triangles: keys of 17 bits, three passes, through the VJP on synthetic forward outputs (the VJP reads nothing else)"""
    rng = np.random.default_rng(5)
    nT, nV, n = 70000, 40000, 6000
    F = rng.integers(0, nV, (nT, 3)).astype(np.uint32)
    tri = rng.integers(-1, nT, n).astype(np.int32)
    tri[:500] = nT - 1
    tri[500:900] = 3
    x = rng.standard_normal((n, 3)); near = rng.standard_normal((n, 3))
    d = rng.standard_normal(n); d[::50] = 0.0
    w = rng.random((n, 3)); g = rng.standard_normal(n)
    assert k10.emu_k10_sort_passes(17) == 3
    gp, gv = run_k10(k10, np.zeros((nV, 3)), F, x, (d, near, None, tri, w), g)
    gx = gr.grad_points(x, d, near, tri, g)
    assert_bits(gp, gx, "grad_points")
    assert_bits(gv, gr.grad_vertices(F, nV, tri, gx, w), "grad_vertices")


def test_refusals(emu, k10):
    V, F = mesh("box")
    m = Mesh(emu, V, F)
    x = queries(V, F, 40, 6)
    r = m.nearest(x, True)
    g = np.ones(len(x))
    for bad in (12, 1000, -2):
        rb = list(r)
        rb[3] = r[3].copy(); rb[3][17] = bad
        rc, gp, gv = m.vjp(x, rb, g)
        assert rc == DG_ERR_INVALID and "triangle ids outside" in emu.dg_last_error().decode()
        assert (gp == 7.0).all() and (gv == 7.0).all(), "nothing is written before a refusal"
        gpk, gvk = np.full((len(x), 3), 7.0), np.full((len(V), 3), 7.0)
        assert k10.emu_k10_vjp(len(x), P(x), P(r[0]), P(r[1]), P(rb[3], I32P), P(r[4]), P(g), P(np.ascontiguousarray(F, np.uint32), U32P),
                               len(F), len(V), P(gpk), P(gvk)) == 1
    n = len(x)
    gv = np.empty((len(V), 3))
    assert emu.dg_mesh_distance_vjp(None, n, P(x), P(r[0]), P(r[1]), P(r[3], I32P), P(r[4]), P(g), None, P(gv)) == DG_ERR_INVALID
    assert emu.dg_last_error().decode().startswith("dg_mesh_distance_vjp:")
    assert emu.dg_mesh_distance_vjp(m.h, n, P(x), P(r[0]), P(r[1]), None, P(r[4]), P(g), None, P(gv)) == DG_ERR_INVALID
    assert emu.dg_mesh_distance_vjp_device(m.h, n, P(x), P(r[0]), P(r[1]), P(r[3], I32P), None, P(g), None, P(gv), None) == DG_ERR_INVALID
    assert emu.dg_last_error().decode().startswith("dg_mesh_distance_vjp_device:")
    assert emu.dg_mesh_distance_bary(None, P(x), n, 1, None, None, None, None, None) == DG_ERR_INVALID
    assert emu.dg_mesh_distance_bary_device(m.h, None, n, 1, None, None, None, None, None, None) == DG_ERR_INVALID
