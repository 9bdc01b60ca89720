"""K8 (the refit, discregrid_b200/csrc/k8_refit.cu) on the CPU: the product's translation unit compiled through tests/emu (build/bin/libk8emu.so)
against the numpy restatement of its contract in tests/refit_ref.py, bit for bit; the refit to the build's own vertices against the host
build; and the refusals of dg_mesh_refit on the emulated library (build/bin/libdgemu.so)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from conftest import ROOT
import refit_ref as rr
import winding_ref as wr

K8EMU = os.path.join(ROOT, "build", "bin", "libk8emu.so")
DGEMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
DP, FP, U32P, I32P, VP = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.c_void_p


def P(a, t=DP):
    return a.ctypes.data_as(t)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a.view(np.uint32) if a.dtype == np.float32 else a


def assert_bits(got, want, what):
    g, w = bits(got), bits(want)
    bad = np.flatnonzero((g != w).reshape(-1))
    assert len(bad) == 0, f"{what}: {len(bad)} of {g.size} differ, first at flat index {bad[0]}: {got.reshape(-1)[bad[0]]!r} vs {want.reshape(-1)[bad[0]]!r}"


@pytest.fixture(scope="module")
def k8():
    if not os.path.exists(K8EMU):
        pytest.skip("build/bin/libk8emu.so not built (make cpp)")
    lib = C.CDLL(K8EMU)
    lib.emu_refit_create.restype = VP
    lib.emu_refit_create.argtypes = [DP, C.c_uint64, U32P, C.c_uint64]
    lib.emu_refit_destroy.argtypes = [VP]
    lib.emu_refit.argtypes = [VP, DP, C.c_int]
    lib.emu_refit_winding_only.argtypes = [VP]
    lib.emu_refit_records.argtypes = [VP, I32P, VP, FP, DP, FP, DP, DP, DP, DP]
    lib.emu_k8_acos.argtypes = [DP, C.c_uint64, DP]
    return lib


class EmuRefit:
    def __init__(self, lib, V, F):
        self.lib, self.F = lib, np.ascontiguousarray(F, np.uint32)
        V = np.ascontiguousarray(V, np.float64)
        self.nV, self.T = len(V), len(self.F)
        self.stride = lib.emu_refit_nodef_stride()
        self.h = lib.emu_refit_create(P(V), len(V), P(self.F, U32P), len(self.F))
        assert self.h

    def refit(self, V, with_k5=True):
        V = np.ascontiguousarray(V, np.float64)
        assert self.lib.emu_refit(self.h, P(V), int(with_k5)) == 0
        return self

    def records(self):
        T = self.T
        r = dict(order=np.empty(T, np.int32), leaves=np.empty((T, 16), np.uint64), leaves_f=np.empty((T, 16), np.float32),
                 spheres=np.empty((T, 8)), nodes_f=np.empty((T, 4 * self.stride), np.float32), normals=np.empty((T, 7, 3)),
                 bounds=np.empty(5), wind_leaves=np.empty((T, 9)), clusters=np.empty((T, 2, 16)))
        self.lib.emu_refit_records(self.h, P(r["order"], I32P), r["leaves"].ctypes.data_as(VP), P(r["leaves_f"], FP), P(r["spheres"]),
                                   P(r["nodes_f"], FP), P(r["normals"]), P(r["bounds"]), P(r["wind_leaves"]), P(r["clusters"]))
        return r

    def close(self):
        self.lib.emu_refit_destroy(self.h)


def check_against_restatement(e, V, F):
    got = e.records()
    want = rr.Refit(V, F, got["order"], e.stride)
    assert_bits(got["bounds"][:3], want.center, "centre")
    assert_bits(got["bounds"][3:4], np.array([want.half_extent]), "half extent")
    assert_bits(got["leaves"], want.leaves, "leaf records")
    assert_bits(got["leaves_f"], want.leaves_f, "fp32 leaf shadows")
    assert_bits(got["spheres"], want.spheres, "sphere pairs")
    assert_bits(got["nodes_f"], want.nodes_f, "fp32 node records")
    assert_bits(got["normals"], want.normals, "per-leaf pseudonormal blocks")
    assert_bits(got["wind_leaves"], want.wind_leaves, "K5 leaf records")
    assert_bits(got["clusters"], want.clusters, "K5 cluster records")
    return got, want


# ---------------------------------------------------------------------------------------------------------------- meshes
def _bunny():
    p = wr.ref_resource(ROOT, "bunny.obj")
    if p is None or not os.path.exists(p):
        pytest.skip("bunny.obj not staged (make -C oracle ref)")
    return wr.read_obj(p)


def _mean_edge(V, F):
    return float(np.linalg.norm(V[F[:, 1]] - V[F[:, 0]], axis=1).mean())


def twist(V, angle):
    lo, hi = V[:, 1].min(), V[:, 1].max()
    t = angle * (V[:, 1] - lo) / (hi - lo)
    c, s = np.cos(t), np.sin(t)
    return np.stack([c * V[:, 0] + s * V[:, 2], V[:, 1], -s * V[:, 0] + c * V[:, 2]], 1)


def deformations(name):
    """(V0, F, [V1, V2, ...]): the build's vertices and the positions to refit to (same topology)"""
    import discregrid_b200 as dg
    rng = np.random.default_rng(11)
    if name == "box":
        m = dg.box(); V, F = m.vertices, m.faces
        return V, F, [V * np.array([1.5, 0.7, 1.1]) + 0.25, V + rng.normal(0, 0.1, V.shape)]
    if name == "uv_sphere":
        m = dg.uv_sphere(12, 24); V, F = m.vertices, m.faces
        return V, F, [V * (1.0 + 0.2 * V[:, :1]), twist(V, 0.7)]
    if name == "bumpy_torus":
        m0 = dg.bumpy_torus(24, 16, amp=0.05)
        return m0.vertices, m0.faces, [dg.bumpy_torus(24, 16, amp=a).vertices for a in (0.0, 0.12, 0.3)]
    if name == "bunny_twist":
        V, F = _bunny()
        return V, F, [twist(V, a) for a in (0.1, 0.5, 1.5)]
    if name == "bunny_noise":
        V, F = _bunny()
        return V, F, [V + rng.normal(0, 0.1 * _mean_edge(V, F), V.shape)]
    if name == "open_bunny":
        V, F = wr.cut_top(*_bunny())
        return V, F, [twist(V, 0.5)]
    if name == "soup":
        V, F = wr.soup()
        return V, F, [V * 1.3 - 0.2, V + rng.normal(0, 0.05, V.shape)]
    if name == "degenerate":
        m = dg.uv_sphere(6, 10); V, F = m.vertices.copy(), m.faces.copy()
        F = np.concatenate([F, [[0, 0, 1], [2, 2, 2]]]).astype(np.uint32)          # a triangle repeating a vertex, one collapsed to a point
        V1 = V.copy(); V1[F[3]] = V1[F[3, 0]]                                       # collapsed to a point
        V1[F[5, 1]] = V1[F[5, 0]]; V1[F[5, 2]] = 0.5 * (V1[F[5, 0]] + V1[F[5, 0]])  # collapsed to an edge
        return V, F, [V1]
    if name == "nonfinite":
        m = dg.uv_sphere(6, 10); V, F = m.vertices, m.faces
        out = []
        for bad in (np.nan, np.inf, -np.inf):
            V1 = V.copy(); V1[5, 1] = bad; out.append(V1)
        return V, F, out
    if name == "scales":
        m = dg.bumpy_torus(16, 12); V, F = m.vertices, m.faces
        return V, F, [twist(V, 0.3) * 1e-200, twist(V, 0.3) * 1e200]
    raise KeyError(name)


MESHES = ["box", "uv_sphere", "bumpy_torus", "bunny_twist", "bunny_noise", "open_bunny", "soup", "degenerate", "nonfinite", "scales"]


@pytest.mark.parametrize("name", MESHES)
def test_records_equal_the_restatement(k8, name):
    V0, F, targets = deformations(name)
    e = EmuRefit(k8, V0, F)
    try:
        for V1 in targets:
            got, _ = check_against_restatement(e.refit(V1), V1, F)
            k5 = wr.Records(V1, F, got["order"])           # the K5 records restated independently of refit_ref
            assert_bits(got["clusters"], k5.as_array(), "K5 clusters vs winding_ref.Records")
            assert_bits(got["wind_leaves"], k5.leaves, "K5 leaves vs winding_ref.Records")
    finally:
        e.close()


@pytest.mark.parametrize("T", [1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128, 129])
def test_tree_sizes_around_powers_of_two(k8, T):
    rng = np.random.default_rng(T)
    V = rng.random((3 * T, 3))
    F = np.arange(3 * T, dtype=np.uint32).reshape(T, 3)
    e = EmuRefit(k8, V, F)
    try:
        V1 = V + rng.normal(0, 0.3, V.shape)
        check_against_restatement(e.refit(V1), V1, F)
    finally:
        e.close()


def test_k5_records_match_the_host_builder_and_winding_ref(k8):
    """the device K5 records equal build_winding_records' (host) bit for bit on the build's vertices, and winding_ref.Records on others"""
    V, F, targets = deformations("soup")
    e = EmuRefit(k8, V, F)
    try:
        host = e.records()
        e.refit(V)
        dev = e.records()
        assert_bits(dev["clusters"], host["clusters"], "K5 clusters, device vs host builder")
        assert_bits(dev["wind_leaves"], host["wind_leaves"], "K5 leaves, device vs host builder")
        for V1 in targets:
            got = e.refit(V1).records()
            want = wr.Records(V1, F, got["order"])
            assert_bits(got["clusters"], want.as_array(), "K5 clusters vs winding_ref.Records")
            assert_bits(got["wind_leaves"], want.leaves, "K5 leaves vs winding_ref.Records")
    finally:
        e.close()


def test_winding_only_pass_equals_the_full_refit(k8):
    V, F, targets = deformations("bumpy_torus")
    e = EmuRefit(k8, V, F)
    try:
        full = e.refit(targets[1]).records()
        e.refit(targets[2], with_k5=False)           # K1 records of targets[2]; K5 records still those of targets[1]
        assert_bits(e.records()["clusters"], full["clusters"], "K5 records untouched without with_k5")
        e.refit(targets[1], with_k5=False)
        assert k8.emu_refit_winding_only(e.h) == 0
        assert_bits(e.records()["clusters"], full["clusters"], "K5-only pass")
    finally:
        e.close()


def test_refit_acos_bounds(k8):
    rng = np.random.default_rng(5)
    x = np.concatenate([rng.random(10 ** 6), [0.0, 1.0, 1.0 + 2 ** -52, 2.0, np.nan, 0.5]])
    got = np.empty_like(x)
    k8.emu_k8_acos(P(x), len(x), P(got))
    want = rr.refit_acos(x)
    assert_bits(got, want, "k8_acos vs restatement")
    assert got[-6] == math.pi / 2 and got[-5] == 0.0
    assert np.isnan(got[-4]) and np.isnan(got[-3]) and np.isnan(got[-2])
    ref = np.arccos(x[:10 ** 6])
    ulp = np.abs(got[:10 ** 6] - ref) / np.spacing(np.maximum(np.abs(ref), 1e-300))
    assert ulp.max() <= 4.0, ulp.max()      # k5_atan2 is within 2 ulp of atan2; the sqrt argument adds at most 2 more near x = 1


@pytest.mark.parametrize("name", ["box", "uv_sphere", "bumpy_torus", "bunny_twist", "soup"])
def test_refit_to_the_build_vertices_equals_the_build(k8, name):
    """leaf records, leaf shadows, leaf spheres, child boxes, centre, half extent and K5 records are those of dg_mesh_create; internal sphere
    centres differ by the sum order (k8_refit.cu), so they and the radii are only close"""
    V, F, _ = deformations(name)
    e = EmuRefit(k8, V, F)
    try:
        b = e.records()
        a = e.refit(V).records()
        for k in ("leaves", "leaves_f", "bounds", "wind_leaves", "clusters"):
            assert_bits(a[k], b[k], k)
        parent, side = rr._leaf_parent(len(F))
        for s_ in (0, 1):
            sel = (parent >= 0) & (side == s_)
            assert_bits(a["spheres"][parent[sel], 4 * s_:4 * s_ + 4], b["spheres"][parent[sel], 4 * s_:4 * s_ + 4], "leaf spheres")
        assert np.array_equal(a["nodes_f"][:, 8:20], b["nodes_f"][:, 8:20]), "child boxes"
        np.testing.assert_allclose(a["spheres"], b["spheres"], rtol=1e-13, atol=1e-15)
    finally:
        e.close()


def test_only_the_current_positions_matter(k8):
    V, F, targets = deformations("bumpy_torus")
    e1, e2 = EmuRefit(k8, V, F), EmuRefit(k8, V, F)
    try:
        a = e1.refit(targets[0]).refit(targets[2]).records()
        b = e2.refit(targets[2]).records()
        for k in a:
            assert_bits(a[k], b[k], k)
    finally:
        e1.close(); e2.close()


# ---------------------------------------------------------------------------------------------------------------- C-ABI refusals
@pytest.fixture(scope="module")
def emu():
    if not os.path.exists(DGEMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    lib = C.CDLL(DGEMU)
    lib.dg_mesh_create.argtypes = [DP, C.c_uint64, U32P, C.c_uint64, C.POINTER(VP)]
    lib.dg_mesh_refit.argtypes = [VP, DP, C.c_uint64]
    lib.dg_mesh_refit_device.argtypes = [VP, VP, C.c_uint64, VP]
    lib.dg_mesh_group_create.argtypes = [VP, C.c_int, C.POINTER(C.c_int), C.POINTER(VP)]
    lib.dg_mesh_group_destroy.argtypes = [VP]
    lib.dg_mesh_destroy.argtypes = [VP]
    lib.dg_mesh_info.argtypes = [VP, C.POINTER(C.c_uint64)]
    lib.dg_mesh_pseudonormals.argtypes = [VP, DP, DP, DP]
    lib.dg_last_error.restype = C.c_char_p
    return lib


def test_refusals(emu):
    import discregrid_b200 as dg
    m = dg.box(); V, F = np.ascontiguousarray(m.vertices, np.float64), np.ascontiguousarray(m.faces, np.uint32)
    h = VP()
    assert emu.dg_mesh_create(P(V), len(V), P(F, U32P), len(F), C.byref(h)) == 0
    try:
        INVALID = -1     # DG_ERR_INVALID
        assert emu.dg_mesh_refit(None, P(V), len(V)) == INVALID
        a = np.empty(9)
        assert emu.dg_mesh_pseudonormals(None, P(a), P(a), P(a)) == INVALID
        assert emu.dg_mesh_refit_device(None, V.ctypes.data, len(V), None) == INVALID
        assert emu.dg_mesh_refit(h, None, len(V)) == INVALID
        assert emu.dg_mesh_refit_device(h, None, len(V), None) == INVALID
        assert emu.dg_mesh_refit(h, P(V), len(V) - 1) == INVALID and b"vertices" in emu.dg_last_error()
        assert emu.dg_mesh_refit(h, P(V), 0) == INVALID
        info = (C.c_uint64 * 8)()
        assert emu.dg_mesh_info(h, info) == 0
        before = info[4]
        g = VP()
        assert emu.dg_mesh_group_create(h, 1, None, C.byref(g)) == 0
        assert emu.dg_mesh_refit(h, P(V), len(V)) == INVALID and b"dg_mesh_group" in emu.dg_last_error()
        assert emu.dg_mesh_group_destroy(g) == 0
        assert emu.dg_mesh_info(h, info) == 0 and info[4] == before          # nothing allocated by a refusal
        assert emu.dg_mesh_refit(h, P(V * 2.0), len(V)) == 0
        assert emu.dg_mesh_info(h, info) == 0 and info[4] > before
    finally:
        emu.dg_mesh_destroy(h)
