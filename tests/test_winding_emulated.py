"""K5 (generalized winding numbers, discregrid_b200/csrc/k5_winding.cu) on the CPU: the product's translation unit compiled through tests/emu
(build/bin/libk5emu.so) against the numpy restatement of its contract in tests/winding_ref.py, bit for bit; and the winding sign mode of the
whole C-ABI on the emulated library (build/bin/libdgemu.so): node values, sentinels and refusals."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from conftest import ROOT, GOLDEN, bits_equal
import winding_ref as wr

K5EMU = os.path.join(ROOT, "build", "bin", "libk5emu.so")
DGEMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
DP, U32P, I32P, VP = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.c_void_p


def P(a, t=DP):
    return a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def k5():
    if not os.path.exists(K5EMU):
        pytest.skip("build/bin/libk5emu.so not built (make cpp)")
    lib = C.CDLL(K5EMU)
    lib.emu_winding_create.restype = VP
    lib.emu_winding_create.argtypes = [DP, C.c_uint64, U32P, C.c_uint64]
    lib.emu_winding_destroy.argtypes = [VP]
    lib.emu_winding_records.argtypes = [VP, I32P, DP, DP]
    lib.emu_winding_number.argtypes = [VP, DP, C.c_uint64, C.c_double, DP]
    lib.emu_k5_atan2.argtypes = [DP, DP, C.c_uint64, DP]
    return lib


class EmuWinding:
    def __init__(self, lib, V, F):
        self.lib, self.V, self.F = lib, np.ascontiguousarray(V, np.float64), np.ascontiguousarray(F, np.uint32)
        self.h = lib.emu_winding_create(P(self.V), len(self.V), P(self.F, U32P), len(self.F))
        T = len(self.F)
        self.order = np.empty(T, np.int32); self.leaves = np.empty((T, 9)); self.clusters = np.empty((T, 2, 16))
        lib.emu_winding_records(self.h, P(self.order, I32P), P(self.leaves), P(self.clusters))

    def w(self, pts, beta):
        pts = np.ascontiguousarray(pts, np.float64).reshape(-1, 3)
        out = np.empty(len(pts))
        assert self.lib.emu_winding_number(self.h, P(pts), len(pts), beta, P(out)) == 0
        return out

    def __del__(self):
        self.lib.emu_winding_destroy(self.h)


def torus_small():
    import discregrid_b200 as dg
    m = dg.bumpy_torus(48, 48, 1.0, 0.4, 0.05, 7, 5)
    return np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)


def mesh(name):
    if name == "box":
        return wr.read_obj(os.path.join(GOLDEN, "box.obj"))
    if name == "torus":
        return torus_small()
    if name == "open_torus":
        return wr.cut_top(*torus_small())
    if name == "soup":
        return wr.soup()
    if name == "open_bunny_small":
        p = wr.ref_resource(ROOT, "bunny.obj")
        if p is None:
            pytest.skip("bunny.obj not staged (make -C oracle ref)")
        V, F = wr.cut_top(*wr.read_obj(p))
        return V, np.ascontiguousarray(F[:3000])
    raise KeyError(name)


MESHES = ["box", "torus", "open_torus", "soup", "open_bunny_small"]


# ---------------------------------------------------------------------------------------------------------------- atan2
def ulp_distance(a, b):
    def ordered(x):
        i = np.ascontiguousarray(x, np.float64).view(np.int64)
        return np.where(i < 0, np.int64(-2 ** 63) - i, i)
    return np.abs(ordered(a) - ordered(b))


def test_atan2_bits_and_accuracy(k5):
    rng = np.random.default_rng(2026)
    n = 1_000_000
    y = rng.standard_normal(n) * np.exp2(rng.integers(-80, 80, n).astype(np.float64))
    x = rng.standard_normal(n) * np.exp2(rng.integers(-80, 80, n).astype(np.float64))
    x[: n // 4] = y[: n // 4] * (1.0 + rng.standard_normal(n // 4) * 1e-3)          # ratios near 1 and -1
    x[n // 4: n // 2] = rng.standard_normal(n // 4)
    y[n // 4: n // 2] = x[n // 4: n // 2] * rng.uniform(0.3, 3.0, n // 4)          # every reduction interval
    out = np.empty(n)
    k5.emu_k5_atan2(P(y), P(x), n, P(out))
    assert bits_equal(out, wr.atan2(y, x))
    ref = np.array([math.atan2(a, b) for a, b in zip(y.tolist(), x.tolist())])
    assert int(ulp_distance(out, ref).max()) <= 2


def test_atan2_special_cases(k5):
    inf, nan = math.inf, math.nan
    vals = [0.0, -0.0, 1.0, -1.0, 1e-310, -1e-310, 1e300, -1e300, inf, -inf, nan, 2.0 ** 61, 2.0 ** -61]
    y = np.array([a for a in vals for _ in vals]); x = np.array([b for _ in vals for b in vals])
    out = np.empty(len(y))
    k5.emu_k5_atan2(P(y), P(x), len(y), P(out))
    assert bits_equal(out, wr.atan2(y, x))
    for a, b, o in zip(y, x, out):
        r = math.atan2(a, b)
        if math.isnan(r):
            assert math.isnan(o)
        else:
            assert ulp_distance(np.array([o]), np.array([r]))[0] <= 2, (a, b, o, r)
            assert math.copysign(1.0, o) == math.copysign(1.0, r)
    s = lambda a, b: float(wr.atan2(np.array([a]), np.array([b]))[0])
    assert math.copysign(1, s(0.0, -1.0)) > 0 and s(0.0, -1.0) == wr.PI and s(-0.0, -1.0) == -wr.PI
    assert bits_equal([s(0.0, 1.0), s(-0.0, 1.0), s(-0.0, -0.0)], [0.0, -0.0, -wr.PI])


# ---------------------------------------------------------------------------------------------------------------- records and sums
@pytest.mark.parametrize("name", MESHES)
def test_records_match_restatement(k5, name):
    V, F = mesh(name)
    e = EmuWinding(k5, V, F)
    rec = wr.Records(V, F, e.order)
    assert sorted(e.order.tolist()) == list(range(len(F)))
    assert bits_equal(e.leaves, rec.leaves)
    assert bits_equal(e.clusters, rec.as_array())


@pytest.mark.parametrize("name", MESHES)
def test_exact_sum_bits(k5, name):
    V, F = mesh(name)
    e = EmuWinding(k5, V, F)
    p = wr.query_points(V, 300, seed=11, near=60)
    w = e.w(p, math.inf)
    leaves = np.ascontiguousarray(V[F[e.order]].reshape(-1, 9))
    assert bits_equal(w, wr.exact_w(leaves, p))
    # the same sum in the original triangle order: only the rounding of the fold differs
    w_orig = wr.exact_w(np.ascontiguousarray(V[F].reshape(-1, 9)), p)
    assert np.max(np.abs(w - w_orig)) <= 1e-12 * len(F)


@pytest.mark.parametrize("name", MESHES)
def test_beta2_bits(k5, name):
    V, F = mesh(name)
    e = EmuWinding(k5, V, F)
    rec = wr.Records(V, F, e.order)
    p = wr.query_points(V, 150, seed=12, near=30)
    for beta in (2.0, 1.0, 3.5):
        assert bits_equal(e.w(p, beta), rec.w(p, beta)), beta
    w2, wi = e.w(p, 2.0), e.w(p, math.inf)
    assert np.max(np.abs(w2 - wi)) <= 0.1


def test_watertight_w_is_integer_away_from_the_surface(k5):
    V, F = mesh("box")
    e = EmuWinding(k5, V, F)
    assert bits_equal(e.w([[0.0, 0.0, 0.0]], math.inf), [1.0]) or abs(e.w([[0.0, 0.0, 0.0]], math.inf)[0] - 1.0) < 1e-15
    p = wr.query_points(V, 200, seed=3)
    inside = np.all(np.abs(p) < 1.0, axis=1)
    for beta in (2.0, math.inf):
        w = e.w(p, beta)
        assert np.all((w > 0.5) == inside)


# ---------------------------------------------------------------------------------------------------------------- the C-ABI on the emulated library
class EmuLib:
    def __init__(self):
        lib = C.CDLL(DGEMU)
        lib.dg_last_error.restype = C.c_char_p
        self.lib = lib

    def check(self, rc):
        assert rc == 0, (rc, self.lib.dg_last_error())

    def mesh(self, V, F):
        h = VP()
        V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
        self.check(self.lib.dg_mesh_create(P(V), C.c_uint64(len(V)), P(F, U32P), C.c_uint64(len(F)), C.byref(h)))
        return h

    def grid(self, V, res):
        mn, mx = (C.c_double * 3)(), (C.c_double * 3)()
        V = np.ascontiguousarray(V, np.float64)
        self.check(self.lib.dg_generate_sdf_domain(P(V), C.c_uint64(len(V)), mn, mx))
        import discregrid_b200._capi as capi
        g = capi.GridDesc()
        self.check(self.lib.dg_grid_init(mn, mx, (C.c_uint32 * 3)(*res), C.byref(g)))
        n = C.c_uint64()
        self.check(self.lib.dg_grid_num_nodes((C.c_uint32 * 3)(*res), C.byref(n)))
        return g, n.value

    def set_mode(self, h, mode, beta=2.0):
        return self.lib.dg_mesh_set_sign_mode(h, C.c_int(mode), C.c_double(beta))

    def sample(self, h, g, n, sign, band=None):
        out = np.empty(n)
        if band is None:
            self.check(self.lib.dg_sample_sdf_device(h, C.byref(g), C.c_double(sign), C.c_uint64(0), C.c_uint64(n), P(out), None))
        else:
            self.check(self.lib.dg_sample_sdf_band_device(h, C.byref(g), C.c_double(sign), C.c_double(band), C.c_uint64(0), C.c_uint64(n),
                                                          P(out), None))
        return out

    def add_function(self, h, g, n, sign, band=None):
        out = np.empty(n)
        if band is None:
            self.check(self.lib.dg_add_function_sdf(h, C.byref(g), C.c_double(sign), P(out), None, None, None))
        else:
            self.check(self.lib.dg_add_function_sdf_band(h, C.byref(g), C.c_double(sign), C.c_double(band), P(out), None, None, None))
        return out

    def distance(self, h, p, signed=True):
        p = np.ascontiguousarray(p, np.float64)
        d = np.empty(len(p)); near = np.empty((len(p), 3)); ent = np.empty(len(p), np.int32); tri = np.empty(len(p), np.int32)
        self.check(self.lib.dg_mesh_distance(h, P(p), C.c_uint64(len(p)), C.c_int(int(signed)), P(d), P(near), P(ent, I32P), P(tri, I32P)))
        return d, near, ent, tri

    def winding(self, h, p, beta):
        p = np.ascontiguousarray(p, np.float64)
        w = np.empty(len(p))
        self.check(self.lib.dg_mesh_winding_number(h, P(p), C.c_uint64(len(p)), C.c_double(beta), P(w)))
        return w


@pytest.fixture(scope="module")
def emu():
    if not os.path.exists(DGEMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    return EmuLib()


@pytest.mark.parametrize("name,res", [("box", (10, 10, 10)), ("torus", (8, 8, 6))])
def test_watertight_node_values_equal_pseudonormal(emu, name, res):
    V, F = mesh(name)
    h = emu.mesh(V, F)
    g, n = emu.grid(V, res)
    cell_diag = math.sqrt(sum(c * c for c in g.cell_size))
    for sign in (1.0, -1.0):
        ref = emu.sample(h, g, n, sign)
        ref_band = emu.sample(h, g, n, sign, band=2 * cell_diag)
        ref_host = emu.add_function(h, g, n, sign, band=2 * cell_diag)
        emu.check(emu.set_mode(h, 1, 2.0))
        got = emu.sample(h, g, n, sign)
        got_band = emu.sample(h, g, n, sign, band=2 * cell_diag)
        got_host = emu.add_function(h, g, n, sign)
        got_host_band = emu.add_function(h, g, n, sign, band=2 * cell_diag)
        emu.check(emu.set_mode(h, 0, 2.0))
        nz = ref != 0.0
        assert bits_equal(got[nz], ref[nz]) and bits_equal(got_host[nz], ref[nz])
        nzb = ref_band != 0.0
        assert bits_equal(got_band[nzb], ref_band[nzb]) and bits_equal(got_host_band[nzb], ref_host[nzb])
        assert np.all(np.abs(got) == np.abs(ref))                    # the magnitude's bits everywhere
        assert np.array_equal(got_band == wr_dbl_max(), ref_band == wr_dbl_max())
        if name == "box":
            assert np.sum(ref_band == wr_dbl_max()) > 0
    emu.lib.dg_mesh_destroy(h)


def wr_dbl_max():
    return np.finfo(np.float64).max


def test_open_mesh_signs_follow_w(emu):
    V, F = mesh("open_torus")
    h = emu.mesh(V, F)
    p = np.concatenate([wr.query_points(V, 400, seed=5), [[np.nan, 0.0, 0.0], [np.inf, 1.0, 2.0]]])
    d_pn, near_pn, ent_pn, tri_pn = emu.distance(h, p, signed=True)
    d_u, near_u, ent_u, tri_u = emu.distance(h, p, signed=False)
    emu.check(emu.set_mode(h, 1, 2.0))
    d_w, near_w, ent_w, tri_w = emu.distance(h, p, signed=True)
    w = emu.winding(h, p, 2.0)
    emu.check(emu.set_mode(h, 0, 2.0))
    assert bits_equal(near_w, near_u) and np.array_equal(ent_w, ent_u) and np.array_equal(tri_w, tri_u)
    assert bits_equal(np.abs(d_w), d_u)
    finite = d_u != wr_dbl_max()
    assert not finite[-1] and not finite[-2] and bits_equal(d_w[~finite], d_pn[~finite])
    assert np.all((d_w[finite] < 0) == (w[finite] > 0.5))
    assert np.any((d_pn[finite] < 0) != (d_w[finite] < 0))          # the open torus: the pseudonormal sign is wrong somewhere
    emu.lib.dg_mesh_destroy(h)


def test_refusals(emu):
    V, F = mesh("box")
    h = emu.mesh(V, F)
    g, n = emu.grid(V, (4, 4, 4))
    for mode, beta in ((1, math.nan), (1, 0.5), (1, -math.inf), (0, math.nan), (2, 2.0), (-1, 2.0)):
        assert emu.set_mode(h, mode, beta) == -1
    w = np.empty(1)
    assert emu.lib.dg_mesh_winding_number(h, P(np.zeros(3)), C.c_uint64(1), C.c_double(math.nan), P(w)) == -1
    assert emu.lib.dg_mesh_winding_number(h, P(np.zeros(3)), C.c_uint64(1), C.c_double(0.99), P(w)) == -1
    emu.check(emu.set_mode(h, 1, math.inf))
    grp = VP()
    assert emu.lib.dg_mesh_group_create(h, C.c_int(1), None, C.byref(grp)) == -1
    assert b"winding" in emu.lib.dg_last_error()
    full = np.empty(n)
    assert emu.lib.dg_sample_sdf_slab_device(h, C.byref(g), C.c_double(1.0), C.c_uint32(0), C.c_uint32(1), P(full), None) == -1
    assert b"winding" in emu.lib.dg_last_error()
    slot = C.c_uint64()
    emu.check(emu.lib.dg_interleaved_slot_elems(C.byref(g), C.c_uint32(1), C.byref(slot)))
    buf = np.empty(slot.value)
    assert emu.lib.dg_sample_sdf_interleaved_device(h, C.byref(g), C.c_double(1.0), C.c_uint32(0), C.c_uint32(1), P(buf), None) == -1
    assert b"winding" in emu.lib.dg_last_error()
    # a mesh that has never used the winding records reports the same device bytes as before
    h2 = emu.mesh(V, F)
    info1, info2 = (C.c_uint64 * 8)(), (C.c_uint64 * 8)()
    emu.check(emu.lib.dg_mesh_info(h2, info1))
    emu.check(emu.set_mode(h2, 1, 2.0))
    emu.check(emu.lib.dg_mesh_info(h2, info2))
    assert info1[4] == info2[4]
    emu.winding(h2, np.zeros((1, 3)), 2.0)
    emu.check(emu.lib.dg_mesh_info(h2, info2))
    assert info2[4] == info1[4] + len(F) * (72 + 256)
    # the group refused above; a group made in the pseudonormal mode refuses once the mesh switches
    emu.check(emu.set_mode(h, 0, 2.0))
    if emu.lib.dg_mesh_group_create(h, C.c_int(1), None, C.byref(grp)) == 0:
        emu.check(emu.set_mode(h, 1, 2.0))
        nodes = np.empty(n)
        assert emu.lib.dg_add_function_sdf_multi(grp, C.byref(g), C.c_double(1.0), P(nodes), None, None, None) == -1
        emu.lib.dg_mesh_group_destroy(grp)
    emu.lib.dg_mesh_destroy(h)
    emu.lib.dg_mesh_destroy(h2)


# ---------------------------------------------------------------------------------------------------------------- tools/k5_fuzz.py, short runs
def _k5_fuzz():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import k5_fuzz
    return k5_fuzz


def test_k5_fuzz_short_run(k5):
    """a short run of tools/k5_fuzz.py on the emulated K5: tree sizes around powers of two, tie-rich meshes (w exactly 1/2, 1/4, 1/8) and a
    zero-area subtree, scales 10^-300 .. 10^300, NaN / inf vertices and queries, every branch of k5_atan2, beta = 1, 2, 3.5, inf and
    prefix counts around the warp and block sizes -- bit for bit with the restatement"""
    f = _k5_fuzz()
    be = f.EmuK5(K5EMU)
    msgs = []
    sizes = [1, 2, 3, 7, 8, 9, 63, 64, 65, 255, 256, 257]
    runs = [f.run_cases(be, f.tree_cases(0, sizes), betas=(2.0, math.inf), counts=f.COUNTS, log=msgs.append, max_points=40),
            f.run_cases(be, f.tie_cases(14, 3), log=msgs.append, max_points=120),
            f.run_cases(be, f.scale_cases(0, (-300, -150, -24, -6, 0, 9, 17, 150, 300)), betas=(2.0, math.inf), log=msgs.append, max_points=60),
            f.run_cases(be, f.nonfinite_cases(), betas=f.BETAS, counts=(33, 129), log=msgs.append),
            f.run_cases(be, f.atan2_cases(), betas=(2.0, math.inf), log=msgs.append)]
    assert sum(r[2] for r in runs) == 0, "\n".join(msgs[:10])
    assert sum(r[0] for r in runs) > 150 and sum(r[1] for r in runs) > 50000


def test_k5_fuzz_atan2_cases_take_every_branch():
    """the one-triangle cases reach every branch of k5_atan2, and |det/den| lands exactly one ulp below and at or one ulp above each of
    7/16, 11/16, 19/16, 39/16 with den of either sign"""
    f = _k5_fuzz()
    seen = f.atan2_coverage(f.atan2_cases())
    assert f.ATAN2_BRANCHES <= seen
    assert all(f"{t}+-ulp,{s}" in seen for t in f.ATAN2_BOUNDS for s in ("den>0", "den<0"))


def test_zero_area_case_has_a_zero_area_subtree(k5):
    f = _k5_fuzz()
    V, F, _ = f.zero_area_case(np.random.default_rng(0))
    e = EmuWinding(k5, V, F)
    assert f.has_zero_area_subtree(V, F, e.order.astype(np.int64))


def test_stack_canary_fails_a_launch_one_entry_short(k5):
    """a perfect tree (T = 2^k) is walked with exactly stack_depth deferred entries: with one entry less the walk writes past the launch's
    shared memory, which the emulation's canary turns into a failed launch; with the tree's own depth the same launch succeeds"""
    f = _k5_fuzz()
    k5.emu_winding_number_with_depth.argtypes = [VP, DP, C.c_uint64, C.c_double, C.c_int, DP]
    k5.emu_winding_stack_depth.argtypes = [VP]
    for T in (8, 64, 1024):
        V, F = f.soup(np.random.default_rng(T), T)
        e = EmuWinding(k5, V, F)
        depth = k5.emu_winding_stack_depth(e.h)
        assert depth == int(math.log2(T))
        p = wr.query_points(V, 40, seed=1)
        w = np.empty(len(p))
        assert k5.emu_winding_number_with_depth(e.h, P(p), len(p), math.inf, depth, P(w)) == 0
        assert bits_equal(w, wr.exact_w(e.leaves, p))
        assert k5.emu_winding_number_with_depth(e.h, P(p), len(p), math.inf, depth - 1, P(w)) != 0


def test_records_and_w_with_an_infinite_vertex(k5):
    """regression: with an infinite vertex a subtree's p~ is +-inf, so every |v - p~|^2 is inf or NaN; r_c is the max over the others (the
    fold from 0 skips NaN), here inf -- the restatement took np.max (NaN), then max(0.0, NaN) = 0 and made such clusters far"""
    f = _k5_fuzz()
    case = next(c for c in f.nonfinite_cases() if c[0] == "awkward 9 x1 vertex inf")
    _, V, F, x = case
    e = EmuWinding(k5, V, F)
    rec = wr.Records(V, F, e.order)
    assert bits_equal(e.clusters, rec.as_array())
    assert np.isinf(e.clusters[..., 15]).any()
    for beta in f.BETAS:
        assert f.same(e.w(x, beta), rec.w(x, beta)).all(), beta


# ---------------------------------------------------------------------------------------------------------------- accuracy of the exact sum
U = 2.0 ** -53


def exact_sum_bound(tris, p):
    """first-order bound on |w - w*| for the exact sum (beta = inf) at points p, from the operation count of the contract; w* is the sum of
    the exact solid angles of the same fp64 inputs.  Per term, with a, b, c = v - x (relative error u each) and first-order error terms:
      det = (ax kx + ay ky) + az kz:  |d det| <= 8u Pdet,  Pdet = sum of |a_i b_j c_k| over the six products of the cross and dot products
      den = ((|a||b||c| + (a.b)|c|) + (b.c)|a|) + (c.a)|b|:  |d den| <= 16u Pden,  Pden = |a||b||c| + P_ab |c| + P_bc |a| + P_ca |b|,
          P_ab = sum |a_i b_i| (|u| carries 3.5u, a.b 5u, each product u, the three additions 3u, 2u, u)
      theta = atan2(det, den):  |d theta| <= (|d det| |den| + |d den| |det|) / (det^2 + den^2) + 4u |theta|  (k5_atan2: 2 ulp)
      Omega = 2 theta exactly.
    The fold adds u |S_k| per addition (k = 2 .. T), the division by FOUR_PI (4 pi (1 + d), |d| <= u) 2u |w|.  So
      |w - w*| <= u [ sum_t 2 (kappa_t + 4 |theta_t|) + sum_k |S_k| ] / 4 pi + 2u |w|,   kappa_t = (8 Pdet |den| + 16 Pden |det|) / (det^2 + den^2)
    -> (w, bound, kappa (n, T), partial sums (n, T))"""
    v = tris[None, :, :]
    a = [v[..., i] - p[:, i:i + 1] for i in range(3)]
    b = [v[..., 3 + i] - p[:, i:i + 1] for i in range(3)]
    c = [v[..., 6 + i] - p[:, i:i + 1] for i in range(3)]
    A = lambda x: np.abs(x)
    pdet = (A(a[0]) * (A(b[1] * c[2]) + A(b[2] * c[1])) + A(a[1]) * (A(b[2] * c[0]) + A(b[0] * c[2])) + A(a[2]) * (A(b[0] * c[1]) + A(b[1] * c[0])))
    n = lambda x: np.sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2])
    la, lb, lc = n(a), n(b), n(c)
    pab = sum(A(a[i] * b[i]) for i in range(3)); pbc = sum(A(b[i] * c[i]) for i in range(3)); pca = sum(A(c[i] * a[i]) for i in range(3))
    pden = la * lb * lc + pab * lc + pbc * la + pca * lb
    det, den = wr.det_den(tris, p)
    kappa = (8.0 * pdet * np.abs(den) + 16.0 * pden * np.abs(det)) / (det * det + den * den)
    theta = wr.atan2(det, den)
    partial = np.cumsum(2.0 * theta, axis=1)
    w = wr.exact_w(tris, p)
    bound = U * ((2.0 * (kappa + 4.0 * np.abs(theta))).sum(1) + np.abs(partial[:, 1:]).sum(1)) / (4 * math.pi) + 2.0 * U * np.abs(w)
    return w, bound, kappa, partial


def exact_w_mp(tris, p, dps=40):
    """sum over the triangles of 2 atan2(det, den) / 4 pi at `dps` digits, from the same fp64 vertices and points"""
    import mpmath as mp
    mp.mp.dps = dps
    out = []
    T = [[[mp.mpf(float(t[3 * k + d])) for d in range(3)] for k in range(3)] for t in tris]
    for x in p:
        X = [mp.mpf(float(v)) for v in x]
        S = []
        for v0, v1, v2 in T:
            a = [v0[d] - X[d] for d in range(3)]; b = [v1[d] - X[d] for d in range(3)]; c = [v2[d] - X[d] for d in range(3)]
            la, lb, lc = (mp.sqrt(u[0] ** 2 + u[1] ** 2 + u[2] ** 2) for u in (a, b, c))
            det = a[0] * (b[1] * c[2] - b[2] * c[1]) + a[1] * (b[2] * c[0] - b[0] * c[2]) + a[2] * (b[0] * c[1] - b[1] * c[0])
            dot = lambda u, q: u[0] * q[0] + u[1] * q[1] + u[2] * q[2]
            den = la * lb * lc + dot(a, b) * lc + dot(b, c) * la + dot(c, a) * lb
            S.append(2 * mp.atan2(det, den))
        out.append(mp.fsum(S) / (4 * mp.pi))
    return out


ACCURACY_MESHES = [("box", 200), ("torus", 12), ("open_torus", 12), ("soup", 200), ("open_bunny_200", 60)]


@pytest.mark.parametrize("name,n_points", ACCURACY_MESHES)
def test_exact_sum_accuracy_against_mpmath(k5, orc, name, n_points):
    """the exact sum (beta = inf; the device returns these bits, see test_gpu_winding.py) against 2 atan2(det, den) / 4 pi summed at 40
    digits from the same fp64 inputs, at points at least 1e-3 of the mesh extent from the surface: within exact_sum_bound, whose
    coefficients come from the operation count, not from this data"""
    pytest.importorskip("mpmath")
    if name == "open_bunny_200":
        V, F = mesh("open_bunny_small")
        F = np.ascontiguousarray(F[:200])
    else:
        V, F = mesh(name)
    e = EmuWinding(k5, V, F)
    ext = float(np.linalg.norm(V.max(0) - V.min(0)))
    p = wr.query_points(V, 6 * n_points, seed=17, near=2 * n_points)
    d = orc.mesh(V, F).distance(p, signed=False)[0]
    p = np.ascontiguousarray(p[d >= 1e-3 * ext][:n_points])
    assert len(p) >= n_points // 2
    w, bound, _kappa, _ = exact_sum_bound(e.leaves, p)
    assert bits_equal(e.w(p, math.inf), w)
    ref = exact_w_mp(e.leaves, p)
    err = np.array([abs(float(r - wi)) for r, wi in zip(ref, w.tolist())])
    assert (err <= bound).all(), (float((err / bound).max()), float(err.max()))
    print(f"{name}: T = {len(F)}, {len(p)} points, max |w - w*| = {err.max():.3g} = {err.max() / U:.1f} u, "
          f"max bound {bound.max() / U:.0f} u, max err / bound = {(err / bound).max():.3g}")
