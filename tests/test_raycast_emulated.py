"""First crossings along rays (K7, discregrid_b200/csrc/k7_raycast.cu) on the CPU: the product's kernels and C-ABI compiled into
build/bin/libdgemu.so (tests/emu).  dg_field_raycast must equal the numpy restatement of the contract (tests/raycast_ref.py) bit for bit on
t_lo, t_hi and status, with the library's own host interpolate as the restatement's evaluator.  Also: every refusal, the thin feature that
the Bernstein test exists for, and properties that do not depend on the restatement (no side change before t_lo under dense sampling, the
sides status states, the guarantee of continuous collision detection).  The GPU runs are tests/test_gpu_raycast.py."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_oracle_golden import read_cdf
from test_isosurface_emulated import Field, dense_field, emu, grid_desc, make_field, same_bits, sphere_sdf  # noqa: F401 (emu: fixture)
import raycast_ref as rr

DBL_MAX = rr.DBL_MAX
DG_ERR_INVALID = -1
INF = float("inf")
_dp, _i32p = C.POINTER(C.c_double), C.POINTER(C.c_int32)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def cast(f, O, Dr, iso=0.0, t_min=0.0, t_max=INF):
    O = np.ascontiguousarray(O, np.float64).reshape(-1, 3)
    Dr = np.ascontiguousarray(Dr, np.float64).reshape(-1, 3)
    lo, hi, st = np.full(len(O), -1.0), np.full(len(O), -1.0), np.full(len(O), -7, np.int32)
    rc = f.emu.dg_field_raycast(f.h, _p(O, _dp), _p(Dr, _dp), len(O), iso, t_min, t_max, _p(lo, _dp), _p(hi, _dp), _p(st, _i32p))
    assert rc == 0, f.emu.dg_last_error()
    return lo, hi, st


def check(f, O, Dr, iso=0.0, t_min=0.0, t_max=INF):
    got = cast(f, O, Dr, iso, t_min, t_max)
    want = rr.raycast(rr.Grid.of_desc(f.desc), f.interpolate, O, Dr, iso, t_min, t_max)
    assert same_bits(got[0], want[0]) and same_bits(got[1], want[1]), (np.nonzero(got[0] != want[0])[0][:10], got[0][:4], want[0][:4])
    assert np.array_equal(got[2], want[2])
    return got


def domain(f):
    return np.array(f.desc.domain_min[:]), np.array(f.desc.domain_max[:]), np.array(f.desc.cell_size[:])


def random_rays(f, n, seed, pad=0.3):
    rng = np.random.default_rng(seed)
    mn, mx, _ = domain(f)
    ext = mx - mn
    O = mn - pad * ext + rng.random((n, 3)) * (1 + 2 * pad) * ext
    Dr = rng.standard_normal((n, 3))
    return O, Dr


def grid_rays(f):
    """rays along grid axes, through faces, edges and corners exactly, and origins on node planes"""
    mn, mx, cell = domain(f)
    n = np.array(f.desc.resolution[:])
    rays = []
    for a in range(3):
        for m in (0, 1, n[a] // 2, n[a]):
            p = mn + cell * np.array([1, 2, 1]) * 0.5
            p[a] = mn[a] + cell[a] * m                          # origin on a node plane
            q = mn + cell * (n // 2)                            # a grid vertex: edges and corners meet there
            e = np.zeros(3); e[a] = 1.0
            rays += [(p, e), (p, -e), (q - 2 * e * cell, e), (q, np.ones(3)), (q, cell), (q, -cell), (p, np.array([0.0, 1.0, 1.0]))]
            f2 = q.copy(); f2[(a + 1) % 3] += 0.5 * cell[(a + 1) % 3]
            rays.append((f2 - e * 3 * cell[a], e))            # along a face
    O = np.array([r[0] for r in rays]); Dr = np.array([r[1] for r in rays])
    return O, Dr


@pytest.mark.parametrize("name", ["box_cdf", "sphere", "torus", "box_band"])
def test_equals_restatement(emu, name):
    f = make_field(emu, name)
    h = float(np.linalg.norm(domain(f)[2]))
    O, Dr = random_rays(f, 160, 1)
    G, Gd = grid_rays(f)
    O, Dr = np.vstack([O, G]), np.vstack([Dr, Gd])
    st_all = []
    for iso in (0.0, 0.3 * h, -0.3 * h):
        st_all.append(check(f, O, Dr, iso)[2])
    st = np.concatenate(st_all)
    assert (st == rr.ENTER).sum() > 0 and (st == rr.MISS).sum() > 0
    # segments x0 -> x1 with t in [0, 1], and the whole line
    mn, mx, cell = domain(f)
    X0 = O
    X1 = X0 + 0.7 * cell * Dr / np.linalg.norm(Dr, axis=1)[:, None]
    check(f, X0, X1 - X0, 0.0, 0.0, 1.0)
    check(f, O, Dr, 0.0, -INF, INF)


def test_density_maps_equal_restatement(emu):
    for name in ("ref_density_bunny_12.cdm", "ref_sphere_reduced.cdm"):
        g = read_cdf(os.path.join(GOLDEN, name))
        d = grid_desc(g["mn"], g["mx"], tuple(int(r) for r in g["res"]))
        k = len(g["nodes"]) - 1
        nodes, cells, cmap = g["nodes"][k], np.ascontiguousarray(g["cells"][k]), np.ascontiguousarray(g["cmap"][k])
        h = C.c_void_p()
        assert emu.dg_field_create(C.byref(d), _p(nodes, _dp), len(nodes), cells.ctypes.data_as(C.POINTER(C.c_uint32)), len(cells),
                                   cmap.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(h)) == 0, emu.dg_last_error()
        f = Field(emu, d, h)
        ok = nodes[(nodes != DBL_MAX) & np.isfinite(nodes)]
        O, Dr = random_rays(f, 120, 2, pad=0.0)
        for iso in (float(np.median(ok)), 0.25 * float(ok.max())):
            st = check(f, O, Dr, iso)[2]
            assert (st != rr.MISS).any(), name


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_non_finite_and_huge_coefficients(emu, seed):
    rng = np.random.default_rng(seed)
    special = np.array([np.nan, np.inf, -np.inf, DBL_MAX, -DBL_MAX, 1.7e308, -1.7e308, 1e308, -1e308, 0.0, -0.0])

    def fn(x):
        v = rng.standard_normal(len(x))
        k = rng.random(len(x)) < 0.1
        v[k] = rng.choice(special, k.sum())
        return v
    f = dense_field(emu, [-1, -2, 0], [1, 1, 0.5], (5, 4, 3), fn)
    O, Dr = random_rays(f, 120, seed)
    for iso in (0.0, 0.25, -1e308, 1.6e308):
        check(f, O, Dr, iso)


def test_special_rays(emu):
    f = make_field(emu, "sphere")
    c = np.array([0.03, -0.02, 0.01])
    O = np.array([[0.1, 0.1, 0.1], [2, 0, 0], [0, 0, 0], [np.nan, 0, 0], [0, np.inf, 0], [0, 0, 0], [5, 5, 5], [-3, 0.2, 0.1],
                  c + [0, 0.6, -2.0], c + [0, 0.6, -2.0], [0, 0, 0], [1.0, -1.0, 0.3]])
    Dr = np.array([[1, 0, 0], [-1, 0, 0], [0, 0, 0], [1, 0, 0], [1, 0, 0], [0, 0, -np.inf], [1, 1, 1], [1, 0, 0],
                   [0, 0, 1], [0, 1e-3, 1], [0, 1e-300, 0], [-1.0, 1.0, 0.0]])
    lo, hi, st = check(f, O, Dr)
    assert (st[2:6] == rr.MISS).all() and (lo[2:6] == INF).all() and (hi[2:6] == INF).all()     # zero / non-finite o or d
    assert st[0] == rr.LEAVE                                   # starts inside: its first crossing leaves
    assert st[1] == rr.ENTER and st[7] == rr.ENTER
    assert st[6] == rr.MISS                                    # misses the domain
    check(f, O, Dr, 0.0, 0.0, 1.0)
    check(f, O, Dr, 0.0, -INF, 0.5)


def test_iso_hit_exactly_at_a_sample(emu):
    """iso equal to f at a depth-0 sample: the side test is strict (f < iso is negative), so the restatement and the kernel must agree"""
    f = make_field(emu, "torus")
    O, Dr = random_rays(f, 60, 4, pad=0.0)
    g = rr.Grid.of_desc(f.desc)
    hit = 0
    for k in (1, 2, 3, 4):                                 # every interior sample position, w_k = k / 5.0 (3 / 5.0 != 3 * 0.2)
        isos = []
        for i in range(len(O)):
            c = rr.clip(g, list(O[i]), list(Dr[i]), 0.0, INF)
            if c is None:
                continue
            b = rr.breakpoints(g, list(O[i]), list(Dr[i]), c[0], c[1])
            t = c[0] + (b[0] - c[0]) * rr.W[k]             # sample k of the ray's first segment
            v = float(f.interpolate(np.array([rr.position(g, list(O[i]), list(Dr[i]), t)]))[0])
            if abs(v) < 0.3:
                isos.append(v)
        for iso in isos[:10]:
            check(f, O, Dr, iso)
            hit += 1
    assert hit >= 20


def test_tangent_ray_to_a_sphere(emu):
    f = dense_field(emu, [-1, -1, -1], [1, 1, 1], (8, 8, 8), lambda x: np.linalg.norm(x, axis=1) - 0.5)
    O = np.array([[-2.0, 0.5, 0.0], [-2.0, 0.5 - 1e-9, 0.0], [-2.0, 0.45, 0.0], [-2.0, 0.51, 0.0]])
    Dr = np.tile([1.0, 0.0, 0.0], (4, 1))
    lo, hi, st = check(f, O, Dr)
    assert st[2] == rr.ENTER and st[3] == rr.MISS


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257])
def test_counts_around_warp_and_block_sizes(emu, n):
    f = make_field(emu, "sphere")
    O, Dr = random_rays(f, n, 100 + n)
    check(f, O, Dr)


def test_empty_call(emu):
    f = make_field(emu, "sphere")
    assert emu.dg_field_raycast(f.h, None, None, 0, 0.0, 0.0, INF, None, None, None) == 0
    assert emu.dg_field_raycast_device(f.h, None, None, 0, 0.0, 0.0, INF, None, None, None, None) == 0


def test_refusals(emu):
    f = make_field(emu, "sphere")
    O = np.zeros((2, 3)); Dr = np.ones((2, 3))
    lo, hi, st = np.empty(2), np.empty(2), np.empty(2, np.int32)
    args = lambda: (_p(O, _dp), _p(Dr, _dp), 2)
    outs = lambda: (_p(lo, _dp), _p(hi, _dp), _p(st, _i32p))
    for fn, tail in ((emu.dg_field_raycast, ()), (emu.dg_field_raycast_device, (None,))):
        for iso in (np.nan, np.inf, -np.inf):
            assert fn(f.h, *args(), iso, 0.0, 1.0, *outs(), *tail) == DG_ERR_INVALID
            assert b"iso" in emu.dg_last_error()
        for t0, t1 in ((np.nan, 1.0), (0.0, np.nan), (np.nan, np.nan)):
            assert fn(f.h, *args(), 0.0, t0, t1, *outs(), *tail) == DG_ERR_INVALID
            assert b"NaN" in emu.dg_last_error()
        assert fn(f.h, *args(), 0.0, 1.0, 0.5, *outs(), *tail) == DG_ERR_INVALID
        assert b"t_min > t_max" in emu.dg_last_error()
        assert fn(None, *args(), 0.0, 0.0, 1.0, *outs(), *tail) == DG_ERR_INVALID
        for k in range(5):
            ptrs = list(args()[:2]) + list(outs())
            ptrs[k] = None
            assert fn(f.h, ptrs[0], ptrs[1], 2, 0.0, 0.0, 1.0, *ptrs[2:], *tail) == DG_ERR_INVALID
            assert b"NULL" in emu.dg_last_error()
        assert fn(f.h, *args(), 0.0, -INF, INF, *outs(), *tail) == 0    # infinite t bounds are fine; so is t_min == t_max
        assert fn(f.h, *args(), 0.0, 0.5, 0.5, *outs(), *tail) == 0
    assert (st == rr.MISS).all()


# ---- the thin feature: a crossing pair strictly between two consecutive depth-0 samples, all six on one side

def thin_field(emu):
    """one cell, phi(x) = (x - 0.45)(x - 0.55)(2 - x): the cubic is reproduced exactly by the interpolant, positive at x = 0, 0.2, .., 1 and
    negative on (0.45, 0.55)"""
    return dense_field(emu, [0, 0, 0], [1, 1, 1], (1, 1, 1), lambda x: (x[:, 0] - 0.45) * (x[:, 0] - 0.55) * (2.0 - x[:, 0]))


def test_thin_feature_between_samples(emu):
    f = thin_field(emu)
    O = np.array([[-0.5, 0.5, 0.5], [-0.5, 0.25, 0.75], [1.5, 0.3, 0.6]])
    Dr = np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [-1.0, 0.0, 0.0]])
    g = rr.Grid.of_desc(f.desc)
    # the six depth-0 samples of every ray are on the non-negative side
    for i in range(len(O)):
        te, tx = rr.clip(g, list(O[i]), list(Dr[i]), 0.0, INF)
        s = [te + (tx - te) * w for w in rr.W]
        assert (f.interpolate(np.array([rr.position(g, list(O[i]), list(Dr[i]), t) for t in s])) > 0).all()
    lo, hi, st = check(f, O, Dr)
    assert (st == rr.ENTER).all()
    x = O[:, 0] + lo * Dr[:, 0]
    assert np.allclose(x, [0.45, 0.45, 0.55], atol=1e-12)
    # a marcher on the same six samples without the Bernstein test misses all three
    _, _, st6 = rr.raycast(g, f.interpolate, O, Dr, bernstein=False)
    assert (st6 == rr.MISS).all()


# ---- properties that do not depend on the restatement

def sides_and_dense_sampling(f, O, Dr, lo, hi, st, iso, per_segment):
    g = rr.Grid.of_desc(f.desc)
    checked = 0
    for i in np.nonzero(st != rr.MISS)[0]:
        o, d = list(O[i]), list(Dr[i])
        flo, fhi = f.interpolate(np.array([rr.position(g, o, d, lo[i]), rr.position(g, o, d, hi[i])]))
        assert (flo >= iso and fhi < iso) if st[i] == rr.ENTER else (flo < iso and fhi >= iso)
        te, tx = rr.clip(g, o, d, 0.0, INF)
        ends = [te] + rr.breakpoints(g, o, d, te, tx)
        ts = np.concatenate([np.linspace(a, b, per_segment) for a, b in zip(ends[:-1], ends[1:]) if a < lo[i]])
        ts = ts[ts <= lo[i]]
        v = f.interpolate(np.array([rr.position(g, o, d, t) for t in ts]))
        if not (np.isfinite(v) & (v != DBL_MAX)).all():
            continue                                        # only rays whose segments are all valid
        side = v < iso
        assert (side == side[0]).all(), i                   # no side change before t_lo
        checked += 1
    return checked


def test_sides_and_no_earlier_crossing_under_dense_sampling(emu):
    f = make_field(emu, "torus")
    O, Dr = random_rays(f, 40, 11)
    lo, hi, st = cast(f, O, Dr)
    assert sides_and_dense_sampling(f, O, Dr, lo, hi, st, 0.0, 10000) >= 5


def test_ccd_guarantee(emu):
    """segments whose ends are valid and on opposite sides, with no invalid cell between them, always report a crossing"""
    f = make_field(emu, "sphere")
    rng = np.random.default_rng(5)
    c = np.array([0.03, -0.02, 0.01])
    u = rng.standard_normal((300, 3)); u /= np.linalg.norm(u, axis=1)[:, None]
    X0 = c + u * (0.6 + rng.uniform(-0.2, 0.2, (300, 1)))
    X1 = X0 + rng.standard_normal((300, 3)) * 0.15
    X1 = np.clip(X1, -0.99, 0.99)
    lo, hi, st = cast(f, X0, X1 - X0, 0.0, 0.0, 1.0)
    g = rr.Grid.of_desc(f.desc)
    f0 = f.interpolate(X0)
    f1 = f.interpolate(np.array([rr.position(g, list(a), list(b - a), 1.0) for a, b in zip(X0, X1)]))
    opposite = (f0 < 0) != (f1 < 0)
    assert opposite.sum() > 30
    assert (st[opposite] != rr.MISS).all()
    assert sides_and_dense_sampling(f, X0, X1 - X0, lo, hi, st, 0.0, 200) > 0


def test_hit_lies_near_the_sphere(emu):
    f = dense_field(emu, [-1, -1, -1], [1, 1, 1], (16, 16, 16), sphere_sdf)
    rng = np.random.default_rng(8)
    u = rng.standard_normal((200, 3)); u /= np.linalg.norm(u, axis=1)[:, None]
    O = -1.5 * u + 0.1 * rng.standard_normal((200, 3))
    lo, hi, st = cast(f, O, u)
    assert (st == rr.ENTER).all()
    x = O + lo[:, None] * u
    err = np.abs(sphere_sdf(x))
    assert err.max() < 1e-3, err.max()
