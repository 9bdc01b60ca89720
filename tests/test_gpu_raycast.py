"""First crossings along rays on the device (K7, discregrid_b200/csrc/k7_raycast.cu): CubicLagrangeDiscreteGrid.raycast against the numpy
restatement of the contract (tests/raycast_ref.py) bit for bit, with the device's own interpolate as the restatement's evaluator; the host
route against the CUDA-tensor route (also from a side stream); dense == reduced band; 10 M rays in one call; the C++ facade; and properties
that do not depend on the restatement: the sides status states, no side change before t_lo under dense sampling, the guarantee of continuous
collision detection, and how close the hits lie to the surface of a sphere and of the bunny."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from test_gpu_isosurface import analytic, diag, field, same_bits, sdf_grid, sphere_sdf
import raycast_ref as rr

pytestmark = pytest.mark.gpu

RAYCAST_CHECK = os.path.join(ROOT, "build", "bin", "raycast_check")
INF = float("inf")


def rays(g, n, seed, pad=0.3):
    rng = np.random.default_rng(seed)
    mn, mx = g.domain()
    ext = mx - mn
    return mn - pad * ext + rng.random((n, 3)) * (1 + 2 * pad) * ext, rng.standard_normal((n, 3))


def axis_rays(g):
    """rays along the grid axes, through grid vertices (edges and corners) and along node planes"""
    mn, _ = g.domain()
    cell = g.cellSize()
    n = np.array(g.resolution(), np.int64)
    O, D = [], []
    for a in range(3):
        e = np.zeros(3); e[a] = 1.0
        for m in (1, n[a] // 2):
            q = mn + cell * (n // 2)
            p = q.copy(); p[a] = mn[a] + cell[a] * m
            O += [q - 2 * e * cell, p, q, q]; D += [e, -e, np.ones(3), cell]
    return np.array(O), np.array(D)


def check(g, O, D, iso=0.0, t_min=0.0, t_max=INF, field_id=0):
    got = g.raycast(field_id, O, D, iso, t_min, t_max)
    want = rr.raycast(rr.Grid.of_grid(g), lambda x: g.interpolate(field_id, x), O, D, iso, t_min, t_max)
    assert same_bits(got[0], want[0]) and same_bits(got[1], want[1]) and np.array_equal(got[2], want[2]), \
        np.nonzero((got[0] != want[0]) | (got[2] != want[2]))[0][:10]
    return got


@pytest.mark.parametrize("name", ["box_cdf", "sphere", "torus", "torus_band"])
def test_equals_restatement(dg, name):
    g = field(dg, name)
    h = diag(g)
    O, D = rays(g, 300, 1)
    A, Ad = axis_rays(g)
    O, D = np.vstack([O, A]), np.vstack([D, Ad])
    st = np.concatenate([check(g, O, D, iso)[2] for iso in (0.0, 0.3 * h, -0.3 * h)])
    assert (st == rr.ENTER).any() and (st == rr.MISS).any()
    X1 = O + 0.7 * g.cellSize() * D / np.linalg.norm(D, axis=1)[:, None]
    check(g, O, X1 - O, 0.0, 0.0, 1.0)
    check(g, O, D, 0.0, -INF, INF)


@pytest.mark.parametrize("res", [128, 256])
def test_bunny_equals_restatement(dg, res):
    g = sdf_grid(dg, "bunny", (res, res, res))[0]
    O, D = rays(g, 400, 2, pad=0.1)
    lo, hi, st = check(g, O, D)
    assert (st == rr.ENTER).sum() > 50
    _, _, _, stats = rr.raycast(rr.Grid.of_grid(g), lambda x: g.interpolate(0, x), O[:100], D[:100], with_stats=True)
    print(f"bunny {res}^3: per ray mean segments {stats['segments'].mean():.1f}, nodes {stats['nodes'].mean():.1f}, "
          f"evaluations {stats['evaluations'].mean():.1f}")


def test_special_fields_equal_restatement(dg):
    g = dg.CubicLagrangeDiscreteGrid(np.array([-1.0, -2.0, 0.0]), np.array([1.0, 1.0, 0.5]), (5, 4, 3))
    rng = np.random.default_rng(3)
    n = g.nNodes()
    v = rng.standard_normal(n)
    k = rng.random(n) < 0.1
    v[k] = rng.choice(np.array([np.nan, np.inf, -np.inf, rr.DBL_MAX, -rr.DBL_MAX, 1.7e308, -1.7e308, 1e308, -1e308, 0.0, -0.0]), k.sum())
    g.addSampledFunction(v)
    O, D = rays(g, 300, 4)
    for iso in (0.0, 0.25, -1e308, 1.6e308):
        check(g, O, D, iso)
    with pytest.raises(dg._capi.DiscregridError):
        g.raycast(0, O, D, float("nan"))
    with pytest.raises(dg._capi.DiscregridError):
        g.raycast(0, O, D, 0.0, 1.0, 0.0)


def test_tensor_route_same_bits_including_a_side_stream(dg):
    import torch
    g = field(dg, "torus_band")
    O, D = rays(g, 5000, 5)
    want = g.raycast(0, O, D, 0.1)
    Ot, Dt = torch.tensor(O, device="cuda"), torch.tensor(D, device="cuda")
    got = g.raycast(0, Ot, Dt, 0.1)
    assert got[0].is_cuda and got[2].dtype == torch.int32
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        O2 = Ot * 1.0                                                # made on the side stream: the cast must see it
        side = g.raycast(0, O2, Dt, 0.1)
    s.synchronize()
    for r in (got, side):
        assert same_bits(r[0].cpu().numpy(), want[0]) and same_bits(r[1].cpu().numpy(), want[1])
        assert np.array_equal(r[2].cpu().numpy(), want[2])
    with pytest.raises(TypeError):
        g.raycast(0, Ot.float(), Dt)


@pytest.mark.parametrize("name,res", [("torus", (32, 32, 16)), ("bunny", (64, 64, 64))])
def test_dense_equals_reduced_band(dg, name, res):
    g, md, V, F = sdf_grid(dg, name, res)
    g.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, 3.0 * diag(g)))
    O, D = rays(g, 20000, 6)
    a, b = g.raycast(0, O, D), g.raycast(1, O, D)
    assert same_bits(a[0], b[0]) and same_bits(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert (a[2] == rr.ENTER).sum() > 1000


def test_large_ten_million_rays(dg):
    import torch
    g = analytic(dg, (64, 64, 64), sphere_sdf)
    n = 10_000_000
    gen = torch.Generator(device="cuda").manual_seed(0)
    O = torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=gen) * 2.4 - 1.2
    D = torch.randn((n, 3), dtype=torch.float64, device="cuda", generator=gen)
    lo, hi, st = g.raycast(0, O, D)
    sample = torch.randint(0, n, (2000,), device="cuda", generator=gen)
    want = g.raycast(0, O[sample].cpu().numpy(), D[sample].cpu().numpy())
    assert same_bits(lo[sample].cpu().numpy(), want[0]) and np.array_equal(st[sample].cpu().numpy(), want[2])
    hit = st == rr.ENTER
    x = O[hit] + lo[hit, None] * D[hit]
    err = (torch.linalg.norm(x - torch.tensor([0.03, -0.02, 0.01], dtype=torch.float64, device="cuda"), dim=1) - 0.6).abs().max().item()
    print(f"10 M rays: {int(hit.sum())} enter, {int((st == rr.LEAVE).sum())} leave; max |sdf(x(t_lo))| = {err:.3e}")
    assert err < 1e-4


def test_facade_equals_python(dg, tmp_path):
    g = field(dg, "torus")
    cdf = tmp_path / "torus.cdf"
    g.save(str(cdf))
    O, D = rays(g, 3000, 7)
    np.hstack([O, D]).tofile(tmp_path / "rays.f64")
    for iso, t0, t1 in ((0.0, 0.0, INF), (0.05, -1.0, 2.0)):
        out = tmp_path / "out.bin"
        subprocess.run([RAYCAST_CHECK, str(cdf), "0", str(tmp_path / "rays.f64"), repr(iso), repr(t0), repr(t1), str(out)], check=True,
                       capture_output=True)
        raw = out.read_bytes()
        t = np.frombuffer(raw[:16 * len(O)], np.float64)
        st = np.frombuffer(raw[16 * len(O):], np.int32)
        lo, hi, s = g.raycast(0, O, D, iso, t0, t1)
        assert same_bits(t[:len(O)], lo) and same_bits(t[len(O):], hi) and np.array_equal(st, s)


# ---- properties that do not depend on the restatement

def sides_and_dense_sampling(g, O, D, lo, hi, st, per_segment, n_rays):
    G = rr.Grid.of_grid(g)
    checked = 0
    for i in np.nonzero(st != rr.MISS)[0][:n_rays]:
        o, d = list(O[i]), list(D[i])
        flo, fhi = g.interpolate(0, np.array([rr.position(G, o, d, lo[i]), rr.position(G, o, d, hi[i])]))
        assert (flo >= 0 and fhi < 0) if st[i] == rr.ENTER else (flo < 0 and fhi >= 0)
        te, tx = rr.clip(G, o, d, 0.0, INF)
        ends = [te] + rr.breakpoints(G, o, d, te, tx)
        ts = np.concatenate([np.linspace(a, b, per_segment) for a, b in zip(ends[:-1], ends[1:]) if a < lo[i]])
        ts = ts[ts <= lo[i]]
        x = o + ts[:, None] * np.asarray(d)
        x = np.clip(x, *g.domain())
        v = g.interpolate(0, x)
        if not (np.isfinite(v) & (v != rr.DBL_MAX)).all():
            continue
        assert ((v < 0) == (v[0] < 0)).all(), i
        checked += 1
    return checked


@pytest.mark.parametrize("name", ["sphere64", "torus", "bunny64"])
def test_sides_and_no_earlier_crossing_under_dense_sampling(dg, name):
    g = analytic(dg, (64, 64, 64), sphere_sdf) if name == "sphere64" else (field(dg, name) if name == "torus" else sdf_grid(dg, "bunny", (64,) * 3)[0])
    O, D = rays(g, 400, 9)
    lo, hi, st = g.raycast(0, O, D)
    assert sides_and_dense_sampling(g, O, D, lo, hi, st, 10000, 40) >= 10


@pytest.mark.parametrize("name", ["sphere64", "bunny64"])
def test_ccd_guarantee(dg, name):
    g = analytic(dg, (64, 64, 64), sphere_sdf) if name == "sphere64" else sdf_grid(dg, "bunny", (64,) * 3)[0]
    rng = np.random.default_rng(10)
    mn, mx = g.domain()
    X0 = mn + rng.random((200000, 3)) * (mx - mn)
    phi0 = g.interpolate(0, X0)
    X0 = X0[np.abs(phi0) < 2 * diag(g)][:50000]
    X1 = np.clip(X0 + rng.standard_normal(X0.shape) * 0.5 * diag(g), mn, mx)
    lo, hi, st = g.raycast(0, X0, X1 - X0, 0.0, 0.0, 1.0)
    f0 = g.interpolate(0, X0)
    f1 = g.interpolate(0, np.clip(X0 + 1.0 * (X1 - X0), mn, mx))
    opposite = (f0 < 0) != (f1 < 0)
    assert opposite.sum() > 1000
    assert (st[opposite] != rr.MISS).all()
    print(f"{name}: {int(opposite.sum())} of {len(X0)} half-cell steps change sides; every one reports a crossing")


def test_hits_lie_near_the_surface(dg):
    g = analytic(dg, (64, 64, 64), sphere_sdf)
    rng = np.random.default_rng(11)
    u = rng.standard_normal((20000, 3)); u /= np.linalg.norm(u, axis=1)[:, None]
    O = np.array([0.03, -0.02, 0.01]) - 1.5 * u + 0.2 * rng.standard_normal((20000, 3))
    lo, hi, st = g.raycast(0, O, u)
    hit = st == rr.ENTER
    err = float(np.abs(sphere_sdf(O[hit] + lo[hit, None] * u[hit])).max())
    print(f"sphere 64^3: {int(hit.sum())} hits, max |sdf(x(t_lo))| = {err:.3e} ({err / diag(g):.2e} cell diagonals)")
    assert hit.sum() > 15000 and err < 1e-3 * diag(g)


def test_bunny_hits_lie_near_the_mesh(dg):
    g, md, V, F = sdf_grid(dg, "bunny", (64, 64, 64))
    O, D = rays(g, 20000, 12, pad=0.1)
    lo, hi, st = g.raycast(0, O, D)
    hit = st == rr.ENTER
    x = O[hit] + lo[hit, None] * D[hit]
    err = float(np.abs(md.signed_distance(x).distance).max())
    print(f"bunny 64^3: {int(hit.sum())} hits, max |mesh distance(x(t_lo))| = {err:.3e} ({err / diag(g):.4f} cell diagonals)")
    assert hit.sum() > 2000 and err < 0.5 * diag(g)
