#!/usr/bin/env python
"""Parity fuzzer for K7 (first crossings of a level set along rays, discregrid_b200/csrc/k7_raycast.cu) against the numpy restatement of
its contract (tests/raycast_ref.py): t_lo and t_hi bit for bit (any NaN equal to any NaN), status exactly, the restatement evaluating the
field through the library's own dg_interpolate_batch.
  fields   k2_fuzz.make_field grids and fields cast from k2_fuzz.queries origins (on faces, on max faces, at corners, outside, non-finite)
           along random, axis-aligned and diagonal directions; iso 0, quartiles of the field's values and values near +-DBL_MAX
  grid     rays along grid axes, through faces, edges and corners and from node planes (as tests/test_raycast_emulated.py); zero, NaN and
           inf origins and directions, subnormal directions; iso equal to a depth-0 sample's value; the thin feature only the Bernstein
           test sees (reported on every ray); tangent rays; the density maps ref_density_bunny_12.cdm and ref_sphere_reduced.cdm
  cursors  domains far from the origin (mn ~ 10^6 .. 10^12, cells ~ 10^-3 .. 1) cast from far outside, so that the entry-cell estimate
           is cells away from the exact breakpoints; one-cell axes; 1 x 1 x 512 grids along the long axis; cubic cells and diagonal rays
           through grid vertices (three axes tie); origins on node planes and t_max equal to a breakpoint
  ulps     cells a few ulps of t wide (|o| ~ 10^15 .. 10^17 with tiny d) and [t_min, t_max] a few ulps wide around a crossing: the a < m < b
           guards of the descent and the bisection
  scales   domains at 10^+-100 and 10^+-150, with scaled and unit directions, clips that overflow to +-inf (a miss by contract) and
           subnormal directions; the restatement must report crossings (a sweep of misses tests nothing)
  holes    reduced fields with scattered removed cells (a checkerboard, random keep fractions): a lane's cached block changes between
           kept and removed cells
  bounds   [0, inf), [-inf, inf), [0, 1], [-0.5, 2], t_min = t_max, t_max just below the first crossing
  counts   the first 1, 127, 128, 129, 257 rays alone give the bits of the whole call (K7_THREADS = 128)
  staging  (`dg`) 2^20 - 1, 2^20 + 1 and 2^21 + 1 rays through the host route (chunks of 2^20) equal the device route; ~3000 of them, the
           first and the last against the restatement
With `dg` every cast also runs through dg_field_raycast_device (torch tensors on the current stream; host memory on the emulated library)
and must give the bits of dg_field_raycast.

usage: tools/k7_fuzz.py [rounds=24] [seed=0] [lib=build/bin/libdgemu.so]
  rounds  k2_fuzz.make_field fields; the other families are fixed lists
  lib     build/bin/libdgemu.so (tests/emu: the whole library with its kernels compiled for the CPU) or `dg`: the product library through its
          C-ABI (dg_field_create, dg_field_raycast[_device], dg_interpolate_batch)
The functions are shared with tests/test_isosurface_raycast_fuzz_emulated.py and tests/test_gpu_isosurface_raycast_fuzz.py."""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import k2_fuzz  # noqa: E402
import k6_fuzz  # noqa: E402
import raycast_ref as rr  # noqa: E402
from oracle_api import Oracle  # noqa: E402

dp, i32p = C.POINTER(C.c_double), C.POINTER(C.c_int32)
INF = float("inf")
DBL_MAX = rr.DBL_MAX
UINT32_MAX = 0xFFFFFFFF
COUNTS = (1, 127, 128, 129, 257)                     # around K7_THREADS = 128
BOUNDS = ((0.0, INF), (-INF, INF), (0.0, 1.0), (-0.5, 2.0))
GOLDEN = os.path.join(ROOT, "tests", "golden")
same = k2_fuzz.same
_p = k6_fuzz._p


class Lib(k6_fuzz.Lib):
    """k6_fuzz.Lib with K7's two routes.  cast() runs the host and the device route and returns the host route's result; device_same
    records whether both gave the same bits"""

    def cast(self, f, O, D, iso, lo, hi):
        n = len(O)
        t0, t1, st = np.full(n, 7.0), np.full(n, 7.0), np.full(n, 7, np.int32)
        self.check(self.lib.dg_field_raycast(f[0], _p(O, dp), _p(D, dp), n, iso, lo, hi, _p(t0, dp), _p(t1, dp), _p(st, i32p)))
        dev = self.cast_device(f, O, D, iso, lo, hi)
        self.device_same = all(np.array_equal(np.asarray(x).view(np.uint8), y.view(np.uint8)) for x, y in zip(dev, (t0, t1, st)))
        return t0, t1, st

    def cast_device(self, f, O, D, iso, lo, hi):
        n = len(O)
        if self.emulated:                                              # "device" memory is host memory
            out = np.full(n, 5.0), np.full(n, 5.0), np.full(n, 5, np.int32)
            self.check(self.lib.dg_field_raycast_device(f[0], O.ctypes.data, D.ctypes.data, n, iso, lo, hi, *(a.ctypes.data for a in out), None))
            return out
        import torch
        Ot, Dt = torch.from_numpy(O).cuda(), torch.from_numpy(D).cuda()
        out = (torch.full((n,), 5.0, dtype=torch.float64, device="cuda"), torch.full((n,), 5.0, dtype=torch.float64, device="cuda"),
               torch.full((n,), 5, dtype=torch.int32, device="cuda"))
        self.check(self.lib.dg_field_raycast_device(f[0], Ot.data_ptr(), Dt.data_ptr(), n, iso, lo, hi, *(a.data_ptr() for a in out),
                                                    torch.cuda.current_stream().cuda_stream))
        return tuple(a.cpu().numpy() for a in out)


def backend(lib):
    return Lib(lib)


# ---------------------------------------------------------------------------------------------------------------- comparison
def restate(be, f, O, D, iso, lo, hi):
    return rr.raycast(rr.Grid.of_desc(f[1]), lambda x: be.interpolate(f, x), O, D, iso, lo, hi)


def compare(got, want):
    return same(got[0], want[0]) & same(got[1], want[1]) & (got[2] == want[2])


def check(be, f, O, D, iso, lo, hi, label, counts=()):
    """one cast against the restatement (and with counts, each prefix alone against the whole call) -> (rays, mismatches, first, want)"""
    O = np.ascontiguousarray(O, np.float64).reshape(-1, 3); D = np.ascontiguousarray(D, np.float64).reshape(-1, 3)
    want = restate(be, f, O, D, iso, lo, hi)
    got = be.cast(f, O, D, iso, lo, hi)
    ok = compare(got, want)
    total, bad, first = len(O), int((~ok).sum()), None
    if bad:
        i = int(np.nonzero(~ok)[0][0])
        first = (f"MISMATCH {label} iso={iso!r} on [{lo!r}, {hi!r}] ray {i} o={O[i].tolist()!r} d={D[i].tolist()!r}: t_lo {got[0][i]!r} vs "
                 f"{want[0][i]!r}, t_hi {got[1][i]!r} vs {want[1][i]!r}, status {got[2][i]} vs {want[2][i]}")
    if not be.device_same:
        bad += 1; first = first or f"MISMATCH {label} iso={iso!r}: dg_field_raycast_device differs from dg_field_raycast"
    for c in counts:
        if c <= len(O):
            pre = be.cast(f, O[:c], D[:c], iso, lo, hi)
            okc = compare(pre, tuple(a[:c] for a in got))
            total += c; bad += int((~okc).sum())
            if not okc.all() and first is None:
                first = f"MISMATCH {label} count {c}: first bad ray {int(np.nonzero(~okc)[0][0])}"
    return total, bad, first, want


def run_cases(be, cases, log=print, counts=(), hits=None):
    """cases: (label, make_field(be) -> field, O, D, isos, bounds) -> (fields, rays checked, mismatches).  hits collects (label, crossings
    the restatement reported).  O and D may be callables of the field"""
    fields = total = bad = 0
    for label, make, O, D, isos, bounds in cases:
        f = make(be)
        try:
            O1 = O(f) if callable(O) else O
            D1 = D(f) if callable(D) else D
            for iso in (isos(f) if callable(isos) else isos):
                for lo, hi in bounds:
                    n, b, msg, want = check(be, f, O1, D1, iso, lo, hi, label, counts)
                    total += n; bad += b
                    if msg: log(msg)
                    if hits is not None:
                        hits.append((label, int((want[2] != rr.MISS).sum())))
        finally:
            be.destroy(f)
        fields += 1
    return fields, total, bad


def domain(f):
    d = f[1]
    return np.array(d.domain_min[:]), np.array(d.domain_max[:]), np.array(d.cell_size[:]), np.array(d.resolution[:], np.int64)


def value_isos(be, f, rng, n=400):
    """0, the quartiles of the valid values at random points of the domain, and values near +-DBL_MAX"""
    mn, mx, _, _ = domain(f)
    v = be.interpolate(f, mn + rng.random((n, 3)) * (mx - mn))
    return k6_fuzz.isos_of(v)[:4] + [1.6e308, -1e308]


def directions(rng, n):
    """random, axis-aligned (both signs) and diagonal directions, n of them"""
    D = rng.standard_normal((n, 3))
    k = rng.integers(0, 6, n)
    ax = np.zeros((n, 3)); ax[np.arange(n), k % 3] = np.where(k < 3, 1.0, -1.0)
    diag = rng.choice([-1.0, 1.0], (n, 3))
    pick = rng.integers(0, 3, n)[:, None]
    return np.where(pick == 0, D, np.where(pick == 1, ax, diag))


# ---------------------------------------------------------------------------------------------------------------- families
def run_fields(be, rounds, seed=0, log=print, n=60):
    """k2_fuzz.make_field fields cast from k2_fuzz.queries origins (n of them and the fixed rows: corners, max faces, NaN, inf, +-0)
    -> (fields, rays checked, mismatches)"""
    rng = np.random.default_rng(seed)
    orc = Oracle()
    tmp = tempfile.mkdtemp(prefix="k7_fuzz_")
    total = bad = 0
    for k in range(rounds):
        gd, r, nodes, cells, cmap, label = k2_fuzz.make_field(orc, rng, k, tmp)
        x = k2_fuzz.queries(rng, gd, r, nodes, cells, cmap)
        fixed = x[len(x) - 13 - 3 * 192:len(x) - 3 * 192] if len(x) > 13 + 3 * 192 else x[:0]
        O = np.ascontiguousarray(np.concatenate([x[rng.integers(0, len(x), n)], fixed]))
        D = directions(rng, len(O))
        f = be.field(gd, r, nodes, cells, cmap)
        try:
            for iso in value_isos(be, f, rng):
                for lo, hi in BOUNDS[k % 4:k % 4 + 1]:
                    m, b, msg, _ = check(be, f, O, D, iso, lo, hi, label)
                    total += m; bad += b
                    if msg: log(msg)
        finally:
            be.destroy(f)
    return rounds, total, bad


# ---- the grid family, after tests/test_raycast_emulated.py
def sphere_sdf(x, c=(0.03, -0.02, 0.01), r=0.6):
    return np.linalg.norm(x - np.asarray(c), axis=1) - r


def torus_sdf(x, R=0.6, r=0.25):
    q = np.hypot(x[:, 0], x[:, 1]) - R
    return np.hypot(q, x[:, 2]) - r


def sphere(be):
    return be.dense_field([-1, -1, -1], [1, 1, 1], (9, 9, 9), sphere_sdf)


def torus(be):
    return be.dense_field([-1, -1, -0.5], [1, 1, 0.5], (12, 12, 6), torus_sdf)


def golden_field(be, name, k=None):
    from test_oracle_golden import read_cdf
    g = read_cdf(os.path.join(GOLDEN, name))
    k = len(g["nodes"]) - 1 if k is None else k
    d = be.grid_desc(g["mn"], g["mx"], tuple(int(v) for v in g["res"]))
    return be.field_desc(d, g["nodes"][k], np.ascontiguousarray(g["cells"][k]), np.ascontiguousarray(g["cmap"][k]))


def random_rays(f, n, seed, pad=0.3):
    rng = np.random.default_rng(seed)
    mn, mx, _, _ = domain(f)
    ext = mx - mn
    return mn - pad * ext + rng.random((n, 3)) * (1 + 2 * pad) * ext, rng.standard_normal((n, 3))


def grid_rays(f):
    """rays along grid axes, through faces, edges and corners exactly, and origins on node planes"""
    mn, mx, cell, n = domain(f)
    rays = []
    for a in range(3):
        for m in (0, 1, n[a] // 2, n[a]):
            p = mn + cell * np.array([1, 2, 1]) * 0.5
            p[a] = mn[a] + cell[a] * m
            q = mn + cell * (n // 2)
            e = np.zeros(3); e[a] = 1.0
            rays += [(p, e), (p, -e), (q - 2 * e * cell, e), (q, np.ones(3)), (q, cell), (q, -cell), (p, np.array([0.0, 1.0, 1.0]))]
            f2 = q.copy(); f2[(a + 1) % 3] += 0.5 * cell[(a + 1) % 3]
            rays.append((f2 - e * 3 * cell[a], e))
    return np.array([r[0] for r in rays]), np.array([r[1] for r in rays])


def with_grid_rays(n, seed):
    def rays(f):
        O, D = random_rays(f, n, seed)
        G, Gd = grid_rays(f)
        return np.vstack([O, G]), np.vstack([D, Gd])
    return rays


def diag_isos(f):
    h = float(np.linalg.norm(domain(f)[2]))
    return [0.0, 0.3 * h, -0.3 * h]


def grid_cases(n=120):
    for label, make in (("box.cdf", lambda be: golden_field(be, "box.cdf", 0)), ("sphere", sphere), ("torus", torus)):
        rays = with_grid_rays(n, 1)
        yield label + " grid rays", make, (lambda f, r=rays: r(f)[0]), (lambda f, r=rays: r(f)[1]), diag_isos, ((0.0, INF), (-INF, INF))
        yield label + " segments", make, (lambda f, r=rays: r(f)[0]), \
            (lambda f, r=rays: 0.7 * domain(f)[2] * r(f)[1] / np.linalg.norm(r(f)[1], axis=1)[:, None]), (0.0,), ((0.0, 1.0),)


SPECIAL_O = np.array([[0.1, 0.1, 0.1], [2, 0, 0], [0, 0, 0], [np.nan, 0, 0], [0, np.inf, 0], [0, 0, 0], [5, 5, 5], [-3, 0.2, 0.1],
                      [0.03, 0.58, -1.99], [0.03, 0.58, -1.99], [0, 0, 0], [1.0, -1.0, 0.3], [0.1, 0.1, 0.1], [-0.5, 0.2, 0.1],
                      [0.2, -0.0, 0.0], [-np.inf, 0, 0]])
SPECIAL_D = np.array([[1, 0, 0], [-1, 0, 0], [0, 0, 0], [1, 0, 0], [1, 0, 0], [0, 0, -np.inf], [1, 1, 1], [1, 0, 0],
                      [0, 0, 1], [0, 1e-3, 1], [0, 1e-300, 0], [-1.0, 1.0, 0.0], [5e-324, 0, 0], [1e-310, 2e-310, -1e-311],
                      [-0.0, np.nan, 1.0], [1, 0, 0]])


def run_special(be, log=print):
    """zero, NaN and inf origins or directions, subnormal directions (tests/test_raycast_emulated.py's rays and more), on the sphere"""
    f = sphere(be)
    total = bad = 0
    try:
        for lo, hi in ((0.0, INF), (0.0, 1.0), (-INF, 0.5), (-INF, INF)):
            n, b, msg, want = check(be, f, SPECIAL_O, SPECIAL_D, 0.0, lo, hi, "special rays")
            total += n; bad += b
            if msg: log(msg)
            st = want[2]
            if (lo, hi) == (0.0, INF):
                expect = (st[2:6] == rr.MISS).all() and st[0] == rr.LEAVE and st[1] == rr.ENTER and st[7] == rr.ENTER and st[6] == rr.MISS
                expect &= st[12] == rr.MISS and st[15] == rr.MISS        # 0.9 / 5e-324 overflows: t_exit = inf, a miss by contract
                if not expect:
                    bad += 1; log(f"MISMATCH special rays: statuses {st.tolist()}")
    finally:
        be.destroy(f)
    return 1, total, bad


def run_iso_at_samples(be, log=print, n=60, per_k=6):
    """iso equal to f at a depth-0 sample of a ray's first segment (w_k = k / 5.0): the strict side test"""
    f = torus(be)
    O, D = random_rays(f, n, 4, pad=0.0)
    g = rr.Grid.of_desc(f[1])
    total = bad = used = 0
    try:
        for k in (1, 2, 3, 4):
            isos = []
            for i in range(len(O)):
                c = rr.clip(g, list(O[i]), list(D[i]), 0.0, INF)
                if c is None:
                    continue
                b = rr.breakpoints(g, list(O[i]), list(D[i]), c[0], c[1])
                t = c[0] + (b[0] - c[0]) * rr.W[k]
                v = float(be.interpolate(f, np.array([rr.position(g, list(O[i]), list(D[i]), t)]))[0])
                if abs(v) < 0.3:
                    isos.append(v)
            for iso in isos[:per_k]:
                m, b, msg, _ = check(be, f, O, D, iso, 0.0, INF, f"iso at sample {k}")
                total += m; bad += b; used += 1
                if msg: log(msg)
    finally:
        be.destroy(f)
    return used, total, bad


def thin_field(be):
    """one cell, phi(x) = (x - 0.45)(x - 0.55)(2 - x): positive at the six depth-0 samples of an x ray, negative on (0.45, 0.55)"""
    return be.dense_field([0, 0, 0], [1, 1, 1], (1, 1, 1), lambda x: (x[:, 0] - 0.45) * (x[:, 0] - 0.55) * (2.0 - x[:, 0]))


def run_thin_and_tangent(be, log=print):
    """the thin feature (every ray reports ENTER at x = 0.45 or 0.55) and rays tangent to a sphere"""
    total = bad = 0
    f = thin_field(be)
    try:
        O = np.array([[-0.5, 0.5, 0.5], [-0.5, 0.25, 0.75], [1.5, 0.3, 0.6], [-0.5, 0.0, 1.0], [1.5, 1.0, 0.0]])
        D = np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [-1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [-1.0, 0.0, 0.0]])
        n, b, msg, want = check(be, f, O, D, 0.0, 0.0, INF, "thin feature")
        got = be.cast(f, O, D, 0.0, 0.0, INF)
        x = O[:, 0] + got[0] * D[:, 0]
        if not ((got[2] == rr.ENTER).all() and np.allclose(x, [0.45, 0.45, 0.55, 0.45, 0.55], atol=1e-12)):
            b += 1; msg = msg or f"MISMATCH thin feature not reported: status {got[2].tolist()}, x {x.tolist()}"
        total += n; bad += b
        if msg: log(msg)
    finally:
        be.destroy(f)
    f = be.dense_field([-1, -1, -1], [1, 1, 1], (8, 8, 8), lambda x: np.linalg.norm(x, axis=1) - 0.5)
    try:
        O = np.array([[-2.0, 0.5, 0.0], [-2.0, 0.5 - 1e-9, 0.0], [-2.0, 0.45, 0.0], [-2.0, 0.51, 0.0], [0.0, -2.0, 0.5],
                      [-2.0, 0.0, 0.5 + 1e-12]])
        D = np.array([[1.0, 0.0, 0.0]] * 4 + [[0.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
        n, b, msg, want = check(be, f, O, D, 0.0, 0.0, INF, "tangent rays")
        if not (want[2][2] == rr.ENTER and want[2][3] == rr.MISS):
            b += 1; msg = msg or f"MISMATCH tangent rays: statuses {want[2].tolist()}"
        total += n; bad += b
        if msg: log(msg)
    finally:
        be.destroy(f)
    return 2, total, bad


def density_cases(n=100):
    for name in ("ref_density_bunny_12.cdm", "ref_sphere_reduced.cdm"):
        def isos(f, name=name):
            from test_oracle_golden import read_cdf
            g = read_cdf(os.path.join(GOLDEN, name))
            v = g["nodes"][-1]
            ok = v[(v != DBL_MAX) & np.isfinite(v)]
            return [float(np.median(ok)), 0.25 * float(ok.max())]
        yield name, (lambda be, name=name: golden_field(be, name)), (lambda f: random_rays(f, n, 2, 0.0)[0]), \
            (lambda f: random_rays(f, n, 2, 0.0)[1]), isos, ((0.0, INF),)


# ---- cursors
def offset_field(mn, cell, res):
    mn = np.asarray(mn, np.float64)
    mx = mn + np.asarray(cell, np.float64) * np.asarray(res, np.float64)
    c = 0.5 * (mn + mx) + 0.1 * (mx - mn)
    return lambda be: be.dense_field(mn, mx, res, lambda x: np.linalg.norm((x - c) / (mx - mn), axis=1) - 0.3)


def far_rays(f, rng, k, n=24):
    """origins R = k * 2^52 cells away (the entry estimate is then ~k cells off), along axes and diagonals, aimed through the domain"""
    mn, mx, cell, _ = domain(f)
    c = 0.5 * (mn + mx)
    R = k * float(cell.max()) * 2.0 ** 52
    O, D = [], []
    for i in range(n):
        a = i % 3
        u = np.zeros(3); u[a] = 1.0 if i % 2 else -1.0
        if i % 4 == 3:
            u = rng.choice([-1.0, 1.0], 3) * (1.0 + 0.1 * rng.random(3))
            u /= np.linalg.norm(u)
        target = mn + (0.2 + 0.6 * rng.random(3)) * (mx - mn)
        O.append(target - R * u); D.append(u)
    return np.array(O), np.array(D)


def cursor_cases(seed=0):
    rng = np.random.default_rng(seed + 5)
    for off, cell in ((1e6, 1e-3), (-3e7, 1e-2), (1e9, 0.25), (-1e12, 1.0), (1e12, 1e-3)):
        mn = off * np.array([1.0, -0.5, 0.25])
        make = offset_field(mn, [cell, 1.3 * cell, 0.7 * cell], (10, 8, 12))
        for k in (1.0 / 64, 1.0, 4.0):
            yield (f"offset {off:g} cell {cell:g}, origins {k:g} * 2^52 cells away", make,
                   (lambda f, k=k, s=int(rng.integers(1 << 30)): far_rays(f, np.random.default_rng(s), k)[0]),
                   (lambda f, k=k, s=int(rng.integers(1 << 30)): far_rays(f, np.random.default_rng(s), k)[1]), (0.0,), ((-INF, INF),))
    for res in ((1, 5, 4), (6, 1, 1), (1, 1, 1), (1, 1, 7), (4, 1, 3)):
        make = lambda be, res=res: be.dense_field([-1, -0.8, -0.6], [1, 0.8, 0.6], res, sphere_sdf)
        yield f"one-cell axes {res}", make, (lambda f: with_grid_rays(60, 6)(f)[0]), (lambda f: with_grid_rays(60, 6)(f)[1]), \
            (0.0, -0.2), ((0.0, INF), (-INF, INF))
    for top in (0.97, 1.5):                                        # a crossing near the far end; none: every breakpoint visited
        make = lambda be, top=top: be.dense_field([0, 0, 0], [1, 1, 64], (1, 1, 512), lambda x: x[:, 2] / 64.0 - top + 0.05 * np.sin(x[:, 0]))
        O = np.array([[0.3, 0.6, -1.0], [0.5, 0.5, 65.0], [0.0, 0.0, -3.0], [1.0, 1.0, 70.0], [0.25, 0.75, 0.0], [0.4, 0.4, 64.0]])
        D = np.array([[0, 0, 1.0], [0, 0, -1.0], [1e-3, 1e-3, 1.0], [-1e-3, -1e-3, -1.0], [0, 0, 0.125], [0, 0, -7.0]])
        yield f"1 x 1 x 512, level at {top} of the length", make, O, D, (0.0,), ((0.0, INF), (-INF, INF))
    make = lambda be: be.dense_field([-1, -1, -1], [1, 1, 1], (6, 6, 6), lambda x: sphere_sdf(x, r=0.5))
    O, D = [], []
    for v in ((2, 2, 2), (1, 3, 2), (3, 3, 3), (0, 0, 0), (6, 6, 6)):
        p = -1.0 + np.array(v) * (2.0 / 6.0)
        for d in ((1, 1, 1), (-1, 1, 1), (1, -1, -1), (-1, -1, -1), (1, 1, 0.37), (1, 0, 1), (0.5, 0.5, 0.5)):
            d = np.array(d, np.float64)
            for back in (0.0, 1.75, 1.0 / 3.0):
                O.append(p - back * d); D.append(d)
    yield "cubic cells, diagonals through grid vertices", make, np.array(O), np.array(D), (0.0, 0.1), ((0.0, INF), (-INF, INF))


def run_plane_bounds(be, log=print):
    """origins on node planes; t_max and t_min equal to a breakpoint shared by every ray of the call"""
    f = torus(be)
    total = bad = 0
    try:
        mn, mx, cell, n = domain(f)
        rng = np.random.default_rng(9)
        for a in range(3):
            m = 2
            O = mn + rng.random((40, 3)) * (mx - mn)
            O[:, a] = mn[a] + cell[a] * (np.arange(40) % (n[a] + 1))            # on node planes
            D = rng.standard_normal((40, 3))
            for lo, hi in ((0.0, INF), (-INF, INF)):
                k, b, msg, _ = check(be, f, O, D, 0.0, lo, hi, f"origins on node planes, axis {a}")
                total += k; bad += b
                if msg: log(msg)
            O2 = O.copy(); O2[:, a] = mn[a] - 0.5 * cell[a]
            D2 = D.copy(); D2[:, a] = 1.0
            t_b = float((mn[a] + float(m) * cell[a]) - O2[0, a])             # t_{a,m} for every ray (d_a = 1)
            for lo, hi in ((0.0, t_b), (t_b, INF), (t_b, t_b), (-INF, t_b)):
                k, b, msg, _ = check(be, f, O2, D2, 0.0, lo, hi, f"a breakpoint as a bound, axis {a}")
                total += k; bad += b
                if msg: log(msg)
    finally:
        be.destroy(f)
    return 1, total, bad


# ---- ulps
def ulp_cases():
    """cells a few ulps of t wide: origins R = 3e13 .. 1e15 away (0.22-wide cells span ~30 .. 1 ulps of t), |d| from 1 to 1e-6"""
    rng = np.random.default_rng(21)
    u = rng.standard_normal((16, 3)); u /= np.linalg.norm(u, axis=1)[:, None]
    c = np.array([0.03, -0.02, 0.01]) + 0.2 * rng.standard_normal((16, 3))
    for R in (3e13, 1e14, 3e14, 1e15):
        for scale in (1.0, 1e-6):
            yield f"origins {R:g} away, |d| = {scale:g}", sphere, c - R * u, u * scale, (0.0, 0.05), ((0.0, INF),)


def run_ulp_bounds(be, log=print, n=40):
    """[t_min, t_max] k ulps on either side of a crossing's t_lo (k = 1, 2, 4), and exactly [t_lo, t_hi]"""
    f = sphere(be)
    total = bad = 0
    try:
        O, D = random_rays(f, n, 23)
        lo, hi, st = be.cast(f, np.ascontiguousarray(O), np.ascontiguousarray(D), 0.0, 0.0, INF)
        for i in np.flatnonzero(st != rr.MISS)[:10]:
            for k in (1, 2, 4):
                a = b_ = lo[i]
                for _ in range(k):
                    a, b_ = np.nextafter(a, -INF), np.nextafter(b_, INF)
                for t0, t1 in ((float(a), float(b_)), (float(lo[i]), float(hi[i])), (float(a), float(lo[i]))):
                    m, b, msg, _ = check(be, f, O[i:i + 1], D[i:i + 1], 0.0, t0, t1, f"ray {i} {k} ulps around t_lo")
                    total += m; bad += b
                    if msg: log(msg)
    finally:
        be.destroy(f)
    return 1, total, bad


# ---- scales
SCALES = (-150, -100, 100, 150)


def dry(hits):
    """labels of the scale cases where the restatement reported no crossing although the clip does not overflow"""
    return sorted({label for label, h in hits if h == 0 and "overflow" not in label})


def scale_cases(exponents=SCALES, n=40):
    """(label, ...) of a sphere on [-1, 1]^3 * 10^k (and offset by 3 * 10^k); directions scaled, unit, and so small that the clip overflows
    (labels with "overflow": misses by contract) or subnormal"""
    rng = np.random.default_rng(31)
    O0 = -1.3 + rng.random((n, 3)) * 2.6
    D0 = rng.standard_normal((n, 3))
    for k in exponents:
        s = 10.0 ** k
        for off in (0.0, 3.0):
            make = lambda be, s=s, off=off: be.dense_field(np.full(3, (off - 1.0) * s), np.full(3, (off + 1.0) * s), (6, 7, 5),
                                                           lambda x, s=s, off=off: sphere_sdf(x / s - off))
            O = (O0 + off) * s
            for dl, D in (("scaled", D0 * s), ("unit", D0 / np.linalg.norm(D0, axis=1)[:, None]),
                          ("subnormal" + (" overflow" if k > 0 else ""), D0 / np.abs(D0).max(1)[:, None] * 1e-310)):
                yield f"sphere@1e{k} off {off:g} {dl} d", make, O, D, (0.0, 0.1), ((0.0, INF), (-INF, INF))
            if k < 0:
                continue
            tiny = 10.0 ** (k - 309)                                  # (mn - o) / d > DBL_MAX
            yield f"sphere@1e{k} off {off:g} overflow", make, O, D0 / np.abs(D0).max(1)[:, None] * tiny, (0.0,), ((0.0, INF),)


# ---- reduced fields with scattered holes
def hole_cases(seed=0):
    rng = np.random.default_rng(seed + 41)
    orc = Oracle()
    for res in ((8, 7, 6), (5, 9, 4)):
        gd, r = orc.grid_desc(np.array([-1.0, -0.9, -0.8]), np.array([1.0, 0.9, 0.8]), res)
        cells = orc.build_cells(r)
        n = np.asarray(res)
        idx = np.arange(len(cells))
        ijk = np.stack([idx % n[0], (idx // n[0]) % n[1], idx // (n[0] * n[1])], 1)
        for kind in ("checkerboard", 0.3, 0.7, 0.9):
            kept = ((ijk.sum(1) % 2) == 0) if kind == "checkerboard" else (rng.random(len(cells)) < kind)
            k = np.nonzero(kept)[0]
            cmap = np.full(len(cells), UINT32_MAX, np.uint32); cmap[k] = np.arange(len(k), dtype=np.uint32)
            used = np.unique(cells[k])
            ncells = np.searchsorted(used, cells[k]).astype(np.uint32)

            def make(be, gd=gd, r=r, used=used, ncells=ncells, cmap=cmap):
                d = be.grid_desc(gd[0:3], gd[3:6], r, gd[6:9], gd[9:12])
                m = C.c_uint64()
                be.check(be.lib.dg_grid_num_nodes(d.resolution, C.byref(m)))
                x = np.empty((m.value, 3))
                be.check(be.lib.dg_node_positions(C.byref(d), 0, m.value, _p(x, dp)))
                return be.field(gd, r, sphere_sdf(x[used]) + 0.05 * np.sin(7 * x[used, 0]), ncells, cmap)
            s = int(rng.integers(1 << 30))
            yield f"holes {kind} {res}", make, (lambda f, s=s: random_rays(f, 80, s, 0.1)[0]), (lambda f, s=s: random_rays(f, 80, s, 0.1)[1]), \
                (0.0, 0.15, -0.1), ((0.0, INF), (-INF, INF))


# ---- bounds and counts
def bound_cases(n=80):
    for label, make in (("sphere", sphere), ("torus", torus)):
        yield label, make, (lambda f: random_rays(f, n, 51)[0]), (lambda f: random_rays(f, n, 51)[1]), (0.0, 0.1), BOUNDS


def run_exact_bounds(be, log=print, n=40):
    """t_min = t_max (inside the domain, at a crossing), and t_max just below the first crossing of every ray"""
    total = bad = 0
    for label, make in (("sphere", sphere), ("torus", torus)):
        f = make(be)
        try:
            O, D = random_rays(f, n, 53)
            lo, _, st = be.cast(f, np.ascontiguousarray(O), np.ascontiguousarray(D), 0.0, 0.0, INF)
            hit = st != rr.MISS
            first = float(lo[hit].min())
            for t0, t1 in ((0.5, 0.5), (first, first), (0.0, float(np.nextafter(first, -INF))), (-INF, float(np.nextafter(first, -INF)))):
                k, b, msg, want = check(be, f, O, D, 0.0, t0, t1, f"{label} exact bounds")
                if t0 == 0.0 and (want[2] != rr.MISS).any():
                    b += 1; msg = msg or f"MISMATCH {label}: a crossing below t_max = {t1!r}"
                total += k; bad += b
                if msg: log(msg)
        finally:
            be.destroy(f)
    return 2, total, bad


def run_counts(be, log=print):
    return run_cases(be, [("torus prefixes", torus, (lambda f: random_rays(f, 300, 55)[0]), (lambda f: random_rays(f, 300, 55)[1]), (0.0,),
                           ((0.0, INF), (-0.5, 2.0)))], log=log, counts=COUNTS)


# ---- host staging
def run_staging(be, n, log=print, sample=3000, seed=0):
    """n rays through the host route (chunks of 2^20) against the device route, and a sample, the first and the last ray against the
    restatement -> (rays checked against the restatement, mismatches)"""
    f = torus(be)
    try:
        rng = np.random.default_rng(seed + 61)
        mn, mx, _, _ = domain(f)
        O = np.ascontiguousarray(mn - 0.3 * (mx - mn) + rng.random((n, 3)) * 1.6 * (mx - mn))
        D = np.ascontiguousarray(rng.standard_normal((n, 3)))
        got = be.cast(f, O, D, 0.05, 0.0, INF)
        bad = int(not be.device_same)
        if bad:
            log(f"MISMATCH {n} rays: the host route differs from the device route")
        idx = np.unique(np.concatenate([[0, n - 1], np.arange(1 << 20, n, 1 << 20), np.arange((1 << 20) - 1, n, 1 << 20),
                                        rng.choice(n, sample, replace=False)]))
        want = restate(be, f, O[idx], D[idx], 0.05, 0.0, INF)
        ok = compare(tuple(a[idx] for a in got), want)
        bad += int((~ok).sum())
        if not ok.all():
            log(f"MISMATCH {n} rays: ray {int(idx[np.nonzero(~ok)[0][0]])} differs from the restatement")
        return len(idx), bad, int((want[2] != rr.MISS).sum())
    finally:
        be.destroy(f)


def run(be, rounds, seed=0, log=print, staging=False):
    """every family through backend `be` -> (fields, rays checked, mismatches)"""
    acc = [0, 0, 0]
    for r in (run_fields(be, rounds, seed, log), run_cases(be, grid_cases(), log), run_special(be, log), run_iso_at_samples(be, log),
              run_thin_and_tangent(be, log), run_cases(be, density_cases(), log), run_cases(be, cursor_cases(seed), log),
              run_plane_bounds(be, log), run_cases(be, ulp_cases(), log), run_ulp_bounds(be, log), run_cases(be, scale_cases(), log),
              run_cases(be, hole_cases(seed), log), run_cases(be, bound_cases(), log), run_exact_bounds(be, log), run_counts(be, log)):
        for i in range(3):
            acc[i] += r[i]
    if staging:
        for n in ((1 << 20) - 1, (1 << 20) + 1, (1 << 21) + 1):
            k, b, _ = run_staging(be, n, log)
            acc[0] += 1; acc[1] += k; acc[2] += b
    return tuple(acc)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 24
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else os.path.join(ROOT, "build", "bin", "libdgemu.so")
    fields, total, bad = run(backend(lib), rounds, seed, staging=lib == "dg")
    print(f"{fields} fields, {total} rays, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
