#!/usr/bin/env python
"""Parity fuzzer for K12 (the ray-cast VJPs, discregrid_b200/csrc/k12_raycast_grad.cu) against the numpy restatement of its contract
(tests/raycast_grad_ref.py; the vertex sums are K10's, the node sums K11's restatement), bit for bit, any NaN equal to any NaN; an invalid
ray's gradients and an untouched vertex or node must be +0.0 exactly (the comparison is on the bits).  Every output combination is asked for.
  mesh     the forward outputs of k9_fuzz's tie, slack, scale, cull, nonfinite and bound cases, cast by the library, with upstreams t, bary,
           both and special values; refits, with the VJP taken at the positions cast against after the mesh was refit elsewhere;
           synthetic outputs (the VJP reads nothing else): triangle ids and t chosen freely, degenerate triangles, directions in a triangle's
           plane (den = 0), subnormal directions, meshes scaled by 10^+-77 .. 10^+-160 so that n . n is inf or 0, n = 1, 127, 128, 129, 257
  field    the forward outputs of k7_fuzz's fields, special rays, thin feature, tangent rays, grid, density, cursor (far-offset), ulp,
           scale, hole and bound cases and the iso-at-sample rays on trainable copies of their fields (dense fields through the
           closed-form table), iso != 0 among them, with grad_nodes; synthetic outputs: crossing points outside the domain (clamped), on a
           max face, in a removed cell, in a DBL_MAX cell, NaN; statuses ENTER, LEAVE and values outside the enum; and a crossing where phi
           is exactly DBL_MAX although no coefficient is (only the DBL_MAX test makes that ray invalid)
With `dg` every VJP runs twice through the host form and once through the _device form on a side stream: all must give the same bits.  On
libdgemu.so the device form takes host memory.

usage: tools/k12_fuzz.py [rounds=8] [seed=0] [lib=emu]
The functions are shared with tests/test_vjp_fuzz_emulated.py and tests/test_gpu_vjp_fuzz.py."""
import ctypes as C
import itertools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import k7_fuzz  # noqa: E402
import k9_fuzz  # noqa: E402
import k10_fuzz  # noqa: E402
import k11_fuzz  # noqa: E402
import raycast_grad_ref as ref  # noqa: E402
import interpolate_vjp_ref  # noqa: E402

dp, u32p, i32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
_p = k11_fuzz._p
same = k11_fuzz.same
_bits = k11_fuzz._bits
INF = np.inf
DBL_MAX = ref.DBL_MAX
COUNTS = (1, 127, 128, 129, 257)                     # around K12_THREADS = 128
SPECIAL = k11_fuzz.SPECIAL
MESH_UP = ("t", "bary", "both", "special")
FIELD_UP = ("lo", "hi", "both", "special")
OUTPUTS = [w for w in itertools.product((False, True), repeat=3) if any(w)]


class Lib(k11_fuzz.Lib):
    """k11_fuzz.Lib with meshes, the two casts and the two VJPs.  The VJPs run the host form twice and the device form once (on a side
    stream on a device) and report whether all gave the same bits"""

    def mesh(self, V, F):
        h = C.c_void_p()
        self.check(self.lib.dg_mesh_create(_p(V), len(V), _p(F, u32p), len(F), C.byref(h)))
        return h

    def mesh_destroy(self, h):
        self.lib.dg_mesh_destroy(h)

    def refit(self, h, V):
        self.check(self.lib.dg_mesh_refit(h, _p(V), len(V)))

    def mesh_cast(self, h, o, d, lo, hi):
        n = len(o)
        t, tid, b, st = np.empty(n), np.empty(n, np.int32), np.empty((n, 3)), np.empty(n, np.int32)
        self.check(self.lib.dg_mesh_raycast(h, _p(o), _p(d), n, lo, hi, _p(t), _p(tid, i32p), _p(b), _p(st, i32p)))
        return t, tid, b, st

    def field_cast(self, h, o, d, iso, lo, hi):
        n = len(o)
        tl, th, st = np.empty(n), np.empty(n), np.empty(n, np.int32)
        self.check(self.lib.dg_field_raycast(h, _p(o), _p(d), n, iso, lo, hi, _p(tl), _p(th), _p(st, i32p)))
        return tl, th, st

    def _runs(self, host, device_fn, ins, outs):
        """host() twice and device_fn(*pointers) once with `ins + outs` in device memory -> (first host result, all equal)"""
        first = host()
        runs = [host()]
        if self.side:
            if self.emulated:
                cp = [None if a is None else a.copy() for a in outs]
                self.check(device_fn(*([None if a is None else a.ctypes.data for a in ins + cp] + [None])))
                runs.append(tuple(cp))
            else:
                import torch
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                dev = [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in ins + outs]
                with torch.cuda.stream(s):
                    self.check(device_fn(*([None if t is None else t.data_ptr() for t in dev] + [s.cuda_stream])))
                s.synchronize()
                runs.append(tuple(None if t is None else t.cpu().numpy() for t in dev[len(ins):]))
        agree = all(all((a is None and b is None) or _bits(a, b) for a, b in zip(r, first)) for r in runs)
        return first, agree

    def mesh_vjp(self, h, nV, d, t, tid, bary, V, gt, gb, want):
        n = len(d)

        def outs():
            return [np.full((n, 3), 7.0) if want[0] else None, np.full((n, 3), 7.0) if want[1] else None,
                    np.full((nV, 3), 7.0) if want[2] else None]

        def host():
            o = outs()
            self.check(self.lib.dg_mesh_raycast_vjp(h, n, _p(d), _p(t), _p(tid, i32p), _p(bary), _p(V), _p(gt), _p(gb), *(_p(a) for a in o)))
            return tuple(o)
        return self._runs(host, lambda *p: self.lib.dg_mesh_raycast_vjp_device(h, n, *p), [d, t, tid, bary, V, gt, gb], outs())

    def field_vjp(self, h, n_nodes, o, d, t_lo, st, glo, ghi, want):
        n = len(o)

        def outs():
            return [np.full((n, 3), 7.0) if want[0] else None, np.full((n, 3), 7.0) if want[1] else None,
                    np.full(n_nodes, 7.0) if want[2] else None]

        def host():
            g = outs()
            self.check(self.lib.dg_field_raycast_vjp(h, n, _p(o), _p(d), _p(t_lo), _p(st, i32p), _p(glo), _p(ghi), *(_p(a) for a in g)))
            return tuple(g)
        return self._runs(host, lambda *p: self.lib.dg_field_raycast_vjp_device(h, n, *p), [o, d, t_lo, st, glo, ghi], outs())


def backend(lib, side=True):
    return Lib("dg" if lib == "dg" else (k11_fuzz.EMU if lib == "emu" else lib), side=side)


def _c(a, dt=np.float64):
    return None if a is None else np.ascontiguousarray(a, dt)


def _compare(got, want, names, label, agree):
    n = bad = 0
    first = None
    for g, w, nm in zip(got, want, names):
        if g is None:
            continue
        ok = same(g, w)
        ok = ok.reshape(len(ok), -1).all(1) if ok.ndim > 1 else ok
        n += len(ok); bad += int((~ok).sum())
        if not ok.all() and first is None:
            i = int(np.nonzero(~ok)[0][0])
            first = f"MISMATCH {label} {nm} row {i}: {np.asarray(g)[i].tolist()!r} vs {np.asarray(w)[i].tolist()!r}"
    if not agree:
        bad += 1; first = first or f"MISMATCH {label}: repeated calls or the device form differ"
    return n, bad, first


# ---------------------------------------------------------------------------------------------------------------- mesh
def mesh_upstreams(rng, n, which):
    gt, gb = rng.standard_normal(n), rng.standard_normal((n, 3))
    if which == "special":
        m = rng.random(n) < 0.4; gt[m] = rng.choice(SPECIAL, int(m.sum()))
        m = rng.random((n, 3)) < 0.4; gb[m] = rng.choice(SPECIAL, int(m.sum()))
    return (None if which == "bary" else gt), (None if which == "t" else gb)


def check_mesh(be, h, V, F, d, fwd, gt, gb, label, outputs=OUTPUTS):
    """every output combination of one VJP against the restatement -> (values, mismatches, first)"""
    t, tid, bary = _c(fwd[0]), _c(fwd[1], np.int32), _c(fwd[2])
    d, V, gt, gb = _c(d), _c(V), _c(gt), _c(gb)
    with np.errstate(all="ignore"):
        go, gd, valid = ref.mesh_ray_grads(V, F, d, t, tid, gt, gb)
        gv = ref.mesh_grad_vertices(F, len(V), tid, bary, go, valid)
    total = bad = 0
    first = None
    for want in outputs:
        got, agree = be.mesh_vjp(h, len(V), d, t, tid, bary, V, gt, gb, want)
        k, b, msg = _compare(got, (go, gd, gv), ("grad_origins", "grad_directions", "grad_vertices"), f"{label} want={want}", agree)
        total += k; bad += b; first = first or msg
    return total, bad, first


def run_mesh_cases(be, cases, seed=0, log=print, outputs=OUTPUTS):
    """k9_fuzz cases: cast by the library on each bound, then the VJP of those outputs"""
    rng = np.random.default_rng(seed + 31)
    acc = k11_fuzz.Acc(log)
    for ci, (label, V, F, o, d, bounds) in enumerate(cases):
        V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
        o = np.ascontiguousarray(o, np.float64); d = np.ascontiguousarray(d, np.float64)
        h = be.mesh(V, F)
        try:
            for bi, (lo, hi) in enumerate(bounds):
                fwd = be.mesh_cast(h, o, d, lo, hi)
                which = MESH_UP[(ci + bi) % len(MESH_UP)]
                acc.add(check_mesh(be, h, V, F, d, fwd, *mesh_upstreams(rng, len(o), which), f"{label} [{lo}, {hi}] {which}", outputs))
        finally:
            be.mesh_destroy(h)
    return acc.result()


def mesh_cases(seed=0, rounds=8, scale_exponents=(-24, -3, 0, 5, 17, -150, 150), n=60):
    yield from k9_fuzz.tie_cases(rounds, seed, n)
    yield from k9_fuzz.slack_cases()
    yield from k9_fuzz.scale_cases(seed, scale_exponents, n)
    yield from k9_fuzz.cull_cases(seed)
    yield from k9_fuzz.nonfinite_cases(seed, n // 2)
    yield from k9_fuzz.bound_cases(seed, n)


def run_mesh_refits(be, seed=0, log=print, n=60):
    """cast at each refit step's positions; refit to the next step; the VJP at the positions cast against (not the mesh's records)"""
    rng = np.random.default_rng(seed + 33)
    acc = k11_fuzz.Acc(log)
    V, F = k9_fuzz.sphere()
    V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
    o, d = k9_fuzz.mixed_rays(V, F, rng, n)
    o = np.ascontiguousarray(o); d = np.ascontiguousarray(d)
    steps = k9_fuzz.refit_steps(V, F)
    h = be.mesh(V, F)
    try:
        for i, (step, V1) in enumerate(steps):
            V1 = np.ascontiguousarray(V1, np.float64)
            be.refit(h, V1)
            fwd = be.mesh_cast(h, o, d, 0.0, INF)
            be.refit(h, np.ascontiguousarray(steps[(i + 1) % len(steps)][1], np.float64))
            which = MESH_UP[i % len(MESH_UP)]
            acc.add(check_mesh(be, h, V1, F, d, fwd, *mesh_upstreams(rng, len(o), which), f"refit {step} {which}"))
    finally:
        be.mesh_destroy(h)
    return acc.result()


MESH_SCALES = (1e-160, 1e-81, 1e-77, 1.0, 1e77, 1e80, 1e160)


def synthetic_mesh(rng, T, scale=1.0):
    """a soup of T triangles with degenerate ones (repeated vertex, collinear, a point) at the given scale"""
    V, F = k10_fuzz.soup(rng, T)
    V = V * scale
    if T >= 8:
        F[1, 2] = F[1, 0]                                                    # a repeated vertex
        F[3] = [F[3, 0], F[3, 0], F[3, 0]]                                   # a point
        V[F[5, 2]] = 0.5 * (V[F[5, 0]] + V[F[5, 1]])                          # collinear (n . n = 0 or a few ulps)
    return np.ascontiguousarray(V), np.ascontiguousarray(F)


def synthetic_rays(rng, V, F, n):
    """(d, t, tid, bary) chosen freely: ids in [-1, T), t from a pool with 0, -0, inf, NaN and huge values, directions in the hit
    triangle's plane (den = 0), subnormal and huge"""
    T = len(F)
    tid = rng.integers(-1, T, n).astype(np.int32)
    tid[::7] = -1
    t = rng.standard_normal(n) * 3.0
    pool = np.array([0.0, -0.0, INF, np.nan, 1e300, -1e-300, 5e-324])
    m = rng.random(n) < 0.2; t[m] = rng.choice(pool, int(m.sum()))
    d = rng.standard_normal((n, 3))
    T0 = F[np.maximum(tid, 0)]
    e1 = V[T0[:, 1]] - V[T0[:, 0]]
    d[1::5] = e1[1::5]                                                    # in the plane: n . d == 0 up to rounding, often exactly
    d[2::11] = rng.choice([5e-324, -1e-310, 2e-308], (len(d[2::11]), 3))
    d[3::13] = 1e300
    bary = rng.dirichlet((1.0, 1.0, 1.0), n)
    bary[tid < 0] = np.nan
    return d, t, tid, bary


def run_mesh_synthetic(be, seed=0, log=print, counts=COUNTS, scales=MESH_SCALES, outputs=OUTPUTS):
    rng = np.random.default_rng(seed + 35)
    acc = k11_fuzz.Acc(log)
    for s in scales:
        V, F = synthetic_mesh(rng, 257, s)
        h = be.mesh(V, F)
        try:
            for ni, n in enumerate(counts):
                d, t, tid, bary = synthetic_rays(rng, V, F, n)
                which = MESH_UP[ni % len(MESH_UP)]
                acc.add(check_mesh(be, h, V, F, d, (t, tid, bary), *mesh_upstreams(rng, n, which), f"synthetic x{s:g} n={n} {which}",
                                   outputs))
        finally:
            be.mesh_destroy(h)
    return acc.result()


# ---------------------------------------------------------------------------------------------------------------- field
class TrainLib(Lib):
    """Lib whose fields (k7_fuzz's and k6_fuzz's makers call field, field_desc, dense_field) are trainable: dense fields through the
    closed-form table (cells NULL).  A field is (handle, descriptor, k11_fuzz.Field)"""

    def __init__(self, lib="dg", side=True):
        super().__init__(lib, side)
        from discregrid_b200.grid import grid_desc
        self.grid_desc = grid_desc
        self.device_same = True

    def field(self, gd, r, nodes, cells, cmap):
        return self.field_desc(self.grid_desc(gd[0:3], gd[3:6], r, gd[6:9], gd[9:12]), nodes, cells, cmap)

    def field_desc(self, d, nodes, cells, cmap):
        fld = k11_fuzz.Field(d, nodes, np.ascontiguousarray(cells, np.uint32), cmap, "")
        return self.create(fld), d, fld

    def dense_field(self, mn, mx, res, fn):
        d = self.grid_desc(np.asarray(mn, np.float64), np.asarray(mx, np.float64), res)
        x = np.empty((self.num_nodes(res), 3))
        self.check(self.lib.dg_node_positions(C.byref(d), 0, len(x), _p(x)))
        fld = k11_fuzz.Field(d, fn(x), None, None, "")
        return self.create(fld), d, fld

    def destroy(self, f):
        super().destroy(f[0] if isinstance(f, tuple) else f)

    def interpolate(self, f, x, chunk=1 << 22):                              # k7_fuzz's value-only evaluation
        return super().interpolate(f[0] if isinstance(f, tuple) else f, x)[0]

    def cast(self, f, O, D, iso, lo, hi):
        return self.field_cast(f[0], O, D, iso, lo, hi)


def field_upstreams(rng, n, which):
    glo, ghi = rng.standard_normal(n), rng.standard_normal(n)
    if which == "special":
        for g in (glo, ghi):
            m = rng.random(n) < 0.4; g[m] = rng.choice(SPECIAL, int(m.sum()))
    return (None if which == "hi" else glo), (None if which == "lo" else ghi)


def check_field(be, f, o, d, t_lo, st, glo, ghi, label, outputs=OUTPUTS):
    """every output combination of one field VJP against the restatement, K2 evaluated by the library at the crossing points"""
    h, dsc, fld = f
    o, d, t_lo, glo, ghi = _c(o), _c(d), _c(t_lo), _c(glo), _c(ghi)
    st = _c(st, np.int32)
    xc = ref.crossing_points(fld.mn, fld.mx, o, d, t_lo, st)
    phi, grad = super(TrainLib, be).interpolate(h, np.ascontiguousarray(xc))
    with np.errstate(all="ignore"):
        go, gd, gphi, valid = ref.field_ray_grads(d, t_lo, st, phi, grad, glo, ghi)
    gn = fld.restate(np.where(valid[:, None], xc, INF), gphi, None)
    total = bad = 0
    first = None
    for want in outputs:
        got, agree = be.field_vjp(h, len(fld.nodes), o, d, t_lo, st, glo, ghi, want)
        k, b, msg = _compare(got, (go, gd, gn), ("grad_origins", "grad_directions", "grad_nodes"), f"{label} want={want}", agree)
        total += k; bad += b; first = first or msg
    return total, bad, first, valid


def run_field_cases(be, cases, seed=0, log=print, outputs=OUTPUTS):
    """k7_fuzz cases (label, make, O, D, isos, bounds) on trainable fields: cast by the library at each iso and bound, then the VJP"""
    rng = np.random.default_rng(seed + 41)
    acc = k11_fuzz.Acc(log)
    for ci, (label, make, O, D, isos, bounds) in enumerate(cases):
        f = make(be)
        try:
            O1 = np.ascontiguousarray(O(f) if callable(O) else O, np.float64).reshape(-1, 3)
            D1 = np.ascontiguousarray(D(f) if callable(D) else D, np.float64).reshape(-1, 3)
            for ii, iso in enumerate(isos(f) if callable(isos) else isos):
                for bi, (lo, hi) in enumerate(bounds):
                    t_lo, _, st = be.cast(f, O1, D1, iso, lo, hi)
                    which = FIELD_UP[(ci + ii + bi) % len(FIELD_UP)]
                    acc.add(check_field(be, f, O1, D1, t_lo, st, *field_upstreams(rng, len(O1), which),
                                        f"{label} iso={iso!r} [{lo}, {hi}] {which}", outputs)[:3])
        finally:
            be.destroy(f)
    return acc.result()


def k2_field_cases(rounds, seed=0, n=60):
    """k2_fuzz.make_field fields cast from k2_fuzz.queries origins along k7_fuzz.directions, iso 0 and a quartile of the values"""
    import tempfile
    from oracle_api import Oracle
    rng = np.random.default_rng(seed + 43)
    orc = Oracle()
    for k in range(rounds):
        with tempfile.TemporaryDirectory(prefix="k12_fuzz_") as tmp:          # make_field's .cdf round trips, removed with the directory
            gd, r, nodes, cells, cmap, label = k7_fuzz.k2_fuzz.make_field(orc, rng, k, tmp)
        x = k7_fuzz.k2_fuzz.queries(rng, gd, r, nodes, cells, cmap)
        O = np.ascontiguousarray(x[rng.integers(0, len(x), n)])
        D = k7_fuzz.directions(rng, n)
        fin = nodes[np.isfinite(nodes) & (nodes != DBL_MAX)]
        isos = (0.0, float(np.quantile(fin, 0.4)) if len(fin) else 0.5)
        yield label, (lambda be, a=(gd, r, nodes, cells, cmap): be.field(*a)), O, D, isos, k7_fuzz.BOUNDS[k % 4:k % 4 + 1]


def field_cases(seed=0, rounds=8):
    yield from k2_field_cases(rounds, seed)
    yield "special rays", k7_fuzz.sphere, k7_fuzz.SPECIAL_O, k7_fuzz.SPECIAL_D, (0.0, 0.2), ((0.0, INF), (-INF, 0.5))
    yield "thin feature", k7_fuzz.thin_field, np.array([[-0.5, 0.5, 0.5], [-0.5, 0.25, 0.75], [1.5, 0.3, 0.6]]), \
        np.array([[1.0, 0.0, 0.0], [1.0, 0.0, 0.0], [-1.0, 0.0, 0.0]]), (0.0,), ((0.0, INF),)
    yield "tangent rays", (lambda be: be.dense_field([-1, -1, -1], [1, 1, 1], (8, 8, 8), lambda x: np.linalg.norm(x, axis=1) - 0.5)), \
        np.array([[-2.0, 0.5, 0.0], [-2.0, 0.5 - 1e-9, 0.0], [-2.0, 0.45, 0.0], [-2.0, 0.51, 0.0], [0.0, -2.0, 0.5], [-2.0, 0.0, 0.5 + 1e-12]]), \
        np.array([[1.0, 0.0, 0.0]] * 4 + [[0.0, 1.0, 0.0], [1.0, 0.0, 0.0]]), (0.0,), ((0.0, INF),)
    yield from k7_fuzz.grid_cases(60)
    yield from k7_fuzz.density_cases(60)
    yield from k7_fuzz.cursor_cases(seed)
    yield from k7_fuzz.ulp_cases()
    yield from k7_fuzz.scale_cases(k7_fuzz.SCALES, 30)
    yield from k7_fuzz.hole_cases(seed)
    yield from k7_fuzz.bound_cases(60)


def run_iso_at_samples(be, seed=0, log=print, n=40):
    """the torus cast at an iso equal to the field at a ray's first depth-0 sample (k7_fuzz's strict side test), then the VJP"""
    rng = np.random.default_rng(seed + 45)
    f = k7_fuzz.torus(be)
    try:
        O, D = k7_fuzz.random_rays(f, n, 4, pad=0.0)
        g = k7_fuzz.rr.Grid.of_desc(f[1])
        isos = []
        for i in range(len(O)):
            c = k7_fuzz.rr.clip(g, list(O[i]), list(D[i]), 0.0, INF)
            if c is None:
                continue
            b = k7_fuzz.rr.breakpoints(g, list(O[i]), list(D[i]), c[0], c[1])
            v = float(be.interpolate(f, np.array([k7_fuzz.rr.position(g, list(O[i]), list(D[i]), c[0] + (b[0] - c[0]) * k7_fuzz.rr.W[2])]))[0])
            if abs(v) < 0.3:
                isos.append(v)
    finally:
        be.destroy(f)
    return run_field_cases(be, [("iso at samples", k7_fuzz.torus, O, D, isos[:4], ((0.0, INF),))], seed, log)


def synthetic_field(be, rng):
    """a trainable 6 x 5 x 4 sphere SDF with three DBL_MAX coefficients and five removed cells"""
    res = (6, 5, 4)
    d = be.desc([-1.0, -0.9, -0.7], [1.1, 0.8, 0.9], res)
    x = np.empty((be.num_nodes(res), 3))
    be.check(be.lib.dg_node_positions(C.byref(d), 0, len(x), _p(x)))
    nodes = np.linalg.norm(x, axis=1) - 0.5
    cells = be.build_cells(res)
    keep = np.ones(len(cells), bool); keep[[3, 17, 40, 61, 100]] = False
    cmap = np.full(len(cells), 0xFFFFFFFF, np.uint32); cmap[keep] = np.arange(keep.sum(), dtype=np.uint32)
    nodes[cells[keep][[5, 50, 90], 7]] = DBL_MAX
    fld = k11_fuzz.Field(d, nodes, cells[keep], cmap, "synthetic field")
    return be.create(fld), d, fld


def synthetic_field_rays(rng, fld, n):
    """(o, d, t_lo, status): x_c inside, outside (clamped), on a max face, in a removed cell, in a DBL_MAX cell, NaN; statuses 0, 1, 2 and
    values outside the enum"""
    mn, mx = fld.mn, fld.mx
    o = mn + rng.random((n, 3)) * (mx - mn)
    d = rng.standard_normal((n, 3))
    t = rng.random(n) * 0.1
    k = np.arange(n) % 6
    t[k == 1] = 50.0 + rng.random(int((k == 1).sum())) * 10                     # far outside: clamped onto a face or edge
    face = k == 2
    o[face, 0] = mx[0]; t[face] = 0.0                                            # on the max face
    cell = np.array(fld.d.cell_size[:])
    res = fld.res
    removed = np.flatnonzero(fld.cmap == 0xFFFFFFFF)
    bad_cells = np.flatnonzero(fld.cmap != 0xFFFFFFFF)[(fld.nodes[fld.cells] == DBL_MAX).any(1)] if len(fld.cells) else removed
    for sel, cs in ((k == 3, removed), (k == 4, bad_cells)):
        c = cs[rng.integers(0, len(cs), int(sel.sum()))]
        ijk = np.stack([c % res[0], (c // res[0]) % res[1], c // (res[0] * res[1])], 1)
        o[sel] = mn + (ijk + 0.5) * cell; t[sel] = 0.0
    nanr = k == 5
    t[nanr] = np.nan
    st = rng.choice(np.array([0, 1, 2, 1, 2, 7, -3], np.int32), n)
    return o, d, t, st


def dbl_max_phi_field(be):
    """one cell on [0, 4]^3 with a single nonzero coefficient c (not DBL_MAX) and a point x where fl(N_j(x) c) is exactly DBL_MAX with a
    finite gradient: a crossing there has phi == DBL_MAX and a finite, nonzero den, so only the DBL_MAX test makes the ray invalid.
    -> (field, x) or None when no such point is found"""
    res = (1, 1, 1)
    d = be.desc([0.0, 0.0, 0.0], [4.0, 4.0, 4.0], res)
    cells = be.build_cells(res)
    rng = np.random.default_rng(47)
    x = rng.random((20000, 3)) * 4.0
    mn, mx = np.zeros(3), np.full(3, 4.0)
    _, _, c0, c1 = interpolate_vjp_ref.locate(mn, mx, d.cell_size[:], d.inv_cell_size[:], d.resolution[:], None, x)
    xi = c0 * x - c1
    N, D = interpolate_vjp_ref.rows(xi[:, 0], xi[:, 1], xi[:, 2])
    q, j = np.unravel_index(int(np.argmax(N)), N.shape)
    if N[q, j] <= 1.0:
        return None
    c = DBL_MAX / N[q, j]
    for _ in range(64):
        p = N[q, j] * c
        if p == DBL_MAX:
            break
        c = np.nextafter(c, INF if p < DBL_MAX else -INF)
    nodes = np.zeros(be.num_nodes(res))
    nodes[cells[0, j]] = c
    fld = k11_fuzz.Field(d, nodes, cells, None, "phi = DBL_MAX")
    f = (be.create(fld), d, fld)
    phi, grad = super(TrainLib, be).interpolate(f[0], x[q:q + 1])
    if not (phi[0] == DBL_MAX and np.isfinite(grad).all() and (grad != 0).any()):
        be.destroy(f)
        return None
    return f, x[q]


def run_field_synthetic(be, seed=0, log=print, counts=COUNTS, outputs=OUTPUTS):
    rng = np.random.default_rng(seed + 49)
    acc = k11_fuzz.Acc(log)
    f = synthetic_field(be, rng)
    try:
        for ni, n in enumerate(counts):
            o, d, t, st = synthetic_field_rays(rng, f[2], n)
            which = FIELD_UP[ni % len(FIELD_UP)]
            acc.add(check_field(be, f, o, d, t, st, *field_upstreams(rng, n, which), f"synthetic n={n} {which}", outputs)[:3])
    finally:
        be.destroy(f)
    made = dbl_max_phi_field(be)
    if made is None:
        acc.add((0, 1, "MISMATCH phi = DBL_MAX: no point with fl(N_j c) == DBL_MAX and a finite gradient was found"))
        return acc.result()
    f, x = made
    try:
        grad = super(TrainLib, be).interpolate(f[0], x[None])[1][0]
        o = np.repeat(x[None], 3, 0); dd = np.array([grad / np.abs(grad).max() * 1e-3, [1.0, 0.0, 0.0], [0.3, -0.2, 0.1]])
        t = np.zeros(3); st = np.array([1, 2, 1], np.int32)
        r = check_field(be, f, o, dd, t, st, np.ones(3), np.full(3, 0.5), "phi = DBL_MAX", outputs)
        acc.add(r[:3])
        if r[3].any():
            acc.add((0, 1, "MISMATCH phi = DBL_MAX: the restatement counts the ray as valid"))
        gp = ref.dot(grad[None], dd[:1])
        if not (np.isfinite(gp).all() and (gp != 0).all()):
            acc.add((0, 1, "MISMATCH phi = DBL_MAX: den is not finite and nonzero, the case tests nothing"))
    finally:
        be.destroy(f)
    return acc.result()


def run(be, rounds, seed=0, log=print):
    tb = be if isinstance(be, TrainLib) else TrainLib(be.name if be.name == "dg" else k11_fuzz.EMU, be.side)
    acc = [0, 0, 0]
    for r in (run_mesh_cases(be, mesh_cases(seed, rounds), seed, log), run_mesh_refits(be, seed, log), run_mesh_synthetic(be, seed, log),
              run_field_cases(tb, field_cases(seed, rounds), seed, log), run_iso_at_samples(tb, seed, log), run_field_synthetic(tb, seed, log)):
        acc = [a + b for a, b in zip(acc, r)]
    return tuple(acc)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 8
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else "emu"
    cases, total, bad = run(TrainLib("dg" if lib == "dg" else (k11_fuzz.EMU if lib == "emu" else lib)), rounds, seed)
    print(f"{cases} cases, {total} values, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
