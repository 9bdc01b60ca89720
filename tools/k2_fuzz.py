#!/usr/bin/env python
"""Parity fuzzer for interpolate: the product's K2 kernel code against the reference's own CubicLagrangeDiscreteGrid::interpolate
(oracle/_ref/libdiscregrid_ref.so; where that is not compiled, the oracle's restatement) on random grids (anisotropic, offset, tiny / huge
cells) and fields: DBL_MAX sentinels, reduced fields, coefficients of +-1e308, -DBL_MAX, NaN, +-inf, subnormals and -0.0, fields with no
kept cell or exactly one.  Queries sit on cell faces, the max faces (the cell-index clamp), domain corners, outside, NaN / infinite, and in
runs of 1, 2 and 3 live lanes between runs of lanes that issue no real copy (out of domain, NaN, removed cell, missing coefficient), at
counts around the warp and block sizes.  Value + gradient and value-only, bit for bit (any NaN equal to any NaN).

usage: tools/k2_fuzz.py [rounds=60] [seed=0] [lib=build/bin/libk23emu.so] [gradient|hessian]
  lib      a build of tests/emu (libk23emu*.so: the K2 translation unit compiled for the CPU, its TMA staging a plain copy), or `dg`: the
           product library through its C-ABI (dg_field_create, dg_interpolate_batch), i.e. the CUDA kernels -- needs a GPU
  hessian  K2's Hessian mode (interpolate_kernel<true, true>; build/bin/libk2hemu.so or `dg`: dg_interpolate_hessian_batch) on the same
           fields and queries: phi and grad are the gradient mode's bits, hess the bits of the numpy restatement of its contract
           (tests/hessian_ref.py), exactly symmetric, and +0.0 in all nine entries wherever phi is DBL_MAX
The functions are shared with tests/test_k23_emulated.py, tests/test_k2_hessian_emulated.py, tests/test_gpu_k23_fuzz.py and
tests/test_gpu_winding_hessian_fuzz.py."""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from oracle_api import Oracle, RefGrid, have_ref_grid  # noqa: E402

dp, u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)
DBL_MAX = np.finfo(np.float64).max
UINT32_MAX = 0xFFFFFFFF
K2_THREADS = 128                                   # csrc/k2_interp.h
COUNTS = (1, 31, 32, 33, K2_THREADS - 1, K2_THREADS + 1)
# coefficient sets that K2 and K3 must carry through exactly as the reference does
EXTREMES = {
    "huge": (1e308, -1e308, -DBL_MAX),
    "nonfinite": (np.nan, np.inf, -np.inf),
    "tiny": (5e-324, -5e-324, 2.2250738585072014e-308 / 3, -1e-310, -0.0),
}


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def same(a, b):
    """bit for bit, any NaN equal to any NaN"""
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def reduce_layout(rng, cells, nodes, keep_frac):
    """a reduced field's arrays without the reference: a random subset of cells kept (renumbered in order), the rest UINT32_MAX in the cell
    map, and only the nodes the kept cells use, renumbered.  -> (nodes, cells, cell map)"""
    n_cells = len(cells)
    kept = np.nonzero(rng.random(n_cells) < keep_frac)[0]
    cmap = np.full(n_cells, UINT32_MAX, np.uint32); cmap[kept] = np.arange(len(kept), dtype=np.uint32)
    used = np.unique(cells[kept]) if len(kept) else np.zeros(0, np.int64)
    new_cells = np.searchsorted(used, cells[kept]).astype(np.uint32).reshape(-1, 32)
    return np.ascontiguousarray(nodes[used], np.float64), np.ascontiguousarray(new_cells), cmap


def plant(rng, v, kind, count=None):
    """v with a few coefficients replaced by the values of EXTREMES[kind] (every value at least once)"""
    v = v.copy()
    vals = EXTREMES[kind]
    count = max(len(vals), int(0.05 * len(v))) if count is None else count
    at = rng.choice(len(v), size=min(count, len(v)), replace=False)
    v[at] = [vals[i % len(vals)] for i in range(len(at))]
    return v


class EmuK2:
    """a build of tests/emu (libk23emu*.so): the K2 kernels and launchers run on the CPU"""

    def __init__(self, so):
        self.name = os.path.basename(so)
        lib = self.lib = C.CDLL(so)
        lib.emu_field_create.restype = C.c_void_p
        lib.emu_field_create.argtypes = [dp, u32p, dp, u32p, C.c_uint64, u32p]
        lib.emu_field_destroy.argtypes = [C.c_void_p]
        lib.emu_interpolate.argtypes = [C.c_void_p, dp, C.c_uint64, dp, dp]
        lib.emu_density_map.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_uint64, dp]
        if hasattr(lib, "emu_interpolate_hessian"):
            lib.emu_interpolate_hessian.argtypes = [C.c_void_p, dp, C.c_uint64, dp, dp, dp]

    def field(self, gd, r, nodes, cells, cmap):
        keep = (gd, r, np.ascontiguousarray(nodes, np.float64), np.ascontiguousarray(cells, np.uint32), np.ascontiguousarray(cmap, np.uint32))
        h = self.lib.emu_field_create(_p(keep[0], dp), _p(keep[1], u32p), _p(keep[2], dp), _p(keep[3], u32p), len(keep[3]), _p(keep[4], u32p))
        assert h
        return (h, keep)

    def destroy(self, f):
        self.lib.emu_field_destroy(f[0])

    def interpolate(self, f, x, grad):
        n = len(x)
        phi = np.full(n, -1.0); g = np.full((n, 3), -1.0) if grad else None
        assert self.lib.emu_interpolate(f[0], _p(x, dp), n, _p(phi, dp), _p(g, dp)) == 0
        return phi, g

    def hessian(self, f, x):
        n = len(x)
        phi, g, h = np.full(n, -1.0), np.full((n, 3), -1.0), np.full((n, 3, 3), -1.0)
        assert self.lib.emu_interpolate_hessian(f[0], _p(x, dp), n, _p(phi, dp), _p(g, dp), _p(h, dp)) == 0
        return phi, g, h

    def density(self, f, h, rho0, no_reduction, l0, l1):
        out = np.full(l1 - l0, -1.0)
        assert self.lib.emu_density_map(f[0], h, rho0, int(no_reduction), l0, l1, _p(out, dp)) == 0
        return out


class DgK2:
    """the product library through its C-ABI: the CUDA kernels on the current device"""

    name = "dg"

    def __init__(self):
        from discregrid_b200 import _capi
        from discregrid_b200.grid import grid_desc
        self.capi, self.lib, self.grid_desc = _capi, _capi.lib, grid_desc

    def field(self, gd, r, nodes, cells, cmap):
        d = self.grid_desc(gd[0:3], gd[3:6], r, gd[6:9], gd[9:12])
        nodes = np.ascontiguousarray(nodes, np.float64); cells = np.ascontiguousarray(cells, np.uint32); cmap = np.ascontiguousarray(cmap, np.uint32)
        h = C.c_void_p()
        self.capi.check(self.lib.dg_field_create(C.byref(d), _p(nodes, dp) if len(nodes) else None, len(nodes), _p(cells, u32p), len(cells),
                                                 _p(cmap, u32p), C.byref(h)))
        return (h, d)

    def destroy(self, f):
        self.capi.check(self.lib.dg_field_destroy(f[0]))

    def interpolate(self, f, x, grad):
        n = len(x)
        phi = np.full(n, -1.0); g = np.full((n, 3), -1.0) if grad else None
        self.capi.check(self.lib.dg_interpolate_batch(f[0], _p(x, dp), n, _p(phi, dp), _p(g, dp)))
        return phi, g

    def hessian(self, f, x):
        n = len(x)
        phi, g, h = np.full(n, -1.0), np.full((n, 3), -1.0), np.full((n, 3, 3), -1.0)
        self.capi.check(self.lib.dg_interpolate_hessian_batch(f[0], _p(x, dp), n, _p(phi, dp), _p(g, dp), _p(h, dp)))
        return phi, g, h

    def density(self, f, h, rho0, no_reduction, l0, l1):
        out = np.full(l1 - l0, -1.0)
        self.capi.check(self.lib.dg_density_map(f[0], h, rho0, int(no_reduction), l0, l1, _p(out, dp)))
        return out


def backend(lib):
    return DgK2() if lib == "dg" else EmuK2(lib)


class Reference:
    """the reference class where oracle/_ref is built (the field goes through a .cdf it loads), else the oracle's restatement"""

    def __init__(self, tmp):
        self.tmp, self.use_ref = tmp, have_ref_grid()
        self.name = "reference CubicLagrangeDiscreteGrid (oracle/_ref)" if self.use_ref else "oracle restatement (oracle/liboracle.so)"
        self.orc = Oracle()

    def interpolate(self, gd, r, nodes, cells, cmap, x, grad):
        if self.use_ref:
            from make_reduce_golden import write_cdf
            src = os.path.join(self.tmp, "ref_in.cdf")
            write_cdf(src, gd[0:3], gd[3:6], r, gd[6:9], gd[9:12], np.ascontiguousarray(nodes, np.float64), np.ascontiguousarray(cells, np.uint32),
                      np.ascontiguousarray(cmap, np.uint32))
            ref = RefGrid(src)
            try:
                return ref.interpolate(0, x, grad=grad)
            finally:
                ref.close()
        return self.orc.interpolate(gd, r, nodes, x, grad=grad, cells=cells, cell_map=cmap)


def make_field(orc, rng, k, tmp):
    """round k's grid and field -> (gd, r, nodes, cells, cmap, label).  k % 3: plain / DBL_MAX sentinels / reduced; k % 4: no extreme
    coefficients / huge / non-finite / tiny; k % 12 == 5: no kept cell, k % 12 == 11: exactly one"""
    res = tuple(int(v) for v in rng.integers(1, 7, 3))
    sc = 10.0 ** rng.integers(-5, 6)
    mn = rng.standard_normal(3) * sc * 10 ** rng.integers(0, 3)
    mx = mn + sc * (0.2 + rng.random(3) * (10 ** rng.integers(0, 2, 3)))
    gd, r = orc.grid_desc(mn, mx, res)
    cells = orc.build_cells(r)
    n = int(cells.max()) + 1
    v = rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4)
    label = f"case {k} res {res}"
    if k % 3 == 1:
        v[rng.random(n) < 0.05] = DBL_MAX                               # missing coefficients
    ck = k % 4
    if ck:
        kind = ("huge", "nonfinite", "tiny")[ck - 1]
        v = plant(rng, v, kind); label += f" {kind}"
    cmap = np.arange(len(cells), dtype=np.uint32)
    if k % 12 == 5:                                                      # no kept cell: n_cells_kept = 0, every cell-map entry UINT32_MAX
        return gd, r, np.zeros(0), np.zeros((0, 32), np.uint32), np.full(len(cells), UINT32_MAX, np.uint32), label + " no kept cell"
    if k % 12 == 11:                                                     # exactly one kept cell
        c = int(rng.integers(len(cells)))
        used = np.unique(cells[c])
        cmap = np.full(len(cells), UINT32_MAX, np.uint32); cmap[c] = 0
        return gd, r, np.ascontiguousarray(v[used]), np.searchsorted(used, cells[c:c + 1]).astype(np.uint32), cmap, label + " one kept cell"
    if k % 3 == 2:                                                       # a reduced field: removed cells, renumbered nodes
        if have_ref_grid():
            from make_reduce_golden import write_cdf
            from test_oracle_golden import read_cdf
            src = os.path.join(tmp, "in.cdf")
            write_cdf(src, mn, mx, res, gd[6:9], gd[9:12], v, cells, cmap)
            fin = v[np.isfinite(v) & (v != DBL_MAX)]
            lo, hi = (float(np.quantile(fin, 0.3)), float(np.quantile(fin, 0.7))) if len(fin) else (0.0, 0.0)
            ref = RefGrid(src); ref.reduce_window(0, lo, hi); ref.save(src); ref.close()
            g = read_cdf(src)
            return gd, r, np.ascontiguousarray(g["nodes"][0]), np.ascontiguousarray(g["cells"][0], np.uint32), \
                np.ascontiguousarray(g["cmap"][0], np.uint32), label + " reduced"
        nodes, cells, cmap = reduce_layout(rng, cells, v, 0.6)
        return gd, r, nodes, cells, cmap, label + " reduced"
    return gd, r, v, cells, cmap, label


def interleave(live, dead, s):
    """runs of s live queries between runs of s dead ones, until the live ones run out"""
    out = []
    j = 0
    for i in range(0, len(live), s):
        out.append(live[i:i + s])
        out.append(dead[np.arange(j, j + s) % len(dead)]); j += s
    return np.concatenate(out)


def queries(rng, gd, r, nodes, cells, cmap):
    mn, mx, cell = gd[0:3], gd[3:6], gd[6:9]
    res = np.asarray(r, np.int64)
    ext = mx - mn
    xs = [mn - 0.1 * ext + rng.random((400, 3)) * 1.2 * ext]
    faces = [mn[d] + cell[d] * np.arange(res[d] + 1) for d in range(3)]
    xs.append(np.stack([rng.choice(faces[0], 200), rng.choice(faces[1], 200), rng.choice(faces[2], 200)], 1))                     # cell corners
    on_face = mn + rng.random((200, 3)) * ext; on_face[:, 0] = rng.choice(faces[0], 200); xs.append(on_face)                      # on x-faces
    on_max = mn + rng.random((150, 3)) * ext                                                                                       # max faces
    for d in range(3):
        on_max[d * 50:(d + 1) * 50, d] = mx[d]
    on_max[::7] = np.where(rng.random((len(on_max[::7]), 3)) < 0.5, mx, on_max[::7])
    xs.append(on_max)
    xs.append(np.array([mn, mx, [mn[0], mx[1], mn[2]], [mx[0], mx[1], mn[2]], 0.5 * (mn + mx), np.nextafter(mx, np.inf), np.nextafter(mn, -np.inf),
                        np.nextafter(mx, -np.inf), [np.nan, mn[1], mn[2]], [np.inf, mn[1], mn[2]], [mn[0], -np.inf, mn[2]], [0.0, 0.0, 0.0],
                        [-0.0, -0.0, -0.0]]))
    # lanes that copy nothing real (K2 issues a dummy copy of cell 0 for them): out of domain, NaN, removed cells, missing coefficients
    idx = np.stack(np.meshgrid(*[np.arange(int(n)) for n in res], indexing="ij"), -1).reshape(-1, 3)        # (i, j, k) of cell i + nx (j + ny k)
    lin = idx[:, 0] + res[0] * (idx[:, 1] + res[1] * idx[:, 2])
    centre = mn + (idx + 0.5) * cell
    order = np.argsort(lin); centre = centre[order]
    removed = centre[cmap == UINT32_MAX]
    has_missing = np.zeros(len(cmap), bool)
    kept = np.nonzero(cmap != UINT32_MAX)[0]
    if len(kept) and len(nodes):
        has_missing[kept] = (nodes[cells[cmap[kept]]] == DBL_MAX).any(1)
    missing = centre[has_missing]
    dead = [mx + ext * (0.5 + rng.random((8, 3))), np.array([[np.nan, mn[1], mn[2]], [mn[0], np.nan, mx[2]], [np.nan] * 3])]
    dead += [removed[:16], missing[:16]]
    dead = np.concatenate([d for d in dead if len(d)])
    rng.shuffle(dead)
    live_ok = np.ones(len(cmap), bool); live_ok[cmap == UINT32_MAX] = False; live_ok &= ~has_missing
    live_cells = centre[live_ok]
    if len(live_cells):
        live = live_cells[rng.integers(len(live_cells), size=96)] + (rng.random((96, 3)) - 0.5) * 0.9 * cell
    else:
        live = mn + rng.random((96, 3)) * ext
    for s in (1, 2, 3):
        xs.append(interleave(live, dead, s))
    return np.ascontiguousarray(np.concatenate(xs), np.float64)


def restate(gd, r, nodes, cells, cmap, x, chunk=1 << 20):
    """tests/hessian_ref.py's restatement of the Hessian on a k2_fuzz field, in chunks of queries"""
    from hessian_ref import restate_hessian        # only the Hessian mode needs it: importing k2_fuzz does not
    return np.concatenate([restate_hessian(gd[0:3], gd[3:6], gd[6:9], gd[9:12], r, nodes, cells, cmap, x[i:i + chunk])
                           for i in range(0, len(x), chunk)] or [np.zeros((0, 3, 3))])


def hessian_ok(phi, grad, hess, phi_g, grad_g, want_hess):
    """per query: the Hessian mode's phi and grad are the gradient mode's bits, hess the restatement's (any NaN equal to any NaN), exactly
    symmetric (the same bits at [a][b] and [b][a], NaN payloads included), and +0.0 in all nine entries where phi is DBL_MAX"""
    hb = hess.reshape(-1, 3, 3).view(np.uint64)
    sym = (hb == hb.transpose(0, 2, 1)).all((1, 2))
    zero = ~(phi == DBL_MAX) | ~hb.any((1, 2))
    return same(phi, phi_g) & same(grad, grad_g).all(1) & same(hess, want_hess).all((1, 2)) & sym & zero


def check_hessian(be, f, gd, r, nodes, cells, cmap, x, label, counts=COUNTS):
    """the Hessian mode at the full count and at the prefix counts -> (queries checked, mismatches, first mismatch)"""
    phi_g, grad_g = be.interpolate(f, x, True)
    want = restate(gd, r, nodes, cells, cmap, x)
    phi, grad, hess = be.hessian(f, x)
    ok = hessian_ok(phi, grad, hess, phi_g, grad_g, want)
    total, bad, first = len(x), int((~ok).sum()), None
    if bad:
        i = int(np.nonzero(~ok)[0][0])
        first = (f"MISMATCH {label} hessian x={x[i]!r}: phi {phi[i]!r} vs {phi_g[i]!r}, grad {grad[i]} vs {grad_g[i]}, "
                 f"hess {hess[i].tolist()} vs {want[i].tolist()}")
    for c in counts:
        if c > len(x):
            continue
        p, g, h = be.hessian(f, x[:c])
        okc = same(p, phi[:c]) & same(g, grad[:c]).all(1) & same(h, hess[:c]).all((1, 2))
        total += c
        if not okc.all():
            bad += int((~okc).sum())
            first = first or f"MISMATCH {label} hessian count {c}: first bad query {int(np.nonzero(~okc)[0][0])}"
    return total, bad, first


def check_field(be, ref, f, gd, r, nodes, cells, cmap, x, label, counts=COUNTS, mode="gradient"):
    """value + gradient and value-only at the full count and at the prefix counts -> (queries checked, mismatches, first mismatch);
    mode "hessian": check_hessian"""
    if mode == "hessian":
        return check_hessian(be, f, gd, r, nodes, cells, cmap, x, label, counts)
    want_phi, want_grad = ref.interpolate(gd, r, nodes, cells, cmap, x, True)
    want_only = ref.interpolate(gd, r, nodes, cells, cmap, x, False)[0]
    phi, grad = be.interpolate(f, x, True)
    only = be.interpolate(f, x, False)[0]
    ok = same(phi, want_phi) & same(grad, want_grad).all(1) & same(only, want_only)
    total, bad, first = len(x), int((~ok).sum()), None
    if bad:
        i = int(np.nonzero(~ok)[0][0])
        first = (f"MISMATCH {label} x={x[i]!r}: phi {phi[i]!r} vs {want_phi[i]!r}, grad {grad[i]} vs {want_grad[i]}, "
                 f"value-only {only[i]!r} vs {want_only[i]!r}")
    for c in counts:
        if c > len(x):
            continue
        p, g = be.interpolate(f, x[:c], c % 2 == 1)
        okc = same(p, want_phi[:c]) & (same(g, want_grad[:c]).all(1) if g is not None else same(p, want_only[:c]))
        total += c
        if not okc.all():
            bad += int((~okc).sum())
            first = first or f"MISMATCH {label} count {c}: first bad query {int(np.nonzero(~okc)[0][0])}"
    return total, bad, first


def run(be, rounds, seed, log=print, mode="gradient"):
    """-> (fields, queries checked, mismatches); mode: "gradient" (value + gradient and value-only against the reference) or "hessian" """
    rng = np.random.default_rng(seed)
    orc = Oracle()
    tmp = tempfile.mkdtemp(prefix="k2_fuzz_")
    ref = Reference(tmp)
    log(f"backend {be.name}, {mode} mode, reference: {ref.name if mode == 'gradient' else 'tests/hessian_ref.py'}")
    total = bad = 0
    for k in range(rounds):
        gd, r, nodes, cells, cmap, label = make_field(orc, rng, k, tmp)
        x = queries(rng, gd, r, nodes, cells, cmap)
        f = be.field(gd, r, nodes, cells, cmap)
        try:
            n, b, msg = check_field(be, ref, f, gd, r, nodes, cells, cmap, x, label, mode=mode)
        finally:
            be.destroy(f)
        total += n; bad += b
        if msg: log(msg)
    return rounds, total, bad


def run_many(be, n_queries=4 << 20, seed=0, log=print, mode="gradient"):
    """one field of every kind of lane and n_queries queries in one call (many warps with copies in flight) -> (queries, mismatches)"""
    rng = np.random.default_rng(seed)
    orc = Oracle()
    tmp = tempfile.mkdtemp(prefix="k2_fuzz_")
    ref = Reference(tmp)
    gd, r = orc.grid_desc(np.array([-1.0, -2.0, -0.5]), np.array([1.5, 1.0, 2.0]), (24, 20, 28))
    full = orc.build_cells(r)
    v = plant(rng, rng.standard_normal(int(full.max()) + 1), "nonfinite", 40)
    v[rng.random(len(v)) < 0.002] = DBL_MAX
    nodes, cells, cmap = reduce_layout(rng, full, v, 0.8)
    base = queries(rng, gd, r, nodes, cells, cmap)
    x = np.ascontiguousarray(base[rng.integers(len(base), size=n_queries)] + np.where(rng.random((n_queries, 1)) < 0.5, 0.0,
                                                                                      1e-3 * rng.standard_normal((n_queries, 3))))
    if mode == "hessian":
        f = be.field(gd, r, nodes, cells, cmap)
        try:
            phi_g, grad_g = be.interpolate(f, x, True)
            phi, grad, hess = be.hessian(f, x)
        finally:
            be.destroy(f)
        ok = hessian_ok(phi, grad, hess, phi_g, grad_g, restate(gd, r, nodes, cells, cmap, x))
        if not ok.all():
            i = int(np.nonzero(~ok)[0][0])
            log(f"MISMATCH {n_queries} queries, hessian: query {i} x={x[i]!r}: hess {hess[i].tolist()}")
        return n_queries, int((~ok).sum())
    want_phi, want_grad = ref.interpolate(gd, r, nodes, cells, cmap, x, True)
    want_only = ref.interpolate(gd, r, nodes, cells, cmap, x, False)[0]
    f = be.field(gd, r, nodes, cells, cmap)
    try:
        phi, grad = be.interpolate(f, x, True)
        only = be.interpolate(f, x, False)[0]
    finally:
        be.destroy(f)
    ok = same(phi, want_phi) & same(grad, want_grad).all(1) & same(only, want_only)
    if not ok.all():
        i = int(np.nonzero(~ok)[0][0])
        log(f"MISMATCH {n_queries} queries: query {i} x={x[i]!r}: phi {phi[i]!r} vs {want_phi[i]!r}")
    return n_queries, int((~ok).sum())


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 60
    seed = int(argv[2]) if len(argv) > 2 else 0
    mode = argv[4] if len(argv) > 4 else "gradient"
    lib = argv[3] if len(argv) > 3 else os.path.join(ROOT, "build", "bin", "libk2hemu.so" if mode == "hessian" else "libk23emu.so")
    fields, total, bad = run(backend(lib), rounds, seed, mode=mode)
    print(f"{fields} fields, {total} queries, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
