#!/usr/bin/env python
"""Parity fuzzer for K6 (level sets by marching tetrahedra, discregrid_b200/csrc/k6_isosurface.cu) against the numpy restatement of its
contract (tests/isosurface_ref.py): vertices as uint64 views (any NaN equal to any NaN) and triangles exactly, the restatement run on the
library's own dg_interpolate_batch values at Lattice.points().
  fields    k2_fuzz.make_field grids and fields (anisotropic, offset, tiny and huge cells; DBL_MAX sentinels; +-1e308, -DBL_MAX, NaN, +-inf
            and subnormal coefficients; reduced fields, no kept cell, exactly one) at s = 1, 2, 3, 16; iso 0, quantiles of the lattice values,
            and values near +-DBL_MAX
  cases     high-frequency random node values on small grids: every one of the 16 cases occurs in even and in odd tetrahedra (counted by
            isosurface_ref.case_counts)
  exact     iso equal to lattice values (f_q == iso: coincident vertices, zero-area triangles); iso = +-0.0 on fields with exact zeros
  sizes     n_cells at 1023, 1024, 1025 (and 2047 .. 2049) mod 1024 -- the count and triangle tiles; 7 Np around multiples of 32 (the
            32-edge chunks that flags_before reads as four words) and of 1024 (the vertex tiles); Np = 2^24 (a 17^3 grid at s = 15) and
            Np = 2^24 + 1 (6 x 16 x 42 at s = 16) -- the K6_CHUNK values pass
  clamp     domains where mn + cell * n rounds above mx, so that the clamp of the lattice coordinate is taken; and domains whose max is
            -0.0 on one axis, where mn + cell * n is +0.0 == mx and the clamp must not be taken (iso at values on that max face)
  large     (`dg`) a 54^3 grid at s = 16: 865^3 = 647,214,625 lattice points, edge ids past 2^32.  The field is 1.0 everywhere (phi > 0 by
            partition of unity) but for three groups of cells: near the origin corner, around the lattice point of lin ceil(2^32 / 7), where
            the crossing edges' ids fall on both sides of 2^32, and at the far corner.  The restatement runs on index windows around them
            (isosurface_ref.extract_windows); outside them no tetrahedron changes sign.  Also the refusal of a lattice of 2^31 points or more (81^3 at s = 16)
With `dg` every result is copied back through dg_isosurface_copy and dg_isosurface_copy_device (torch tensors on the device; host memory
on the emulated library), and both must give the same bits.

usage: tools/k6_fuzz.py [rounds=24] [seed=0] [lib=build/bin/libdgemu.so]
  rounds  k2_fuzz.make_field fields; the other families are fixed lists
  lib     build/bin/libdgemu.so (the whole library with its kernels compiled for the CPU, tests/emu) or `dg`: the product library through
          its C-ABI (dg_field_create, dg_isosurface_create, dg_isosurface_copy[_device], dg_interpolate_batch)
The functions are shared with tests/test_isosurface_raycast_fuzz_emulated.py and tests/test_gpu_isosurface_raycast_fuzz.py."""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import isosurface_ref as ir  # noqa: E402
import k2_fuzz  # noqa: E402
from oracle_api import Oracle  # noqa: E402

dp, u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)
DBL_MAX = ir.DBL_MAX
UINT32_MAX = 0xFFFFFFFF
DG_ERR_INVALID = -1
SUBDIVISIONS = (1, 2, 3, 16)
same = k2_fuzz.same


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


class Lib:
    """the library through its C-ABI: `dg` (the product: CUDA kernels on the current device) or the path of build/bin/libdgemu.so"""

    def __init__(self, lib="dg"):
        from discregrid_b200 import _capi
        from discregrid_b200.grid import grid_desc
        self.grid_desc = grid_desc
        if lib == "dg":
            self.name, self.lib, self.emulated = "dg", _capi.lib, _capi.EMULATED
        else:
            self.name, self.lib, self.emulated = os.path.basename(lib), C.CDLL(lib), True
            for nm, (res, args) in _capi.SIGNATURES.items():
                f = getattr(self.lib, nm)
                f.restype, f.argtypes = res, args

    def check(self, rc):
        if rc != 0:
            raise RuntimeError(f"rc {rc}: {self.lib.dg_last_error()}")

    # ---- fields
    def field(self, gd, r, nodes, cells, cmap):
        """a k2_fuzz field (gd: mn, mx, cell, inv) -> (handle, descriptor, the arrays)"""
        return self.field_desc(self.grid_desc(gd[0:3], gd[3:6], r, gd[6:9], gd[9:12]), nodes, cells, cmap)

    def field_desc(self, d, nodes, cells, cmap):
        keep = (np.ascontiguousarray(nodes, np.float64), np.ascontiguousarray(cells, np.uint32), np.ascontiguousarray(cmap, np.uint32))
        h = C.c_void_p()
        self.check(self.lib.dg_field_create(C.byref(d), _p(keep[0], dp) if len(keep[0]) else None, len(keep[0]), _p(keep[1], u32p),
                                            len(keep[1]), _p(keep[2], u32p), C.byref(h)))
        return h, d, keep

    def dense_field(self, mn, mx, res, fn):
        """a dense field whose node values are fn(node positions) -> (handle, descriptor, nodes)"""
        d = self.grid_desc(np.asarray(mn, np.float64), np.asarray(mx, np.float64), res)
        n = C.c_uint64()
        self.check(self.lib.dg_grid_num_nodes(d.resolution, C.byref(n)))
        x = np.empty((n.value, 3))
        self.check(self.lib.dg_node_positions(C.byref(d), 0, n.value, _p(x, dp)))
        nodes = np.ascontiguousarray(fn(x), np.float64)
        h = C.c_void_p()
        self.check(self.lib.dg_field_create(C.byref(d), _p(nodes, dp), len(nodes), None, int(np.prod(np.asarray(res, np.int64))), None,
                                            C.byref(h)))
        return h, d, nodes

    def destroy(self, f):
        self.check(self.lib.dg_field_destroy(f[0]))

    def interpolate(self, f, x, chunk=1 << 22):
        x = np.ascontiguousarray(x, np.float64)
        phi = np.empty(len(x))
        for b in range(0, len(x), chunk):
            e = min(len(x), b + chunk)
            self.check(self.lib.dg_interpolate_batch(f[0], _p(x[b:e], dp), e - b, _p(phi[b:e], dp), None))
        return phi

    # ---- K6
    def create(self, f, iso, s):
        """dg_isosurface_create -> (handle or None, rc)"""
        r = C.c_void_p()
        rc = self.lib.dg_isosurface_create(f[0], float(iso), int(s), C.byref(r), None)
        return (r if rc == 0 else None), rc

    def sizes(self, r):
        nv, nt = C.c_uint64(), C.c_uint64()
        self.check(self.lib.dg_isosurface_sizes(r, C.byref(nv), C.byref(nt)))
        return nv.value, nt.value

    def copy(self, r):
        """(V, T) through dg_isosurface_copy, and whether dg_isosurface_copy_device gave the same bits"""
        nv, nt = self.sizes(r)
        V, T = np.full((nv, 3), 7.0), np.full((nt, 3), 7, np.uint32)
        self.check(self.lib.dg_isosurface_copy(r, _p(V, dp), _p(T, u32p)))
        if self.emulated:                                                 # "device" memory is host memory
            Vd, Td = np.full((nv, 3), 5.0), np.full((nt, 3), 5, np.uint32)
            self.check(self.lib.dg_isosurface_copy_device(r, Vd.ctypes.data if nv else None, Td.ctypes.data if nt else None, None))
        else:
            import torch
            Vt = torch.full((nv, 3), 5.0, dtype=torch.float64, device="cuda")
            Tt = torch.full((nt, 3), 5, dtype=torch.int32, device="cuda")
            st = torch.cuda.current_stream()
            self.check(self.lib.dg_isosurface_copy_device(r, Vt.data_ptr() if nv else None, Tt.data_ptr() if nt else None, st.cuda_stream))
            st.synchronize()
            Vd, Td = Vt.cpu().numpy(), Tt.cpu().numpy().view(np.uint32)
        device_same = np.array_equal(V.view(np.uint64), Vd.view(np.uint64)) and np.array_equal(T, Td)
        return V, T, device_same

    def release(self, r):
        self.check(self.lib.dg_isosurface_destroy(r))

    def extract(self, f, iso, s):
        r, rc = self.create(f, iso, s)
        self.check(rc)
        try:
            return self.copy(r)
        finally:
            self.release(r)


def backend(lib):
    return Lib(lib)


def lattice(d, s):
    return ir.Lattice(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.resolution[:], s)


# ---------------------------------------------------------------------------------------------------------------- comparison
def check(be, f, L, vals, iso, label):
    """one extraction against the restatement -> (1, mismatches, first mismatch, restated triangle count)"""
    V, T, device_same = be.extract(f, iso, L.s)
    Vr, Tr = ir.extract(L, vals, iso)
    ok = V.shape == Vr.shape and same(V, Vr).all() and T.shape == Tr.shape and np.array_equal(T, Tr)
    msg = None
    if not ok:
        msg = f"MISMATCH {label} s={L.s} iso={iso!r}: {len(V)} / {len(Vr)} vertices, {len(T)} / {len(Tr)} triangles"
        if V.shape == Vr.shape:
            bad = np.nonzero(~same(V, Vr).all(1))[0]
            if len(bad):
                msg += f"; vertex {bad[0]} {V[bad[0]].tolist()!r} vs {Vr[bad[0]].tolist()!r}"
        if T.shape == Tr.shape:
            bad = np.nonzero((T != Tr).any(1))[0]
            if len(bad):
                msg += f"; triangle {bad[0]} {T[bad[0]].tolist()} vs {Tr[bad[0]].tolist()}"
    elif not device_same:
        ok, msg = False, f"MISMATCH {label} s={L.s} iso={iso!r}: dg_isosurface_copy_device differs from dg_isosurface_copy"
    return 1, int(not ok), msg, len(Tr)


def isos_of(vals):
    """0, the quartiles of the valid lattice values (0 where there is none), and values near +-DBL_MAX"""
    ok = vals[np.isfinite(vals) & (vals != DBL_MAX)]
    q = [float(np.quantile(ok, p)) if len(ok) else 0.0 for p in (0.25, 0.5, 0.75)]
    return [0.0] + q + [1.6e308, -1e308, DBL_MAX, -DBL_MAX]


def run_checks(be, f, d, plan, label, log, tris=None):
    """plan: [(s, isos or None)] (None: isos_of the lattice values) -> (extractions, mismatches)"""
    total = bad = 0
    for s, isos in plan:
        L = lattice(d, s)
        vals = be.interpolate(f, L.points())
        for iso in (isos_of(vals) if isos is None else isos):
            n, b, msg, nt = check(be, f, L, vals, iso, label)
            total += n; bad += b
            if msg: log(msg)
            if tris is not None:
                tris.append((label, s, iso, nt))
    return total, bad


# ---------------------------------------------------------------------------------------------------------------- families
def run_fields(be, rounds, seed=0, log=print, subdivisions=SUBDIVISIONS, tris=None):
    """k2_fuzz.make_field fields at every s; at s = 16 only iso = 0 and the median -> (fields, extractions, mismatches)"""
    rng = np.random.default_rng(seed)
    orc = Oracle()
    tmp = tempfile.mkdtemp(prefix="k6_fuzz_")
    total = bad = 0
    for k in range(rounds):
        gd, r, nodes, cells, cmap, label = k2_fuzz.make_field(orc, rng, k, tmp)
        f = be.field(gd, r, nodes, cells, cmap)
        try:
            for s in subdivisions:
                L = lattice(f[1], s)
                vals = be.interpolate(f, L.points())
                isos = isos_of(vals)
                if s == 16:
                    isos = [isos[0], isos[2], isos[5]]                       # 0, the median, -1e308
                n, b = run_checks(be, f, f[1], [(s, isos)], label, log, tris)
                total += n; bad += b
        finally:
            be.destroy(f)
    return rounds, total, bad


def run_cases(be, seed=0, log=print, grids=((2, 2, 2), (3, 2, 1), (1, 3, 2)), subdivisions=(1, 2, 3)):
    """high-frequency random node values on small grids -> (fields, extractions, mismatches, case counts (16, 2) summed)"""
    rng = np.random.default_rng(seed + 1)
    counts = np.zeros((16, 2), np.int64)
    total = bad = 0
    for res in grids:
        f = be.dense_field([-1.0, -0.5, 0.0], [1.0, 0.5, 0.75], res, lambda x: rng.standard_normal(len(x)))
        try:
            for s in subdivisions:
                L = lattice(f[1], s)
                vals = be.interpolate(f, L.points())
                for iso in (0.0, float(np.median(vals))):
                    counts += ir.case_counts(L, vals, iso)
                    n, b, msg, _ = check(be, f, L, vals, iso, f"cases {res}")
                    total += n; bad += b
                    if msg: log(msg)
        finally:
            be.destroy(f)
    return len(grids), total, bad, counts


def run_exact(be, seed=0, log=print):
    """iso equal to lattice values (coincident vertices); iso = +0.0 and -0.0 on a field that is exactly 0 on a block of cells.  K2 never
    returns -0.0 (its sum starts at +0.0), so iso = -0.0 against +0.0 values stands in for iso = 0.0 against -0.0 values: both test that
    f < iso is strict on signed zeros -> (fields, extractions, mismatches, lattice values equal to the iso used)"""
    rng = np.random.default_rng(seed + 2)
    total = bad = hits = 0

    def zero_block(x):
        v = np.linalg.norm(x - [0.1, -0.05, 0.2], axis=1) - 0.5
        v[(np.abs(x) <= 0.5).all(1)] = 0.0
        return v
    for label, res, fn in (("sphere", (6, 6, 6), lambda x: np.linalg.norm(x - [0.03, -0.02, 0.01], axis=1) - 0.6),
                           ("zero block", (4, 4, 4), zero_block),
                           ("random", (3, 3, 3), lambda x: np.round(rng.standard_normal(len(x)), 1))):
        f = be.dense_field([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0], res, fn)
        try:
            for s in (1, 2, 3):
                L = lattice(f[1], s)
                vals = be.interpolate(f, L.points())
                ok = vals[np.isfinite(vals)]
                near = ok[np.argsort(np.abs(ok))[:len(ok) // 3]]
                isos = [0.0, -0.0] + [float(v) for v in rng.choice(near, 4, replace=False)]
                for iso in isos:
                    hits += int((vals == iso).sum())
                    n, b, msg, _ = check(be, f, L, vals, iso, f"exact {label}")
                    total += n; bad += b
                    if msg: log(msg)
        finally:
            be.destroy(f)
    return 3, total, bad, hits


def size_plan():
    """(label, res, s): n_cells at -1, 0, +1 mod 1024 (1023 .. 1025 and 2047 .. 2049), 7 Np at -1, 0, +1 mod 32 and mod 1024, Np = 2^24
    and 2^24 + 1"""
    out = [("n_cells 1023", (3, 11, 31), 1), ("n_cells 1024", (4, 4, 8), 2), ("n_cells 1025", (5, 5, 41), 1),
           ("n_cells 2047", (1, 23, 89), 1), ("n_cells 2048", (4, 8, 8), 2), ("n_cells 2049", (1, 3, 683), 1)]
    want = {(32, -1): None, (32, 0): None, (32, 1): None, (1024, -1): None, (1024, 0): None, (1024, 1): None}
    for s in (1, 2, 3):
        for a in range(1, 12):
            for b in range(a, 12):
                for c in range(b, 40):
                    e = 7 * (s * a + 1) * (s * b + 1) * (s * c + 1)
                    for (m, r) in want:
                        if want[(m, r)] is None and (e - r) % m == 0 and e > 2 * m:
                            want[(m, r)] = ((a, b, c), s, e)
    for (m, r), (res, s, e) in sorted(want.items()):
        out.append((f"7 Np = {e} ({r:+d} mod {m})", res, s))
    out += [("Np = 2^24", (17, 17, 17), 15), ("Np = 2^24 + 1", (6, 16, 42), 16)]
    return out


def run_sizes(be, log=print, big=True, tris=None):
    """the size plan on a sphere whose surface crosses the top face (the last values chunk has crossings), at iso 0 and (on the small
    lattices, some of which are one cell thick) the median of the lattice values -> (fields, extractions, mismatches)"""
    total = bad = fields = 0
    for label, res, s in size_plan():
        if not big and label.startswith("Np"):
            continue
        ext = np.asarray(res, np.float64) / max(res)
        fn = lambda x, ext=ext: np.linalg.norm((x - ext * [0.5, 0.5, 0.9]) / ext, axis=1) - 0.35
        f = be.dense_field([0.0, 0.0, 0.0], ext, res, fn)
        try:
            L = lattice(f[1], s)
            vals = be.interpolate(f, L.points())
            for iso in ((0.0,) if L.n_points > 1 << 20 else (0.0, float(np.median(vals)))):
                n, b, msg, nt = check(be, f, L, vals, iso, f"size {label} res {res}")
                total += n; bad += b
                if msg: log(msg)
                if tris is not None:
                    tris.append((label, s, iso, nt))
        finally:
            be.destroy(f)
        fields += 1
    return fields, total, bad


def clamp_domains(rng, count=6):
    """(mn, mx, res, s) whose lattice coordinate mn + cell * (I / s) rounds above mx on some axis"""
    from discregrid_b200.grid import grid_desc
    out = []
    while len(out) < count:
        res = tuple(int(v) for v in rng.integers(1, 7, 3))
        sc = 10.0 ** rng.integers(-3, 4)
        mn = rng.standard_normal(3) * sc * 10.0 ** rng.integers(0, 4)
        mx = mn + sc * (0.1 + rng.random(3))
        d = grid_desc(mn, mx, res)
        for s in (1, 3):
            L = ir.Lattice(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.resolution[:], s)
            raw = [L.mn[a] + L.cell[a] * (np.arange(L.np[a]) / float(s)) for a in range(3)]
            if any((raw[a] > L.mx[a]).any() for a in range(3)):
                out.append((mn, mx, res, s))
                break
    return out


def run_clamp(be, seed=0, log=print, count=6):
    """clamp_domains, then run_zero_max -> (fields, extractions, mismatches)"""
    rng = np.random.default_rng(seed + 3)
    total = bad = 0
    for mn, mx, res, s in clamp_domains(rng, count):
        c = 0.5 * (mn + mx) + 0.2 * (mx - mn)                               # off centre: the surface reaches the max faces
        f = be.dense_field(mn, mx, res, lambda x: np.linalg.norm((x - c) / (mx - mn), axis=1) - 0.4)
        try:
            n, b = run_checks(be, f, f[1], [(s, None)], f"clamp {res} mn {mn.tolist()}", log)
            total += n; bad += b
        finally:
            be.destroy(f)
    fields, n, b = run_zero_max(be, seed, log)
    return count + fields, total + n, bad + b


def run_zero_max(be, seed=0, log=print):
    """a domain whose max is -0.0 on one axis: mn + cell * n computes to +0.0 there, which equals mx, so the lattice coordinate keeps its
    +0.0 while a clamp taken on equality would give -0.0.  iso equal to values on that max face: an edge in the face whose lower end p has
    f_p == iso and whose upper end is negative has t = +0.0 / (f_q - f_p) = -0.0, and its vertex's coordinate on that axis is
    x_p + (-0.0 * 0.0), whose sign is x_p's -> (fields, extractions, mismatches)"""
    rng = np.random.default_rng(seed + 4)
    total = bad = 0
    for a in range(3):
        mx = np.ones(3); mx[a] = -0.0
        b, c = (a + 1) % 3, (a + 2) % 3
        f = be.dense_field([-1.0, -1.0, -1.0], mx, (4, 4, 4), lambda x: 0.37 * x[:, c] - x[:, b] + 0.05 * x[:, a])
        try:
            assert np.signbit(f[1].domain_max[a]), "the descriptor must keep the -0.0 maximum"
            for s in (1, 2):
                L = lattice(f[1], s)
                raw = L.mn[a] + L.cell[a] * (np.arange(L.np[a]) / float(s))
                assert raw[-1] == 0.0 and not np.signbit(raw[-1]), raw[-1]      # the top coordinate is +0.0, equal to mx = -0.0
                vals = be.interpolate(f, L.points())
                face = vals.reshape(L.np[2], L.np[1], L.np[0])[tuple(slice(-1, None) if k == 2 - a else slice(None) for k in range(3))]
                isos = [float(v) for v in rng.choice(np.unique(face), 6, replace=False)]
                for iso in isos:
                    n, m, msg, _ = check(be, f, L, vals, iso, f"max -0.0 on axis {a}")
                    total += n; bad += m
                    if msg: log(msg)
        finally:
            be.destroy(f)
    return 3, total, bad


# ---------------------------------------------------------------------------------------------------------------- large lattice
LARGE_RES, LARGE_S = (54, 54, 54), 16            # 865^3 = 647,214,625 lattice points, 4,530,502,375 edge ids
LARGE_BYTES = 12 << 30                           # values, flags, counts, chunk ranks, one positions chunk
REFUSED_RES = (81, 81, 81)                       # 1297^3 = 2,181,825,073 >= 2^31 at s = 16


def large_groups(res=LARGE_RES, s=LARGE_S):
    """grid cells whose 32 nodes turn negative: near the origin corner, the cell holding the lattice point of lin ceil(2^32 / 7) (7 lin + d
    passes 2^32 there), at the far corner.  phi is -1 on a whole such cell, so its crossing edges lie in the neighbouring cells; around the
    middle group their ids fall on both sides of 2^32 (run_large checks that)"""
    np_ = [s * r + 1 for r in res]
    lin = -(-(1 << 32) // 7)
    P = (lin % np_[0], (lin // np_[0]) % np_[1], lin // (np_[0] * np_[1]))
    return [(1, 1, 1), tuple(int(v) // s for v in P), tuple(r - 1 for r in res)], P


def run_large(be, log=print, res=LARGE_RES, s=LARGE_S):
    """-> (extractions, mismatches, largest edge id, restated triangles); skips (returns None) when the device lacks 2x LARGE_BYTES"""
    if not be.emulated:
        import torch
        free, _ = torch.cuda.mem_get_info()
        if free < 2 * LARGE_BYTES:
            log(f"large lattice skipped: {free / 2**30:.1f} GB free on the device, {2 * LARGE_BYTES / 2**30:.0f} GB wanted")
            return None
    orc = Oracle()
    gd, r = orc.grid_desc(np.zeros(3), np.asarray(res, np.float64) / max(res), res)
    cells = orc.build_cells(r)
    nodes = np.ones(int(cells.max()) + 1)
    groups, P = large_groups(res, s)
    n = np.asarray(res, np.int64)
    for g in groups:
        lin = g[0] + n[0] * (g[1] + n[1] * g[2])
        nodes[cells[lin]] = -1.0                                             # the 32 nodes of one cell: phi < 0 around its centre
    f = be.field(gd, r, nodes, cells, np.arange(len(cells), dtype=np.uint32))
    try:
        L = lattice(f[1], s)
        windows = []
        for g in groups:                                                     # cells g - 2 .. g + 2: the changed nodes reach g +- 1
            lo = np.array([max(0, (c - 2) * s) for c in g]); hi = np.array([min(s * n[a], (g[a] + 3) * s) for a, c in enumerate(g)])
            W = ir.Lattice(np.zeros(3), np.zeros(3), np.zeros(3), hi - lo, 1)
            I, J, K = W.unlin(np.arange(W.n_points))
            pts = np.stack([L.coord(0, I + lo[0]), L.coord(1, J + lo[1]), L.coord(2, K + lo[2])], axis=1)
            windows.append((lo, hi, be.interpolate(f, pts)))
        Vr, Tr, E = ir.extract_windows(L, windows, 0.0)
        emax = int(E.max())
        Em = ir.extract_windows(L, windows[1:2], 0.0)[2]                    # the middle group alone
        below, above = int((Em < 1 << 32).sum()), int((Em >= 1 << 32).sum())
        log(f"large lattice {L.np.tolist()}: {L.n_points} points, {7 * L.n_points} edge ids; groups at cells {groups} (lattice point "
            f"{tuple(int(v) for v in P)}); restated {len(Vr)} vertices, {len(Tr)} triangles, largest edge id {emax} (2^32 = {1 << 32}); "
            f"the middle group's crossing edges: {below} below 2^32 (largest {int(Em[Em < 1 << 32].max()) if below else None}), {above} at or "
            f"above (smallest {int(Em[Em >= 1 << 32].min()) if above else None})")
        h, rc = be.create(f, 0.0, s)
        be.check(rc)
        try:
            nv, nt = be.sizes(h)
            V, T, device_same = be.copy(h)
        finally:
            be.release(h)
        bad = int(not ((nv, nt) == (len(Vr), len(Tr)) and same(V, Vr).all() and np.array_equal(T, Tr) and device_same and below and above))
        if bad:
            log(f"MISMATCH large lattice: {nv} / {len(Vr)} vertices, {nt} / {len(Tr)} triangles, device copy same: {device_same}, "
                f"middle group's edge ids on both sides of 2^32: {bool(below and above)}")
    finally:
        be.destroy(f)
    return 1, bad, emax, len(Tr)


def run_refusal(be, log=print, res=REFUSED_RES):
    """a lattice of 2^31 points or more is refused, with no handle -> (1, mismatches)"""
    d = be.grid_desc(np.zeros(3), np.ones(3), res)
    cells = np.zeros((1, 32), np.uint32)
    cmap = np.full(int(np.prod(np.asarray(res, np.int64))), UINT32_MAX, np.uint32)
    h = C.c_void_p()
    be.check(be.lib.dg_field_create(C.byref(d), None, 0, _p(cells, u32p), 0, _p(cmap, u32p), C.byref(h)))
    try:
        r = C.c_void_p()
        rc = be.lib.dg_isosurface_create(h, 0.0, 16, C.byref(r), None)
        ok = rc == DG_ERR_INVALID and not r.value and b"2^31" in be.lib.dg_last_error()
    finally:
        be.lib.dg_field_destroy(h)
    if not ok:
        log(f"MISMATCH {res} at s = 16 was not refused (rc {rc})")
    return 1, int(not ok)


def run(be, rounds, seed=0, log=print, large=False):
    """every family through backend `be` -> (fields, extractions, mismatches)"""
    acc = [0, 0, 0]
    for r in (run_fields(be, rounds, seed, log), run_cases(be, seed, log)[:3], run_exact(be, seed, log)[:3], run_sizes(be, log),
              run_clamp(be, seed, log)):
        for i in range(3):
            acc[i] += r[i]
    if large:
        r = run_large(be, log)
        if r:
            acc[0] += 1; acc[1] += r[0]; acc[2] += r[1]
        n, b = run_refusal(be, log)
        acc[1] += n; acc[2] += b
    return tuple(acc)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 24
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else os.path.join(ROOT, "build", "bin", "libdgemu.so")
    fields, total, bad = run(backend(lib), rounds, seed, large=lib == "dg")
    print(f"{fields} fields, {total} extractions, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
