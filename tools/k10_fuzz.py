#!/usr/bin/env python
"""Parity fuzzer for K10 (the mesh distance's forward with weights and its vector-Jacobian product, discregrid_b200/csrc/k10_distance_grad.cu,
radix_sort.cu and K1's mesh_distance_bary_kernel) against the numpy restatement of the contract (tests/mesh_distance_grad_ref.py), bit for bit,
a NaN equal to any NaN (the sign and payload of a NaN made by an invalid operation are not promised); grad_points of a query with t = -1 or
d = 0 must be +0.0 exactly.
  forward  k1_fuzz's tie-rich meshes, scale sweep and awkward meshes (with NaN, infinite and huge queries), in the pseudonormal and the winding
           sign mode, signed and unsigned: fields 0-3 of dg_mesh_distance_bary equal dg_mesh_distance bit for bit, and the weights equal
           gr.weights(gr.leaf_params(...)) on the returned triangle; then the VJP of those outputs
  vjp      synthetic forward outputs (the VJP reads nothing else): meshes of T = 1, 255, 256, 257, 65535, 65536, 65537 triangles (keys of 1, 8,
           9, 16, 17 bits: 1, 2 and 3 sort passes) and happy_buddha.obj where it is staged; triangle ids all equal, all distinct, descending,
           all -1, -1 interleaved, only the low digit varying, only the high digit varying, uniform; n = 0, 1, 31, 32, 33, 1023, 1024, 1025,
           2^17 - 1, 2^17 + 1 (RS_TILE = RS_SCAN_CHUNK = 1024, more than 32 scan chunks)
  segments one segment of 31, 32, 33, 1023, 1024, 1025, 32768, 32769 queries among others (the 32^k boundaries of the level tree); with `dg`
           large, one segment of 2^22 + 1 queries (five levels)
  fan      a vertex shared by 10^4 triangles
  values   g with +-0, subnormals, +-1e308, +-inf, NaN; subnormal d; x - p near overflow
Outputs grad_points (or none) and grad_vertices (or none) against gr.grad_points / gr.grad_vertices.  With `dg` every VJP runs twice through
dg_mesh_distance_vjp, and, with `side`, once more through dg_mesh_distance_vjp_device on a side stream: all must give the same bits.

usage: tools/k10_fuzz.py [rounds=40] [seed=0] [lib=emu]
  rounds  tie-rich meshes for the forward (k1_fuzz.make_case); the other families are fixed lists
  lib     `emu`: build/bin/libdgemu.so (the whole C-ABI emulated on the CPU) for the forward and build/bin/libk10emu.so (emu_k10_vjp, the
          sort and VJP passes alone) for the VJP; or `dg`: the product library through its C-ABI, i.e. the CUDA kernels
The functions are shared with tests/test_mesh_raycast_grad_fuzz_emulated.py and tests/test_gpu_mesh_raycast_grad_fuzz.py."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import k1_fuzz  # noqa: E402
import mesh_distance_grad_ref as gr  # noqa: E402
import winding_ref as wr  # noqa: E402

dp, u32p, i32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
same = k1_fuzz._same
DG_SIGN_PSEUDONORMAL, DG_SIGN_WINDING = 0, 1
TREE_T = (1, 255, 256, 257, 65535, 65536, 65537)
COUNTS = (0, 1, 31, 32, 33, 1023, 1024, 1025, (1 << 17) - 1, (1 << 17) + 1)
SEGMENTS = (31, 32, 33, 1023, 1024, 1025, 32768, 32769)
PATTERNS = ("equal", "distinct", "descending", "none", "none interleaved", "low digit", "high digit", "uniform")


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _dg_calls(lib):
    """the forward and the VJP through a library that exports the C-ABI (the product or libdgemu.so)"""
    class Calls:
        def __init__(self):
            self.lib = lib

        def check(self, rc):
            assert rc == 0, (lib.dg_last_error() or b"").decode()

        def mesh(self, V, F, mode=DG_SIGN_PSEUDONORMAL):
            h = C.c_void_p()
            self.check(lib.dg_mesh_create(_p(V, dp), len(V), _p(F, u32p), len(F), C.byref(h)))
            if mode == DG_SIGN_WINDING:
                self.check(lib.dg_mesh_set_sign_mode(h, DG_SIGN_WINDING, C.c_double(2.0)))
            return h

        def destroy(self, h):
            lib.dg_mesh_destroy(h)

        def distance(self, h, x, signed):
            n = len(x)
            out = np.full(n, 7.0), np.full((n, 3), 7.0), np.full(n, 7, np.int32), np.full(n, 7, np.int32)
            self.check(lib.dg_mesh_distance(h, _p(x, dp), n, int(signed), _p(out[0], dp), _p(out[1], dp), _p(out[2], i32p), _p(out[3], i32p)))
            return out

        def distance_bary(self, h, x, signed):
            n = len(x)
            out = np.full(n, 7.0), np.full((n, 3), 7.0), np.full(n, 7, np.int32), np.full(n, 7, np.int32), np.full((n, 3), 7.0)
            self.check(lib.dg_mesh_distance_bary(h, _p(x, dp), n, int(signed), _p(out[0], dp), _p(out[1], dp), _p(out[2], i32p),
                                                 _p(out[3], i32p), _p(out[4], dp)))
            return out

        def vjp(self, h, nV, q, points, vertices):
            x, d, p, tri, w, g = q
            n = len(x)
            gp = np.full((n, 3), 7.0) if points else None
            gv = np.full((nV, 3), 7.0) if vertices else None
            self.check(lib.dg_mesh_distance_vjp(h, n, _p(x, dp), _p(d, dp), _p(p, dp), _p(tri, i32p), _p(w, dp), _p(g, dp), _p(gp, dp),
                                                _p(gv, dp)))
            return gp, gv
    return Calls()


class EmuK10:
    """build/bin/libdgemu.so for the forward, build/bin/libk10emu.so for the VJP (emu_k10_vjp: the same passes, launched on F directly)"""

    name = "emu"

    def __init__(self, dgemu=None, k10emu=None):
        dgemu = dgemu or os.path.join(ROOT, "build", "bin", "libdgemu.so")
        k10emu = k10emu or os.path.join(ROOT, "build", "bin", "libk10emu.so")
        lib = C.CDLL(dgemu)
        for nm, res, args in (("dg_mesh_create", C.c_int, [dp, C.c_uint64, u32p, C.c_uint64, C.POINTER(C.c_void_p)]),
                              ("dg_mesh_destroy", C.c_int, [C.c_void_p]), ("dg_last_error", C.c_char_p, []),
                              ("dg_mesh_set_sign_mode", C.c_int, [C.c_void_p, C.c_int, C.c_double]),
                              ("dg_mesh_distance", C.c_int, [C.c_void_p, dp, C.c_uint64, C.c_int, dp, dp, i32p, i32p]),
                              ("dg_mesh_distance_bary", C.c_int, [C.c_void_p, dp, C.c_uint64, C.c_int, dp, dp, i32p, i32p, dp]),
                              ("dg_mesh_distance_vjp", C.c_int, [C.c_void_p, C.c_uint64, dp, dp, dp, i32p, dp, dp, dp, dp])):
            f = getattr(lib, nm)
            f.restype, f.argtypes = res, args
        self.fwd = _dg_calls(lib)
        self.k10 = C.CDLL(k10emu)
        self.k10.emu_k10_vjp.argtypes = [C.c_uint64, dp, dp, dp, i32p, dp, dp, u32p, C.c_uint64, C.c_uint64, dp, dp]

    def mesh(self, V, F, mode=DG_SIGN_PSEUDONORMAL):
        return self.fwd.mesh(V, F, mode)

    def destroy(self, h):
        self.fwd.destroy(h)

    def distance(self, h, x, signed):
        return self.fwd.distance(h, x, signed)

    def distance_bary(self, h, x, signed):
        return self.fwd.distance_bary(h, x, signed)

    def vjp_mesh(self, V, F):
        return (len(V), F)                                       # emu_k10_vjp takes the triangles themselves

    def vjp_destroy(self, m):
        pass

    def vjp(self, m, q, points=True, vertices=True):
        nV, F = m
        x, d, p, tri, w, g = q
        n = len(x)
        gp = np.full((n, 3), 7.0) if points else None
        gv = np.full((nV, 3), 7.0) if vertices else None
        assert self.k10.emu_k10_vjp(n, _p(x, dp), _p(d, dp), _p(p, dp), _p(tri, i32p), _p(w, dp), _p(g, dp), _p(F, u32p), len(F), nV,
                                    _p(gp, dp), _p(gv, dp)) == 0
        return gp, gv, True


class DgK10:
    """the product library through its C-ABI.  vjp() calls dg_mesh_distance_vjp twice (and, with side, dg_mesh_distance_vjp_device once on
    a side stream) and reports whether all calls gave the same bits"""

    name = "dg"

    def __init__(self, side=False):
        from discregrid_b200 import _capi
        self.capi = _capi
        self.fwd = _dg_calls(_capi.lib)
        self.side = side

    def mesh(self, V, F, mode=DG_SIGN_PSEUDONORMAL):
        return self.fwd.mesh(V, F, mode)

    def destroy(self, h):
        self.fwd.destroy(h)

    def distance(self, h, x, signed):
        return self.fwd.distance(h, x, signed)

    def distance_bary(self, h, x, signed):
        return self.fwd.distance_bary(h, x, signed)

    def vjp_mesh(self, V, F):
        return (len(V), self.mesh(V, F))

    def vjp_destroy(self, m):
        self.destroy(m[1])

    def vjp(self, m, q, points=True, vertices=True):
        nV, h = m
        gp, gv = self.fwd.vjp(h, nV, q, points, vertices)
        runs = [self.fwd.vjp(h, nV, q, points, vertices)]
        if self.side:
            runs.append(self._side(h, nV, q, points, vertices))
        agree = all(_bits_eq(a, gp) and _bits_eq(b, gv) for a, b in runs)
        return gp, gv, agree

    def _side(self, h, nV, q, points, vertices):
        import torch
        x, d, p, tri, w, g = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in q)
        n = len(q[0])
        gp = torch.full((n, 3), 7.0, dtype=torch.float64, device="cuda") if points else None
        gv = torch.full((nV, 3), 7.0, dtype=torch.float64, device="cuda") if vertices else None
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self.capi.check(self.capi.lib.dg_mesh_distance_vjp_device(
                h, n, x.data_ptr(), d.data_ptr(), p.data_ptr(), tri.data_ptr(), w.data_ptr(), g.data_ptr(),
                gp.data_ptr() if gp is not None else None, gv.data_ptr() if gv is not None else None, s.cuda_stream))
        s.synchronize()
        return (gp.cpu().numpy() if gp is not None else None), (gv.cpu().numpy() if gv is not None else None)


def _bits_eq(a, b):
    if a is None or b is None:
        return a is None and b is None
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


def backend(lib, side=False):
    return DgK10(side) if lib == "dg" else EmuK10()


# ---------------------------------------------------------------------------------------------------------------- checks
def check_vjp(be, m, F, nV, q, label, outputs=((True, True), (True, False), (False, True))):
    """the VJP of the forward outputs q = (x, d, p, tri, w, g) against the restatement -> (values checked, mismatches, first)"""
    x, d, p, tri, w, g = q
    with np.errstate(all="ignore"):
        want_gx = gr.grad_points(x, d, p, tri, g)
        want_gv = gr.grad_vertices(F, nV, tri, want_gx, w)
    total = bad = 0
    first = None
    for points, vertices in outputs:
        gp, gv, agree = be.vjp(m, q, points, vertices)
        for got, want, nm in ((gp, want_gx, "grad_points"), (gv, want_gv, "grad_vertices")):
            if got is None:
                continue
            ok = same(got, want).all(1)
            total += len(ok); bad += int((~ok).sum())
            if not ok.all() and first is None:
                i = int(np.nonzero(~ok)[0][0])
                first = f"MISMATCH {label} {nm} (points={points}, vertices={vertices}) row {i}: {got[i].tolist()!r} vs {want[i].tolist()!r}"
        if not agree:
            bad += 1
            first = first or f"MISMATCH {label} (points={points}, vertices={vertices}): repeated calls differ"
    return total, bad, first


def check_forward(be, V, F, x, label, modes=(DG_SIGN_PSEUDONORMAL, DG_SIGN_WINDING), seed=0):
    """fields 0-3 of dg_mesh_distance_bary == dg_mesh_distance; weights == the restatement's; then the VJP of those outputs"""
    total = bad = 0
    first = None
    rng = np.random.default_rng(seed)
    for mode in modes:
        h = be.mesh(V, F, mode)
        try:
            for signed in (1, 0):
                want = be.distance(h, x, signed)
                r = be.distance_bary(h, x, signed)
                ok = np.ones(len(x), bool)
                for k in range(4):
                    ok &= (np.asarray(r[k]).view(np.uint8).reshape(len(x), -1) == np.asarray(want[k]).view(np.uint8).reshape(len(x), -1)).all(1)
                s, t, _ = gr.leaf_params(V, F, r[3], x)
                ok &= same(r[4], gr.weights(s, t)).all(1)
                total += len(x); bad += int((~ok).sum())
                if not ok.all() and first is None:
                    i = int(np.nonzero(~ok)[0][0])
                    first = (f"MISMATCH {label} mode={mode} signed={signed} x={x[i].tolist()!r}: d {r[0][i]!r} vs {want[0][i]!r}, tri {r[3][i]} vs "
                             f"{want[3][i]}, w {r[4][i].tolist()!r}")
                g = rng.standard_normal(len(x))
                if signed and len(x):
                    q = (x, r[0], r[1], r[3], r[4], g)
                    n, b, msg = check_vjp(be, be.vjp_mesh(V, F) if isinstance(be, EmuK10) else (len(V), h), F, len(V), q, label,
                                          outputs=((True, True),))
                    total += n; bad += b
                    first = first or msg
        finally:
            be.destroy(h)
    return total, bad, first


# ---------------------------------------------------------------------------------------------------------------- cases
def forward_cases(rounds, seed=0, scale_exponents=k1_fuzz.SCALE_EXPONENTS):
    """(label, V, F, x): k1_fuzz's tie-rich meshes, its scale sweep, its awkward meshes with the queries no triangle accepts"""
    rng = np.random.default_rng(seed)
    for k in range(rounds):
        V, F, x = k1_fuzz.make_case(rng, k)
        yield f"case {k} (kind {k % 7}, {len(F)} tris)", V, F, x
    for label, V, F in k1_fuzz.scale_cases(seed, scale_exponents):
        with np.errstate(over="ignore", invalid="ignore"):
            x = k1_fuzz.queries(rng, V, F, flat=0.25)
        yield label, V, F, x
    for n_tri, scale, offset, degenerate in k1_fuzz.AWKWARD:
        V, F, x, lost = k1_fuzz.awkward_case(n_tri, scale, offset, degenerate)
        yield f"awkward {n_tri} x{scale:g}+{offset:g}", V, F, np.ascontiguousarray(np.concatenate([x, lost]))


def soup(rng, T, nV=None):
    """T triangles over few vertices: the VJP reads only the triangles"""
    nV = nV or max(3, min(T, 997))
    V = rng.standard_normal((nV, 3))
    F = rng.integers(0, nV, (T, 3)).astype(np.uint32)
    F[:, 1] = (F[:, 0] + 1 + rng.integers(0, nV - 1, T)) % nV                  # no repeated vertex in most triangles
    return np.ascontiguousarray(V), np.ascontiguousarray(F)


def ids(rng, pattern, n, T):
    if pattern == "equal":
        return np.full(n, T - 1, np.int32)
    if pattern == "distinct":
        return (rng.permutation(max(n, T))[:n] % T).astype(np.int32)
    if pattern == "descending":
        return ((T - 1) - np.arange(n) * max(1, T // max(n, 1)) % T).astype(np.int32)
    if pattern == "none":
        return np.full(n, -1, np.int32)
    if pattern == "none interleaved":
        t = rng.integers(0, T, n).astype(np.int32); t[::2] = -1
        return t
    if pattern == "low digit":
        base = (T - 1) & ~0xff
        return np.minimum(base + rng.integers(0, 256, n), T - 1).astype(np.int32)
    if pattern == "high digit":
        return np.minimum(rng.integers(0, max(1, T >> 8) + 1, n) << 8, T - 1).astype(np.int32)
    return rng.integers(-1, T, n).astype(np.int32)


def synthetic(rng, tri, values=False):
    """forward outputs for triangle ids tri: random x, p, w (finite), d; with values, the awkward g, d and x - p"""
    n = len(tri)
    x = rng.standard_normal((n, 3)); p = rng.standard_normal((n, 3))
    d = rng.standard_normal(n); d[::37] = 0.0
    w = rng.random((n, 3)); g = rng.standard_normal(n)
    w[tri < 0] = np.nan
    if values and n:
        special = np.array([0.0, -0.0, 5e-324, -2.5e-310, 1e308, -1e308, np.inf, -np.inf, np.nan, 1.0])
        g[::3] = special[rng.integers(0, len(special), len(g[::3]))]
        d[1::5] = rng.choice([5e-324, -1e-310, 2.2e-308, 1e-300], len(d[1::5]))
        x[2::7] = 1e308; p[2::7] = -1e308                                           # x - p overflows
        x[3::7] = 8.9e307; p[3::7] = -8.9e307                                       # x - p just below DBL_MAX
        w[4::9] = rng.choice([0.0, -0.0, 1e308, 5e-324], (len(w[4::9]), 3))
    return (np.ascontiguousarray(x), np.ascontiguousarray(d), np.ascontiguousarray(p), np.ascontiguousarray(tri, np.int32),
            np.ascontiguousarray(w), np.ascontiguousarray(g))


def vjp_meshes(seed=0, sizes=TREE_T):
    rng = np.random.default_rng(seed + 21)
    for T in sizes:
        V, F = soup(rng, T)
        yield f"T={T}", V, F
    p = wr.ref_resource(ROOT, "happy_buddha.obj")
    if p and sizes == TREE_T:
        V, F = wr.read_obj(p)
        yield "happy_buddha", V, np.ascontiguousarray(F, np.uint32)


def run_vjp(be, seed=0, log=print, counts=COUNTS, sizes=TREE_T, per_mesh=None):
    """every id pattern at every count on every mesh (per_mesh: only that many (pattern, count) pairs per mesh, rotating) -> (cases, values,
    mismatches)"""
    rng = np.random.default_rng(seed + 23)
    cases = total = bad = 0
    for mi, (label, V, F) in enumerate(vjp_meshes(seed, sizes)):
        m = be.vjp_mesh(V, F)
        try:
            pairs = [(p, n) for p in PATTERNS for n in counts]
            if per_mesh is not None:
                pairs = [pairs[(mi * 7 + 11 * j) % len(pairs)] for j in range(per_mesh)]
            for j, (pattern, n) in enumerate(pairs):
                q = synthetic(rng, ids(rng, pattern, n, len(F)), values=(j % 4 == 3))
                k, b, msg = check_vjp(be, m, F, len(V), q, f"{label} ids {pattern} n={n}", outputs=((True, True), (False, True)))
                cases += 1; total += k; bad += b
                if msg: log(msg)
        finally:
            be.vjp_destroy(m)
    return cases, total, bad


def run_segments(be, seed=0, log=print, lengths=SEGMENTS):
    """one segment of each length, in a shuffled run of other ids, -1 and a fan vertex shared by 10^4 triangles"""
    rng = np.random.default_rng(seed + 25)
    V, F = soup(rng, 10000, nV=600)
    F[:, 0] = 0                                                                      # vertex 0: in every triangle
    F[:, 1] = 1 + rng.integers(0, 599, 10000); F[:, 2] = 1 + (F[:, 1] + rng.integers(0, 598, 10000)) % 599
    m = be.vjp_mesh(V, F)
    cases = total = bad = 0
    try:
        for L in lengths:
            others = rng.integers(-1, len(F), L // 3 + 5).astype(np.int32)
            tri = np.concatenate([np.full(L, int(rng.integers(0, len(F))), np.int32), others])
            tri = tri[rng.permutation(len(tri))]
            for values in (False, True):
                k, b, msg = check_vjp(be, m, F, len(V), synthetic(rng, tri, values), f"segment of {L} (fan), values={values}",
                                      outputs=((True, True),))
                cases += 1; total += k; bad += b
                if msg: log(msg)
    finally:
        be.vjp_destroy(m)
    return cases, total, bad


def run_values(be, seed=0, log=print):
    """the awkward values on a mesh of 257 triangles, uniform and equal ids"""
    rng = np.random.default_rng(seed + 27)
    V, F = soup(rng, 257)
    m = be.vjp_mesh(V, F)
    cases = total = bad = 0
    try:
        for pattern in ("uniform", "equal", "none interleaved"):
            for n in (33, 1025, 5000):
                k, b, msg = check_vjp(be, m, F, len(V), synthetic(rng, ids(rng, pattern, n, len(F)), True), f"values ids {pattern} n={n}")
                cases += 1; total += k; bad += b
                if msg: log(msg)
    finally:
        be.vjp_destroy(m)
    return cases, total, bad


def run_large_segment(be, n=(1 << 22) + 1, seed=0, log=print):
    """one segment of n queries (2^22 + 1: five levels) -> (values, mismatches)"""
    rng = np.random.default_rng(seed + 29)
    V, F = soup(rng, 5)
    tri = np.full(n, 3, np.int32)
    tri[rng.integers(0, n, 1000)] = -1
    m = be.vjp_mesh(V, F)
    try:
        k, b, msg = check_vjp(be, m, F, len(V), synthetic(rng, tri), f"one segment of {n}", outputs=((True, True),))
    finally:
        be.vjp_destroy(m)
    if msg: log(msg)
    return k, b


def run_forward(be, rounds, seed=0, log=print, scale_exponents=k1_fuzz.SCALE_EXPONENTS):
    meshes = total = bad = 0
    for i, (label, V, F, x) in enumerate(forward_cases(rounds, seed, scale_exponents)):
        V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32); x = np.ascontiguousarray(x, np.float64)
        n, b, msg = check_forward(be, V, F, x, label, seed=seed + i)
        meshes += 1; total += n; bad += b
        if msg: log(msg)
    return meshes, total, bad


def run(be, rounds, seed=0, log=print, large=False):
    acc = [0, 0, 0]

    def add(r):
        for i in range(3):
            acc[i] += r[i]
    add(run_forward(be, rounds, seed, log))
    add(run_vjp(be, seed, log))
    add(run_segments(be, seed, log))
    add(run_values(be, seed, log))
    if large:
        k, b = run_large_segment(be, seed=seed, log=log)
        acc[0] += 1; acc[1] += k; acc[2] += b
    return tuple(acc)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 40
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else "emu"
    be = backend(lib, side=(lib == "dg"))
    cases, total, bad = run(be, rounds, seed, large=(lib == "dg"))
    print(f"{cases} cases, {total} values, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
