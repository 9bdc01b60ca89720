#!/usr/bin/env python
"""Parity fuzzer for K9 (first hits of rays on a mesh, discregrid_b200/csrc/k9_mesh_raycast.cu) against the brute-force numpy restatement of
its contract (tests/mesh_raycast_ref.py), on all four outputs: t and barycentric bit for bit (a NaN of a hit equal to any NaN; a miss's
weights must be 0x7ff8000000000000), triangle id and status exactly.
  trees   T = 1, 2, 3 and 2^k - 1, 2^k, 2^k + 1 for k <= 12 (a perfect tree fills the walk's stack), and happy_buddha.obj where it is staged
  ties    k1_fuzz.make_case meshes and coplanar grids (flat and tilted) with their triangle ids shuffled against the tree's leaf order; stacked
          duplicates (the lower id wins at equal t); k5_fuzz.zero_area_case; rays aimed at shared vertices, edge points and centroids, rays in
          a triangle's plane; and a flat grid too small for an fp32 half extent (no culling slack along z) cast from its own plane, where every
          accepted triangle has t = 0 and a pushed subtree enters at exactly t = 0
  slack   meshes built so that an fp32 child box, rounded outward from a double difference that was itself rounded, lies 1 - 2 ulp inside
          the vertex it bounds; rays through that vertex along an axis are culled unless the 2^-50 slack covers the gap
  scales  10^-45 .. 10^-38 (half_extent subnormal or 0 in fp32), 10^-24 .. 10^17 and 10^+-100, 10^+-150, centred and offset, with scaled and
          unit directions; the restatement's hit count must be > 0 (a sweep of misses only tests nothing)
  cull    origins and meshes at 2^1019, 2^1020, 2^1021 (culling switches off above 2^1020), and direction components so small that Sz is inf
  nonfinite  k5_fuzz.nonfinite_cases (NaN / inf vertices), and NaN, +-inf, zero and huge ray components
  bounds  [0, inf), [-inf, inf), [0, 1], [-0.5, 2], t_min = t_max at a hit's t, t_max just below every hit
  counts  the first 1, 127, 128, 129, 257 rays alone give the bits of the whole call
  refits  (`dg`) refit to scaled, mirrored, translated positions, a subtree collapsed to a point, one vertex NaN and back; cast after each
  large   (`dg`) one call of 2^22 rays on bunny.obj (a bumpy torus where it is not staged), a sample against the restatement
With `dg` every cast also runs through dg_mesh_raycast_device (torch tensors on the current stream; host memory on the emulated library) and
must give the bits of dg_mesh_raycast.

usage: tools/k9_fuzz.py [rounds=40] [seed=0] [lib=build/bin/libk9emu.so]
  rounds  tie-rich meshes (k1_fuzz.make_case); the other families are fixed lists
  lib     build/bin/libk9emu.so or libk9emu_nocull.so (tests/emu/k9_emu.cpp: the K9 translation unit compiled for the CPU, with culling and
          without), or `dg`: the product library through its C-ABI (dg_mesh_create, dg_mesh_raycast[_device], dg_mesh_refit)
The functions are shared with tests/test_mesh_raycast_grad_fuzz_emulated.py and tests/test_gpu_mesh_raycast_grad_fuzz.py."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import k1_fuzz  # noqa: E402
import k5_fuzz  # noqa: E402
import mesh_raycast_ref as mr  # noqa: E402
import winding_ref as wr  # noqa: E402

dp, u32p, i32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
INF = np.inf
MISS_BARY = np.uint64(0x7ff8000000000000)
COUNTS = (1, 127, 128, 129, 257)                     # around K9_THREADS = 128
BOUNDS = ((0.0, INF), (-INF, INF), (0.0, 1.0), (-0.5, 2.0))
same = k1_fuzz._same
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


class EmuK9:
    """a build of tests/emu/k9_emu.cpp: the K9 kernel and launcher run on the CPU"""

    def __init__(self, so):
        self.name = os.path.basename(so)
        lib = self.lib = C.CDLL(so)
        lib.emu_k9_create.restype = C.c_void_p
        lib.emu_k9_create.argtypes = [dp, C.c_uint64, u32p, C.c_uint64]
        lib.emu_k9_destroy.argtypes = [C.c_void_p]
        lib.emu_k9_raycast.argtypes = [C.c_void_p, dp, dp, C.c_uint64, C.c_double, C.c_double, dp, i32p, dp, i32p]

    def mesh(self, V, F):
        h = self.lib.emu_k9_create(_p(V, dp), len(V), _p(F, u32p), len(F))
        assert h
        return h

    def destroy(self, h):
        self.lib.emu_k9_destroy(h)

    def cast(self, h, o, d, lo, hi):
        n = len(o)
        t, tid, b, st = np.full(n, 7.0), np.full(n, 7, np.int32), np.full((n, 3), 7.0), np.full(n, 7, np.int32)
        assert self.lib.emu_k9_raycast(h, _p(o, dp), _p(d, dp), n, lo, hi, _p(t, dp), _p(tid, i32p), _p(b, dp), _p(st, i32p)) == 0
        return t, tid, b, st


class DgK9(k1_fuzz.DgK1):
    """the product library through its C-ABI: the CUDA kernels on the current device.  cast() runs the host and the device form and
    returns the host form's result with a flag: both forms gave the same bits"""

    def cast(self, h, o, d, lo, hi):
        n = len(o)
        t, tid, b, st = np.full(n, 7.0), np.full(n, 7, np.int32), np.full((n, 3), 7.0), np.full(n, 7, np.int32)
        self.capi.check(self.lib.dg_mesh_raycast(h, _p(o, dp), _p(d, dp), n, lo, hi, _p(t, dp), _p(tid, i32p), _p(b, dp), _p(st, i32p)))
        dev = self.cast_device(h, o, d, lo, hi)
        self.device_same = all(np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)) for x, y in zip(dev, (t, tid, b, st)))
        return t, tid, b, st

    def cast_device(self, h, o, d, lo, hi):
        n = len(o)
        if self.capi.EMULATED:                                   # "device" memory is host memory
            out = np.full(n, 7.0), np.full(n, 7, np.int32), np.full((n, 3), 7.0), np.full(n, 7, np.int32)
            self.capi.check(self.lib.dg_mesh_raycast_device(h, o.ctypes.data, d.ctypes.data, n, lo, hi, *(a.ctypes.data for a in out), None))
            return out
        import torch
        ot, dt = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
        out = (torch.full((n,), 7.0, dtype=torch.float64, device="cuda"), torch.full((n,), 7, dtype=torch.int32, device="cuda"),
               torch.full((n, 3), 7.0, dtype=torch.float64, device="cuda"), torch.full((n,), 7, dtype=torch.int32, device="cuda"))
        self.capi.check(self.lib.dg_mesh_raycast_device(h, ot.data_ptr(), dt.data_ptr(), n, lo, hi, *(a.data_ptr() for a in out),
                                                        torch.cuda.current_stream().cuda_stream))
        return tuple(a.cpu().numpy() for a in out)

    def refit(self, h, V):
        self.capi.check(self.lib.dg_mesh_refit(h, _p(V, dp), len(V)))


def backend(lib):
    return DgK9() if lib == "dg" else EmuK9(lib)


# ---------------------------------------------------------------------------------------------------------------- comparison
def compare(got, want):
    """per ray: all four outputs equal (t, barycentric: bits, any NaN of a hit equal to any NaN; a miss's weights exactly 0x7ff8...)"""
    t, tid, b, st = got
    wt, wid, wb, wst = want
    miss = wst == mr.MISS
    ok = same(t, wt) & (tid == wid) & (st == wst) & same(b, wb).all(1)
    ok &= ~miss | (b.view(np.uint64) == MISS_BARY).all(1)
    return ok


def check(be, h, V, F, o, d, lo, hi, label, counts=()):
    """one cast against the restatement (and, with counts, each prefix alone against the whole call) -> (rays, mismatches, first, want)"""
    o = np.ascontiguousarray(o, np.float64); d = np.ascontiguousarray(d, np.float64)
    want = mr.raycast(V, F, o, d, lo, hi)
    got = be.cast(h, o, d, lo, hi)
    ok = compare(got, want)
    total, bad, first = len(o), int((~ok).sum()), None
    if not ok.all():
        i = int(np.nonzero(~ok)[0][0])
        first = (f"MISMATCH {label} on [{lo!r}, {hi!r}] ray {i} o={o[i].tolist()!r} d={d[i].tolist()!r}: t {got[0][i]!r} vs {want[0][i]!r}, "
                 f"id {got[1][i]} vs {want[1][i]}, status {got[3][i]} vs {want[3][i]}, bary {got[2][i].tolist()!r} vs {want[2][i].tolist()!r}")
    if not getattr(be, "device_same", True):
        bad += 1; first = first or f"MISMATCH {label} on [{lo!r}, {hi!r}]: dg_mesh_raycast_device differs from dg_mesh_raycast"
    for c in counts:
        if c <= len(o):
            pre = be.cast(h, o[:c], d[:c], lo, hi)
            okc = np.ones(c, bool)
            for x, y in zip(pre, got):
                okc &= (np.asarray(x).view(np.uint8).reshape(c, -1) == np.asarray(y)[:c].view(np.uint8).reshape(c, -1)).all(1)
            total += c; bad += int((~okc).sum())
            if not okc.all() and first is None:
                first = f"MISMATCH {label} count {c}: first bad ray {int(np.nonzero(~okc)[0][0])}"
    return total, bad, first, want


# ---------------------------------------------------------------------------------------------------------------- rays
def feature_rays(V, F, rng, n):
    """rays from around the mesh aimed exactly at vertices, edge points (midpoints and random) and centroids"""
    E = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]).astype(np.int64)
    s = rng.random((len(E), 1))
    with np.errstate(all="ignore"):
        targets = np.concatenate([V, 0.5 * (V[E[:, 0]] + V[E[:, 1]]), V[E[:, 0]] + s * (V[E[:, 1]] - V[E[:, 0]]), V[F].mean(1)])
    targets = targets[rng.integers(0, len(targets), n)]
    o, _ = mr.random_rays(V, n, rng, 2.0)
    return o, targets - o


def mixed_rays(V, F, rng, n):
    """random, aimed, axis-aligned, in-plane and feature rays: about 2.5 n"""
    Vf = np.where(np.isfinite(V), V, 0.0)
    with np.errstate(all="ignore"):
        parts = [mr.random_rays(Vf, n, rng), mr.aimed_rays(Vf, F, n // 2, rng), mr.axis_rays(Vf, n // 4, rng),
                 mr.in_plane_rays(Vf, F, n // 4, rng), feature_rays(Vf, F, rng, n // 2)]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def shuffled(rng, F):
    """the triangles in a random id order, so that ids and the tree's leaf order disagree"""
    return np.ascontiguousarray(F[rng.permutation(len(F))])


# ---------------------------------------------------------------------------------------------------------------- cases
# a case: (label, V, F, o, d, bounds)
def sphere():
    return wr.read_obj(os.path.join(GOLDEN, "sphere.obj"))


def tree_cases(seed=0, sizes=k5_fuzz.TREE_SIZES, n=60):
    rng = np.random.default_rng(seed + 11)
    for label, V, F, _ in k5_fuzz.tree_cases(seed, sizes):
        o, d = mixed_rays(V, F, rng, n)
        yield label, V, F, o, d, ((0.0, INF),)


def buddha_case(seed=0, n=80):
    p = wr.ref_resource(ROOT, "happy_buddha.obj")
    if p:
        V, F = wr.read_obj(p)
        o, d = mixed_rays(V, F, np.random.default_rng(seed), n)
        yield "happy_buddha", V, F, o, d, ((0.0, INF),)


def tiny_flat_case(rng, scale=1e-46):
    """a 4 x 4 coplanar grid in z = 0 whose half extent rounds to 0 in fp32, so that the box slack along z is 0; rays cast from points of
    its plane (vertices, edge points, interior) with kz = z: every accepted triangle has t = +-0, the subtrees enter at exactly t = 0, and
    at a shared vertex or edge the lowest id must still be found in a pushed subtree"""
    V, F = mr.grid_mesh(4, tilt=False)
    V = np.ascontiguousarray(V * scale)
    F = shuffled(rng, F)
    E = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]).astype(np.int64)
    on = np.concatenate([V, 0.5 * (V[E[:, 0]] + V[E[:, 1]]), V[F].mean(1)])
    o = np.repeat(on, 3, axis=0)
    d = np.tile(np.array([[0.0, 0.0, 1.0], [0.3, -0.2, -1.0], [-0.1, 0.25, 2.0]]), (len(on), 1))
    return V, F, o, d


def tie_cases(rounds, seed=0, n=80):
    """k1_fuzz.make_case meshes (every other one with shuffled ids), coplanar grids, stacked duplicates, zero-area triangles, the tiny
    flat grid"""
    rng = np.random.default_rng(seed)
    for k in range(rounds):
        V, F, _ = k1_fuzz.make_case(rng, k)
        if k % 2:
            F = shuffled(rng, F)
        o, d = mixed_rays(V, F, rng, n)
        yield f"case {k} (kind {k % 7}, {len(F)} tris)", V, F, o, d, BOUNDS[k % 4:k % 4 + 1]
        if k % 7 == 6:
            V, F, _ = k5_fuzz.zero_area_case(rng)
            o, d = mixed_rays(V, F, rng, n)
            yield f"case {k} zero-area", V, F, o, d, ((0.0, INF),)
    for tilt in (False, True):
        V, F = mr.grid_mesh(6, tilt)
        F = shuffled(rng, F)
        o, d = mixed_rays(V, F, rng, 3 * n)
        yield f"grid tilt={tilt}", V, F, o, d, ((0.0, INF), (-INF, INF))
        F2 = np.ascontiguousarray(np.concatenate([F, F, F[:, [1, 2, 0]]]))      # duplicates: identical t, the lower id wins
        o, d = feature_rays(V, F2, rng, 3 * n)
        yield f"grid tilt={tilt} stacked duplicates", V, F2, o, d, ((0.0, INF),)
    V, F = sphere()
    F2 = shuffled(rng, np.concatenate([F, F, F[:, [2, 0, 1]]]))
    o, d = mixed_rays(V, F2, rng, 2 * n)
    yield "sphere stacked duplicates, shuffled", V, F2, o, d, ((0.0, INF), (-INF, INF))
    for s in (1e-46, 3e-47):
        V, F, o, d = tiny_flat_case(rng, s)
        yield f"flat grid x{s:g} from its plane", V, F, o, d, ((0.0, INF), (-INF, INF), (0.0, 0.0))


def _rec_down(x):
    f = np.float32(x)
    return np.nextafter(f, np.float32(-np.inf)) if float(f) > x else f


def slack_cases():
    """two-triangle meshes whose box centre c is fixed by a wide frame triangle, and a small triangle whose lowest vertex coordinate b
    (on axis a) makes fl(b - c) round up onto an fp32 value: the child box's lo_f is then above the exact b - c, and only the slack keeps
    the box around the vertex.  Rays through b along the other axes"""
    from fractions import Fraction
    for a in range(3):
        for C0, F0 in ((1000.0, -999.5), (3.0e5, -299999.75), (1.0, -0.75)):
            half = np.spacing(abs(F0)) / 2
            for k in (0.9, 0.6):
                b = 0.0 + (C0 + F0) - k * half                  # fl(b - C0) == F0 although b - C0 < F0
                if float(b - C0) != F0 or Fraction(b) - Fraction(C0) >= Fraction(F0) or float(_rec_down(b - C0)) != F0:
                    continue
                P = np.zeros((6, 3))
                P[0, a], P[1, a], P[2, a] = 0.0, 2 * C0, C0                       # the frame: spans [0, 2 C0] on axis a
                e1, e2 = (a + 1) % 3, (a + 2) % 3
                P[0:3, e1] = -5.0; P[2, e2] = 1.0
                P[3, a], P[4, a], P[5, a] = b, b, b + 0.5                         # the small triangle: an edge at coordinate b
                P[3, e1], P[4, e1], P[5, e1] = 1.0, 3.0, 2.0
                P[3, e2], P[4, e2], P[5, e2] = 0.0, 0.0, 0.0
                F = np.array([[0, 1, 2], [3, 4, 5]], np.uint32)
                m = 24
                o = np.zeros((m, 3)); d = np.zeros((m, 3))
                o[:, a] = b
                o[:, e1] = np.linspace(1.0, 3.0, m)
                o[:, e2] = 2.0
                d[:, e2] = -1.0
                d[::3, e1] = 1e-3                                                 # and a slightly slanted one
                yield f"slack axis {a} c={C0:g} f={F0:g} k={k}", P, F, o, d, ((0.0, INF),)


SCALE_EXPONENTS = tuple(range(-45, -37)) + tuple(range(-24, 18)) + (-150, -100, 100, 150)


def scale_cases(seed=0, exponents=SCALE_EXPONENTS, n=40):
    """(label, V, F, o, d, bounds, hits_required) of sphere.obj at 10^k: centred, offset by 0.3 and by 10^3 of its size, with directions
    scaled along and of unit length"""
    V0, F = sphere()
    V0 = V0 - 0.5 * (V0.min(0) + V0.max(0))
    rng = np.random.default_rng(seed + 3)
    o0, d0 = mixed_rays(V0, F, rng, n)
    for k in exponents:
        s = 10.0 ** k
        for off in (0.0, 0.3, 1e3):
            for unit in (False, True):
                with np.errstate(all="ignore"):
                    V = (V0 + off) * s
                    o = (o0 + off) * s
                    d = d0 / np.linalg.norm(d0, axis=1, keepdims=True) if unit else d0 * s
                yield f"sphere@1e{k} off {off:g} {'unit' if unit else 'scaled'} d", np.ascontiguousarray(V), F, o, d, ((0.0, INF),)


def cull_cases(seed=0):
    """origins at 2^1019, 2^1020, 2^1021 aimed at a unit mesh (culling on, on the boundary, off); meshes placed at those coordinates; and
    directions whose largest component is subnormal (Sz = 1 / d[kz] = inf switches culling off) or tiny but normal"""
    rng = np.random.default_rng(seed + 5)
    V, F = sphere()
    for e in (1019, 1020, 1021):
        big = 2.0 ** e
        for axis in range(3):
            for sgn in (1.0, -1.0):
                targets = V[rng.integers(0, len(V), 16)] * rng.random((16, 1))
                o = np.zeros((16, 3)); o[:, axis] = sgn * big
                o[1::2, (axis + 1) % 3] = 0.25
                yield f"origins at {'-' if sgn < 0 else ''}2^{e} on axis {axis}", V, F, o, targets - o, ((0.0, INF), (-INF, INF))
        for spread in (2.0 ** (e - 30), 2.0 ** (e - 2)):
            Vb = V * spread + big
            o, d = mixed_rays(Vb, F, rng, 20)
            yield f"mesh at 2^{e}, size {spread:g}", np.ascontiguousarray(Vb), F, o, d, ((0.0, INF),)
    o, d = mixed_rays(V, F, rng, 40)
    for tiny in (5e-324, 1e-310, 2.2250738585072014e-308, 1e-300):
        dd = d / np.abs(d).max(1, keepdims=True) * tiny
        yield f"directions scaled to {tiny:g}", V, F, o, np.ascontiguousarray(dd), ((0.0, INF), (-INF, INF))


SPECIAL_O = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e308, 0, 0], [-1.7976931348623157e308, 1e308, 0], [0, 0, 0],
                      [0.1, 0.2, 0.3], [1e300, 1e300, 1e300], [0.0, -0.0, 0.0]])
SPECIAL_D = np.array([[0, 0, 0.0], [np.nan, 0, 1], [0, -np.inf, 1], [1e308, 1e308, 1e308], [-0.0, 0.0, -0.0], [1, 0, 0], [0, 1e300, 0],
                      [1e-320, 0, 0], [1, 1, 1]])


def nonfinite_cases(seed=0, n=40):
    """k5_fuzz.nonfinite_cases meshes (NaN / inf / huge vertices), with mixed rays and every pairing of special origins and directions"""
    rng = np.random.default_rng(seed + 7)
    so = np.repeat(SPECIAL_O, len(SPECIAL_D), axis=0)
    sd = np.tile(SPECIAL_D, (len(SPECIAL_O), 1))
    for label, V, F, _ in k5_fuzz.nonfinite_cases():
        o, d = mixed_rays(V, F, rng, n)
        yield label, V, F, np.concatenate([o, so]), np.concatenate([d, sd]), ((0.0, INF), (-INF, INF))


def bound_cases(seed=0, n=80):
    """sphere.obj and a coplanar grid under the four standard bounds"""
    rng = np.random.default_rng(seed + 9)
    for label, (V, F) in (("sphere", sphere()), ("grid", mr.grid_mesh(5, True))):
        o, d = mixed_rays(V, F, rng, n)
        yield label, V, F, o, d, BOUNDS


def run_cases(be, cases, log=print, counts=(), hits=None):
    """every case through backend `be` -> (meshes, rays checked, mismatches).  hits: a list that collects (label, restatement hits)"""
    meshes = total = bad = 0
    for label, V, F, o, d, bounds in cases:
        V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
        h = be.mesh(V, F)
        try:
            for lo, hi in bounds:
                n, b, msg, want = check(be, h, V, F, o, d, lo, hi, label, counts)
                total += n; bad += b
                if msg: log(msg)
                if hits is not None:
                    hits.append((label, int((want[3] != mr.MISS).sum())))
        finally:
            be.destroy(h)
        meshes += 1
    return meshes, total, bad


def run_exact_bounds(be, seed=0, log=print, n=60):
    """t_min = t_max exactly at each hit's t (the same hit must come back), and t_max just below every hit (no hit)"""
    rng = np.random.default_rng(seed + 13)
    meshes = total = bad = 0
    for label, (V, F) in (("sphere", sphere()), ("grid", mr.grid_mesh(5, True))):
        o, d = mr.aimed_rays(V, F, n, rng)
        t, tid, _, st = mr.raycast(V, F, o, d)
        h = be.mesh(V, F)
        try:
            for i in np.flatnonzero(st != mr.MISS)[:12]:
                for lo, hi in ((t[i], t[i]), (0.0, t[i]), (t[i], INF)):
                    k, b, msg, want = check(be, h, V, F, o[i:i + 1], d[i:i + 1], lo, hi, f"{label} ray {i}")
                    if want[1][0] != tid[i]:
                        b += 1; msg = msg or f"MISMATCH {label} ray {i} on [{lo!r}, {hi!r}]: the restatement lost its hit"
                    total += k; bad += b
                    if msg: log(msg)
            below = float(np.nextafter(t[st != mr.MISS].min(), -INF))
            k, b, msg, want = check(be, h, V, F, o, d, 0.0, below, f"{label} t_max below every hit")
            if (want[3] != mr.MISS).any():
                b += 1; msg = msg or f"MISMATCH {label}: hits below t_max = {below!r}"
            total += k; bad += b
            if msg: log(msg)
        finally:
            be.destroy(h)
        meshes += 1
    return meshes, total, bad


def run_counts(be, seed=0, log=print):
    """ray counts around multiples of 128: each prefix alone gives the bits of the whole call"""
    rng = np.random.default_rng(seed + 15)
    V, F = sphere()
    o, d = mixed_rays(V, F, rng, 120)
    return run_cases(be, [("sphere prefixes", V, F, o, d, ((0.0, INF), (-0.5, 2.0)))], log=log, counts=COUNTS)


def refit_steps(V, F):
    """(label, positions) of the refits, in order: scaled, mirrored, translated, a subtree collapsed to a point, one vertex NaN, back"""
    cen = V[F].mean(1)
    far = np.unique(F[cen[:, 0] > np.median(cen[:, 0])].reshape(-1))      # the vertices of the triangles right of the median
    Vc = V.copy(); Vc[far] = V[far].mean(0)
    Vn = V.copy(); Vn[len(V) // 3] = np.nan
    return [("scaled x2.5", V * 2.5), ("mirrored in x", V * [-1.0, 1.0, 1.0]), ("translated", V + [3.0, -1.0, 0.5]),
            ("half the triangles collapsed to a point", Vc), ("one vertex NaN", Vn), ("back", V.copy())]


def run_refits(be, seed=0, log=print, n=60):
    """K8's refit, then a cast: the restatement on the new vertices (the culling proof on the refit's boxes).  A mirror flips every status"""
    rng = np.random.default_rng(seed + 17)
    meshes = total = bad = 0
    from discregrid_b200.mesh import bumpy_torus
    m = bumpy_torus(24, 20)
    for label, (V, F) in (("sphere", sphere()), ("torus", (np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)))):
        V = np.ascontiguousarray(V); F = np.ascontiguousarray(F, np.uint32)
        o0, d0 = mixed_rays(V, F, rng, n)
        h = be.mesh(V, F)
        try:
            for step, V1 in refit_steps(V, F):
                V1 = np.ascontiguousarray(V1, np.float64)
                be.refit(h, V1)
                mirror = step.startswith("mirrored")
                o, d = (o0 * [-1.0, 1.0, 1.0], d0 * [-1.0, 1.0, 1.0]) if mirror else (o0, d0)
                if step.startswith("scaled"):
                    o = o0 * 2.5
                if step == "translated":
                    o = o0 + [3.0, -1.0, 0.5]
                o = np.ascontiguousarray(o); d = np.ascontiguousarray(d)
                k, b, msg, want = check(be, h, V1, F, o, d, 0.0, INF, f"{label} refit {step}")
                if mirror:                                               # the same triangle hit from the mirrored side: status flips
                    _, tid0, _, st0 = mr.raycast(V, F, o0, d0)
                    both = (st0 != mr.MISS) & (want[1] == tid0)
                    if both.sum() < 10 or not (want[3][both] == np.where(st0[both] == mr.ENTER, mr.LEAVE, mr.ENTER)).all():
                        b += 1; msg = msg or f"MISMATCH {label} mirrored: the status did not flip"
                total += k; bad += b
                if msg: log(msg)
        finally:
            be.destroy(h)
        meshes += 1
    return meshes, total, bad


def large_mesh():
    p = wr.ref_resource(ROOT, "bunny.obj")
    if p:
        return ("bunny",) + tuple(wr.read_obj(p))
    from discregrid_b200.mesh import bumpy_torus
    m = bumpy_torus(80, 60)
    return "torus", np.asarray(m.vertices, np.float64), np.asarray(m.faces, np.uint32)


def run_large(be, n=1 << 22, seed=0, log=print, sample=3000):
    """one call of n rays; the first and last rays and a random sample against the restatement, and the sample cast alone"""
    label, V, F = large_mesh()
    rng = np.random.default_rng(seed + 19)
    o, d = mr.random_rays(V, n, rng, 1.3)
    k = n // 4
    o2, d2 = mr.aimed_rays(V, F, k, rng)
    o[:k], d[:k] = o2, d2
    h = be.mesh(V, F)
    try:
        got = be.cast(h, o, d, 0.0, INF)
        idx = np.unique(np.concatenate([np.arange(200), np.arange(n - 200, n), rng.integers(0, n, sample)]))
        want = mr.raycast(V, F, o[idx], d[idx])
        ok = compare(tuple(np.asarray(x)[idx] for x in got), want)
        alone = be.cast(h, np.ascontiguousarray(o[idx]), np.ascontiguousarray(d[idx]), 0.0, INF)
        ok &= compare(alone, want)
        ok &= bool(getattr(be, "device_same", True))
    finally:
        be.destroy(h)
    if not ok.all():
        i = int(idx[np.nonzero(~ok)[0][0]])
        log(f"MISMATCH {n} rays on {label}: ray {i}")
    return len(idx), int((~ok).sum()), int((want[3] != mr.MISS).sum())


def run(be, rounds, seed=0, log=print, large=None):
    """every family through backend `be` -> (meshes, rays checked, mismatches)"""
    acc = [0, 0, 0]

    def add(r):
        for i in range(3):
            acc[i] += r[i]
    add(run_cases(be, tree_cases(seed), log=log))
    add(run_cases(be, buddha_case(seed), log=log))
    add(run_cases(be, tie_cases(rounds, seed), log=log))
    add(run_cases(be, slack_cases(), log=log))
    add(run_cases(be, scale_cases(seed), log=log))
    add(run_cases(be, cull_cases(seed), log=log))
    add(run_cases(be, nonfinite_cases(seed), log=log))
    add(run_cases(be, bound_cases(seed), log=log))
    add(run_exact_bounds(be, seed, log))
    add(run_counts(be, seed, log))
    if isinstance(be, DgK9):
        add(run_refits(be, seed, log))
        if large:
            n, b, _ = run_large(be, large, seed, log)
            acc[0] += 1; acc[1] += n; acc[2] += b
    return tuple(acc)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 40
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else os.path.join(ROOT, "build", "bin", "libk9emu.so")
    meshes, total, bad = run(backend(lib), rounds, seed)
    print(f"{meshes} meshes, {total} rays, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
