#!/usr/bin/env python
"""Parity fuzzer: the product's K1 kernel code against the reference's own TriangleMeshDistance.h (oracle/_ref/libdgref.so; where that is
not compiled, the oracle port pinned to it) on meshes built to provoke exact ties and awkward arithmetic -- regular grids of coplanar
triangles, cubes / octahedra with queries on symmetry planes, duplicated triangles, slivers, lattice-aligned queries, random soups at scales
1e-24 .. 1e17 -- signed and unsigned, distance bits, nearest point, entity and triangle id.

usage: tools/k1_fuzz.py [rounds=200] [seed=0] [lib=build/bin/libk1emu.so] [points|grid|scales] [band]
  lib    a build of tests/emu/k1_emu.cpp (the K1 translation unit compiled for the CPU), or `dg`: the product library through its C-ABI
         (dg_mesh_create, dg_mesh_distance, dg_node_positions, dg_sample_sdf), i.e. the CUDA kernels -- needs a GPU
  points mesh_distance on arbitrary points (the per-lane walk)
  grid   the addFunction NODE LOOP (sdf_sample_nodes_kernel: bricks of lattice nodes, the packet walk when built with K1_PACKET) on lattices
         laid over the same meshes -- half-integer lattices through the symmetric ones -- sign * distance compared bit for bit with the
         reference evaluated at the node positions
  scales the scale sweep (`rounds` is ignored): soups, strips and coplanar grids at scales 10^k, k = -24 .. 17, with and without an offset
         large against the mesh, and meshes whose half extent lies just below / just above the 1e18 limit of the fp32 filters; both forms
  band   grid / scales only: the node loop in its narrow-band form (addFunction with pred(x) = |distance| <= band; classifier + band kernel,
         k1_launch_sample_nodes_band) with band = `band` times the largest cell size; compared with the reference's distance where it is
         <= band and DBL_MAX elsewhere.  Needs a build of tests/emu/k1_band_emu.cpp or `dg`
The functions are shared with tests/test_k1_emulated.py and tests/test_gpu_k1_scales.py."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle_api import Oracle, RefMesh, have_ref  # noqa: E402

dp, u32p, i32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def num_nodes(res):
    nx, ny, nz = (int(r) for r in res)
    return (nx + 1) * (ny + 1) * (nz + 1) + 2 * (nx * (ny + 1) * (nz + 1) + (nx + 1) * ny * (nz + 1) + (nx + 1) * (ny + 1) * nz)


class EmuK1:
    """a build of tests/emu/k1_emu.cpp: the K1 kernels and launchers run on the CPU"""

    def __init__(self, so):
        self.name = os.path.basename(so)
        lib = self.lib = C.CDLL(so)
        lib.emu_mesh_create.restype = C.c_void_p
        lib.emu_mesh_create.argtypes = [dp, C.c_uint64, u32p, C.c_uint64]
        lib.emu_mesh_destroy.argtypes = [C.c_void_p]
        lib.emu_mesh_distance.argtypes = [C.c_void_p, dp, C.c_uint64, C.c_int, dp, dp, i32p, i32p]
        lib.emu_sample_sdf.argtypes = [C.c_void_p, dp, u32p, C.c_double, C.c_uint64, C.c_uint64, dp]
        lib.emu_node_positions.argtypes = [dp, u32p, C.c_uint64, C.c_uint64, dp]
        if hasattr(lib, "emu_sample_sdf_band"):
            lib.emu_sample_sdf_band.argtypes = [C.c_void_p, dp, u32p, C.c_double, C.c_double, C.c_uint64, C.c_uint64, dp]

    def mesh(self, V, F):
        h = self.lib.emu_mesh_create(_p(V, dp), len(V), _p(F, u32p), len(F))
        assert h
        return h

    def destroy(self, h):
        self.lib.emu_mesh_destroy(h)

    def distance(self, h, x, signed, near=True):
        n = len(x)
        d = np.zeros(n); nr = np.zeros((n, 3)) if near else None; e = np.zeros(n, np.int32) if near else None; t = np.zeros(n, np.int32)
        assert self.lib.emu_mesh_distance(h, _p(x, dp), n, int(signed), _p(d, dp), _p(nr, dp), _p(e, i32p), _p(t, i32p)) == 0
        return d, nr, e, t

    def grid(self, mn, mx, res):
        return Oracle.grid_desc(mn, mx, res)

    def node_positions(self, g, n):
        gd, r = g
        xs = np.empty((n, 3))
        assert self.lib.emu_node_positions(_p(gd, dp), _p(r, u32p), 0, n, _p(xs, dp)) == 0
        return xs

    def sample(self, h, g, sign, n, band=None):
        gd, r = g
        out = np.full(n, np.nan)
        if band is None:
            assert self.lib.emu_sample_sdf(h, _p(gd, dp), _p(r, u32p), sign, 0, n, _p(out, dp)) == 0
        else:
            assert self.lib.emu_sample_sdf_band(h, _p(gd, dp), _p(r, u32p), sign, band, 0, n, _p(out, dp)) == 0
        return out

    def cell_size(self, g):
        return g[0][6:9]


class DgK1:
    """the product library through its C-ABI: the CUDA kernels on the current device"""

    name = "dg"

    def __init__(self):
        from discregrid_b200 import _capi
        self.capi, self.lib = _capi, _capi.lib

    def mesh(self, V, F):
        h = C.c_void_p()
        self.capi.check(self.lib.dg_mesh_create(_p(V, dp), len(V), _p(F, u32p), len(F), C.byref(h)))
        return h

    def destroy(self, h):
        self.capi.check(self.lib.dg_mesh_destroy(h))

    def distance(self, h, x, signed, near=True):
        n = len(x)
        d = np.zeros(n); nr = np.zeros((n, 3)) if near else None; e = np.zeros(n, np.int32) if near else None; t = np.zeros(n, np.int32)
        self.capi.check(self.lib.dg_mesh_distance(h, _p(x, dp), n, int(signed), _p(d, dp), _p(nr, dp), _p(e, i32p), _p(t, i32p)))
        return d, nr, e, t

    def grid(self, mn, mx, res):
        desc = self.capi.GridDesc()
        self.capi.check(self.lib.dg_grid_init(_p(np.ascontiguousarray(mn, np.float64), dp), _p(np.ascontiguousarray(mx, np.float64), dp),
                                              _p(np.ascontiguousarray(res, np.uint32), u32p), C.byref(desc)))
        return desc

    def node_positions(self, g, n):
        xs = np.empty((n, 3))
        self.capi.check(self.lib.dg_node_positions(C.byref(g), 0, n, _p(xs, dp)))
        return xs

    def sample(self, h, g, sign, n, band=None):
        out = np.full(n, np.nan)
        if band is None:
            self.capi.check(self.lib.dg_sample_sdf(h, C.byref(g), sign, 0, n, _p(out, dp)))
        else:
            self.capi.check(self.lib.dg_add_function_sdf_band(h, C.byref(g), sign, band, _p(out, dp), None, None, None))
        return out

    def cell_size(self, g):
        return np.array(g.cell_size[:])


def backend(lib):
    return DgK1() if lib == "dg" else EmuK1(lib)


def reference(V, F):
    """the reference's own header where it is compiled (oracle/_ref), else the oracle port pinned to it"""
    return RefMesh(V, F) if have_ref() else Oracle().mesh(V, F)


def _same(a, b):
    """bit for bit, any NaN equal to any NaN"""
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def check_points(be, h, ref, x, label=""):
    """signed and unsigned queries: distance bits, nearest point, entity, triangle id.  -> (queries checked, mismatches, first mismatch)"""
    bad, first = 0, None
    for signed in (1, 0):
        wd, wn, we, wt = ref.distance(x, signed=bool(signed))
        d, nr, e, t = be.distance(h, x, signed)
        ok = _same(d, wd) & _same(nr, wn).all(1) & (e == we) & (t == wt)
        if not ok.all():
            i = int(np.nonzero(~ok)[0][0]); bad += int((~ok).sum())
            first = first or (f"MISMATCH {label} signed={signed} x={x[i]!r}: d {d[i]!r} vs {wd[i]!r}, tri {t[i]} vs {wt[i]}, ent {e[i]} vs {we[i]}")
    return 2 * len(x), bad, first


def band_expect(wd, sign, band):
    """addFunction(func, pred) with pred(x) = |d| <= band: sign * d where it holds, DBL_MAX elsewhere (NaN fails the predicate)"""
    return np.where(np.abs(wd) <= band, wd if sign == 1.0 else sign * wd, np.finfo(np.float64).max)


def check_grid(be, h, ref, mn, mx, res, sign, label="", band_cells=None):
    """the node loop over the lattice (mn, mx, res) == sign * the reference's signed distance at the node positions, bit for bit; with
    band_cells, the narrow-band form with band = band_cells * the largest cell size"""
    g = be.grid(mn, mx, res)
    nn = num_nodes(res)
    xs = be.node_positions(g, nn)
    wd = ref.distance(xs, signed=True)[0]
    band = None if band_cells is None else band_cells * float(np.max(be.cell_size(g)))
    want = (wd if sign == 1.0 else sign * wd) if band is None else band_expect(wd, sign, band)
    got = be.sample(h, g, sign, nn, band) if band is not None else be.sample(h, g, sign, nn)
    ok = _same(got, want)
    if ok.all():
        return nn, 0, None
    i = int(np.nonzero(~ok)[0][0])
    return nn, int((~ok).sum()), f"MISMATCH {label} grid {tuple(res)} node {i} x={xs[i]!r}: {got[i]!r} vs {want[i]!r}"


def grid_mesh(rng, nx, ny, jitter=0.0, z=0.0):
    xs, ys = np.meshgrid(np.arange(nx + 1, dtype=float), np.arange(ny + 1, dtype=float), indexing="ij")
    V = np.stack([xs.ravel(), ys.ravel(), np.full(xs.size, z)], 1)
    V[:, :2] += jitter * rng.standard_normal((len(V), 2))
    F = []
    for i in range(nx):
        for j in range(ny):
            a, b, c, d = i * (ny + 1) + j, (i + 1) * (ny + 1) + j, (i + 1) * (ny + 1) + j + 1, i * (ny + 1) + j + 1
            F += [[a, b, c], [a, c, d]] if (i + j) % 2 else [[a, b, d], [b, c, d]]
    return V, np.array(F, np.uint32)


def cube():
    V = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], float)
    F = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.uint32)
    return V, F


def octa():
    V = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], float)
    F = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], np.uint32)
    return V, F


def queries(rng, V, F, extra=(), flat=1e-12):
    """around the mesh (box of twice its extent; a flat side counts as `flat` times the longest), a 7^3 lattice through it, the vertices,
    edge midpoints and centroids"""
    lo, hi = V.min(0), V.max(0)
    ext = np.maximum(hi - lo, flat * max(1.0, float((hi - lo).max())))
    q = [lo - 0.5 * ext + rng.random((150, 3)) * 2 * ext]
    lat = np.stack(np.meshgrid(*[np.linspace(lo[d] - ext[d], hi[d] + ext[d], 7) for d in range(3)], indexing="ij"), -1).reshape(-1, 3)
    q += [lat, V, 0.5 * (V[F[:, 0]] + V[F[:, 1]]), (V[F[:, 0]] + V[F[:, 1]] + V[F[:, 2]]) / 3.0]
    q += list(extra)
    return np.ascontiguousarray(np.concatenate(q))


def make_case(rng, k):
    kind = k % 7
    if kind == 0: V, F = grid_mesh(rng, int(rng.integers(1, 7)), int(rng.integers(1, 7)))
    elif kind == 1: V, F = grid_mesh(rng, int(rng.integers(2, 6)), int(rng.integers(2, 6)), jitter=1e-3)
    elif kind == 2: V, F = cube()
    elif kind == 3: V, F = octa()
    elif kind == 4:                                              # two stacked sheets + duplicated triangles
        V1, F1 = grid_mesh(rng, 3, 3); V2, F2 = grid_mesh(rng, 3, 3, z=1.0)
        V = np.concatenate([V1, V2]); F = np.concatenate([F1, F2 + len(V1), F1[:4]])
    elif kind == 5:                                              # slivers and near-degenerate triangles
        n = int(rng.integers(3, 30)); V = rng.standard_normal((n + 2, 3)); V[:, 2] *= 1e-7
        F = np.array([[i, i + 1, i + 2] for i in range(n)], np.uint32)
    else:                                                        # random soup, random scale / offset
        n = int(rng.integers(1, 60)); sc = 10.0 ** rng.integers(-24, 18); off = rng.standard_normal(3) * sc * 10 ** rng.integers(0, 4)
        V = rng.standard_normal((3 * n, 3)) * sc + off; F = np.arange(3 * n, dtype=np.uint32).reshape(n, 3)
    V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
    extra = []
    if kind in (0, 2, 3, 4):                                     # half-integer lattice: symmetric, tie-rich queries
        extra.append(np.stack(np.meshgrid(*[np.arange(-1.0, 2.51, 0.5)] * 3, indexing="ij"), -1).reshape(-1, 3))
    return V, F, queries(rng, V, F, extra)


def case_lattice(k, V):
    """the node lattice of fuzz case k: half-integer through the symmetric meshes, else (9, 7, 6) over the mesh's box + 30 %"""
    lo, hi = V.min(0), V.max(0)
    if k % 7 in (0, 2, 3, 4):                                    # nodes on the half-integer lattice: ties by symmetry
        mn = np.floor(lo) - 1.0; mx = mn + 4.0 * np.ceil((hi - mn + 1.0) / 4.0)
        return mn, mx, tuple(int(r) for r in ((mx - mn) * 2))
    ext = np.maximum(hi - lo, 1e-9 * max(1.0, float((hi - lo).max())))
    return lo - 0.3 * ext, hi + 0.3 * ext, (9, 7, 6)


SCALE_EXPONENTS = tuple(range(-24, 18))


def scale_cases(seed=0, exponents=SCALE_EXPONENTS):
    """(label, V, F) of the scale sweep: per 10^k a random soup, a strip (neighbours share edges and vertices) and a coplanar grid, each once
    centred near the origin and once with an offset 10^3 - 10^6 times the mesh size (fewer fp64 bits left for the mesh itself); then soups
    whose half extent is 1e18 (1 -+ 1e-3): the queries near them lie on both sides of the fp32 filters' upper limit"""
    rng = np.random.default_rng(seed)
    for k in exponents:
        s = 10.0 ** k
        for off_exp in (None, float(rng.uniform(3, 6))):
            off = np.zeros(3) if off_exp is None else rng.standard_normal(3) * s * 10.0 ** off_exp
            n = int(rng.integers(4, 41))
            soup = (rng.standard_normal((3 * n, 3)), np.arange(3 * n, dtype=np.uint32).reshape(n, 3))
            n = int(rng.integers(4, 81))
            strip = (rng.standard_normal((n + 2, 3)), np.array([[i, i + 1, i + 2] for i in range(n)], np.uint32))
            plane = grid_mesh(rng, int(rng.integers(2, 7)), int(rng.integers(2, 7)))
            for kind, (V, F) in (("soup", soup), ("strip", strip), ("grid", plane)):
                tag = "" if off_exp is None else f"+off1e{off_exp:.1f}"
                yield f"{kind}@1e{k}{tag}", np.ascontiguousarray(V * s + off), np.ascontiguousarray(F, np.uint32)
    for h in (0.999e18, 1.001e18):
        n = int(rng.integers(4, 41))
        V = rng.standard_normal((3 * n, 3))
        V = (V - 0.5 * (V.max(0) + V.min(0))) * (h / (0.5 * (V.max(0) - V.min(0)).max()))
        yield f"soup@half_extent{h:.4g}", np.ascontiguousarray(V), np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def run_scales(be, seed=0, modes=("points", "grid"), exponents=SCALE_EXPONENTS, log=print, band_cells=None):
    """the scale sweep through backend `be` -> (meshes, queries + nodes checked, mismatches); band_cells: the grid form in its narrow-band form"""
    rng = np.random.default_rng(seed + 1)
    meshes = total = bad = 0
    for i, (label, V, F) in enumerate(scale_cases(seed, exponents)):
        ref = reference(V, F)
        h = be.mesh(V, F)
        meshes += 1
        if "points" in modes:
            n, b, msg = check_points(be, h, ref, queries(rng, V, F, flat=0.25), label)
            total += n; bad += b
            if msg: log(msg)
        if "grid" in modes:
            lo, hi = V.min(0), V.max(0)
            ext = np.maximum(hi - lo, 0.25 * (hi - lo).max())
            n, b, msg = check_grid(be, h, ref, lo - 0.3 * ext, hi + 0.3 * ext, (9, 7, 6), -1.0 if i % 2 else 1.0, label, band_cells)
            total += n; bad += b
            if msg: log(msg)
        be.destroy(h)
    return meshes, total, bad


# one- and two-triangle meshes (the root is a leaf / has leaf children), tiny and huge coordinates, large offsets, degenerate triangles
AWKWARD = [(1, 1.0, 0.0, False), (2, 1.0, 0.0, False), (3, 1.0, 0.0, False), (7, 1e-9, 0.0, False), (40, 1.0, 1e9, False), (33, 1e6, -3e7, False),
           (9, 1.0, 0.0, True), (64, 1.0, 0.0, True)]


def strip_mesh(rng, n_tri, scale=1.0, offset=0.0, degenerate=False):
    V = rng.standard_normal((n_tri + 2, 3)) * scale + offset
    F = np.array([[i, i + 1, i + 2] for i in range(n_tri)], np.uint32)        # a strip: neighbours share edges and vertices (ties)
    if degenerate and n_tri >= 3:
        V[3] = V[2]                                                            # zero-length edge -> zero-area triangles
        F[-1] = [0, 0, 1]                                                      # a triangle with a repeated vertex
    return np.ascontiguousarray(V), F


def awkward_case(n_tri, scale, offset, degenerate):
    """(V, F, queries the reference answers, queries it accepts no triangle for).  The second set -- NaN, infinite, or so large that the
    squared distance overflows -- makes the reference index triangles[-1] (undefined behaviour: it crashes for some meshes), so it is not
    sent there; the kernels must answer DBL_MAX / triangle -1"""
    rng = np.random.default_rng(1000 + n_tri)
    V, F = strip_mesh(rng, n_tri, scale, offset, degenerate)
    x = np.concatenate([rng.standard_normal((300, 3)) * scale * 2 + offset,                    # around the mesh
                        V[:min(len(V), 20)],                                                  # exactly on vertices
                        0.5 * (V[F[:, 0]] + V[F[:, 1]])[:20],                                  # on edges
                        rng.standard_normal((40, 3)) * scale * 1e6 + offset,                   # far
                        np.array([[1e19, -1e19, 3e18], [0.0, 0.0, 0.0], [-0.0, 0.0, -0.0]])])
    lost = np.array([[1e300, 0, 0], [np.nan, 0, 0], [np.inf, 1, 2], [0, -np.inf, 0]])
    return V, F, np.ascontiguousarray(x), np.ascontiguousarray(lost)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 200
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else os.path.join(ROOT, "build", "bin", "libk1emu.so")
    mode = argv[4] if len(argv) > 4 else "points"
    band_cells = float(argv[5]) if len(argv) > 5 else None
    be = backend(lib)
    if mode == "scales":
        meshes, total, bad = run_scales(be, seed, band_cells=band_cells)
        print(f"{meshes} meshes, {total} queries, {bad} mismatches")
        return 1 if bad else 0
    rng = np.random.default_rng(seed)
    bad = total = 0
    for k in range(rounds):
        V, F, x = make_case(rng, k)
        try:
            ref = reference(V, F)
        except Exception as ex:
            print("reference refused the mesh", ex); continue
        h = be.mesh(V, F)
        label = f"case {k} (kind {k % 7}, {len(F)} tris)"
        if mode == "grid":
            mn, mx, res = case_lattice(k, V)
            n, b, msg = check_grid(be, h, ref, mn, mx, res, 1.0 if k % 2 else -1.0, label, band_cells)
        else:
            n, b, msg = check_points(be, h, ref, x, label)
        total += n; bad += b
        if msg: print(msg)
        be.destroy(h)
    print(f"{rounds} meshes, {total} queries, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
