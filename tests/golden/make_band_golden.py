"""Narrow-band fixtures from the reference's own classes (oracle/_ref/libdiscregrid_ref.so).  addFunction(func, false, pred) with
func = sign * md.signed_distance(x).distance and pred(x) = |md.signed_distance(x).distance| <= band stores func(x) where pred(x) holds and
DBL_MAX elsewhere (cubic_lagrange_discrete_grid.cpp:806-817).  func and pred evaluate the same deterministic query at the same node position,
so that field is exactly the reference's own dense addFunction(func) output (refg_add_function_sdf) with DBL_MAX wherever |value| > band
(|sign * d| = |d|; a NaN distance fails the predicate).  The band field is then handed to a reference grid object (refg_grid_from_nodes:
the reference's connectivity and cell map) and, unless dense, reduced by the reference's reduceField with the window [-inf, +inf] -- every
non-NaN value passes, which is the always-true predicate on these meshes -- and written by its save().  Meshes are read with the reference's
TriangleMesh loader, domains are GenerateSDF's padded boxes (dg_generate_sdf_domain) unless given.  Writes ref_band_*.cdf and
ref_band_cases.json (the cases and their band widths) next to this file.

usage: python tests/golden/make_band_golden.py      (needs oracle/_ref, i.e. `make -C oracle ref` with the reference sources present)"""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF_GRID_SO = os.path.join(ROOT, "oracle", "_ref", "libdiscregrid_ref.so")
RESOURCES = os.path.join(ROOT, "oracle", "_ref", "resources")
_dp, _u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)

# name -> mesh, resolution, domain (None: GenerateSDF's), invert, band (a number, or ("diag", k): k cell diagonals), reduce
CASES = {
    # nodes on the planes x, y, z = +-1.5 lie exactly 0.5 from the faces of the cube [-1, 1]^3: the `<=` edge of the predicate
    "box_edge": dict(mesh="golden/box.obj", res=(8, 8, 8), domain=((-2.0, -2.0, -2.0), (2.0, 2.0, 2.0)), invert=False, band=0.5, reduce=False),
    "bunny_20": dict(mesh="bunny.obj", res=(20, 20, 20), domain=None, invert=False, band=("diag", 1.0), reduce=True),
    "dragon_12_inverted": dict(mesh="dragon.obj", res=(12, 12, 12), domain=None, invert=True, band=("diag", 2.0), reduce=False),
    "sphere_aniso": dict(mesh="golden/sphere.obj", res=(19, 6, 11), domain=None, invert=False, band=("diag", 0.5), reduce=True),
}


def mesh_path(name):
    return os.path.join(ROOT, "tests", name) if name.startswith("golden/") else os.path.join(RESOURCES, name)


def ref_mesh(lib, path):
    """vertices / triangles as the reference's TriangleMesh(path) reads them"""
    lib.refm_open.restype = C.c_void_p; lib.refm_open.argtypes = [C.c_char_p, _dp]
    lib.refm_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.refm_copy.argtypes = [C.c_void_p, _dp, _u32p]; lib.refm_close.argtypes = [C.c_void_p]
    t = C.c_double()
    h = lib.refm_open(path.encode(), C.byref(t))
    nv, nf = C.c_uint64(), C.c_uint64()
    lib.refm_sizes(h, C.byref(nv), C.byref(nf))
    V = np.empty((nv.value, 3)); F = np.empty((nf.value, 3), np.uint32)
    lib.refm_copy(h, V.ctypes.data_as(_dp), F.ctypes.data_as(_u32p))
    lib.refm_close(h)
    return V, F


def case_geometry(case, V):
    """(domain min, domain max, band) of a case: GenerateSDF's domain through the library's host helper (no GPU) unless given"""
    if case["domain"] is None:
        sys.path.insert(0, ROOT)
        from discregrid_b200 import generate_sdf_domain
        mn, mx = generate_sdf_domain(V)
    else:
        mn, mx = (np.array(case["domain"][0], float), np.array(case["domain"][1], float))
    band = case["band"]
    if isinstance(band, (tuple, list)):
        cell = (mx - mn) / np.array(case["res"], float)
        band = float(band[1] * np.sqrt((cell * cell).sum()))
    return mn, mx, float(band)


def reference_band_grid(V, F, mn, mx, res, invert, band, reduce):
    """a reference grid object holding the reference's band field (reduced unless `reduce` is false); the caller saves / queries it"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from oracle_api import RefAddFunction, RefGridInMemory
    ref = RefAddFunction(V, F)
    _, nodes, _ = ref.add_function(mn, mx, res, invert=invert, want_nodes=True)
    ref.close()
    nodes = np.where(np.abs(nodes) <= band, nodes, np.finfo(np.float64).max)
    g = RefGridInMemory(mn, mx, res, nodes)
    if reduce:
        g.reduce_window(0, -np.inf, np.inf)
    return g


def main():
    lib = C.CDLL(REF_GRID_SO)
    meta = {}
    for name, case in CASES.items():
        V, F = ref_mesh(lib, mesh_path(case["mesh"]))
        mn, mx, band = case_geometry(case, V)
        out = os.path.join(HERE, f"ref_band_{name}.cdf")
        g = reference_band_grid(V, F, mn, mx, case["res"], case["invert"], band, case["reduce"])
        g.save(out)
        g.close()
        meta[name] = dict(case, domain=[list(map(float, mn)), list(map(float, mx))], band=band, band_hex=float.hex(band), file=os.path.basename(out))
        print(name, out, os.path.getsize(out), "bytes, band", band)
    with open(os.path.join(HERE, "ref_band_cases.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
