"""Narrow-band K1 (addFunction with pred(x) = |md.signed_distance(x).distance| <= band): the product's classifier passes and the band form
of the node loop (k1_sdf.cu, k1_launch_sample_nodes_band) compiled for the CPU by tests/emu, against the reference bit for bit -- its own
addFunction(func, pred) (+ reduceField) as committed fixtures, its own header at the node positions elsewhere.  The GPU runs are
tests/test_gpu_k1_band.py."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, grid_for
from test_oracle_golden import read_cdf, read_obj

sys.path.insert(0, os.path.join(ROOT, "tools"))
import k1_fuzz  # noqa: E402

LIBS = [os.path.join(ROOT, "build", "bin", n) for n in ("libk1emu_band.so", "libk1emu_band_perlane.so")]
DBL_MAX = np.finfo(np.float64).max
CASES = json.load(open(os.path.join(GOLDEN, "ref_band_cases.json")))
_dp, _u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


@pytest.fixture(scope="module", params=LIBS, ids=[os.path.basename(p) for p in LIBS])
def be(request):
    if not os.path.exists(request.param):
        pytest.skip(f"{request.param} not built (make cpp)")
    return k1_fuzz.EmuK1(request.param)


def band_sample(be, h, gd, r, sign, band, l0, l1, out=None):
    out = np.full(l1 - l0, np.nan) if out is None else out
    assert be.lib.emu_sample_sdf_band(h, _p(gd, _dp), _p(r, _u32p), sign, band, l0, l1, _p(out, _dp)) == 0
    return out


def case_mesh(case):
    path = os.path.join(ROOT, "tests", case["mesh"]) if case["mesh"].startswith("golden/") else os.path.join(ROOT, "oracle", "_ref", "resources", case["mesh"])
    if not os.path.exists(path):
        pytest.skip(f"{path} missing (oracle/_ref resources)")
    V, F = read_obj(path)
    return np.ascontiguousarray(V, np.float64), np.ascontiguousarray(F, np.uint32)


def reduced_values(orc, res, dense):
    """the node values reduceField(always true) keeps (:1065-1174): every node of every cell that owns a node != DBL_MAX, as a sorted multiset"""
    cells = orc.build_cells(res)
    kept = (dense[cells] != DBL_MAX).any(1)
    return np.sort(dense[np.unique(cells[kept])])


@pytest.mark.parametrize("name", sorted(CASES))
def test_band_fields_equal_reference_fixtures(be, orc, name):
    """the reference's own addFunction(func, pred) -- dense, or reduced with an always-true predicate -- on the box (nodes exactly at the band
    edge), bunny, dragon inverted and an anisotropic grid: same coefficients bit for bit"""
    case = CASES[name]
    g = read_cdf(os.path.join(GOLDEN, case["file"]))
    V, F = case_mesh(case)
    gd, res = orc.grid_desc(g["mn"], g["mx"], g["res"], g["cell"], g["inv"])
    nn = orc.num_nodes(res)
    h = be.mesh(V, F)
    got = band_sample(be, h, gd, res, -1.0 if case["invert"] else 1.0, float.fromhex(case["band_hex"]), 0, nn)
    be.destroy(h)
    want = g["nodes"][0]
    if case["reduce"]:
        assert len(g["cells"][0]) < int(np.prod(res))                          # the fixture is really reduced
        assert np.array_equal(reduced_values(orc, res, got).view(np.uint64), np.sort(want).view(np.uint64))
    else:
        assert bits_equal(got, want)
    if name == "box_edge":                                                    # the `<=` edge: nodes exactly at distance band are kept
        assert (np.abs(got) == 0.5).sum() > 100 and (got == DBL_MAX).any()


def test_band_edges_nextafter_zero_and_everything(be, orc):
    """band just below / exactly at a node's distance drops / keeps it; band 0 keeps only nodes on the surface; a band wider than the
    domain (and +inf) equals the plain node loop"""
    V, F = case_mesh(CASES["box_edge"])
    gd, r = orc.grid_desc(np.array([-2.0, -2, -2]), np.array([2.0, 2, 2]), (8, 8, 8))
    nn = orc.num_nodes(r)
    h = be.mesh(V, F)
    full = be.sample(h, (gd, r), 1.0, nn)
    rng = np.random.default_rng(3)
    for i in rng.choice(np.nonzero(np.abs(full) > 0)[0], 6, replace=False):
        w = abs(full[i])
        at = band_sample(be, h, gd, r, 1.0, w, 0, nn)
        below = band_sample(be, h, gd, r, 1.0, float(np.nextafter(w, 0.0)), 0, nn)
        assert at[i] == full[i] and below[i] == DBL_MAX
        assert bits_equal(at, np.where(np.abs(full) <= w, full, DBL_MAX)) and bits_equal(below, np.where(np.abs(full) < w, full, DBL_MAX))
    zero = band_sample(be, h, gd, r, -1.0, 0.0, 0, nn)
    assert (full == 0).sum() > 50 and bits_equal(zero, np.where(full == 0, -full, DBL_MAX))
    for w in (100.0, np.inf):
        assert bits_equal(band_sample(be, h, gd, r, -1.0, w, 0, nn), -full)
    be.destroy(h)


def test_band_sub_ranges_leave_the_rest_untouched(be, orc):
    """node ranges that cut through blocks: the range holds the band field, a sentinel-filled buffer is untouched outside it"""
    import discregrid_b200 as dg
    t = dg.bumpy_torus(24, 20, 1.0, 0.4, 0.05, 7, 5)
    mn, mx, gd, r = grid_for(orc, t.vertices, (11, 9, 6))
    want_full = orc.mesh(t.vertices, t.faces).sample_sdf(gd, r)
    n = len(want_full)
    h = be.mesh(t.vertices, t.faces)
    band = 0.15
    want = np.where(np.abs(want_full) <= band, want_full, DBL_MAX)
    for (a, b) in [(0, 1), (5, 77), (n // 3, n // 3 + 1000), (n - 13, n), (0, n)]:
        buf = np.full(n + 64, 7.25)
        band_sample(be, h, gd, r, 1.0, band, a, b, out=buf[32 + a:])
        assert bits_equal(buf[32 + a:32 + b], want[a:b])
        assert (buf[:32 + a] == 7.25).all() and (buf[32 + b:] == 7.25).all()
    be.destroy(h)


def test_classifier_drops_blocks_and_keeps_all_for_non_finite_meshes(be, orc):
    """a thin band leaves most blocks unsampled (the node loop runs only the listed blocks, in launch order); a mesh with NaN / inf vertices
    keeps every block, and its band field still equals the reference's"""
    import discregrid_b200 as dg
    from oracle_api import RefMesh, have_ref
    be.lib.emu_block_trace.restype = C.c_uint64
    be.lib.emu_block_trace.argtypes = [_u32p, C.c_uint64]
    buf = np.zeros(1 << 16, np.uint32)
    t = dg.bumpy_torus(24, 20, 1.0, 0.4, 0.05, 7, 5)
    mn, mx, gd, r = grid_for(orc, t.vertices, (32, 32, 16))
    nn = orc.num_nodes(r)
    h = be.mesh(t.vertices, t.faces)
    be.lib.emu_block_trace(_p(buf, _u32p), len(buf))
    full = be.sample(h, (gd, r), 1.0, nn)
    n_full = be.lib.emu_block_trace(_p(buf, _u32p), len(buf))
    got = band_sample(be, h, gd, r, 1.0, 0.05, 0, nn)
    n_band = be.lib.emu_block_trace(_p(buf, _u32p), len(buf))
    order = buf[:n_band].astype(np.int64)
    assert bits_equal(got, np.where(np.abs(full) <= 0.05, full, DBL_MAX))
    assert 0 < n_band < 0.9 * n_full and (np.diff(order) > 0).all()
    be.destroy(h)
    V = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [np.nan, 2, 2], [3, 3, np.inf], [2, 2, 2]], float)
    F = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5], [6, 0, 2], [7, 8, 4]], np.uint32)
    ref = RefMesh(V, F) if have_ref() else orc.mesh(V, F)
    gd, r = orc.grid_desc(np.array([-2.0, -2, -2]), np.array([2.0, 2, 2]), (8, 8, 8))
    nn = orc.num_nodes(r)
    xs = orc.node_positions(gd, r, 0, nn)
    wd = ref.distance(xs, signed=True)[0]
    h = be.mesh(V, F)
    be.lib.emu_block_trace(_p(buf, _u32p), len(buf))
    be.sample(h, (gd, r), 1.0, nn)
    n_full = be.lib.emu_block_trace(_p(buf, _u32p), len(buf))
    got = band_sample(be, h, gd, r, 1.0, 0.01, 0, nn)
    assert be.lib.emu_block_trace(_p(buf, _u32p), len(buf)) == n_full
    assert bits_equal(got, k1_fuzz.band_expect(wd, 1.0, 0.01))
    be.destroy(h)


@pytest.mark.parametrize("mode", ["grid", "scales"])
def test_band_fuzz_tie_lattices_and_scales(mode):
    """tools/k1_fuzz.py with a band of 3 cells: the tie-rich lattices (coplanar grids, cubes, octahedra on half-integer lattices, duplicated
    triangles, slivers, soups) and the 1e-24 .. 1e17 scale sweep, band form == the reference header, 0 differences"""
    from oracle_api import REF_SO
    so = LIBS[0]
    if not os.path.exists(REF_SO) or not os.path.exists(so):
        pytest.skip("needs oracle/_ref/libdgref.so and build/bin/libk1emu_band.so")
    args = ["14", "5", so, "grid", "3"] if mode == "grid" else ["0", "0", so, "scales", "3"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "k1_fuzz.py")] + args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and " 0 mismatches" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_band_c_abi_validation_and_launch_counts():
    """through the whole library built for the CPU (build/bin/libdgemu.so): a negative or NaN band is DG_ERR_INVALID; a call without a band
    launches what it always launched; dg_add_function_sdf_band == dg_add_function_sdf where |d| <= band, with the same index tables"""
    so = os.path.join(ROOT, "build", "bin", "libdgemu.so")
    if not os.path.exists(so):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    from discregrid_b200._capi import GridDesc
    lib = C.CDLL(so)
    lib.dg_kernel_launch_count.restype = C.c_uint64
    V, F = read_obj(os.path.join(GOLDEN, "sphere.obj"))
    V = np.ascontiguousarray(V); F = np.ascontiguousarray(F, np.uint32)
    h = C.c_void_p()
    assert lib.dg_mesh_create(_p(V, _dp), C.c_uint64(len(V)), _p(F, _u32p), C.c_uint64(len(F)), C.byref(h)) == 0
    d = GridDesc()
    mn, mx, res = np.array([-1.5, -1.5, -1.5]), np.array([1.5, 1.5, 1.5]), np.array([7, 6, 5], np.uint32)
    assert lib.dg_grid_init(_p(mn, _dp), _p(mx, _dp), _p(res, _u32p), C.byref(d)) == 0
    nn = (8 * 7 * 6) + 2 * (7 * 7 * 6 + 8 * 6 * 6 + 8 * 7 * 5)
    nc = 7 * 6 * 5
    fn = lib.dg_add_function_sdf_band
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, _dp, _u32p, _u32p, _dp]
    lib.dg_add_function_sdf.argtypes = [C.c_void_p, C.c_void_p, C.c_double, _dp, _u32p, _u32p, _dp]
    full, band = np.empty(nn), np.empty(nn)
    c1, c2 = np.empty((nc, 32), np.uint32), np.empty((nc, 32), np.uint32)
    m1, m2 = np.empty(nc, np.uint32), np.empty(nc, np.uint32)
    for bad in (-1.0, -0.0 - 1e-300, float("nan")):
        assert fn(h, C.byref(d), 1.0, bad, _p(band, _dp), None, None, None) == -1
    n0 = lib.dg_kernel_launch_count()
    assert lib.dg_add_function_sdf(h, C.byref(d), 1.0, _p(full, _dp), _p(c1, _u32p), _p(m1, _u32p), None) == 0
    assert lib.dg_kernel_launch_count() - n0 == 1                              # one K1 chunk on a grid this small, as before
    assert fn(h, C.byref(d), 1.0, 0.2, _p(band, _dp), _p(c2, _u32p), _p(m2, _u32p), None) == 0
    assert bits_equal(band, np.where(np.abs(full) <= 0.2, full, DBL_MAX))
    assert np.array_equal(c1, c2) and np.array_equal(m1, m2)
    lib.dg_mesh_destroy.argtypes = [C.c_void_p]
    lib.dg_mesh_destroy(h)
