"""The reduced narrow band in one call (dg_reduced_band_create: addFunction(func, band predicate) + reduceField(always true)) on the CPU:
the product's kernels and C-ABI compiled into build/bin/libdgemu.so (tests/emu).  The device swap walk (build/bin/libk4emu.so) must equal
the reference's serial walk (reduce_swap_walk), and the whole entry point must equal dg_add_function_sdf_band followed by dg_reduce_field, bit for bit.  The GPU
runs are tests/test_gpu_band_reduced.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal
from test_oracle_golden import read_cdf, read_obj

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
CASES = json.load(open(os.path.join(GOLDEN, "ref_band_cases.json")))
DBL_MAX = np.finfo(np.float64).max
REFERENCE_SORT, HOST_PASSES = 1, 2
_dp, _u32p, _u8p, _u64p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def emu():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    from discregrid_b200._capi import SIGNATURES
    lib = C.CDLL(EMU)
    for name, (res, args) in SIGNATURES.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def walk_lib():
    so = os.path.join(ROOT, "build", "bin", "libk4emu.so")
    if not os.path.exists(so):
        pytest.skip("build/bin/libk4emu.so not built (make cpp)")
    lib = C.CDLL(so)
    lib.emu_k4_swap_walk.restype = C.c_uint64
    lib.emu_k4_swap_walk.argtypes = [_u8p, C.c_uint64, _u32p, C.POINTER(C.c_uint)]
    lib.emu_reduce_swap_walk.restype = C.c_uint64
    lib.emu_reduce_swap_walk.argtypes = [_u8p, C.c_uint64, _u32p]
    return lib


# ------------------------------------------------------------------------------------------------ the swap walk
def walks(walk_lib, used):
    used = np.ascontiguousarray(used, np.uint8)
    n = len(used)
    a, b = np.full(n + 1, 0xDEADBEEF, np.uint32), np.full(n + 1, 0xDEADBEEF, np.uint32)
    rounds = C.c_uint()
    m_dev = walk_lib.emu_k4_swap_walk(_p(used, _u8p), n, _p(a, _u32p), C.byref(rounds))
    m_ref = walk_lib.emu_reduce_swap_walk(_p(used, _u8p), n, _p(b, _u32p))
    return m_dev, a[:m_dev], m_ref, b[:m_ref], rounds.value


def chain_length(used):
    """longest chain of the parallel form (a dead position p < m: q0 = m + dead(p), q_{i+1} = m + dead(q_i) until a used position)"""
    used = np.asarray(used, bool)
    m = int(used.sum())
    dead_before = np.cumsum(~used) - (~used)
    longest = 0
    for p in np.nonzero(~used[:m])[0]:
        q, steps = m + dead_before[p], 1
        while not used[q]:
            q, steps = m + dead_before[q], steps + 1
        longest = max(longest, steps)
    return longest


@pytest.mark.parametrize("n", [1, 31, 33, 1000, 1025, 3077])
@pytest.mark.parametrize("density", [0.02, 0.3, 0.7, 0.97])
def test_device_swap_walk_equals_the_serial_walk_on_random_flags(walk_lib, n, density):
    rng = np.random.default_rng(n * 100 + int(density * 100))
    for _ in range(3):
        used = rng.random(n) < density
        m_dev, a, m_ref, b, _ = walks(walk_lib, used)
        assert m_dev == m_ref == used.sum() and np.array_equal(a, b)


def test_device_swap_walk_edge_patterns(walk_lib):
    """all used, none used, one survivor at 0 and at n - 1, and a pattern whose chain is n - 2 long (one dead position before m, every
    position from m on dead except the last one): ceil(log2(n - m)) rounds"""
    n = 5000
    for used in (np.ones(n, bool), np.zeros(n, bool)):
        m_dev, a, m_ref, b, _ = walks(walk_lib, used)
        assert m_dev == m_ref and np.array_equal(a, b)
    assert walks(walk_lib, np.ones(n, bool))[4] == 0 and walks(walk_lib, np.zeros(n, bool))[0] == 0
    for pos in (0, n - 1):
        used = np.zeros(n, bool); used[pos] = True
        m_dev, a, m_ref, b, _ = walks(walk_lib, used)
        assert m_dev == m_ref == 1 and np.array_equal(a, b) and a[0] == pos
    used = np.zeros(n, bool); used[1] = True; used[n - 1] = True
    assert chain_length(used) == n - 2
    m_dev, a, m_ref, b, rounds = walks(walk_lib, used)
    assert m_dev == m_ref == 2 and np.array_equal(a, b) and list(a) == [n - 1, 1]
    assert rounds == int(np.ceil(np.log2(n - 2)))
    rng = np.random.default_rng(11)
    for _ in range(20):                                                      # long chains with random prefixes
        k = int(rng.integers(2, 40))
        used = np.zeros(n, bool); used[rng.choice(k, k // 2, replace=False)] = True; used[n - k // 2 - (k - k // 2):] = True
        m_dev, a, m_ref, b, _ = walks(walk_lib, used)
        assert m_dev == m_ref and np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ the whole entry point
def emu_mesh(emu, V, F):
    V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
    h = C.c_void_p()
    assert emu.dg_mesh_create(_p(V, _dp), len(V), _p(F, _u32p), len(F), C.byref(h)) == 0
    return h


def desc_of(mn, mx, res, cell=None, inv=None):
    from discregrid_b200 import _capi as capi
    from discregrid_b200.grid import grid_desc
    return grid_desc(mn, mx, res, cell, inv), capi


def reduced_band(emu, h, d, sign, band, flags=0):
    """dg_reduced_band_create + sizes + copy: (nodes, cells, cell_map, timings)"""
    r = C.c_void_p()
    tm = np.full(7, -1.0)
    rc = emu.dg_reduced_band_create(h, C.byref(d), sign, band, flags, C.byref(r), _p(tm, _dp))
    assert rc == 0, emu.dg_last_error()
    nn, nc = C.c_uint64(), C.c_uint64()
    assert emu.dg_reduced_band_sizes(r, C.byref(nn), C.byref(nc)) == 0
    nodes = np.empty(nn.value); cells = np.empty((nc.value, 32), np.uint32)
    cmap = np.empty(int(np.prod(np.array(d.resolution[:], np.uint64))), np.uint32)
    assert emu.dg_reduced_band_copy(r, _p(nodes, _dp), _p(cells, _u32p), _p(cmap, _u32p)) == 0
    assert emu.dg_reduced_band_destroy(r) == 0
    return nodes, cells, cmap, tm


def old_route(emu, h, d, sign, band, flags=0):
    """dg_add_function_sdf_band + keep flags (always-true predicate and :1073) + dg_reduce_field with every pass on the host"""
    nn = C.c_uint64()
    emu.dg_grid_num_nodes(d.resolution, C.byref(nn))
    nc = int(np.prod(np.array(d.resolution[:], np.uint64)))
    nodes = np.empty(nn.value); cells = np.empty((nc, 32), np.uint32); cmap = np.empty(nc, np.uint32)
    assert emu.dg_add_function_sdf_band(h, C.byref(d), sign, band, _p(nodes, _dp), _p(cells, _u32p), _p(cmap, _u32p), None) == 0
    keep = np.ascontiguousarray(nodes != DBL_MAX, np.uint8)
    n_out, c_out = C.c_uint64(), C.c_uint64()
    tm = np.zeros(5)
    assert emu.dg_reduce_field(C.byref(d), _p(nodes, _dp), len(nodes), _p(keep, _u8p), _p(cells, _u32p), nc, _p(cmap, _u32p), flags | HOST_PASSES,
                               C.byref(n_out), C.byref(c_out), _p(tm, _dp)) == 0
    return nodes[:n_out.value], cells[:c_out.value], cmap, tm


def case_setup(emu, name):
    case = CASES[name]
    path = os.path.join(ROOT, "tests", case["mesh"]) if case["mesh"].startswith("golden/") else os.path.join(ROOT, "oracle", "_ref", "resources", case["mesh"])
    if not os.path.exists(path):
        pytest.skip(f"{path} missing (oracle/_ref resources)")
    V, F = read_obj(path)
    g = read_cdf(os.path.join(GOLDEN, case["file"]))
    d, _ = desc_of(g["mn"], g["mx"], g["res"], g["cell"], g["inv"])
    return case, g, emu_mesh(emu, V, F), d


def write_reduced_cdf(path, g, nodes, cells, cmap):
    import struct
    with open(path, "wb") as fh:
        fh.write(struct.pack("<6d", *g["mn"], *g["mx"])); fh.write(struct.pack("<3I", *[int(r) for r in g["res"]]))
        fh.write(struct.pack("<3d", *g["cell"])); fh.write(struct.pack("<3d", *g["inv"]))
        fh.write(struct.pack("<QQ", int(np.prod(g["res"].astype(np.uint64))), 1))
        for a in (nodes, cells, cmap):
            fh.write(struct.pack("<QQ", 1, len(a))); fh.write(np.ascontiguousarray(a).tobytes())


@pytest.mark.parametrize("flags", [0, REFERENCE_SORT])
@pytest.mark.parametrize("name", sorted(CASES))
def test_entry_point_equals_band_then_reduce_field(emu, tmp_path, name, flags):
    """the four band fixtures (box with nodes at the band edge, bunny, dragon inverted, anisotropic sphere): same nodes, cells and cell
    map as the two-step route; the two reduced fixtures are byte-identical once written"""
    case, g, h, d = case_setup(emu, name)
    sign, band = (-1.0 if case["invert"] else 1.0), float.fromhex(case["band_hex"])
    nodes, cells, cmap, tm = reduced_band(emu, h, d, sign, band, flags)
    want = old_route(emu, h, d, sign, band, flags)
    emu.dg_mesh_destroy(h)
    assert bits_equal(nodes, want[0]) and np.array_equal(cells, want[1]) and np.array_equal(cmap, want[2])
    assert tm[5] == want[3][4] and (tm[:5] >= 0).all() and tm[6] >= tm[:5].sum() - 1e-6
    if name == "sphere_aniso":
        assert tm[5] == 1.0                                                    # the anisotropic cells give equal Z-curve keys: the tie path
    if case["reduce"]:
        out = str(tmp_path / "out.cdf")
        write_reduced_cdf(out, g, nodes, cells, cmap)
        assert open(out, "rb").read() == open(os.path.join(GOLDEN, case["file"]), "rb").read()


def test_entry_point_widths_zero_infinite_and_empty(emu):
    """w = 0, w = +inf (every node kept: all cells, all nodes, only reordered) and a width at which nothing survives (no nodes, no cells,
    cell map all 0xffffffff), with and without the reference sort"""
    V, F = read_obj(os.path.join(GOLDEN, "sphere.obj"))
    h = emu_mesh(emu, V, F)
    d, _ = desc_of([-1.5, -1.5, -1.5], [1.5, 1.5, 1.5], (7, 6, 5))
    for flags in (0, REFERENCE_SORT):
        for w in (0.0, float("inf"), 1e-3):
            got = reduced_band(emu, h, d, 1.0, w, flags)
            want = old_route(emu, h, d, 1.0, w, flags)
            assert bits_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), w
            if w == float("inf"):
                assert len(got[1]) == 7 * 6 * 5 and np.array_equal(got[2], np.arange(7 * 6 * 5, dtype=np.uint32))
            if w == 1e-3:
                assert len(got[0]) == 0 and len(got[1]) == 0 and (got[2] == 0xFFFFFFFF).all()
    emu.dg_mesh_destroy(h)


def test_entry_point_refuses_invalid_input(emu):
    """a negative or NaN band, NULL arguments, unknown flags and a grid of 2^31 nodes or more are refused; the handle calls check theirs"""
    V, F = read_obj(os.path.join(GOLDEN, "sphere.obj"))
    h = emu_mesh(emu, V, F)
    d, capi = desc_of([-1.5, -1.5, -1.5], [1.5, 1.5, 1.5], (7, 6, 5))
    r = C.c_void_p()
    for bad in (-1.0, float("nan"), -1e-300):
        assert emu.dg_reduced_band_create(h, C.byref(d), 1.0, bad, 0, C.byref(r), None) == capi.DG_ERR_INVALID and not r.value
    assert emu.dg_reduced_band_create(None, C.byref(d), 1.0, 0.1, 0, C.byref(r), None) == capi.DG_ERR_INVALID
    assert emu.dg_reduced_band_create(h, None, 1.0, 0.1, 0, C.byref(r), None) == capi.DG_ERR_INVALID
    assert emu.dg_reduced_band_create(h, C.byref(d), 1.0, 0.1, 0, None, None) == capi.DG_ERR_INVALID
    assert emu.dg_reduced_band_create(h, C.byref(d), 1.0, 0.1, HOST_PASSES, C.byref(r), None) == capi.DG_ERR_INVALID
    big, _ = desc_of([0, 0, 0], [1, 1, 1], (7, 7, 7))
    for k in range(3):                                                       # 700^3: 2,408,356,301 nodes, in [2^31, 2^32)
        big.resolution[k] = 700; big.cell_size[k] = 1.0 / 700; big.inv_cell_size[k] = 700.0
    assert emu.dg_reduced_band_create(h, C.byref(big), 1.0, 0.1, 0, C.byref(r), None) == capi.DG_ERR_INVALID and not r.value
    assert b"grid too large" in emu.dg_last_error()
    n1, n2 = C.c_uint64(), C.c_uint64()
    assert emu.dg_reduced_band_sizes(None, C.byref(n1), C.byref(n2)) == capi.DG_ERR_INVALID
    assert emu.dg_reduced_band_create(h, C.byref(d), 1.0, 0.3, 0, C.byref(r), None) == 0
    assert emu.dg_reduced_band_sizes(r, None, C.byref(n2)) == capi.DG_ERR_INVALID
    assert emu.dg_reduced_band_sizes(r, C.byref(n1), C.byref(n2)) == 0 and n1.value > 0
    cmap = np.empty(7 * 6 * 5, np.uint32)
    assert emu.dg_reduced_band_copy(r, None, None, _p(cmap, _u32p)) == capi.DG_ERR_INVALID
    assert emu.dg_reduced_band_copy(None, None, None, _p(cmap, _u32p)) == capi.DG_ERR_INVALID
    assert emu.dg_reduced_band_destroy(r) == 0 and emu.dg_reduced_band_destroy(None) == 0
    emu.dg_mesh_destroy(h)
