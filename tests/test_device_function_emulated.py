"""User functions on the GPU -- dg_add_function_device, dg_reduced_function_create, dg_reduce_field_device -- on the CPU: the product's
kernels and C-ABI compiled into build/bin/libdgemu.so (tests/emu), where "device" pointers are host memory, so the callbacks here are numpy
over the library's buffers.  Every entry point must equal the host route (dg_node_positions, the function and predicates evaluated in
numpy, dg_build_cells + identity map, dg_reduce_field with every pass on the host) bit for bit, and rebuild the reference's own fixtures
(tests/golden/make_device_function_golden.py) byte for byte.  The GPU runs are tests/test_gpu_device_function.py."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal, ref_resource
from test_oracle_golden import read_cdf

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
CASES = json.load(open(os.path.join(GOLDEN, "ref_devfn_cases.json")))
DBL_MAX = np.finfo(np.float64).max
REFERENCE_SORT, HOST_PASSES = 1, 2
DG_ERR_INVALID, DG_ERR_CALLBACK = -1, -7
_dp, _u32p, _u8p, _vp = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), C.c_void_p


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


def capi():
    from discregrid_b200 import _capi
    return _capi


# ------------------------------------------------------------------------------------------------ the analytic case, in numpy
def func_np(x, p):
    """std::sqrt((dx*dx + dy*dy) + dz*dz) - r, operation for operation"""
    dx, dy, dz = x[:, 0] - p["centre"][0], x[:, 1] - p["centre"][1], x[:, 2] - p["centre"][2]
    return np.sqrt((dx * dx + dy * dy) + dz * dz) - p["r"]


def sample_np(x, p):
    return x[:, 0] + 0.5 * x[:, 1] < p["c"]


def reduce_np(x, v, p):
    return (v <= p["vmax"]) & (x[:, 2] > p["z0"])


def desc_of(case):
    from discregrid_b200.grid import grid_desc
    return grid_desc(case["mn"], case["mx"], case["res"])


def n_grid_cells(d):
    return int(np.prod(np.array(d.resolution[:], np.uint64)))


def n_nodes_of(emu, d):
    nn = C.c_uint64()
    assert emu.dg_grid_num_nodes(d.resolution, C.byref(nn)) == 0
    return nn.value


def arr(addr, n, ctype, shape=None):
    return np.ctypeslib.as_array(C.cast(addr, C.POINTER(ctype)), shape=shape or (n,))


class Callbacks:
    """numpy callbacks over the emulated library's buffers; every chunk each callback sees is recorded"""

    def __init__(self, func=None, sample=None, node=None, fail=None):
        cap = capi()
        self.seen = {"function": [], "sample": [], "node": []}
        self.fail = fail or {}

        def pos(x, n):
            return arr(x, n, C.c_double, (n, 3)).copy()

        def run(kind, n, body):
            self.seen[kind].append(n)
            if self.fail.get(kind) == len(self.seen[kind]):
                return 3
            body()
            return 0

        def f(_u, x, keep, n, values, _s):
            def body():
                k = None if not keep else arr(keep, n, C.c_uint8).copy()
                arr(values, n, C.c_double)[:] = func(pos(x, n), k)
            return run("function", n, body)

        def s(_u, x, n, keep, _s):
            return run("sample", n, lambda: arr(keep, n, C.c_uint8).__setitem__(slice(None), sample(pos(x, n))))

        def q(_u, x, values, n, keep, _s):
            return run("node", n, lambda: arr(keep, n, C.c_uint8).__setitem__(slice(None), node(pos(x, n), arr(values, n, C.c_double).copy())))

        self.func = cap.DEVICE_FUNCTION(f) if func else cap.DEVICE_FUNCTION()
        self.sample = cap.DEVICE_SAMPLE_PREDICATE(s) if sample else cap.DEVICE_SAMPLE_PREDICATE()
        self.node = cap.DEVICE_NODE_PREDICATE(q) if node else cap.DEVICE_NODE_PREDICATE()


def as_u8(mask):
    return np.asarray(mask, bool).astype(np.uint8)


def add_new(emu, d, cb, chunk=0):
    n = n_nodes_of(emu, d)
    nodes, cells, cmap, tm = np.empty(n), np.empty((n_grid_cells(d), 32), np.uint32), np.empty(n_grid_cells(d), np.uint32), np.full(6, -1.0)
    rc = emu.dg_add_function_device(C.byref(d), cb.func, None, cb.sample, None, chunk, _p(nodes, _dp), _p(cells, _u32p), _p(cmap, _u32p), _p(tm, _dp))
    return rc if rc else ((nodes, cells, cmap), tm)


def read_handle(emu, h, d):
    nn, nc = C.c_uint64(), C.c_uint64()
    assert emu.dg_reduced_band_sizes(h, C.byref(nn), C.byref(nc)) == 0
    f = (np.empty(nn.value), np.empty((nc.value, 32), np.uint32), np.empty(n_grid_cells(d), np.uint32))
    assert emu.dg_reduced_band_copy(h, _p(f[0], _dp), _p(f[1], _u32p), _p(f[2], _u32p)) == 0
    assert emu.dg_reduced_band_destroy(h) == 0
    return f


def reduced_new(emu, d, cb, chunk=0, flags=0):
    h, tm = _vp(), np.full(8, -1.0)
    rc = emu.dg_reduced_function_create(C.byref(d), cb.func, None, cb.sample, None, cb.node, None, chunk, flags, C.byref(h), _p(tm, _dp))
    if rc:
        assert not h.value
        return rc
    return read_handle(emu, h, d), tm


def reduce_field_new(emu, d, nodes, cells, cb, chunk=0, flags=0):
    nodes, cells = np.ascontiguousarray(nodes, np.float64), np.ascontiguousarray(cells, np.uint32)
    h, tm = _vp(), np.full(8, -1.0)
    rc = emu.dg_reduce_field_device(C.byref(d), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), cb.node, None, chunk, flags, C.byref(h),
                                    _p(tm, _dp))
    if rc:
        assert not h.value
        return rc
    return read_handle(emu, h, d), tm


def positions(emu, d, n):
    x = np.empty((n, 3))
    assert emu.dg_node_positions(C.byref(d), 0, n, _p(x, _dp)) == 0
    return x


def closed_cells(emu, d):
    res = np.array(d.resolution[:], np.uint32)
    cells = np.empty((n_grid_cells(d), 32), np.uint32)
    assert emu.dg_build_cells(_p(res, _u32p), 0, len(cells), _p(cells, _u32p)) == 0
    return cells


def reduce_host(emu, d, nodes, cells, keep, flags):
    nodes = np.ascontiguousarray(nodes, np.float64).copy(); cells = np.ascontiguousarray(cells, np.uint32).copy()
    keep = np.ascontiguousarray(keep, np.uint8)
    cmap = np.empty(n_grid_cells(d), np.uint32)
    n_out, c_out, tm = C.c_uint64(), C.c_uint64(), np.zeros(5)
    assert emu.dg_reduce_field(C.byref(d), _p(nodes, _dp), len(nodes), _p(keep, _u8p), _p(cells, _u32p), len(cells), _p(cmap, _u32p),
                               flags | HOST_PASSES, C.byref(n_out), C.byref(c_out), _p(tm, _dp)) == 0, emu.dg_last_error()
    return (nodes[:n_out.value].copy(), cells[:c_out.value].copy(), cmap), tm[4]


def host_route(emu, d, func, sample=None, node=None, flags=0):
    """addSampledFunction of numpy values at dg_node_positions, then dg_reduce_field (host passes) with keep = node && v != DBL_MAX"""
    n = n_nodes_of(emu, d)
    x = positions(emu, d, n)
    with np.errstate(invalid="ignore"):
        v = func(x, None) if sample is None else np.where(sample(x) != 0, func(x, None), DBL_MAX)
    dense = (v, closed_cells(emu, d), np.arange(n_grid_cells(d), dtype=np.uint32))
    if node is None:
        return dense, None
    with np.errstate(invalid="ignore"):
        keep = (np.asarray(node(x, v)) != 0) & (v != DBL_MAX)
    return dense, reduce_host(emu, d, v, dense[1], keep, flags)


def same_field(a, b):
    return bits_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def write_cdf(path, d, f):
    """the reference's save() of a one-field grid (cubic_lagrange_discrete_grid.cpp:678-719)"""
    with open(path, "wb") as fh:
        fh.write(struct.pack("<6d", *d.domain_min[:], *d.domain_max[:])); fh.write(struct.pack("<3I", *d.resolution[:]))
        fh.write(struct.pack("<3d", *d.cell_size[:])); fh.write(struct.pack("<3d", *d.inv_cell_size[:]))
        fh.write(struct.pack("<QQ", n_grid_cells(d), 1))
        for k in range(3):
            fh.write(struct.pack("<QQ", 1, len(f[k]))); fh.write(np.ascontiguousarray(f[k]).tobytes())


def case_callbacks(case):
    f = (lambda x, k: func_np(x, case))
    s = (lambda x: as_u8(sample_np(x, case))) if case["sample"] else None
    q = (lambda x, v: as_u8(reduce_np(x, v, case))) if case["reduce"] else None
    return f, s, q


# ------------------------------------------------------------------------------------------------ fixtures and the host route
@pytest.mark.parametrize("flags", [0, REFERENCE_SORT])
@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_equal_host_route_and_reference(emu, tmp_path, name, flags):
    """all three entry points against the host route, bit for bit, and the reference's own .cdf byte for byte"""
    case = CASES[name]
    d = desc_of(case)
    f, s, q = case_callbacks(case)
    want = open(os.path.join(GOLDEN, case["file"]), "rb").read()
    dense, reduced = host_route(emu, d, f, s, q, flags)
    got, tm = add_new(emu, d, Callbacks(f, s))
    assert same_field(got, dense)
    assert tm[0] >= tm[1] >= 0 and tm[4] >= 1 and tm[5] >= 0
    if not case["reduce"]:
        out = str(tmp_path / "dense.cdf"); write_cdf(out, d, got)
        assert open(out, "rb").read() == want
        return
    one, tm = reduced_new(emu, d, Callbacks(f, s, q), flags=flags)
    assert same_field(one, reduced[0]) and tm[5] == reduced[1]
    assert (tm >= 0).all() and tm[6] >= tm[:5].sum() - 1e-6
    if name == "aniso_reduced":
        assert tm[5] == 1.0                                                  # survivors share Z-curve keys: the tie order is exercised
    two, _ = reduce_field_new(emu, d, dense[0], dense[1], Callbacks(node=q), flags=flags)
    assert same_field(two, reduced[0])
    for field in (one, two):
        out = str(tmp_path / "reduced.cdf"); write_cdf(out, d, field)
        assert open(out, "rb").read() == want


@pytest.mark.parametrize("flags", [0, REFERENCE_SORT])
def test_reduce_field_device_rebuilds_ref_aniso_reduced(emu, tmp_path, flags):
    """reduceField(0, 0.3 <= v <= 0.9) of ref_aniso_field.cdf through a device node predicate: the reference's ref_aniso_reduced.cdf"""
    g = read_cdf(os.path.join(GOLDEN, "ref_aniso_field.cdf"))
    from discregrid_b200.grid import grid_desc
    d = grid_desc(g["mn"], g["mx"], g["res"], g["cell"], g["inv"])
    got, tm = reduce_field_new(emu, d, g["nodes"][0], g["cells"][0], Callbacks(node=lambda x, v: as_u8((0.3 <= v) & (v <= 0.9))), flags=flags)
    out = str(tmp_path / "out.cdf"); write_cdf(out, d, got)
    assert open(out, "rb").read() == open(os.path.join(GOLDEN, "ref_aniso_reduced.cdf"), "rb").read()


def test_chunk_sizes_give_identical_outputs_and_complete_ascending_chunks(emu):
    """chunk_nodes 1, 7, 1000 and the default: the same bits; every callback sees chunks that are contiguous, ascending and cover the grid
    (checked through the positions it receives, which must be the chunk's own node positions)"""
    case = CASES["aniso_reduced"]
    d = desc_of(case)
    n = n_nodes_of(emu, d)
    xall = positions(emu, d, n)
    f, s, q = case_callbacks(case)
    ids = []

    def f_checked(x, k):
        b = sum(len(i) for i in ids)
        assert bits_equal(x, xall[b:b + len(x)])                             # the chunk [b, b + n) in order, positions of dg_node_positions
        ids.append(np.arange(b, b + len(x)))
        return f(x, k)
    results = []
    for chunk in (1, 7, 1000, 0):
        ids.clear()
        cb = Callbacks(f_checked, s, q)
        got, tm = reduced_new(emu, d, cb, chunk=chunk)
        want_sizes = [min(chunk or n, n - b) for b in range(0, n, chunk or n)]
        assert cb.seen["function"] == want_sizes and cb.seen["sample"] == want_sizes and cb.seen["node"] == want_sizes
        assert np.array_equal(np.concatenate(ids), np.arange(n))
        ids.clear()
        dense, _ = add_new(emu, d, Callbacks(f_checked, s), chunk=chunk)
        results.append((got, dense))
    for got, dense in results[1:]:
        assert same_field(got, results[0][0]) and same_field(dense, results[0][1])


def test_masks_other_than_0_1_nan_and_dbl_max_values(emu):
    """mask bytes 2, 128 and 255 mean keep; the function itself returns NaN and DBL_MAX at some nodes (DBL_MAX is then never kept, a NaN
    only when the node predicate says so); the function sees the sample mask as given"""
    case = CASES["box_reduced"]
    d = desc_of(case)
    n = n_nodes_of(emu, d)
    x = positions(emu, d, n)
    rng = np.random.default_rng(5)
    smask = rng.choice(np.array([0, 1, 2, 128, 255], np.uint8), size=n)
    nmask = rng.choice(np.array([0, 3, 255], np.uint8), size=n)
    base = func_np(x, case)
    special = base.copy()
    special[::7] = np.nan
    special[3::11] = DBL_MAX
    lookup = {tuple(r): i for i, r in enumerate(x)}

    def idx(xc):
        return np.array([lookup[tuple(r)] for r in xc])

    def f(xc, k):
        i = idx(xc)
        assert k is not None and np.array_equal(k, smask[i])
        return special[i]
    s = (lambda xc: smask[idx(xc)])
    q = (lambda xc, v: nmask[idx(xc)])
    for flags in (0, REFERENCE_SORT):
        dense, reduced = host_route(emu, d, lambda xx, k: special, lambda xx: smask, lambda xx, v: nmask, flags)
        got, _ = add_new(emu, d, Callbacks(f, s), chunk=13)
        assert same_field(got, dense)
        one, tm = reduced_new(emu, d, Callbacks(f, s, q), chunk=13, flags=flags)
        assert same_field(one, reduced[0]) and len(one[0]) > 0
        two, _ = reduce_field_new(emu, d, dense[0], dense[1], Callbacks(node=q), chunk=5, flags=flags)
        assert same_field(two, reduced[0])
        assert np.isnan(one[0]).any()


def test_nothing_kept_and_everything_kept(emu):
    case = CASES["aniso_reduced"]
    d = desc_of(case)
    n = n_nodes_of(emu, d)
    f = (lambda x, k: func_np(x, case))
    none = (lambda x, v: np.zeros(len(x), np.uint8))
    every = (lambda x, v: np.ones(len(x), np.uint8))
    got, _ = reduced_new(emu, d, Callbacks(f, node=none))
    assert len(got[0]) == 0 and len(got[1]) == 0 and (got[2] == 0xFFFFFFFF).all()
    got, _ = reduced_new(emu, d, Callbacks(f, node=every))
    dense, reduced = host_route(emu, d, f, None, every)
    assert same_field(got, reduced[0]) and len(got[0]) == n and np.array_equal(got[2], np.arange(n_grid_cells(d), dtype=np.uint32))
    got, _ = reduced_new(emu, d, Callbacks(f))                               # no reduce predicate: always true
    assert same_field(got, reduced[0])
    got, _ = reduced_new(emu, d, Callbacks(f, sample=lambda x: np.zeros(len(x), np.uint8)))     # every node DBL_MAX
    assert len(got[0]) == 0 and (got[2] == 0xFFFFFFFF).all()


def test_refusals(emu):
    """NULL callbacks, unknown flags, an already reduced field, more rows than cells, a row naming a node >= n_nodes, a grid of 2^31 nodes or
    more, and a callback returning nonzero (DG_ERR_CALLBACK naming the callback and the chunk, no handle)"""
    case = CASES["box_reduced"]
    d = desc_of(case)
    f, s, q = case_callbacks(case)
    none = Callbacks()
    assert add_new(emu, d, none) == DG_ERR_INVALID and b"function callback is NULL" in emu.dg_last_error()
    assert reduced_new(emu, d, Callbacks(node=q)) == DG_ERR_INVALID
    dense, reduced = host_route(emu, d, f, s, q)
    assert reduce_field_new(emu, d, dense[0], dense[1], Callbacks(f)) == DG_ERR_INVALID and b"node predicate callback is NULL" in emu.dg_last_error()
    for flags in (HOST_PASSES, 4, 0x80000000):
        assert reduced_new(emu, d, Callbacks(f, s, q), flags=flags) == DG_ERR_INVALID and b"unknown flags" in emu.dg_last_error()
        assert reduce_field_new(emu, d, dense[0], dense[1], Callbacks(node=q), flags=flags) == DG_ERR_INVALID
    assert reduce_field_new(emu, d, reduced[0][0], reduced[0][1], Callbacks(node=q)) == DG_ERR_INVALID
    assert b"already reduced" in emu.dg_last_error()
    assert reduce_field_new(emu, d, dense[0], np.concatenate([dense[1], dense[1][:1]]), Callbacks(node=q)) == DG_ERR_INVALID
    bad = dense[1].copy(); bad[17, 4] = len(dense[0])
    assert reduce_field_new(emu, d, dense[0], bad, Callbacks(node=q)) == DG_ERR_INVALID and b"node id >= n_nodes" in emu.dg_last_error()
    h = _vp()
    cb = Callbacks(f, s, q)
    assert emu.dg_reduced_function_create(C.byref(d), cb.func, None, cb.sample, None, cb.node, None, 0, 0, None, None) == DG_ERR_INVALID
    big = desc_of(case)
    for k in range(3):                                                       # 700^3: 2,408,356,301 nodes, in [2^31, 2^32)
        big.resolution[k] = 700; big.cell_size[k] = 1.0 / 700; big.inv_cell_size[k] = 700.0
    assert emu.dg_reduced_function_create(C.byref(big), cb.func, None, cb.sample, None, cb.node, None, 0, 0, C.byref(h), None) == DG_ERR_INVALID
    assert b"grid too large" in emu.dg_last_error() and not h.value and cb.seen["function"] == []
    n = n_nodes_of(emu, d)
    s = (lambda x: as_u8(sample_np(x, dict(case, c=1.2))))
    for kind, which in (("function", 2), ("sample", 1), ("node", 3)):
        cb = Callbacks(f, s, q, fail={kind: which})
        assert reduced_new(emu, d, cb, chunk=100) == DG_ERR_CALLBACK
        msg = emu.dg_last_error().decode()
        b = 100 * (which - 1)
        assert "returned 3" in msg and f"[{b}, {min(b + 100, n)})" in msg and {"function": "function", "sample": "sample predicate",
                                                                               "node": "node predicate"}[kind] in msg, msg
        assert len(cb.seen[kind]) == which                                   # nothing is called after the failure
        if kind != "node":
            assert add_new(emu, d, Callbacks(f, s, fail={kind: which}), chunk=100) == DG_ERR_CALLBACK
    assert reduce_field_new(emu, d, dense[0], dense[1], Callbacks(node=q, fail={"node": 1})) == DG_ERR_CALLBACK


# ------------------------------------------------------------------------------------------------ a callback that calls the library
def mesh_sdf_callback(emu, mesh):
    """a DeviceFunction that calls dg_mesh_distance_device on the positions: the route must equal dg_add_function_sdf bit for bit"""
    def f(_u, x, keep, n, values, stream):
        return emu.dg_mesh_distance_device(mesh, x, n, 1, values, None, None, None, stream)
    return capi().DEVICE_FUNCTION(f)


@pytest.mark.parametrize("which", ["box", "bunny"])
def test_mesh_distance_callback_equals_add_function_sdf(emu, which):
    from discregrid_b200.grid import grid_desc
    if which == "box":
        from discregrid_b200.mesh import box
        m = box()
        V, F = np.ascontiguousarray(m.vertices, np.float64), np.ascontiguousarray(m.faces, np.uint32)
        res = (5, 4, 6)
    else:
        path = ref_resource("bunny.obj")
        if path is None:
            pytest.skip("bunny.obj not staged (make -C oracle ref)")
        pv, nv, pf, nf = _dp(), C.c_uint64(), _u32p(), C.c_uint64()
        assert emu.dg_obj_read(path.encode(), C.byref(pv), C.byref(nv), C.byref(pf), C.byref(nf)) == 0
        V = np.ctypeslib.as_array(pv, (nv.value, 3)).copy(); F = np.ctypeslib.as_array(pf, (nf.value, 3)).copy()
        emu.dg_obj_free(pv, pf)
        res = (6, 6, 6)
    mesh = _vp()
    assert emu.dg_mesh_create(_p(V, _dp), len(V), _p(F, _u32p), len(F), C.byref(mesh)) == 0
    try:
        mn, mx = np.empty(3), np.empty(3)
        assert emu.dg_generate_sdf_domain(_p(V, _dp), len(V), _p(mn, _dp), _p(mx, _dp)) == 0
        d = grid_desc(mn, mx, res)
        n = n_nodes_of(emu, d)
        want = (np.empty(n), np.empty((n_grid_cells(d), 32), np.uint32), np.empty(n_grid_cells(d), np.uint32))
        assert emu.dg_add_function_sdf(mesh, C.byref(d), 1.0, _p(want[0], _dp), _p(want[1], _u32p), _p(want[2], _u32p), None) == 0
        cb = Callbacks()
        cb.func = mesh_sdf_callback(emu, mesh)
        got, _ = add_new(emu, d, cb, chunk=50)
        assert same_field(got, want)
    finally:
        emu.dg_mesh_destroy(mesh)
