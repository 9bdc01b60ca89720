#!/usr/bin/env python
"""Parity fuzzer for K11 (the VJP of interpolate in the node values, discregrid_b200/csrc/k11_field_grad.cu: key, radix-sort, segment, level
and node passes, and the trainable field's incidence table) against the numpy restatement of its contract (tests/interpolate_vjp_ref.py), bit
for bit, any NaN equal to any NaN; an untouched node must be +0.0 exactly (the comparison is on the bits).
  fields   k2_fuzz.make_field rounds (plain, DBL_MAX, reduced, huge / non-finite / tiny coefficients, no kept cell, exactly one) made
           trainable, k2_fuzz.queries points, upstreams phi, grad and both, at n = 0, 1, 31, 32, 33, 127, 129 (K11_THREADS = 128) and all
  tables   tables no grid makes (the contract is defined on the table): permuted node ids, node arrays padded with unreferenced nodes (long
           runs in the inc_begin pass), a hub node in one slot of every one of 2^12 cells (and a whole row of it in 32 cells), largest node
           id exactly 2^8, 2^16, 2^24 (n_nodes = 2^k + 1: the incidence sort needs k + 1 key bits)
  passes   n_cells_kept = 2^8 (8 x 8 x 4), 2^16 (64 x 64 x 16), 2^16 - 1 and 2^16 + 1 (reduced), with a query in the last kept cell, whose key
           n_cells_kept needs one more bit than n_cells_kept - 1; with `big`, 2^24 (256^3, below)
  closed   cells == NULL (the closed-form table, cell_node_id) against the uploaded table of the same grid: VJP, interpolate and set_nodes
           give the same bits, on 1 x 1 x 1, 1 x 1 x N, N x 1 x 1, 7 x 5 x 3; with `big`, 256^3 (n_cells_kept = 2^24, 25 key bits, 4 passes
           of the query sort; node ids up to 118 M, 27 bits, 4 passes of the incidence sort)
  depth    cells holding 31, 32, 33, 1023, 1025, 32767, 32769 queries in one call (levels S = 1, 32, 1024); with `big`, one cell holding
           2^20 + 1 queries among others (32769 groups: the level with S = 32768)
  strides  (`big`) 2^20 queries on 128^3 (~10^6 groups, more than the first level's 16384 warps); 2^19 + 2^16 singleton cells and deep
           cells at the highest cell ids (more than the 2^19 threads of a higher level, the deep groups past them)
  values   +-0, subnormal, +-1e308, +-inf, NaN upstreams; a set_nodes_device that plants a DBL_MAX, then a VJP on the same stream
With `dg` every VJP runs twice through dg_interpolate_vjp and, with `side`, once through dg_interpolate_vjp_device on a side stream: all must
give the same bits.  On libdgemu.so the device form takes host memory.

usage: tools/k11_fuzz.py [rounds=24] [seed=0] [lib=emu] [big]
  lib   `emu`: build/bin/libdgemu.so (the whole C-ABI with its kernels compiled for the CPU), a path to such a build, or `dg`: the product
        library through its C-ABI, i.e. the CUDA kernels
  big   also the 256^3, 2^20-query-cell and stride families
The functions are shared with tests/test_vjp_fuzz_emulated.py and tests/test_gpu_vjp_fuzz.py."""
import ctypes as C
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import k2_fuzz  # noqa: E402
import interpolate_vjp_ref as ref  # noqa: E402
from oracle_api import Oracle  # noqa: E402

dp, u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)
DBL_MAX = ref.DBL_MAX
UINT32_MAX = 0xFFFFFFFF
K11_THREADS = 128                                    # csrc/k11_field_grad.h
COUNTS = (0, 1, 31, 32, 33, K11_THREADS - 1, K11_THREADS + 1)
DEPTHS = (31, 32, 33, 1023, 1025, 32767, 32769)
UPSTREAMS = ("phi", "grad", "both")
SPECIAL = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2e-308, 1e308, -1e308, np.inf, -np.inf, np.nan])
same = k2_fuzz.same
EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")


def _p(a, t=dp):
    return None if a is None else a.ctypes.data_as(t)


def _bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


class Lib:
    """the C-ABI of the product (`dg`) or of a libdgemu.so build.  vjp() runs the host form twice and the device form once (on a side stream
    with `side` on a device; with host memory and the default stream on the emulated library) and reports whether all gave the same bits"""

    def __init__(self, lib="dg", side=True):
        from discregrid_b200 import _capi
        self.GridDesc = _capi.GridDesc
        if lib == "dg":
            self.name, self.lib, self.emulated = "dg", _capi.lib, _capi.EMULATED
        else:
            self.name, self.lib, self.emulated = os.path.basename(lib), C.CDLL(lib), True
            for nm, (res, args) in _capi.SIGNATURES.items():
                f = getattr(self.lib, nm)
                f.restype, f.argtypes = res, args
        self.side = side

    def check(self, rc):
        if rc != 0:
            raise RuntimeError(f"rc {rc}: {self.lib.dg_last_error()}")

    def desc(self, mn, mx, res, cell=None, inv=None):
        d = self.GridDesc()
        mn = np.ascontiguousarray(mn, np.float64); mx = np.ascontiguousarray(mx, np.float64); r = np.ascontiguousarray(res, np.uint32)
        self.check(self.lib.dg_grid_init(_p(mn), _p(mx), _p(r, u32p), C.byref(d)))
        if cell is not None:
            for k in range(3):
                d.cell_size[k] = float(cell[k]); d.inv_cell_size[k] = float(inv[k])
        return d

    def num_nodes(self, res):
        n = C.c_uint64()
        self.check(self.lib.dg_grid_num_nodes(_p(np.ascontiguousarray(res, np.uint32), u32p), C.byref(n)))
        return n.value

    def build_cells(self, res):
        n = int(np.prod(np.asarray(res, np.int64)))
        cells = np.empty((n, 32), np.uint32)
        self.check(self.lib.dg_build_cells(_p(np.ascontiguousarray(res, np.uint32), u32p), 0, n, _p(cells, u32p)))
        return cells

    def create(self, fld, trainable=True):
        h = C.c_void_p()
        fn = self.lib.dg_field_create_trainable if trainable else self.lib.dg_field_create
        cells = None if fld.cells is None else np.ascontiguousarray(fld.cells, np.uint32)
        self.check(fn(C.byref(fld.d), _p(fld.nodes) if len(fld.nodes) else None, len(fld.nodes), _p(cells, u32p), fld.n_cells_kept,
                      _p(fld.cmap, u32p), C.byref(h)))
        return h

    def destroy(self, h):
        self.check(self.lib.dg_field_destroy(h))

    def set_nodes(self, h, nodes):
        nodes = np.ascontiguousarray(nodes, np.float64)
        self.check(self.lib.dg_field_set_nodes(h, _p(nodes), len(nodes)))

    def interpolate(self, h, x):
        x = np.ascontiguousarray(x, np.float64)
        phi, grad = np.full(len(x), 7.0), np.full((len(x), 3), 7.0)
        self.check(self.lib.dg_interpolate_batch(h, _p(x), len(x), _p(phi), _p(grad)))
        return phi, grad

    def _host(self, h, n_nodes, x, gphi, ggrad):
        out = np.full(n_nodes, 7.0)
        self.check(self.lib.dg_interpolate_vjp(h, _p(x), len(x), _p(gphi), _p(ggrad), _p(out)))
        return out

    def _device(self, h, n_nodes, x, gphi, ggrad, new_nodes=None):
        """dg_interpolate_vjp_device (after dg_field_set_nodes_device of new_nodes on the same stream, if given)"""
        if self.emulated:
            out = np.full(n_nodes, 5.0)
            if new_nodes is not None:
                self.check(self.lib.dg_field_set_nodes_device(h, new_nodes.ctypes.data, len(new_nodes), None))
            self.check(self.lib.dg_interpolate_vjp_device(h, x.ctypes.data, len(x), None if gphi is None else gphi.ctypes.data,
                                                          None if ggrad is None else ggrad.ctypes.data, out.ctypes.data, None))
            return out
        import torch
        # an empty tensor has a NULL data pointer, and NULL means "no upstream": give n = 0 calls a one-element buffer instead
        t = [None if a is None else torch.from_numpy(a if a.size else np.zeros(1)).cuda() for a in (x, gphi, ggrad, new_nodes)]
        out = torch.full((n_nodes,), 5.0, dtype=torch.float64, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            if new_nodes is not None:
                self.check(self.lib.dg_field_set_nodes_device(h, t[3].data_ptr(), len(new_nodes), s.cuda_stream))
            self.check(self.lib.dg_interpolate_vjp_device(h, t[0].data_ptr(), len(x), None if t[1] is None else t[1].data_ptr(),
                                                          None if t[2] is None else t[2].data_ptr(), out.data_ptr(), s.cuda_stream))
        s.synchronize()
        return out.cpu().numpy()

    def vjp(self, h, n_nodes, x, gphi, ggrad, repeat=True):
        x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
        gphi = None if gphi is None else np.ascontiguousarray(gphi, np.float64)
        ggrad = None if ggrad is None else np.ascontiguousarray(ggrad, np.float64)
        out = self._host(h, n_nodes, x, gphi, ggrad)
        if not repeat:
            return out, True
        runs = [self._host(h, n_nodes, x, gphi, ggrad)]
        if self.side:
            runs.append(self._device(h, n_nodes, x, gphi, ggrad))
        return out, all(_bits(r, out) for r in runs)

    def set_nodes_then_vjp(self, h, nodes, x, gphi, ggrad):
        """dg_field_set_nodes_device then dg_interpolate_vjp_device, queued on one stream with no synchronisation between them"""
        return self._device(h, len(nodes), np.ascontiguousarray(x, np.float64), None if gphi is None else np.ascontiguousarray(gphi),
                            None if ggrad is None else np.ascontiguousarray(ggrad), np.ascontiguousarray(nodes, np.float64))


def backend(lib, side=True):
    return Lib("dg" if lib == "dg" else (EMU if lib == "emu" else lib), side=side)


class Field:
    """a field's arrays: descriptor d, nodes, cells ([n_cells_kept, 32] or None: the closed-form table), cmap (None: the identity)"""

    def __init__(self, d, nodes, cells, cmap, label, n_cells_kept=None):
        self.d, self.nodes, self.cells, self.cmap, self.label = d, np.ascontiguousarray(nodes, np.float64), cells, cmap, label
        self.res = np.array(d.resolution[:], np.int64)
        self.n_cells_kept = len(cells) if cells is not None else (n_cells_kept or int(np.prod(self.res)))
        if cmap is not None:
            self.cmap = np.ascontiguousarray(cmap, np.uint32)

    @property
    def mn(self):
        return np.array(self.d.domain_min[:])

    @property
    def mx(self):
        return np.array(self.d.domain_max[:])

    def rows(self):
        return (lambda c, r=self.res: ref.closed_form_cells(r, c)) if self.cells is None else self.cells

    def restate(self, x, gphi, ggrad, nodes=None):
        d = self.d
        args = (d.domain_min[:], d.domain_max[:], d.cell_size[:], d.inv_cell_size[:], d.resolution[:], self.nodes if nodes is None else nodes)
        if self.cells is not None and len(x) <= 1 << 14 and 32 * self.n_cells_kept <= 1 << 22:
            return ref.interpolate_vjp(*args, self.cells, self.cmap, x, gphi, ggrad)
        return ref.interpolate_vjp_touched(*args, self.rows(), self.cmap, x, gphi, ggrad)

    def points(self, rng, n):
        return self.mn + rng.random((n, 3)) * (self.mx - self.mn)

    def cell_points(self, rng, c, m):
        """m points inside grid cell c (unreduced index)"""
        i, j, k = c % self.res[0], (c // self.res[0]) % self.res[1], c // (self.res[0] * self.res[1])
        cell = np.array(self.d.cell_size[:])
        return self.mn + (np.array([i, j, k]) + 0.05 + 0.9 * rng.random((m, 3))) * cell


def upstreams(rng, n, which, special=False):
    def vals(shape):
        v = rng.standard_normal(shape)
        if special:
            mask = rng.random(shape) < 0.35
            v[mask] = rng.choice(SPECIAL, size=int(mask.sum()))
        return v
    return (vals(n) if which in ("phi", "both") else None), (vals((n, 3)) if which in ("grad", "both") else None)


def check(be, fld, h, x, gphi, ggrad, label, repeat=True):
    """one VJP against the restatement -> (values checked, mismatches, first)"""
    x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
    want = fld.restate(x, gphi, ggrad)
    got, agree = be.vjp(h, len(fld.nodes), x, gphi, ggrad, repeat)
    ok = same(got, want)
    bad, first = int((~ok).sum()), None
    if bad:
        i = int(np.nonzero(~ok)[0][0])
        first = f"MISMATCH {fld.label} {label} n={len(x)}: node {i} {got[i]!r} vs {want[i]!r} ({bad} nodes)"
    if not agree:
        bad += 1; first = first or f"MISMATCH {fld.label} {label} n={len(x)}: repeated calls or the device form differ"
    return len(got), bad, first


class Acc:
    def __init__(self, log):
        self.cases = self.total = self.bad = 0
        self.log = log

    def add(self, r):
        n, b, msg = r
        self.cases += 1; self.total += n; self.bad += b
        if msg: self.log(msg)

    def result(self):
        return self.cases, self.total, self.bad


def run_with(be, fld, fn):
    h = be.create(fld)
    try:
        fn(h)
    finally:
        be.destroy(h)


# ---------------------------------------------------------------------------------------------------------------- families
def run_fields(be, rounds, seed=0, log=print, counts=COUNTS):
    """k2_fuzz.make_field rounds, trainable; every upstream at the prefix counts and at all of k2_fuzz.queries; special upstreams"""
    rng = np.random.default_rng(seed)
    orc = Oracle()
    acc = Acc(log)
    for k in range(rounds):
        with tempfile.TemporaryDirectory(prefix="k11_fuzz_") as tmp:          # make_field's .cdf round trips, removed with the directory
            gd, r, nodes, cells, cmap, label = k2_fuzz.make_field(orc, rng, k, tmp)
        fld = Field(be.desc(gd[0:3], gd[3:6], r, gd[6:9], gd[9:12]), nodes, np.ascontiguousarray(cells, np.uint32), cmap, label)
        x = k2_fuzz.queries(rng, gd, r, nodes, cells, cmap)

        def body(h):
            for which in UPSTREAMS:
                for n in counts:
                    sel = rng.choice(len(x), n, replace=False)
                    acc.add(check(be, fld, h, x[sel], *upstreams(rng, n, which), f"{which} n={n}"))
                acc.add(check(be, fld, h, x, *upstreams(rng, len(x), which), f"{which} all"))
                acc.add(check(be, fld, h, x, *upstreams(rng, len(x), which, True), f"{which} special"))
        run_with(be, fld, body)
    return acc.result()


def _grid(be, res, mn=(-1.0, -0.5, 0.25), ext=(2.0, 1.3, 0.9)):
    mn = np.asarray(mn, np.float64)
    return be.desc(mn, mn + np.asarray(ext, np.float64), res)


HUB = ((16, 16, 16), 6000)                                           # the hub's grid (2^12 cells) and its query count


def table_fields(be, seed=0, id_bits=(8, 16, 24), hub=HUB):
    """(Field, queries) of the tables no grid makes; hub: (resolution, queries) of the hub-node table"""
    rng = np.random.default_rng(seed + 3)
    res = (6, 5, 4)
    d = _grid(be, res)
    cells = be.build_cells(res).astype(np.int64)
    nn = be.num_nodes(res)
    perm = rng.permutation(nn)
    f = Field(d, rng.standard_normal(nn), perm[cells].astype(np.uint32), None, "permuted ids")
    yield f, f.points(rng, 700)
    res = (5, 4, 3)
    d = _grid(be, res)
    cells = be.build_cells(res).astype(np.int64)
    nn = be.num_nodes(res)
    big = 5 * nn + 1000
    spread = np.sort(rng.choice(big, nn, replace=False))
    spread[-1] = big - 1                                                 # the last node referenced, unreferenced runs before it
    f = Field(d, rng.standard_normal(big), spread[cells].astype(np.uint32), None, f"padded to {big} nodes")
    yield f, f.points(rng, 500)
    res = hub[0]
    d = _grid(be, res)
    cells = be.build_cells(res).astype(np.int64)
    nn = be.num_nodes(res)
    v = int(rng.integers(nn))
    cells[np.arange(len(cells)), np.arange(len(cells)) % 32] = v        # the hub in one slot of every cell, every slot in turn
    cells[rng.choice(len(cells), 32, replace=False)] = v                # and whole rows of it
    f = Field(d, rng.standard_normal(nn), cells.astype(np.uint32), None, f"hub node in {len(cells)} cells")
    yield f, f.points(rng, hub[1])
    for bits in id_bits:
        res = (3, 2, 2)
        d = _grid(be, res)
        top = 1 << bits
        cells = rng.integers(0, top + 1, (12, 32))
        cells[rng.integers(0, 12, 6), rng.integers(0, 32, 6)] = top
        cells[0, 0] = 0
        f = Field(d, rng.standard_normal(top + 1), cells.astype(np.uint32), None, f"largest node id 2^{bits}")
        yield f, f.points(rng, 300)


def run_tables(be, seed=0, log=print, id_bits=(8, 16, 24), hub=HUB):
    acc = Acc(log)
    rng = np.random.default_rng(seed + 5)
    for fld, x in table_fields(be, seed, id_bits, hub):
        def body(h):
            for which in UPSTREAMS:
                acc.add(check(be, fld, h, x, *upstreams(rng, len(x), which), which))
        run_with(be, fld, body)
    return acc.result()


def _reduced(be, res, n_keep, rng, label):
    """a reduced field of res keeping n_keep cells, the last grid cell among them, nodes renumbered"""
    cells = be.build_cells(res)
    n = len(cells)
    keep = np.zeros(n, bool)
    keep[rng.choice(n - 1, n_keep - 1, replace=False)] = True
    keep[n - 1] = True
    kept = np.flatnonzero(keep)
    cmap = np.full(n, UINT32_MAX, np.uint32); cmap[kept] = np.arange(len(kept), dtype=np.uint32)
    used = np.unique(cells[kept])
    ncells = np.searchsorted(used, cells[kept]).astype(np.uint32)
    return Field(_grid(be, res), rng.standard_normal(len(used)), ncells, cmap, label)


PASS_DENSE = ((8, 8, 4), (64, 64, 16))


def pass_fields(be, seed=0, dense=PASS_DENSE, reduced=True):
    rng = np.random.default_rng(seed + 7)
    for res in dense:
        n = int(np.prod(res))
        yield Field(_grid(be, res), rng.standard_normal(be.num_nodes(res)), be.build_cells(res), None,
                    f"dense {res}: n_cells_kept = 2^{n.bit_length() - 1}")
    if reduced:
        yield _reduced(be, (64, 64, 16), (1 << 16) - 1, rng, "reduced: n_cells_kept = 2^16 - 1")
        yield _reduced(be, (65, 64, 16), (1 << 16) + 1, rng, "reduced: n_cells_kept = 2^16 + 1")


def _last_cell_queries(fld, rng, m=5):
    """m points in the grid cell that holds the last kept cell"""
    c = int(np.flatnonzero(fld.cmap == fld.n_cells_kept - 1)[0]) if fld.cmap is not None else fld.n_cells_kept - 1
    return fld.cell_points(rng, c, m)


def run_passes(be, seed=0, log=print, n=3000, dense=PASS_DENSE, reduced=True):
    """pass boundaries of the query sort: queries in the last kept cell, among random ones and sentinels (key 0, outside or NaN), which a
    sort short of the top key bit would mix with the last cell's"""
    acc = Acc(log)
    rng = np.random.default_rng(seed + 9)
    for fld in pass_fields(be, seed, dense, reduced):
        out = fld.mx + rng.random((n // 10, 3)) * (fld.mx - fld.mn)
        out[::3, 1] = np.nan
        x = np.concatenate([fld.points(rng, n), _last_cell_queries(fld, rng), out])
        x = x[rng.permutation(len(x))]

        def body(h):
            for which in UPSTREAMS:
                acc.add(check(be, fld, h, x, *upstreams(rng, len(x), which), which))
            acc.add(check(be, fld, h, _last_cell_queries(fld, rng, 1), *upstreams(rng, 1, "both"), "the last cell alone"))
        run_with(be, fld, body)
    return acc.result()


CLOSED = ((1, 1, 1), (1, 1, 9), (9, 1, 1), (7, 5, 3))


def check_closed(be, res, rng, nq, label, log, measure=None):
    """cells == NULL against the uploaded table of the same grid: the VJP (both against the restatement), interpolate and set_nodes (a
    DBL_MAX planted) -> (cases, values, mismatches)"""
    acc = Acc(log)
    d = _grid(be, res)
    nn = be.num_nodes(res)
    nodes = rng.standard_normal(nn)
    closed = Field(d, nodes, None, None, f"closed form {res}")
    x = np.concatenate([closed.points(rng, nq), _last_cell_queries(closed, rng), closed.cell_points(rng, 0, 3)])
    x = x[rng.permutation(len(x))]
    ups = {w: upstreams(rng, len(x), w) for w in UPSTREAMS}
    new = nodes.copy()
    new[rng.choice(nn, 3, replace=False)] = DBL_MAX
    new[0] = -2.5
    results = []
    for fld in (closed, None):
        if fld is None:
            fld = Field(d, nodes, be.build_cells(res), None, f"uploaded table {res}")
        t0 = time.perf_counter()
        h = be.create(fld) if measure is None else measure(lambda: be.create(fld), fld.label)
        t1 = time.perf_counter()
        try:
            out = {}
            for w, (gp, gg) in ups.items():
                acc.add(check(be, fld, h, x, gp, gg, w, repeat=(fld.cells is None)))
                out[w] = be.vjp(h, nn, x, gp, gg, repeat=False)[0]
            out["interpolate"] = be.interpolate(h, x)
            be.set_nodes(h, new)
            out["set_nodes interpolate"] = be.interpolate(h, x)
            got, agree = be.vjp(h, nn, x, *ups["both"], repeat=False)
            want = fld.restate(x, *ups["both"], nodes=new)
            ok = same(got, want)
            acc.add((len(got), int((~ok).sum()), None if ok.all() else f"MISMATCH {fld.label} after set_nodes"))
            out["set_nodes vjp"] = got
            results.append(out)
        finally:
            be.destroy(h)
        if measure is not None:
            log(f"{fld.label}: created in {t1 - t0:.2f} s")
    for key in results[0]:
        a, b = results[0][key], results[1][key]
        a, b = (a if isinstance(a, tuple) else (a,)), (b if isinstance(b, tuple) else (b,))
        ok = all(_bits(u, v) for u, v in zip(a, b))
        acc.add((sum(len(u) for u in a), 0 if ok else 1, None if ok else f"MISMATCH closed form {res}: {key} differs from the uploaded table"))
    return acc.result()


def run_closed(be, seed=0, log=print, sizes=CLOSED):
    rng = np.random.default_rng(seed + 11)
    acc = [0, 0, 0]
    for res in sizes:
        r = check_closed(be, res, rng, 400, str(res), log)
        acc = [a + b for a, b in zip(acc, r)]
    return tuple(acc)


def run_256(be, seed=0, log=print, nq=200000):
    """256^3, closed form and uploaded: n_cells_kept = 2^24 (the query sort's 25 key bits), the last cell touched; creation time and peak
    device memory of each (sampled by a thread polling cudaMemGetInfo while the creation runs)"""
    rng = np.random.default_rng(seed + 13)
    measure = None
    if not be.emulated:
        import threading
        import torch

        def measure(fn, label):
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            low = [free0]
            done = threading.Event()

            def poll():
                while not done.is_set():
                    low[0] = min(low[0], torch.cuda.mem_get_info()[0])
                    time.sleep(0.0005)
            th = threading.Thread(target=poll)
            th.start()
            t0 = time.perf_counter()
            try:
                h = fn()
            finally:
                done.set(); th.join()
            dt = time.perf_counter() - t0
            info = (C.c_uint64 * 4)()
            be.check(be.lib.dg_field_info(h, info))
            kept = free0 - torch.cuda.mem_get_info()[0]
            log(f"MEASURE {label}: dg_field_create_trainable {dt:.3f} s, field {info[2] / 2**30:.2f} GiB (dg_field_info), "
                f"held after {kept / 2**30:.2f} GiB, peak during {(free0 - low[0]) / 2**30:.2f} GiB")
            return h
    return check_closed(be, (256, 256, 256), rng, nq, "256^3", log, measure)


def run_depth(be, seed=0, log=print, depths=DEPTHS, huge=False):
    """cells holding each of `depths` queries in one call, among 300 scattered ones; huge: one cell of 2^20 + 1 queries among 5000 others"""
    acc = Acc(log)
    rng = np.random.default_rng(seed + 15)
    res = (5, 4, 3)
    fld = Field(_grid(be, res), rng.standard_normal(be.num_nodes(res)), be.build_cells(res), None, "depth")
    if huge:
        parts = [fld.cell_points(rng, 37, (1 << 20) + 1), fld.points(rng, 5000)]
    else:
        parts = [fld.cell_points(rng, int(c), L) for c, L in zip(rng.permutation(60)[:len(depths)], depths)] + [fld.points(rng, 300)]
    x = np.concatenate(parts)
    x = x[rng.permutation(len(x))]

    def body(h):
        for which in (("both",) if huge else UPSTREAMS):
            acc.add(check(be, fld, h, x, *upstreams(rng, len(x), which, special=(which == "grad")),
                          f"{'2^20 + 1 in one cell' if huge else 'depths ' + str(depths)} {which}"))
    run_with(be, fld, body)
    return acc.result()


def run_strides(be, seed=0, log=print):
    """128^3 (closed form): 2^20 random queries (~10^6 groups); 2^19 + 2^16 singleton cells at the lowest ids and deep cells at the highest"""
    acc = Acc(log)
    rng = np.random.default_rng(seed + 17)
    res = (128, 128, 128)
    fld = Field(_grid(be, res), rng.standard_normal(be.num_nodes(res)), None, None, "128^3")
    n_cells = 128 ** 3
    single = (1 << 19) + (1 << 16)
    cs = np.arange(single)
    i, j, k = cs % 128, (cs // 128) % 128, cs // (128 * 128)
    cell = np.array(fld.d.cell_size[:])
    xs = fld.mn + (np.stack([i, j, k], 1) + 0.1 + 0.8 * rng.random((single, 3))) * cell
    deep = [fld.cell_points(rng, n_cells - 1 - m, L) for m, L in enumerate((1025, 100, 33, 32769, 64))]
    x2 = np.concatenate([xs] + deep)
    x2 = x2[rng.permutation(len(x2))]

    def body(h):
        x1 = fld.points(rng, 1 << 20)
        acc.add(check(be, fld, h, x1, *upstreams(rng, len(x1), "both"), "2^20 random queries"))
        acc.add(check(be, fld, h, x2, *upstreams(rng, len(x2), "phi"), f"{single} singletons and deep top cells"))
    run_with(be, fld, body)
    return acc.result()


def run_values(be, seed=0, log=print):
    """special upstreams on a dense and a reduced field; set_nodes_device planting a DBL_MAX, then the VJP on the same stream"""
    acc = Acc(log)
    rng = np.random.default_rng(seed + 19)
    res = (6, 5, 4)
    dense = Field(_grid(be, res), rng.standard_normal(be.num_nodes(res)), be.build_cells(res), None, "values dense")
    red = _reduced(be, res, 70, rng, "values reduced")
    for fld in (dense, red):
        x = np.concatenate([fld.points(rng, 900), fld.cell_points(rng, 0, 40)])

        def body(h):
            for which in UPSTREAMS:
                acc.add(check(be, fld, h, x, *upstreams(rng, len(x), which, special=True), f"special {which}"))
            new = fld.nodes.copy()
            new[rng.choice(len(new), 4, replace=False)] = DBL_MAX
            gp, gg = upstreams(rng, len(x), "both")
            got = be.set_nodes_then_vjp(h, new, x, gp, gg)
            want = fld.restate(x, gp, gg, nodes=new)
            ok = same(got, want)
            acc.add((len(got), int((~ok).sum()), None if ok.all() else f"MISMATCH {fld.label}: set_nodes_device then the VJP on its stream"))
            acc.add(check(be, Field(fld.d, new, fld.cells, fld.cmap, fld.label + " after set_nodes_device"), h, x, gp, gg, "again"))
        run_with(be, fld, body)
    return acc.result()


def run(be, rounds, seed=0, log=print, big=False):
    acc = [0, 0, 0]
    fams = [run_fields(be, rounds, seed, log), run_tables(be, seed, log), run_passes(be, seed, log), run_closed(be, seed, log),
            run_depth(be, seed, log), run_values(be, seed, log)]
    if big:
        fams += [run_depth(be, seed, log, huge=True), run_strides(be, seed, log), run_256(be, seed, log)]
    for r in fams:
        acc = [a + b for a, b in zip(acc, r)]
    return tuple(acc)


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 24
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else "emu"
    big = "big" in argv[4:]
    be = backend(lib)
    cases, total, bad = run(be, rounds, seed, big=big)
    print(f"{cases} cases, {total} values, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
