"""K13 (discregrid_b200/csrc/k13_isosurface_grad.cu) on the CPU: the product's kernels and C-ABI compiled into build/bin/libdgemu.so (tests/emu).
dg_isosurface_vjp, host and device forms, must equal the numpy restatement of the contract (tests/isosurface_grad_ref.py) bit for bit on
every family; independently of it, the edge ids must be K6's (isosurface_ref.extract_windows), the node sums K11's (dg_interpolate_vjp),
and the gradient must satisfy partition of unity and central differences of the forward.  The families are shared with the device run
(tests/test_gpu_isosurface_grad.py), which passes the CUDA library instead."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT
import isosurface_grad_ref as ref
import isosurface_ref as ir

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
DBL_MAX = np.finfo(np.float64).max
UINT32_MAX = 0xFFFFFFFF
DG_ERR_INVALID = -1
_dp, _u32p, _u64p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


def _p(a, t=_dp):
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


def same_bits(a, b):
    """bit for bit, any NaN equal to any NaN (the sign and payload of a NaN are not part of the contract, as in tools/k11_fuzz.py)"""
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def _ok(lib, rc):
    assert rc == 0, lib.dg_last_error()


def call_device_form(lib, fn, arrays, outputs):
    """fn(*pointers) with every array of `arrays` (None stays NULL) in device memory: host memory itself on the emulated library, CUDA
    tensors on the product library; the arrays at the indices `outputs` are copied back afterwards.  Returns fn's status."""
    if hasattr(lib, "emu_mesh_create"):
        return fn(*(None if a is None else a.ctypes.data for a in arrays))
    import torch
    dev = [None if a is None else torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else np.ascontiguousarray(a)).cuda()
           for a in arrays]
    rc = fn(*(None if t is None else t.data_ptr() for t in dev))
    torch.cuda.synchronize()
    for k in outputs:
        if arrays[k] is not None:
            arrays[k][...] = dev[k].cpu().numpy()
    return rc


# ------------------------------------------------------------------------------------------------ fields
class Field:
    """node values from a function of the node positions on a grid, dense or reduced to the cells within `band` of the level set 0"""

    def __init__(self, lib, fn, mn, mx, res, band=None):
        from discregrid_b200._capi import GridDesc
        self.lib = lib
        self.mn, self.mx, self.res = np.asarray(mn, np.float64), np.asarray(mx, np.float64), np.asarray(res, np.uint32)
        self.desc = GridDesc()
        _ok(lib, lib.dg_grid_init(_p(self.mn), _p(self.mx), _p(self.res, _u32p), C.byref(self.desc)))
        nn = C.c_uint64()
        _ok(lib, lib.dg_grid_num_nodes(_p(self.res, _u32p), C.byref(nn)))
        X = np.empty((nn.value, 3))
        _ok(lib, lib.dg_node_positions(C.byref(self.desc), 0, nn.value, _p(X)))
        self.nodes = np.ascontiguousarray(fn(X), np.float64)
        n_cells = int(np.prod(self.res.astype(np.int64)))
        cells = np.empty((n_cells, 32), np.uint32)
        _ok(lib, lib.dg_build_cells(_p(self.res, _u32p), 0, n_cells, _p(cells, _u32p)))
        cmap = np.arange(n_cells, dtype=np.uint32)
        if band is not None:
            keep = (np.abs(self.nodes[cells]) <= band).any(axis=1)
            assert 0 < keep.sum() < n_cells
            cmap = np.full(n_cells, UINT32_MAX, np.uint32); cmap[keep] = np.arange(keep.sum(), dtype=np.uint32)
            cells = cells[keep]
        self.cells, self.cmap = np.ascontiguousarray(cells), cmap
        self.handles = []

    def lattice(self, s):
        d = self.desc
        return ir.Lattice(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.resolution[:], s)

    def create(self, trainable=True, nodes=None):
        nodes = np.ascontiguousarray(self.nodes if nodes is None else nodes, np.float64)
        h = C.c_void_p()
        fn = self.lib.dg_field_create_trainable if trainable else self.lib.dg_field_create
        _ok(self.lib, fn(C.byref(self.desc), _p(nodes), len(nodes), _p(self.cells, _u32p), len(self.cells), _p(self.cmap, _u32p), C.byref(h)))
        self.handles.append(h)
        return h

    def close(self):
        for h in self.handles:
            self.lib.dg_field_destroy(h)
        self.handles = []

    def extract(self, h, iso, s):
        """(V, T, edge ids) of dg_isosurface_create"""
        lib, out = self.lib, C.c_void_p()
        _ok(lib, lib.dg_isosurface_create(h, iso, s, C.byref(out), None))
        try:
            nv, nt = C.c_uint64(), C.c_uint64()
            _ok(lib, lib.dg_isosurface_sizes(out, C.byref(nv), C.byref(nt)))
            V, T, E = np.empty((nv.value, 3)), np.empty((nt.value, 3), np.uint32), np.empty(nv.value, np.uint64)
            _ok(lib, lib.dg_isosurface_copy(out, _p(V), _p(T, _u32p)))
            _ok(lib, lib.dg_isosurface_copy_edges(out, _p(E, _u64p)))
            return V, T, E
        finally:
            lib.dg_isosurface_destroy(out)

    def values(self, h, x):
        x = np.ascontiguousarray(x, np.float64).reshape(-1, 3)
        phi = np.empty(len(x))
        _ok(self.lib, self.lib.dg_interpolate_batch(h, _p(x), len(x), _p(phi), None))
        return phi

    def vjp(self, h, iso, s, E, gV, device_form=False):
        E = np.ascontiguousarray(E, np.uint64); gV = np.ascontiguousarray(gV, np.float64).reshape(-1, 3)
        gn = np.full(len(self.nodes), np.nan)
        if device_form:
            rc = call_device_form(self.lib, lambda *p: self.lib.dg_isosurface_vjp_device(h, iso, s, len(E), *p, None), [E, gV, gn], (2,))
        else:
            rc = self.lib.dg_isosurface_vjp(h, iso, s, len(E), _p(E, _u64p), _p(gV), _p(gn))
        _ok(self.lib, rc)
        return gn

    def restate(self, h, iso, s, E, gV, nodes=None):
        """(grad_nodes, (gphi_p, gphi_q, valid, t, x_p, x_q)) of the contract, with f_p and f_q from the value-only interpolate"""
        L = self.lattice(s)
        xp, xq = ref.endpoints(L, E)
        f = self.values(h, ref.points(xp, xq)).reshape(-1, 2)
        gp, gq, valid, t = ref.vertex_grads(iso, f[:, 0], f[:, 1], xp, xq, gV)
        d = self.desc
        gn = ref.grad_nodes(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.inv_cell_size[:], d.resolution[:],
                            self.nodes if nodes is None else nodes, self.cells, self.cmap, xp, xq, gp, gq, valid)
        return gn, (gp, gq, valid, t, xp, xq)


def sphere(c=(0.1, -0.05, 0.07), r=0.55):
    c = np.asarray(c)
    return lambda X: np.sqrt(((X - c) ** 2).sum(1)) - r


def noisy_sphere(seed):
    rng = np.random.default_rng(seed)
    f = sphere()
    return lambda X: f(X) + 0.05 * rng.standard_normal(len(X))


def check(f, h, iso, s, E, gV, what, nodes=None):
    """both forms against the restatement; returns the restated parts"""
    want, parts = f.restate(h, iso, s, E, gV, nodes)
    for dev in (False, True):
        got = f.vjp(h, iso, s, E, gV, device_form=dev)
        assert same_bits(got, want), f"{what} device_form={dev}"
    return want, parts


def dense_specs(lib):
    """(name, field, subdivisions) of the dense families"""
    return [("1x1x1", Field(lib, noisy_sphere(1), [-1.0] * 3, [1.0] * 3, [1, 1, 1]), (1, 2, 3, 16)),
            ("3x4x5", Field(lib, noisy_sphere(2), [-0.9, -1.0, -1.1], [1.0, 0.8, 1.2], [3, 4, 5]), (1, 2, 3, 16)),
            ("16^3", Field(lib, noisy_sphere(3), [-1.0] * 3, [1.0] * 3, [16, 16, 16]), (1, 2, 3))]


def run_families(lib, seed=0):
    rng = np.random.default_rng(seed)
    specs = dense_specs(lib)
    specs.append(("band", Field(lib, sphere(), [-1.0] * 3, [1.0] * 3, [12, 12, 12], band=0.2), (1, 2)))
    try:
        for name, f, subs in specs:
            ht = f.create(True)
            # after set_nodes: the backward reads the values the field holds
            c = f.nodes + 0.03 * rng.standard_normal(len(f.nodes))
            hs = f.create(True)
            _ok(lib, lib.dg_field_set_nodes(hs, _p(c), len(c)))
            for s in subs:
                for label, h, nodes in (("trainable", ht, None), ("set_nodes", hs, c)):
                    V, T, E = f.extract(h, 0.0, s)
                    assert len(E) > 0 or name == "1x1x1", f"{name} s={s}: no vertex"
                    check(f, h, 0.0, s, E, rng.standard_normal((len(E), 3)), f"{name} s={s} {label}", nodes)
    finally:
        for _, f, _ in specs:
            f.close()


def run_exact_values(lib):
    """iso equal to lattice values: t = 0 and t = 1, coincident vertices"""
    f = Field(lib, sphere(), [-1.0] * 3, [1.0] * 3, [6, 6, 6])
    try:
        h = f.create(True)
        rng = np.random.default_rng(5)
        seen = np.zeros(2, bool)
        vals = np.sort(f.values(h, f.lattice(2).points()))
        for iso in vals[len(vals) // 3::len(vals) // 7][:4]:
            V, T, E = f.extract(h, float(iso), 2)
            _, (gp, gq, valid, t, _, _) = check(f, h, float(iso), 2, E, rng.standard_normal((len(E), 3)), f"iso {iso}")
            seen |= [(t == 0.0).any(), (t == 1.0).any()]
        assert seen.all(), "want t = 0 and t = 1"
    finally:
        f.close()


def run_huge_values(lib):
    """values near +-DBL_MAX: delta overflows and the vertex is invalid (0 at both ends)"""
    f = Field(lib, lambda X: np.clip(sphere()(X) * 1e309, -1.7e308, 1.7e308), [-1.0] * 3, [1.0] * 3, [5, 5, 5])
    try:
        h = f.create(True)
        rng = np.random.default_rng(6)
        bad = 0
        for s in (1, 2):
            V, T, E = f.extract(h, 0.0, s)
            _, (_, _, valid, _, _, _) = check(f, h, 0.0, s, E, rng.standard_normal((len(E), 3)), f"huge s={s}")
            bad += int((~valid).sum())
        assert bad > 0, "want invalid vertices"
    finally:
        f.close()


def clamp_domain(rng):
    """(mn, mx, res, s) whose lattice coordinate mn + cell * (I / s) rounds above mx on some axis"""
    from discregrid_b200.grid import grid_desc
    while True:
        res = tuple(int(v) for v in rng.integers(1, 6, 3))
        sc = 10.0 ** rng.integers(-3, 4)
        mn = rng.standard_normal(3) * sc * 10.0 ** rng.integers(0, 4)
        mx = mn + sc * (0.1 + rng.random(3))
        d = grid_desc(mn, mx, res)
        for s in (1, 3):
            L = ir.Lattice(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.resolution[:], s)
            if any((L.mn[a] + L.cell[a] * (np.arange(L.np[a]) / float(s)) > L.mx[a]).any() for a in range(3)):
                return mn, mx, res, s


def run_clamp(lib, count=3):
    """the clamp of the lattice coordinate taken (random domains) and not taken (the plain [-1, 1] domain)"""
    rng = np.random.default_rng(7)
    for k in range(count):
        mn, mx, res, s = clamp_domain(rng)
        c = 0.5 * (mn + mx) + 0.2 * (mx - mn)
        f = Field(lib, lambda x: np.linalg.norm((x - c) / (mx - mn), axis=1) - 0.4, mn, mx, res)
        try:
            h = f.create(True)
            V, T, E = f.extract(h, 0.0, s)
            check(f, h, 0.0, s, E, rng.standard_normal((len(E), 3)), f"clamp {k} {res} s={s}")
            assert len(E) > 0
        finally:
            f.close()
    f = Field(lib, sphere(), [-1.0] * 3, [1.0] * 3, [4, 4, 4])
    try:
        L = f.lattice(2)
        assert not any((L.mn[a] + L.cell[a] * (np.arange(L.np[a]) / 2.0) > L.mx[a]).any() for a in range(3))
        h = f.create(True)
        V, T, E = f.extract(h, 0.0, 2)
        check(f, h, 0.0, 2, E, rng.standard_normal((len(E), 3)), "no clamp")
    finally:
        f.close()


def run_special_upstreams_and_sizes(lib):
    """upstreams +-0.0, NaN, +-inf; n = 0, 1, 33; arbitrary lattice edges that do not cross"""
    f = Field(lib, noisy_sphere(8), [-1.0] * 3, [1.0] * 3, [5, 5, 5])
    try:
        h = f.create(True)
        rng = np.random.default_rng(8)
        V, T, E = f.extract(h, 0.0, 2)
        assert len(E) > 40
        specials = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1.0])
        gV = specials[rng.integers(0, len(specials), (len(E), 3))]
        check(f, h, 0.0, 2, E, gV, "special upstreams")
        for n in (0, 1, 33):
            check(f, h, 0.0, 2, E[:n], rng.standard_normal((n, 3)), f"n={n}")
        gn = f.vjp(h, 0.0, 2, E[:0], np.zeros((0, 3)))
        assert same_bits(gn, np.zeros(len(f.nodes)))
        L = f.lattice(2)
        lp = rng.integers(0, L.n_points, 400)
        d = rng.integers(0, 7, 400)
        e = (7 * lp + d).astype(np.uint64)
        e = e[[ref.bad_edges(L, [x]) == 0 for x in e]]
        assert len(e) > 100
        check(f, h, 0.0, 2, e, rng.standard_normal((len(e), 3)), "arbitrary edges")
        check(f, h, 0.3, 2, e, rng.standard_normal((len(e), 3)), "arbitrary edges, iso 0.3")
    finally:
        f.close()


def run_refusals(lib):
    f = Field(lib, sphere(), [-1.0] * 3, [1.0] * 3, [4, 4, 4])
    try:
        hd, ht = f.create(False), f.create(True)
        V, T, E = f.extract(ht, 0.0, 1)
        n = len(E)
        gV = np.ones((n, 3))
        gn = np.full(len(f.nodes), 7.0)
        L = f.lattice(1)

        def refused(h, iso, s, e, g, out, msg):
            e = None if e is None else np.ascontiguousarray(e, np.uint64)
            rc = lib.dg_isosurface_vjp(h, iso, s, n if e is None else len(e), _p(e, _u64p), _p(g), _p(out))
            err = lib.dg_last_error().decode()
            assert rc == DG_ERR_INVALID and msg in err, (msg, err)
        refused(hd, 0.0, 1, E, gV, gn, "dg_field_create_trainable")
        refused(None, 0.0, 1, E, gV, gn, "field is NULL")
        refused(ht, 0.0, 1, None, gV, gn, "NULL")
        refused(ht, 0.0, 1, E, None, gn, "NULL")
        refused(ht, 0.0, 1, E, gV, None, "grad_nodes is NULL")
        refused(ht, np.nan, 1, E, gV, gn, "iso must be finite")
        refused(ht, np.inf, 1, E, gV, gn, "iso must be finite")
        refused(ht, 0.0, 0, E, gV, gn, "subdivisions must be 1..16")
        refused(ht, 0.0, 17, E, gV, gn, "subdivisions must be 1..16")
        for e in ([7 * L.n_points], [7 * (L.n_points - 1) + 1], [7 * (L.np[0] - 1)], [7 * (L.np[0] * (L.np[1] - 1)) + 1],
                  [7 * (L.np[0] * L.np[1] * (L.np[2] - 1)) + 2], [2 ** 64 - 1]):
            e = np.concatenate([E, np.asarray(e, np.uint64)])
            assert ref.bad_edges(L, e) == 1
            rc = lib.dg_isosurface_vjp(ht, 0.0, 1, len(e), _p(e, _u64p), _p(np.ones((len(e), 3))), _p(gn))
            assert rc == DG_ERR_INVALID and "1 edge ids are not edges" in lib.dg_last_error().decode()
        # the device form refuses the same edge ids
        e = np.concatenate([E, np.asarray([7 * L.n_points], np.uint64)])
        rc = call_device_form(lib, lambda *p: lib.dg_isosurface_vjp_device(ht, 0.0, 1, len(e), *p, None), [e, np.ones((len(e), 3)), gn], ())
        assert rc == DG_ERR_INVALID and "not edges" in lib.dg_last_error().decode()
        assert (gn == 7.0).all(), "nothing is written before a refusal"
        # copy_edges: NULL only when there are no vertices
        out = C.c_void_p()
        _ok(lib, lib.dg_isosurface_create(ht, 0.0, 1, C.byref(out), None))
        try:
            assert lib.dg_isosurface_copy_edges(out, None) == DG_ERR_INVALID and "NULL output" in lib.dg_last_error().decode()
            assert lib.dg_isosurface_copy_edges_device(out, None, None) == DG_ERR_INVALID
        finally:
            lib.dg_isosurface_destroy(out)
        assert lib.dg_isosurface_copy_edges(None, None) == DG_ERR_INVALID
        _ok(lib, lib.dg_isosurface_create(ht, 100.0, 1, C.byref(out), None))
        try:
            _ok(lib, lib.dg_isosurface_copy_edges(out, None))
        finally:
            lib.dg_isosurface_destroy(out)
    finally:
        f.close()


def run_large_lattice_refusal(lib):
    """a lattice of 2^31 points or more (81^3 cells at s = 16) is refused before anything is written"""
    big = Field(lib, lambda X: X[:, 0], [-1.0] * 3, [1.0] * 3, [81, 81, 81])
    try:
        hb = big.create(True)
        g = np.full(len(big.nodes), 7.0)
        rc = lib.dg_isosurface_vjp(hb, 0.0, 16, 0, None, None, _p(g))
        assert rc == DG_ERR_INVALID and "2^31 points or more" in lib.dg_last_error().decode()
        assert (g == 7.0).all()
    finally:
        big.close()


# ------------------------------------------------------------------------------------------------ the tests
def test_families_equal_the_restatement(emu):
    run_families(emu)


def test_iso_at_lattice_values(emu):
    run_exact_values(emu)


def test_values_near_dbl_max(emu):
    run_huge_values(emu)


def test_lattice_coordinate_clamp(emu):
    run_clamp(emu)


def test_special_upstreams_sizes_and_arbitrary_edges(emu):
    run_special_upstreams_and_sizes(emu)


def test_refusals(emu):
    run_refusals(emu)


def test_edge_ids_and_vertices_are_k6s(emu):
    """the edge ids equal those the K6 restatement gives for one window over the whole lattice, and x_p + t (x_q - x_p) from the restated t
    has the bits of the forward's vertices"""
    for name, f, subs in dense_specs(emu) + [("band", Field(emu, sphere(), [-1.0] * 3, [1.0] * 3, [8, 8, 8], band=0.3), (1, 2))]:
        try:
            h = f.create(True)
            for s in subs[:3]:
                V, T, E = f.extract(h, 0.0, s)
                L = f.lattice(s)
                vals = f.values(h, L.points())
                Vw, Tw, Ew = ir.extract_windows(L, [((0, 0, 0), L.np - 1, vals)], 0.0)
                assert np.array_equal(E, Ew.astype(np.uint64)), f"{name} s={s}"
                assert (np.diff(E.astype(np.int64)) > 0).all()
                _, (_, _, _, t, xp, xq) = f.restate(h, 0.0, s, E, np.zeros((len(E), 3)))
                with np.errstate(all="ignore"):
                    Vr = xp + t[:, None] * (xq - xp)
                assert same_bits(Vr, V), f"{name} s={s}"
        finally:
            f.close()


def test_node_sums_are_k11s(emu):
    """grad_nodes equals dg_interpolate_vjp on the restated 2n points and gphi, bit for bit"""
    f = Field(emu, noisy_sphere(9), [-1.0] * 3, [1.0] * 3, [7, 6, 5], band=0.4)
    try:
        h = f.create(True)
        rng = np.random.default_rng(9)
        for s in (1, 3):
            V, T, E = f.extract(h, 0.0, s)
            gV = rng.standard_normal((len(E), 3))
            got = f.vjp(h, 0.0, s, E, gV)
            _, (gp, gq, valid, _, xp, xq) = f.restate(h, 0.0, s, E, gV)
            x = ref.points(np.where(valid[:, None], xp, np.inf), np.where(valid[:, None], xq, np.inf))
            g = np.ascontiguousarray(np.stack([gp, gq], axis=1).reshape(-1))
            want = np.empty(len(f.nodes))
            _ok(emu, emu.dg_interpolate_vjp(h, _p(x), len(x), _p(g), None, _p(want)))
            assert same_bits(got, want), f"s={s}"
    finally:
        f.close()


def test_partition_of_unity(emu):
    """adding delta to every node value shifts every lattice value by delta, so sum(grad_nodes) = -sum_v g_t,v / delta_v"""
    f = Field(emu, noisy_sphere(10), [-1.0] * 3, [1.0] * 3, [8, 8, 8])
    try:
        h = f.create(True)
        rng = np.random.default_rng(10)
        for s in (1, 2):
            V, T, E = f.extract(h, 0.0, s)
            gV = rng.standard_normal((len(E), 3))
            gn = f.vjp(h, 0.0, s, E, gV)
            _, (gp, gq, valid, _, xp, xq) = f.restate(h, 0.0, s, E, gV)
            fvals = f.values(h, ref.points(xp, xq)).reshape(-1, 2)
            r = ((gV * (xq - xp)).sum(1) / (fvals[:, 1] - fvals[:, 0]))[valid]
            assert abs(gn.sum() + r.sum()) <= 1e-9 * np.abs(r).sum(), (gn.sum(), -r.sum())
    finally:
        f.close()


def test_central_differences(emu):
    """sum(gV . V) of a re-extraction, differenced in single node values, against the VJP; iso keeps every lattice value at least 1e-3
    away, so the topology is fixed over the step"""
    f = Field(emu, sphere(), [-1.0] * 3, [1.0] * 3, [8, 8, 8])
    try:
        h = f.create(True)
        rng = np.random.default_rng(11)
        for s in (1, 2):
            L = f.lattice(s)
            vals = f.values(h, L.points())
            iso = 0.0
            while np.abs(vals - iso).min() < 1e-3:
                iso += 1.7e-3
            V, T, E = f.extract(h, iso, s)
            gV = rng.standard_normal((len(E), 3))
            gn = f.vjp(h, iso, s, E, gV)
            hs = 1e-6
            for j in np.argsort(-np.abs(gn))[:4]:
                out = []
                for sg in (1.0, -1.0):
                    c = f.nodes.copy(); c[j] += sg * hs
                    _ok(emu, emu.dg_field_set_nodes(h, _p(c), len(c)))
                    Vp, Tp, Ep = f.extract(h, iso, s)
                    assert np.array_equal(Ep, E)
                    out.append((gV * Vp).sum())
                _ok(emu, emu.dg_field_set_nodes(h, _p(f.nodes), len(f.nodes)))
                fd = (out[0] - out[1]) / (2 * hs)
                assert abs(fd - gn[j]) <= 1e-5 * max(1.0, abs(gn[j])), (s, j, fd, gn[j])
    finally:
        f.close()
