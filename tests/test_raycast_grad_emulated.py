"""K12 (discregrid_b200/csrc/k12_raycast_grad.cu) on the CPU: the product's kernels and C-ABI compiled into build/bin/libdgemu.so (tests/emu).
dg_mesh_raycast_vjp and dg_field_raycast_vjp, host and device forms, must equal the numpy restatement of the contract
(tests/raycast_grad_ref.py) bit for bit for every output combination; independently of it, the gradients must match exact geometry,
translation invariance, the implicit-function rule and central differences of the forward casts.  The families are shared with the device
run (tests/test_gpu_raycast_grad.py), which passes the CUDA library instead."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

from conftest import ROOT, GOLDEN
import raycast_grad_ref as ref

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")
DBL_MAX = np.finfo(np.float64).max
UINT32_MAX = 0xFFFFFFFF
DG_ERR_INVALID = -1
_dp, _u32p, _i32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)


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


same_bits = ref.same_bits


def _ok(lib, rc):
    assert rc == 0, lib.dg_last_error()


def call_device_form(lib, fn, arrays, outputs):
    """fn(*pointers) with every array of `arrays` (None stays NULL) in device memory: host memory itself on the emulated library, CUDA
    tensors on the product library; the arrays at the indices `outputs` are copied back afterwards.  Returns fn's status."""
    if hasattr(lib, "emu_mesh_create"):
        return fn(*(None if a is None else a.ctypes.data for a in arrays))
    import torch
    dev = [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    rc = fn(*(None if t is None else t.data_ptr() for t in dev))
    torch.cuda.synchronize()
    for k in outputs:
        if arrays[k] is not None:
            arrays[k][...] = dev[k].cpu().numpy()
    return rc


# ------------------------------------------------------------------------------------------------ meshes
class Mesh:
    def __init__(self, lib, V, F):
        self.lib = lib
        self.V = np.ascontiguousarray(V, np.float64).reshape(-1, 3)
        self.F = np.ascontiguousarray(F, np.uint32).reshape(-1, 3)
        self.h = C.c_void_p()
        _ok(lib, lib.dg_mesh_create(_p(self.V), len(self.V), _p(self.F, _u32p), len(self.F), C.byref(self.h)))

    def close(self):
        self.lib.dg_mesh_destroy(self.h)

    def cast(self, o, d, t_min=0.0, t_max=np.inf):
        o = np.ascontiguousarray(o, np.float64); d = np.ascontiguousarray(d, np.float64)
        n = len(o)
        t, tid, b, st = np.empty(n), np.empty(n, np.int32), np.empty((n, 3)), np.empty(n, np.int32)
        _ok(self.lib, self.lib.dg_mesh_raycast(self.h, _p(o), _p(d), n, t_min, t_max, _p(t), _p(tid, _i32p), _p(b), _p(st, _i32p)))
        return t, tid, b, st

    def vjp(self, d, t, tid, bary, gt, gb, want=(True, True, True), V=None, device_form=False):
        """(grad_origins, grad_directions, grad_vertices), None where not wanted"""
        V = self.V if V is None else np.ascontiguousarray(V, np.float64)
        n = len(d)
        d = np.ascontiguousarray(d, np.float64); t = np.ascontiguousarray(t, np.float64)
        tid = np.ascontiguousarray(tid, np.int32); bary = np.ascontiguousarray(bary, np.float64)
        gt = None if gt is None else np.ascontiguousarray(gt, np.float64)
        gb = None if gb is None else np.ascontiguousarray(gb, np.float64)
        go = np.full((n, 3), np.nan) if want[0] else None
        gd = np.full((n, 3), np.nan) if want[1] else None
        gv = np.full((len(self.V), 3), np.nan) if want[2] else None
        if device_form:
            rc = call_device_form(self.lib, lambda *p: self.lib.dg_mesh_raycast_vjp_device(self.h, n, *p, None),
                                  [d, t, tid, bary, V, gt, gb, go, gd, gv], (7, 8, 9))
        else:
            rc = self.lib.dg_mesh_raycast_vjp(self.h, n, _p(d), _p(t), _p(tid, _i32p), _p(bary), _p(V), _p(gt), _p(gb), _p(go), _p(gd), _p(gv))
        _ok(self.lib, rc)
        return go, gd, gv


def box_mesh():
    from discregrid_b200.mesh import TriangleMesh
    m = TriangleMesh(os.path.join(GOLDEN, "box.obj"))
    return m.vertices, m.faces


def sphere_mesh():
    from discregrid_b200.mesh import TriangleMesh
    m = TriangleMesh(os.path.join(GOLDEN, "sphere.obj"))
    return m.vertices, m.faces


def torus_mesh():
    from discregrid_b200.mesh import bumpy_torus
    m = bumpy_torus(24, 16)
    return m.vertices, m.faces


def mesh_rays(V, F, rng, n):
    """camera rays, CCD segments near the surface and misses: (origins, directions, t_max) per family"""
    V = np.asarray(V); lo, hi = V.min(0), V.max(0); c, ext = (lo + hi) / 2, (hi - lo).max()
    eye = c + np.array([0.31, 0.23, 2.1]) * ext
    tgt = c + (rng.random((n, 3)) - 0.5) * ext * 1.1
    cam = (np.repeat(eye[None], n, 0), tgt - eye, np.inf)
    x0 = V[rng.integers(0, len(V), n)] + rng.normal(0, 0.05 * ext, (n, 3))
    ccd = (x0, rng.normal(0, 0.08 * ext, (n, 3)), 1.0)
    miss = (np.repeat(eye[None], 8, 0), np.repeat((eye - c)[None], 8, 0) + rng.normal(0, 0.01, (8, 3)), np.inf)
    return {"camera": cam, "ccd": ccd, "miss": miss}


def shared_edge_ray(V, F):
    """a ray from outside through the midpoint of the first edge two triangles share"""
    V = np.asarray(V); F = np.asarray(F, np.int64)
    seen = {}
    for tri in F:
        for a, b in ((tri[0], tri[1]), (tri[1], tri[2]), (tri[2], tri[0])):
            k = (min(a, b), max(a, b))
            if k in seen:
                mid = 0.5 * (V[a] + V[b])
                c = V.mean(0)
                return (mid + 2.0 * (mid - c))[None], (-2.0 * (mid - c))[None]
            seen[k] = True
    raise AssertionError("no shared edge")


def upstreams(rng, n):
    return {"t": (rng.standard_normal(n), None), "bary": (None, rng.standard_normal((n, 3))),
            "both": (rng.standard_normal(n), rng.standard_normal((n, 3)))}


def check_mesh(m, o, d, hit, gt, gb, what):
    """every output combination, both forms, against the restatement"""
    t, tid, bary, _ = hit
    go_w, gd_w, valid = ref.mesh_ray_grads(m.V, m.F, d, t, tid, gt, gb)
    gv_w = ref.mesh_grad_vertices(m.F, len(m.V), tid, bary, go_w, valid)
    for want in itertools.product((False, True), repeat=3):
        if not any(want):
            continue
        for dev in (False, True):
            got = m.vjp(d, t, tid, bary, gt, gb, want, device_form=dev)
            for g, w, nm in zip(got, (go_w, gd_w, gv_w), ("grad_origins", "grad_directions", "grad_vertices")):
                if g is not None:
                    assert same_bits(g, w), f"{what} {nm} want={want} device_form={dev}"
    return go_w, gd_w, gv_w, valid


def run_mesh_families(lib, n=300, seed=0):
    rng = np.random.default_rng(seed)
    for name, (V, F) in {"box": box_mesh(), "sphere": sphere_mesh(), "torus": torus_mesh()}.items():
        m = Mesh(lib, V, F)
        try:
            fams = mesh_rays(V, F, rng, n)
            fams["edge"] = shared_edge_ray(V, F) + (np.inf,)
            for fam, (o, d, t_max) in fams.items():
                hit = m.cast(o, d, 0.0, t_max)
                if fam in ("camera", "ccd"):
                    assert (hit[1] >= 0).sum() > 0, f"{name} {fam}: no hit"
                if fam == "miss":
                    assert (hit[1] < 0).all()
                if fam == "edge":
                    assert hit[1][0] >= 0, f"{name}: the ray through a shared edge was lost"
                for up, (gt, gb) in upstreams(rng, len(o)).items():
                    check_mesh(m, o, d, hit, gt, gb, f"{name} {fam} {up}")
        finally:
            m.close()


def run_mesh_edge_cases(lib):
    V, F = box_mesh()
    m = Mesh(lib, V, F)
    try:
        rng = np.random.default_rng(7)
        # every ray on one triangle: long segments straight down onto the top face, more than 32^2 rays (two levels of K10's tree)
        t0, tid0, _, _ = m.cast(np.array([[0.3, 0.2, 5.0]]), np.array([[0.0, 0.0, -1.0]]))
        T = m.F[tid0[0]]
        w = rng.dirichlet((2.0, 2.0, 2.0), 2100)
        o = w @ m.V[T]; o[:, 2] = 3.0
        d = np.tile([0.0, 0.0, -100.0], (len(o), 1))
        hit = m.cast(o, d, 0.0, 1.0)
        assert (hit[1] >= 0).all() and len(np.unique(hit[1])) <= 2
        check_mesh(m, o, d, hit, rng.standard_normal(len(o)), rng.standard_normal((len(o), 3)), "one triangle")
        # a direction in the triangle's plane (den = 0) and a degenerate triangle give zeros and no vertex contribution
        tid = np.array([tid0[0], tid0[0], -1], np.int32)
        d = np.array([[1.0, 0.5, 0.0], [0.0, 0.0, -1.0], [0.0, 0.0, -1.0]])
        bary = np.array([[0.2, 0.3, 0.5], [0.2, 0.3, 0.5], [np.nan] * 3])
        t = np.array([0.5, 2.0, np.inf])
        gt, gb = np.ones(3), np.ones((3, 3))
        go, gd, gv = m.vjp(d, t, tid, bary, gt, gb)
        assert same_bits(go[[0, 2]], np.zeros((2, 3))) and same_bits(gd[[0, 2]], np.zeros((2, 3)))
        go1, _, gv1 = m.vjp(d[1:2], t[1:2], tid[1:2], bary[1:2], gt[1:2], gb[1:2])
        assert same_bits(gv, gv1), "the in-plane ray and the miss must not reach the vertex sums"
        Vd = m.V.copy(); Vd[m.F[tid0[0], 1]] = Vd[m.F[tid0[0], 0]]; Vd[m.F[tid0[0], 2]] = Vd[m.F[tid0[0], 0]]
        go, gd, gv = m.vjp(d[1:2], t[1:2], tid[1:2], bary[1:2], gt[1:2], gb[1:2], V=Vd)
        assert same_bits(go, np.zeros((1, 3))) and same_bits(gv, np.zeros_like(m.V)), "a degenerate triangle (n . n = 0) gives zeros"
        # n = 0 writes zeros into grad_vertices; NULL upstreams equal zero upstreams
        e = np.empty((0, 3))
        _, _, gv = m.vjp(e, np.empty(0), np.empty(0, np.int32), e, np.empty(0), None)
        assert same_bits(gv, np.zeros_like(m.V))
        fam = mesh_rays(m.V, m.F, rng, 200)["camera"]
        t, tid, bary, _ = m.cast(fam[0], fam[1])
        gt = rng.standard_normal(len(t))
        a = m.vjp(fam[1], t, tid, bary, gt, None)
        b = m.vjp(fam[1], t, tid, bary, gt, np.zeros((len(t), 3)))
        c = m.vjp(fam[1], t, tid, bary, None, np.zeros((len(t), 3)))
        z = m.vjp(fam[1], t, tid, bary, np.zeros(len(t)), np.zeros((len(t), 3)))
        for x, y in zip(a, b):
            assert same_bits(x, y), "grad_barycentric NULL must equal zeros"
        for x, y in zip(c, z):
            assert same_bits(x, y), "grad_t NULL must equal zeros"
    finally:
        m.close()


def run_mesh_refusals(lib):
    V, F = box_mesh()
    m = Mesh(lib, V, F)
    try:
        n = 2
        d = np.tile([0.0, 0.0, -1.0], (n, 1)); t = np.ones(n); tid = np.array([0, 1], np.int32); b = np.full((n, 3), 1 / 3)
        gt = np.ones(n); go = np.full((n, 3), 7.0)
        def call(**kw):
            a = dict(d=d, t=t, tid=tid, b=b, V=m.V, gt=gt, gb=None, go=go)
            a.update(kw)
            return lib.dg_mesh_raycast_vjp(m.h, kw.get("n", n), _p(a["d"]), _p(a["t"]), _p(a["tid"], _i32p), _p(a["b"]), _p(a["V"]), _p(a["gt"]),
                                           _p(a["gb"]), _p(a["go"]), None, None)
        for k in ("d", "t", "tid", "b", "V"):
            assert call(**{k: None}) == DG_ERR_INVALID and "NULL" in lib.dg_last_error().decode()
        assert call(gt=None) == DG_ERR_INVALID and "grad_t" in lib.dg_last_error().decode()
        for bad in (len(m.F), -2):
            assert call(tid=np.array([0, bad], np.int32)) == DG_ERR_INVALID
            assert "triangle ids outside" in lib.dg_last_error().decode()
        assert (go == 7.0).all(), "nothing is written before a refusal"
        assert lib.dg_mesh_raycast_vjp(None, 0, None, None, None, None, None, _p(gt), None, None, None, None) == DG_ERR_INVALID
        assert lib.dg_mesh_raycast_vjp(m.h, 0, None, None, None, None, None, _p(gt), None, None, None, None) == 0, "no output: a no-op"
    finally:
        m.close()


# ------------------------------------------------------------------------------------------------ fields
class Field:
    """an analytic SDF sampled at the nodes of a grid, dense or reduced to a band of 3 cell diagonals"""

    def __init__(self, lib, sdf, mn, mx, res, band=False):
        from discregrid_b200._capi import GridDesc
        self.lib = lib
        self.mn, self.mx, self.res = np.asarray(mn, np.float64), np.asarray(mx, np.float64), np.asarray(res, np.uint32)
        self.desc = GridDesc()
        _ok(lib, lib.dg_grid_init(_p(self.mn), _p(self.mx), _p(self.res, _u32p), C.byref(self.desc)))
        nn = C.c_uint64()
        _ok(lib, lib.dg_grid_num_nodes(_p(self.res, _u32p), C.byref(nn)))
        X = np.empty((nn.value, 3))
        _ok(lib, lib.dg_node_positions(C.byref(self.desc), 0, nn.value, _p(X)))
        self.nodes = sdf(X)
        n_cells = int(np.prod(self.res.astype(np.int64)))
        cells = np.empty((n_cells, 32), np.uint32)
        _ok(lib, lib.dg_build_cells(_p(self.res, _u32p), 0, n_cells, _p(cells, _u32p)))
        cmap = np.arange(n_cells, dtype=np.uint32)
        if band:
            diag = float(np.sqrt((np.asarray(self.desc.cell_size[:]) ** 2).sum()))
            keep = (np.abs(self.nodes[cells]) <= 3 * diag).any(axis=1)
            assert 0 < keep.sum() < n_cells
            cmap = np.full(n_cells, UINT32_MAX, np.uint32); cmap[keep] = np.arange(keep.sum(), dtype=np.uint32)
            cells = cells[keep]
        self.cells, self.cmap = np.ascontiguousarray(cells), cmap
        self.handles = []

    def create(self, trainable, nodes=None):
        nodes = np.ascontiguousarray(self.nodes if nodes is None else nodes, np.float64)
        h = C.c_void_p()
        fn = self.lib.dg_field_create_trainable if trainable else self.lib.dg_field_create
        _ok(self.lib, fn(C.byref(self.desc), _p(nodes), len(nodes), _p(self.cells, _u32p), len(self.cells), _p(self.cmap, _u32p), C.byref(h)))
        self.handles.append(h)
        return h

    def close(self):
        for h in self.handles:
            self.lib.dg_field_destroy(h)

    def cast(self, h, o, d, iso=0.0, t_min=0.0, t_max=np.inf):
        o = np.ascontiguousarray(o, np.float64); d = np.ascontiguousarray(d, np.float64)
        n = len(o)
        tl, th, st = np.empty(n), np.empty(n), np.empty(n, np.int32)
        _ok(self.lib, self.lib.dg_field_raycast(h, _p(o), _p(d), n, iso, t_min, t_max, _p(tl), _p(th), _p(st, _i32p)))
        return tl, th, st

    def interpolate(self, h, x, gradient=True):
        x = np.ascontiguousarray(x, np.float64)
        phi, grad = np.empty(len(x)), (np.empty((len(x), 3)) if gradient else None)
        _ok(self.lib, self.lib.dg_interpolate_batch(h, _p(x), len(x), _p(phi), _p(grad)))
        return phi, grad

    def vjp(self, h, o, d, t_lo, st, glo, ghi, want=(True, True, False), device_form=False, n_nodes=None):
        n = len(o)
        o, d, t_lo = (np.ascontiguousarray(a, np.float64) for a in (o, d, t_lo))
        st = np.ascontiguousarray(st, np.int32)
        glo = None if glo is None else np.ascontiguousarray(glo, np.float64)
        ghi = None if ghi is None else np.ascontiguousarray(ghi, np.float64)
        go = np.full((n, 3), np.nan) if want[0] else None
        gd = np.full((n, 3), np.nan) if want[1] else None
        gn = np.full(len(self.nodes) if n_nodes is None else n_nodes, np.nan) if want[2] else None
        if device_form:
            rc = call_device_form(self.lib, lambda *p: self.lib.dg_field_raycast_vjp_device(h, n, *p, None),
                                  [o, d, t_lo, st, glo, ghi, go, gd, gn], (6, 7, 8))
        else:
            rc = self.lib.dg_field_raycast_vjp(h, n, _p(o), _p(d), _p(t_lo), _p(st, _i32p), _p(glo), _p(ghi), _p(go), _p(gd), _p(gn))
        _ok(self.lib, rc)
        return go, gd, gn

    def restate(self, h, o, d, t_lo, st, glo, ghi, nodes=None):
        xc = ref.crossing_points(self.mn, self.mx, o, d, t_lo, st)
        phi, grad = self.interpolate(h, xc)
        go, gd, gphi, valid = ref.field_ray_grads(d, t_lo, st, phi, grad, glo, ghi)
        dd = self.desc
        gn = ref.field_grad_nodes(dd.domain_min[:], dd.domain_max[:], dd.cell_size[:], dd.inv_cell_size[:], dd.resolution[:],
                                  self.nodes if nodes is None else nodes, self.cells, self.cmap, xc, gphi, valid)
        return go, gd, gn, valid


def sphere_sdf(X):
    return np.sqrt((X ** 2).sum(1)) - 0.55


def torus_sdf(X):
    q = np.sqrt(X[:, 0] ** 2 + X[:, 1] ** 2) - 0.55
    return np.sqrt(q ** 2 + X[:, 2] ** 2) - 0.22


def field_rays(rng, n):
    eye = np.array([0.21, -0.17, 2.4])
    tgt = (rng.random((n, 3)) - 0.5) * 1.6
    x0 = rng.normal(0, 0.45, (n, 3))
    return {"camera": (np.repeat(eye[None], n, 0), tgt - eye, np.inf), "ccd": (x0, rng.normal(0, 0.3, (n, 3)), 1.0)}


def field_specs(lib):
    return {"sphere": Field(lib, sphere_sdf, [-1.0] * 3, [1.0] * 3, [10, 10, 10]),
            "torus": Field(lib, torus_sdf, [-1.0, -1.0, -0.5], [1.0, 1.0, 0.5], [12, 12, 6]),
            "sphere_band": Field(lib, sphere_sdf, [-1.0] * 3, [1.0] * 3, [16, 16, 16], band=True),
            "torus_band": Field(lib, torus_sdf, [-1.0, -1.0, -0.5], [1.0, 1.0, 0.5], [28, 28, 14], band=True)}


def check_field(f, h, o, d, hit, glo, ghi, trainable, what, nodes=None):
    t_lo, _, st = hit
    go_w, gd_w, gn_w, valid = f.restate(h, o, d, t_lo, st, glo, ghi, nodes)
    for want in itertools.product((False, True), repeat=3):
        if not any(want) or (want[2] and not trainable):
            continue
        for dev in (False, True):
            got = f.vjp(h, o, d, t_lo, st, glo, ghi, want, device_form=dev)
            for g, w, nm in zip(got, (go_w, gd_w, gn_w), ("grad_origins", "grad_directions", "grad_nodes")):
                if g is not None:
                    assert same_bits(g, w), f"{what} {nm} want={want} device_form={dev}"
    return go_w, gd_w, gn_w, valid


def run_field_families(lib, n=200, seed=1):
    rng = np.random.default_rng(seed)
    specs = field_specs(lib)
    try:
        for name, f in specs.items():
            hd, ht = f.create(False), f.create(True)
            # a trainable field after set_nodes: the backward reads the values the field holds
            c = f.nodes + 0.05 * rng.standard_normal(len(f.nodes))
            hs = f.create(True)
            _ok(lib, lib.dg_field_set_nodes(hs, _p(c), len(c)))
            for fam, (o, d, t_max) in field_rays(rng, n).items():
                for label, h, trainable, nodes in (("dense", hd, False, None), ("trainable", ht, True, None), ("set_nodes", hs, True, c)):
                    hit = f.cast(h, o, d, 0.0, 0.0, t_max)
                    assert (hit[2] != 0).sum() > 0 and (hit[2] == 0).sum() > 0, f"{name} {fam}: want hits and misses"
                    for up, (glo, ghi) in {"lo": (rng.standard_normal(n), None), "hi": (None, rng.standard_normal(n)),
                                           "both": (rng.standard_normal(n), rng.standard_normal(n))}.items():
                        check_field(f, h, o, d, hit, glo, ghi, trainable, f"{name} {fam} {label} {up}", nodes)
    finally:
        for f in specs.values():
            f.close()


def run_field_edge_cases(lib):
    f = field_specs(lib)["sphere"]
    try:
        h = f.create(True)
        rng = np.random.default_rng(3)
        o, d, _ = field_rays(rng, 100)["camera"]
        t_lo, t_hi, st = f.cast(h, o, d)
        g = rng.standard_normal(100)
        # NULL upstreams equal zero upstreams; g_lo + g_hi on both ends equals their sum on one end (both follow the crossing)
        want = (True, True, True)
        a = f.vjp(h, o, d, t_lo, st, g, None, want)
        b = f.vjp(h, o, d, t_lo, st, g, np.zeros(100), want)
        c = f.vjp(h, o, d, t_lo, st, None, g, want)
        for x, y in zip(a, b):
            assert same_bits(x, y)
        for x, y in zip(a, c):
            assert same_bits(x, y)
        g2 = rng.standard_normal(100)
        s = f.vjp(h, o, d, t_lo, st, g, g2, want)
        one = f.vjp(h, o, d, t_lo, st, g + g2, None, want)
        for x, y in zip(s, one):
            assert same_bits(x, y)
        # a ray tangent to the level set (grad . d = 0) and a miss give zeros and take no part in the node sum
        i = int(np.flatnonzero(st != 0)[0])
        xc = ref.crossing_points(f.mn, f.mx, o[i:i + 1], d[i:i + 1], t_lo[i:i + 1], st[i:i + 1])
        _, gr = f.interpolate(h, xc)
        o2 = np.array([xc[0], [0.0, 0.0, 2.0]]); d2 = np.array([[gr[0, 1], -gr[0, 0], 0.0], [0.0, 0.0, -1.0]])   # g0 g1 - g1 g0 = 0
        t2 = np.array([0.0, 1.45]); st2 = np.array([1, 0], np.int32)
        go, gd, gn = f.vjp(h, o2, d2, t2, st2, np.ones(2), None, want)
        assert same_bits(go, np.zeros((2, 3))) and same_bits(gd, np.zeros((2, 3))) and same_bits(gn, np.zeros(len(f.nodes)))
        # n = 0 writes zeros into grad_nodes
        e = np.empty((0, 3))
        _, _, gn = f.vjp(h, e, e, np.empty(0), np.empty(0, np.int32), np.empty(0), None, (False, False, True))
        assert same_bits(gn, np.zeros(len(f.nodes)))
    finally:
        f.close()


def run_field_refusals(lib):
    f = field_specs(lib)["sphere"]
    try:
        hd, ht = f.create(False), f.create(True)
        n = 2
        o = np.zeros((n, 3)); d = np.tile([0.0, 0.0, 1.0], (n, 1)); t = np.ones(n); st = np.ones(n, np.int32); g = np.ones(n)
        gn = np.full(len(f.nodes), 7.0)
        rc = lib.dg_field_raycast_vjp(hd, n, _p(o), _p(d), _p(t), _p(st, _i32p), _p(g), None, None, None, _p(gn))
        assert rc == DG_ERR_INVALID and "dg_field_create_trainable" in lib.dg_last_error().decode()
        assert (gn == 7.0).all()
        for k in range(4):
            args = [_p(o), _p(d), _p(t), _p(st, _i32p)]
            args[k] = None
            assert lib.dg_field_raycast_vjp(ht, n, *args, _p(g), None, None, None, _p(gn)) == DG_ERR_INVALID
            assert "NULL" in lib.dg_last_error().decode()
        assert lib.dg_field_raycast_vjp(ht, n, _p(o), _p(d), _p(t), _p(st, _i32p), None, None, None, None, _p(gn)) == DG_ERR_INVALID
        assert lib.dg_field_raycast_vjp(None, n, _p(o), _p(d), _p(t), _p(st, _i32p), _p(g), None, None, None, _p(gn)) == DG_ERR_INVALID
        assert (gn == 7.0).all(), "nothing is written before a refusal"
    finally:
        f.close()


# ------------------------------------------------------------------------------------------------ the tests
def test_mesh_families_equal_the_restatement(emu):
    run_mesh_families(emu)


def test_mesh_one_triangle_in_plane_degenerate_empty_and_null_upstreams(emu):
    run_mesh_edge_cases(emu)


def test_mesh_refusals(emu):
    run_mesh_refusals(emu)


def test_field_families_equal_the_restatement(emu):
    run_field_families(emu)


def test_field_implicit_rule_tangent_miss_empty_and_null_upstreams(emu):
    run_field_edge_cases(emu)


def test_field_refusals(emu):
    run_field_refusals(emu)


def test_mesh_exact_geometry_on_an_axis_aligned_face(emu):
    """t = (z_face - o_z) / d_z on the box's top face: dt/do = (0, 0, -1/d_z), dt/dd = t dt/do, dt/dV_i = -b_i dt/do"""
    V, F = box_mesh()
    m = Mesh(emu, V, F)
    try:
        rng = np.random.default_rng(11)
        o = np.column_stack([rng.uniform(-0.9, 0.9, 50), rng.uniform(-0.9, 0.9, 50), np.full(50, 3.0)])
        d = np.tile([0.0, 0.0, -0.5], (50, 1))
        t, tid, bary, _ = m.cast(o, d)
        assert np.array_equal(t, np.full(50, 4.0))
        go, gd, _ = m.vjp(d, t, tid, bary, np.ones(50), None)
        assert np.array_equal(go, np.tile([0.0, 0.0, 2.0], (50, 1))) and np.array_equal(gd, np.tile([0.0, 0.0, 8.0], (50, 1)))
        for i in range(5):
            _, _, gv = m.vjp(d[i:i + 1], t[i:i + 1], tid[i:i + 1], bary[i:i + 1], np.ones(1), None, (False, False, True))
            want = np.zeros_like(m.V)
            for k in range(3):
                want[m.F[tid[i], k]] += -bary[i, k] * go[i]
            np.testing.assert_allclose(gv, want, rtol=1e-15, atol=1e-15)
    finally:
        m.close()


def test_mesh_translation_invariance(emu):
    """per ray, the vertex gradients and the origin gradient sum to zero (for t and for the weights)"""
    V, F = torus_mesh()
    m = Mesh(emu, V, F)
    try:
        rng = np.random.default_rng(12)
        o, d, _ = mesh_rays(V, F, rng, 60)["camera"]
        t, tid, bary, _ = m.cast(o, d)
        for i in np.flatnonzero(tid >= 0)[:25]:
            for gt, gb in ((np.ones(1), None), (None, rng.standard_normal((1, 3)))):
                go, _, gv = m.vjp(d[i:i + 1], t[i:i + 1], tid[i:i + 1], bary[i:i + 1], gt, gb)
                s = gv.sum(0) + go[0]
                assert np.abs(s).max() <= 64 * np.finfo(float).eps * max(1.0, np.abs(go).max()), (i, s, go)
    finally:
        m.close()


def test_mesh_central_differences(emu):
    """t and the weights of a re-cast, differenced in o, d and V, against the VJP, at rays away from edges"""
    V, F = torus_mesh()
    m = Mesh(emu, V, F)
    try:
        rng = np.random.default_rng(13)
        o, d, _ = mesh_rays(V, F, rng, 200)["camera"]
        t, tid, bary, _ = m.cast(o, d)
        rays = np.flatnonzero((tid >= 0) & (np.nan_to_num(bary, nan=0).min(1) > 0.15))[:6]
        assert len(rays) >= 3
        h = 1e-6
        for i in rays:
            gt, gb = rng.standard_normal(1), rng.standard_normal((1, 3))
            go, gd, gv = m.vjp(d[i:i + 1], t[i:i + 1], tid[i:i + 1], bary[i:i + 1], gt, gb)
            loss = lambda r: gt[0] * r[0][0] + (gb[0] * r[2][0]).sum()
            for k in range(3):
                e = np.zeros((1, 3)); e[0, k] = h
                fd_o = (loss(m.cast(o[i:i + 1] + e, d[i:i + 1])) - loss(m.cast(o[i:i + 1] - e, d[i:i + 1]))) / (2 * h)
                fd_d = (loss(m.cast(o[i:i + 1], d[i:i + 1] + e)) - loss(m.cast(o[i:i + 1], d[i:i + 1] - e))) / (2 * h)
                assert abs(fd_o - go[0, k]) <= 1e-5 * max(1.0, abs(go[0, k])), (i, k, fd_o, go[0, k])
                assert abs(fd_d - gd[0, k]) <= 1e-5 * max(1.0, abs(gd[0, k])), (i, k, fd_d, gd[0, k])
            vi = int(m.F[tid[i], 1])
            for k in range(3):
                out = []
                for s in (1.0, -1.0):
                    Vp = m.V.copy(); Vp[vi, k] += s * h
                    mp = Mesh(emu, Vp, m.F)
                    try:
                        out.append(loss(mp.cast(o[i:i + 1], d[i:i + 1])))
                    finally:
                        mp.close()
                fd_v = (out[0] - out[1]) / (2 * h)
                assert abs(fd_v - gv[vi, k]) <= 1e-5 * max(1.0, abs(gv[vi, k])), (i, k, fd_v, gv[vi, k])
    finally:
        m.close()


def test_field_crossing_point_values_and_sides(emu):
    """phi(x_c) from K2's gradient mode has the bits of the value-only interpolate K7 samples with, on the side the status says"""
    f = field_specs(emu)["torus_band"]
    try:
        h = f.create(False)
        rng = np.random.default_rng(14)
        for fam, (o, d, t_max) in field_rays(rng, 300).items():
            t_lo, t_hi, st = f.cast(h, o, d, 0.0, 0.0, t_max)
            hit = st != 0
            xc = ref.crossing_points(f.mn, f.mx, o, d, t_lo, st)[hit]
            phi_g, _ = f.interpolate(h, xc, True)
            phi_v, _ = f.interpolate(h, xc, False)
            assert same_bits(phi_g, phi_v)
            assert (phi_v[st[hit] == 1] >= 0).all() and (phi_v[st[hit] == 2] < 0).all(), fam
    finally:
        f.close()


def test_field_central_differences(emu):
    """t_lo of a re-cast, differenced in o, d and node values, against the VJP, at crossings away from cell faces"""
    f = field_specs(emu)["torus"]
    try:
        h = f.create(True)
        rng = np.random.default_rng(15)
        o, d, _ = field_rays(rng, 200)["camera"]
        t_lo, _, st = f.cast(h, o, d)
        xc = ref.crossing_points(f.mn, f.mx, o, d, t_lo, st)
        with np.errstate(invalid="ignore"):
            frac = np.where(np.isfinite(xc), ((xc - f.mn) * np.asarray(f.desc.inv_cell_size[:])) % 1.0, 0.0)
        rays = np.flatnonzero((st != 0) & (frac.min(1) > 0.1) & (frac.max(1) < 0.9))[:5]
        assert len(rays) >= 3
        hs = 1e-6
        for i in rays:
            sl = slice(i, i + 1)
            go, gd, gn = f.vjp(h, o[sl], d[sl], t_lo[sl], st[sl], np.ones(1), None, (True, True, True))
            for k in range(3):
                e = np.zeros((1, 3)); e[0, k] = hs
                fd_o = (f.cast(h, o[sl] + e, d[sl])[0][0] - f.cast(h, o[sl] - e, d[sl])[0][0]) / (2 * hs)
                fd_d = (f.cast(h, o[sl], d[sl] + e)[0][0] - f.cast(h, o[sl], d[sl] - e)[0][0]) / (2 * hs)
                assert abs(fd_o - go[0, k]) <= 1e-5 * max(1.0, abs(go[0, k])), (i, k, fd_o, go[0, k])
                assert abs(fd_d - gd[0, k]) <= 1e-5 * max(1.0, abs(gd[0, k])), (i, k, fd_d, gd[0, k])
            for j in np.argsort(-np.abs(gn))[:3]:
                out = []
                for s in (1.0, -1.0):
                    c = f.nodes.copy(); c[j] += s * hs
                    _ok(emu, emu.dg_field_set_nodes(h, _p(c), len(c)))
                    out.append(f.cast(h, o[sl], d[sl])[0][0])
                _ok(emu, emu.dg_field_set_nodes(h, _p(f.nodes), len(f.nodes)))
                fd_c = (out[0] - out[1]) / (2 * hs)
                assert abs(fd_c - gn[j]) <= 1e-5 * max(1.0, abs(gn[j])), (i, j, fd_c, gn[j])
    finally:
        f.close()
