"""The volume map (dg_volume_map, dg_reduced_volume_map_create: K3's volume-map kernel) on the CPU: the product's kernels and C-ABI compiled
into build/bin/libdgemu.so (tests/emu).  Held bit for bit to orc_volume_map (tests/cpp/volume_oracle.cpp, the contract restated over the
oracle's interpolate, every Gauss point visited) and to the reference-side generator's .cdm files (tests/golden/make_volume_golden.py), and
to closed forms that need no oracle.  The GPU runs are tests/test_gpu_volume_map.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, bits_equal
from test_density_reduced_emulated import (DG_ERR_INVALID, REFERENCE_SORT, _dp, _p, _u32p, _vp, box_grid, cdm_equal, cell_diag, dense_layout,
                                           emu, load_sdf, n_grid_cells, positions, reduce_host, same_field, write_cdm)  # noqa: F401 (emu)
from test_oracle_golden import read_cdf

ORC = os.path.join(ROOT, "build", "bin", "liborcvolume.so")
CASES = json.load(open(os.path.join(GOLDEN, "ref_volume_cases.json")))
DBL_MAX = np.finfo(np.float64).max
GA16 = np.array([-0.989400934991649938510249739920, -0.944575023073232600268056557979, -0.865631202387831755196145877562,
                 -0.755404408355002998654015300417, -0.617876244402643770570193737512, -0.458016777657227369680015272024,
                 -0.281603550779258915426339626720, -0.095012509837637426635126303154, 0.095012509837637426635126303154,
                 0.281603550779258915426339626720, 0.458016777657227369680015272024, 0.617876244402643770570193737512,
                 0.755404408355002998654015300417, 0.865631202387831755196145877562, 0.944575023073232600268056557979,
                 0.989400934991649938510249739920])
GW16 = np.array([0.027152459411758110563450685504, 0.062253523938649010793788818319, 0.095158511682492036287683845330,
                 0.124628971255533488315947465708, 0.149595988816575764523975067277, 0.169156519395001675443168664970,
                 0.182603415044922529064663763165, 0.189450610455067447457366824892, 0.189450610455067447457366824892,
                 0.182603415044922529064663763165, 0.169156519395001675443168664970, 0.149595988816575764523975067277,
                 0.124628971255533488315947465708, 0.095158511682492036287683845330, 0.062253523938649010793788818319,
                 0.027152459411758110563450685504])


@pytest.fixture(scope="module")
def orcv():
    if not os.path.exists(ORC):
        pytest.skip("build/bin/liborcvolume.so not built (make cpp)")
    lib = C.CDLL(ORC)
    lib.orc_volume_map.restype = None
    lib.orc_volume_map.argtypes = [_dp, _u32p, _dp, _u32p, _u32p, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_uint64, _dp, C.c_int]
    lib.orc_num_nodes.restype, lib.orc_num_nodes.argtypes = C.c_uint64, [_u32p]
    return lib


K3VEMU = os.path.join(ROOT, "build", "bin", "libk3vemu.so")


@pytest.fixture(scope="module")
def k3v():
    """the K3 translation unit alone, emulated (tests/emu/k3_volume_emu.cpp): emu_field_create + emu_volume_map"""
    if not os.path.exists(K3VEMU):
        pytest.skip("build/bin/libk3vemu.so not built (make cpp)")
    lib = C.CDLL(K3VEMU)
    lib.emu_field_create.restype = _vp
    lib.emu_field_create.argtypes = [_dp, _u32p, _dp, _u32p, C.c_uint64, _u32p]
    lib.emu_field_destroy.argtypes = [_vp]
    lib.emu_volume_map.argtypes = [_vp, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_uint64, _dp]
    return lib


def gd_res(d):
    gd = np.concatenate([d.domain_min[:], d.domain_max[:], d.cell_size[:], d.inv_cell_size[:]]).astype(np.float64)
    return gd, np.array(d.resolution[:], np.uint32)


def oracle(orcv, d, nodes, cells, cmap, h, scale, no_reduction, l0=0, l1=None):
    gd, res = gd_res(d)
    nodes = np.ascontiguousarray(nodes, np.float64); cells = np.ascontiguousarray(cells, np.uint32); cmap = np.ascontiguousarray(cmap, np.uint32)
    l1 = int(orcv.orc_num_nodes(_p(res, _u32p))) if l1 is None else l1      # the grid's nodes (the SDF may be reduced)
    out = np.empty(l1 - l0)
    orcv.orc_volume_map(_p(gd, _dp), _p(res, _u32p), _p(nodes, _dp), _p(cells, _u32p), _p(cmap, _u32p), h, scale, int(no_reduction), l0, l1,
                        _p(out, _dp), 0)
    return out


class Field:
    """dg_field_create on the emulated library, for a grid with n_nodes nodes (the SDF may be reduced)"""

    def __init__(self, emu, d, nodes, cells, cmap):
        self.emu, self.d = emu, d
        self.nodes = np.ascontiguousarray(nodes, np.float64); cells = np.ascontiguousarray(cells, np.uint32)
        cmap = np.ascontiguousarray(cmap, np.uint32)
        self.h = _vp()
        assert emu.dg_field_create(C.byref(d), _p(self.nodes, _dp), len(self.nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p),
                                   C.byref(self.h)) == 0, emu.dg_last_error()
        nn = C.c_uint64()
        assert emu.dg_grid_num_nodes(d.resolution, C.byref(nn)) == 0
        self.n_grid = nn.value

    def volume(self, h, scale, no_reduction, l0=0, l1=None):
        l1 = self.n_grid if l1 is None else l1
        out = np.empty(l1 - l0)
        rc = self.emu.dg_volume_map(self.h, h, scale, int(no_reduction), l0, l1, _p(out, _dp))
        return out if rc == 0 else rc

    def close(self):
        self.emu.dg_field_destroy(self.h)


def volume_dense(emu, d, nodes, cells, cmap, h, scale, no_reduction=False):
    f = Field(emu, d, nodes, cells, cmap)
    try:
        out = f.volume(h, scale, no_reduction)
        assert not isinstance(out, int), emu.dg_last_error()
        return out
    finally:
        f.close()


def call_new(emu, d, nodes, cells, cmap, h, scale, flags=0):
    """dg_reduced_volume_map_create -> status, or ((nodes, cells, cmap) of field 0, of field 1, timings)"""
    nodes = np.ascontiguousarray(nodes, np.float64); cells = np.ascontiguousarray(cells, np.uint32); cmap = np.ascontiguousarray(cmap, np.uint32)
    r0, r1 = _vp(), _vp()
    tm = np.full(13, -1.0)
    rc = emu.dg_reduced_volume_map_create(C.byref(d), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), h, scale, flags,
                                          C.byref(r0), C.byref(r1), _p(tm, _dp))
    if rc != 0:
        assert not r0.value and not r1.value
        return rc
    out = []
    for r in (r0, r1):
        nn, nc = C.c_uint64(), C.c_uint64()
        assert emu.dg_reduced_band_sizes(r, C.byref(nn), C.byref(nc)) == 0
        f = (np.empty(nn.value), np.empty((nc.value, 32), np.uint32), np.empty(n_grid_cells(d), np.uint32))
        assert emu.dg_reduced_band_copy(r, _p(f[0], _dp), _p(f[1], _u32p), _p(f[2], _u32p)) == 0
        assert emu.dg_reduced_band_destroy(r) == 0
        out.append(f)
    return out[0], out[1], tm


def call_old(emu, d, nodes, cells, cmap, h, scale, flags=0):
    """the two-step route: dg_volume_map with the predicate, closed-form cells + identity map, then dg_reduce_field (host passes) on each
    field with GenerateDensityMap's p0 and with 0 <= v, both with != DBL_MAX (:1073)"""
    vol = volume_dense(emu, d, nodes, cells, cmap, h, scale)
    diag = cell_diag(d)
    with np.errstate(invalid="ignore", over="ignore"):
        keep0 = (-6.0 * h < nodes + diag) & (nodes - diag < 2.0 * h) & (nodes != DBL_MAX)
        keep1 = (0.0 <= vol) & (vol != DBL_MAX)
    f0, tie0 = reduce_host(emu, d, nodes, cells, keep0, flags)
    res = np.array(d.resolution[:], np.uint32)
    cells1 = np.empty((n_grid_cells(d), 32), np.uint32)
    assert emu.dg_build_cells(_p(res, _u32p), 0, len(cells1), _p(cells1, _u32p)) == 0
    f1, tie1 = reduce_host(emu, d, vol, cells1, keep1, flags)
    return f0, f1, (tie0, tie1)


def in_ball_weight_sum(h):
    """sum of wijk = (wi * wj) * wk over the Gauss points inside the ball, in quadrature order, then * c0^3 (no contraction in numpy)"""
    c0, c1 = 0.5 * (h - (-h)), 0.5 * ((-h) + h)
    off = c0 * GA16 + c1
    s = 0.0
    for i in range(16):
        for j in range(16):
            wij = GW16[i] * GW16[j]
            for k in range(16):
                if (off[i] * off[i] + off[j] * off[j]) + off[k] * off[k] > h * h:
                    continue
                s = s + wij * GW16[k]
    return s, c0 * c0 * c0


# ------------------------------------------------------------------------------------------------ reference-side generator fixtures
@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_equal_reference_generator(emu, orcv, tmp_path, name):
    """each fixture of the reference-side generator, reduced (both sorts; equal to the two-step route) or --no-reduction, written
    byte-identical to its .cdm; the dense volume field also equals orc_volume_map bit for bit"""
    c = CASES[name]
    h, scale = float.fromhex(c["h_hex"]), c["scale"]
    g, d, nodes, cells, cmap = load_sdf(c["sdf"])
    want = os.path.join(GOLDEN, c["file"])
    vol = volume_dense(emu, d, nodes, cells, cmap, h, scale, c["no_reduction"])
    assert bits_equal(vol, oracle(orcv, d, nodes, cells, cmap, h, scale, c["no_reduction"]))
    out = str(tmp_path / "out.cdm")
    if c["no_reduction"]:
        n, cells1, cmap1 = dense_layout(emu, d)
        write_cdm(out, g, (nodes, cells, cmap), (vol, cells1, cmap1))
        assert cdm_equal(out, want)
        return
    for flags in (0, REFERENCE_SORT):
        f0, f1, tm = call_new(emu, d, nodes, cells, cmap, h, scale, flags)
        assert len(f0[0]) < len(nodes) and len(f1[0]) < len(vol)      # both reductions drop nodes
        old = call_old(emu, d, nodes, cells, cmap, h, scale, flags)
        assert same_field(f0, old[0]) and same_field(f1, old[1]) and (tm[10], tm[11]) == old[2]
        assert (tm[:10] >= 0).all() and tm[12] >= tm[:10].sum() - 1e-6
        write_cdm(out, g, f0, f1)
        assert cdm_equal(out, want), flags


@pytest.mark.parametrize("src", ["ref_bunny_12.cdf", "ref_sphere_reduced.cdm"])
def test_k3_entry_point_equals_oracle_and_capi(emu, orcv, k3v, src):
    """emu_volume_map (K3's launcher on an emulated field, as emu_density_map is for the density map) equals the oracle and dg_volume_map"""
    g, d, nodes, cells, cmap = load_sdf(src)
    gd, res = gd_res(d)
    nodes = np.ascontiguousarray(nodes, np.float64); cells = np.ascontiguousarray(cells, np.uint32); cmap = np.ascontiguousarray(cmap, np.uint32)
    fh = k3v.emu_field_create(_p(gd, _dp), _p(res, _u32p), _p(nodes, _dp), _p(cells, _u32p), len(cells), _p(cmap, _u32p))
    assert fh
    try:
        for h_cells, no_reduction in ((0.4, False), (1.5, True)):
            h = h_cells * float(cell_diag(d))
            want = oracle(orcv, d, nodes, cells, cmap, h, 0.8, no_reduction)
            got = np.empty(len(want))
            assert k3v.emu_volume_map(fh, h, 0.8, int(no_reduction), 0, len(got), _p(got, _dp)) == 0
            assert bits_equal(got, want) and bits_equal(got, volume_dense(emu, d, nodes, cells, cmap, h, 0.8, no_reduction))
    finally:
        k3v.emu_field_destroy(fh)


# ------------------------------------------------------------------------------------------------ the oracle on more inputs
SDFS = ["ref_sphere.cdf", "ref_bunny_12.cdf", "ref_band_dragon_12_inverted.cdf", "ref_aniso_reduced.cdf", "ref_sphere_reduced.cdm"]


@pytest.mark.parametrize("h_cells", [0.3, 1.0, 2.5])
@pytest.mark.parametrize("no_reduction", [False, True])
@pytest.mark.parametrize("src", SDFS)
def test_equals_oracle(emu, orcv, src, no_reduction, h_cells):
    """dense and reduced SDFs (field 0), with and without the predicate, h from below a cell diagonal to several: bit for bit"""
    g, d, nodes, cells, cmap = load_sdf(src)
    h = h_cells * float(cell_diag(d))
    got = volume_dense(emu, d, nodes, cells, cmap, h, 0.8, no_reduction)
    want = oracle(orcv, d, nodes, cells, cmap, h, 0.8, no_reduction)
    assert bits_equal(got, want)
    assert (got > 0).any()


def test_non_finite_coefficients(emu, orcv):
    """an SDF holding NaN, +inf, -inf and -DBL_MAX: gamma maps them to 1 or 0, so every value stays finite and >= 0 (or DBL_MAX)"""
    g, d, nodes, cells, cmap = load_sdf("ref_sphere.cdf")
    nodes = nodes.copy()
    rng = np.random.default_rng(7)
    idx = rng.choice(len(nodes), 40, replace=False)
    nodes[idx[:10]] = np.nan; nodes[idx[10:20]] = np.inf; nodes[idx[20:30]] = -np.inf; nodes[idx[30:]] = -DBL_MAX
    h = float(cell_diag(d))
    for no_reduction in (False, True):
        got = volume_dense(emu, d, nodes, cells, cmap, h, 0.8, no_reduction)
        assert bits_equal(got, oracle(orcv, d, nodes, cells, cmap, h, 0.8, no_reduction))
        v = got[got != DBL_MAX]
        assert np.isfinite(v).all() and (v >= 0).all() and len(v) > 0


def test_range_slices(emu, orcv):
    """sub-ranges [l0, l1) give the same bits as the whole range and as the oracle on that range"""
    g, d, nodes, cells, cmap = load_sdf("ref_bunny_12.cdf")
    h = float(cell_diag(d))
    f = Field(emu, d, nodes, cells, cmap)
    try:
        whole = f.volume(h, 0.8, False)
        for l0, l1 in ((0, 1), (5, 133), (1000, 4097), (len(nodes) - 7, len(nodes)), (17, 17)):
            part = f.volume(h, 0.8, False, l0, l1)
            assert bits_equal(part, whole[l0:l1]) and bits_equal(part, oracle(orcv, d, nodes, cells, cmap, h, 0.8, False, l0, l1))
    finally:
        f.close()


# ------------------------------------------------------------------------------------------------ closed forms
@pytest.mark.parametrize("h", [0.7, 2.0, 3.3])
def test_inside_everywhere_is_the_weight_sum(emu, h):
    """an SDF of -1000 everywhere, no predicate: a node whose whole ball lies in the domain is s * ((sum of in-ball wijk) * c0^3) exactly;
    every other node is smaller (points outside the domain give gamma(DBL_MAX) = 0) and still >= 0"""
    d = box_grid((4, 4, 4), (3.0, 4.0, 12.0))
    n, cells, cmap = dense_layout(emu, d)
    x = positions(emu, d, n)
    s, c0p = in_ball_weight_sum(h)
    vol = volume_dense(emu, d, np.full(n, -1000.0), cells, cmap, h, 0.8, True)
    mx = np.array(d.domain_max[:])
    inside = ((x - h >= 0.0) & (x + h <= mx)).all(axis=1)
    assert inside.sum() > 10
    assert (vol[inside] == 0.8 * (s * c0p)).all()
    assert (vol[~inside] < 0.8 * (s * c0p)).all() and (vol >= 0).all()


def test_far_outside_is_zero_and_values_are_bounded(emu):
    """d(x) > 2h gives exactly +0.0; with a plane SDF every value lies in [0, s * 4.2991 * h^3]"""
    d = box_grid((3, 2, 2))
    n, cells, cmap = dense_layout(emu, d)
    x = positions(emu, d, n)
    vol = volume_dense(emu, d, np.full(n, 50.0), cells, cmap, 2.0, 0.8, True)
    assert bits_equal(vol, np.zeros(n))
    plane = x[:, 2] - 12.0 + 0.25 * x[:, 0]
    for h, scale in ((1.0, 0.8), (4.0, 1.0), (13.0, 0.5)):
        vol = volume_dense(emu, d, plane, cells, cmap, h, scale, True)
        assert (vol >= 0).all() and (vol <= scale * 4.2991 * h ** 3).all() and (vol > 0).any()
        far = plane > 2.0 * h
        assert bits_equal(vol[far], np.zeros(int(far.sum())))


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(emu):
    """h <= 0, NaN or +-inf; a non-finite scale; a NULL output; a bad range; a NULL field: DG_ERR_INVALID.  The one-call route refuses
    the same h and scale before anything is allocated."""
    g, d, nodes, cells, cmap = load_sdf("ref_sphere.cdf")
    f = Field(emu, d, nodes, cells, cmap)
    try:
        for h in (0.0, -0.1, float("nan"), float("inf"), -float("inf")):
            assert f.volume(h, 0.8, False) == DG_ERR_INVALID, h
        for s in (float("nan"), float("inf"), -float("inf")):
            assert f.volume(0.1, s, False) == DG_ERR_INVALID, s
        assert not isinstance(f.volume(0.1, -2.0, False, 0, 10), int)           # a negative finite scale is allowed
        assert emu.dg_volume_map(f.h, 0.1, 0.8, 0, 0, 10, None) == DG_ERR_INVALID
        out = np.empty(10)
        assert emu.dg_volume_map(f.h, 0.1, 0.8, 0, 10, 5, _p(out, _dp)) == DG_ERR_INVALID
        assert emu.dg_volume_map(f.h, 0.1, 0.8, 0, 0, f.n_grid + 1, _p(np.empty(f.n_grid + 1), _dp)) == DG_ERR_INVALID
        assert emu.dg_volume_map(None, 0.1, 0.8, 0, 0, 10, _p(out, _dp)) == DG_ERR_INVALID
        assert emu.dg_volume_map_device(f.h, 0.1, 0.8, 0, 0, 10, None, None) == DG_ERR_INVALID
        assert emu.dg_volume_map_device(f.h, float("inf"), 0.8, 0, 0, 10, _p(out, _dp), None) == DG_ERR_INVALID
        assert emu.dg_volume_map(f.h, 0.1, 0.8, 0, 7, 7, None) == 0                # an empty range needs no output
    finally:
        f.close()
    for h, s in ((0.0, 0.8), (float("nan"), 0.8), (float("inf"), 0.8), (0.15, float("nan")), (0.15, float("inf"))):
        assert call_new(emu, d, nodes, cells, cmap, h, s) == DG_ERR_INVALID, (h, s)
    red = read_cdf(os.path.join(GOLDEN, "ref_sphere_reduced.cdm"))
    assert call_new(emu, d, red["nodes"][0], red["cells"][0], red["cmap"][0], 0.15, 0.8) == DG_ERR_INVALID
    assert b"already reduced" in emu.dg_last_error()
    r0, r1 = _vp(), _vp()
    assert emu.dg_reduced_volume_map_create(C.byref(d), None, len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), 0.15, 0.8, 0,
                                            C.byref(r0), C.byref(r1), None) == DG_ERR_INVALID
    assert emu.dg_reduced_volume_map_create(C.byref(d), _p(nodes, _dp), len(nodes), _p(cells, _u32p), len(cells), _p(cmap, _u32p), 0.15, 0.8, 4,
                                            C.byref(r0), C.byref(r1), None) == DG_ERR_INVALID
