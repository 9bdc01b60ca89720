"""K2 (interpolate) and K3 (density map) fuzzed on the device.  The CPU emulation of the kernels (tests/test_k23_emulated.py) replaces K2's TMA
staging (cp.async.bulk + a per-warp mbarrier) by a plain copy and runs K3 one lane at a time, so the fuzzers run here through the product's
C-ABI too (tools/k2_fuzz.py, tools/k3_fuzz.py, backend `dg`): extreme coefficients (+-1e308, -DBL_MAX, NaN, +-inf, subnormals, -0.0),
fields with no kept cell or one, warps that mix live lanes with lanes that copy nothing real, query counts around the warp and block sizes
and 4 M queries in one call; K3 on reduced inputs, h on both sides of the fast division's range, h = +inf / subnormal, rho0 of 0, -1,
+inf, NaN.  Then the same fields through the CUDA-tensor route of interpolate, the one-call reduced density map, and GenerateDensityMap
against the reference tool where build() compiled it.  Bar: bit-exact, any NaN equal to any NaN (which payload an operation on two NaNs
returns is left to the hardware by IEEE 754)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import k2_fuzz  # noqa: E402
import k3_fuzz  # noqa: E402

pytestmark = pytest.mark.gpu

REF_TOOL = os.path.join(ROOT, "oracle", "_ref", "bin", "GenerateDensityMap")
OUR_TOOL = os.path.join(ROOT, "build", "bin", "GenerateDensityMap")


@pytest.fixture(scope="module")
def be(dg):
    return k2_fuzz.DgK2()


def test_k2_fuzz_on_device(capsys, dg):
    """tools/k2_fuzz.py on the device: every field kind and query pattern of the fuzzer, value + gradient and value-only, prefix counts"""
    rc = k2_fuzz.main(["k2_fuzz", "36", "5", "dg"])
    out = capsys.readouterr().out
    assert rc == 0 and "0 mismatches" in out, out[-3000:]


def test_k2_many_queries_on_device(be):
    """4 M queries in one call on a reduced field with NaN / inf / DBL_MAX coefficients: many warps with copies in flight"""
    msgs = []
    n, bad = k2_fuzz.run_many(be, 4 << 20, seed=2, log=msgs.append)
    assert n == 4 << 20 and bad == 0, "\n".join(msgs)


def test_k3_fuzz_on_device(capsys, dg):
    """tools/k3_fuzz.py on the device: four rounds of every kind, both predicate modes"""
    rc = k3_fuzz.main(["k3_fuzz", "40", "3", "dg"])
    out = capsys.readouterr().out
    assert rc == 0 and "0 mismatches" in out, out[-3000:]


def _grid_file(tmp_path, orc, case, name):
    from make_reduce_golden import write_cdf
    gd, r, nodes, cells, cmap = case[:5]
    path = str(tmp_path / name)
    write_cdf(path, gd[0:3], gd[3:6], r, gd[6:9], gd[9:12], nodes, cells, cmap)
    return path


@pytest.mark.parametrize("k", [1, 2, 3, 5, 11])
def test_interpolate_tensor_route_on_extreme_fields(dg, orc, tmp_path, k):
    """interpolate on float64 CUDA tensors (also a view at an odd element offset) == the host route, bit for bit, on k2_fuzz's fields:
    huge / non-finite / tiny coefficients, sentinels, a reduced field, no kept cell"""
    import torch
    rng = np.random.default_rng(100 + k)
    case = k2_fuzz.make_field(orc, rng, k, str(tmp_path))
    x = k2_fuzz.queries(rng, *case[:5])
    grid = dg.CubicLagrangeDiscreteGrid(_grid_file(tmp_path, orc, case, "f.cdf"))
    phi_h, grad_h = grid.interpolate(0, x, gradient=True)
    only_h = grid.interpolate(0, x)
    xt = torch.from_numpy(np.concatenate([np.full((1, 3), 7.0), x])).to("cuda").reshape(-1)
    view = xt.reshape(-1, 3)[1:]                                             # starts 3 elements (24 bytes) into its storage
    assert view.storage_offset() == 3
    for xd in (view, view.clone()):
        phi, grad = grid.interpolate(0, xd, gradient=True)
        only = grid.interpolate(0, xd)
        assert phi.is_cuda and grad.is_cuda
        assert k2_fuzz.same(phi.cpu().numpy(), phi_h).all() and k2_fuzz.same(grad.cpu().numpy(), grad_h).all()
        assert k2_fuzz.same(only.cpu().numpy(), only_h).all()


@pytest.mark.parametrize("k", [0, 4, 5, 6, 7, 9])
def test_reduced_density_map_on_extreme_fields(dg, orc, k):
    """dg_reduced_density_map_create == dg_density_map + dg_reduce_field on each field, bit for bit, on k3_fuzz's unreduced fields:
    -DBL_MAX, +-1e308 / 1e306, NaN, +-inf / subnormal / -0.0 coefficients, h = +inf"""
    from discregrid_b200.grid import grid_desc
    from test_density_reduced_emulated import same_field
    from test_gpu_density_reduced import capi_new, capi_old
    rng = np.random.default_rng(200 + k)
    c = k3_fuzz.make_case(orc, rng, k)
    assert len(c["cells"]) == int(np.prod(c["r"].astype(np.int64)))       # an unreduced SDF
    gd = c["gd"]
    d = grid_desc(gd[0:3], gd[3:6], c["r"], gd[6:9], gd[9:12])
    with np.errstate(invalid="ignore", over="ignore"):
        new = capi_new(d, c["nodes"], c["cells"], c["cmap"], c["h"], c["rho0"])
        old = capi_old(d, c["nodes"], c["cells"], c["cmap"], c["h"], c["rho0"])
    assert same_field(new[0], old[0]) and same_field(new[1], old[1]) and (new[2][10], new[2][11]) == old[2]


def _tool_inputs(orc):
    """small sphere SDFs on [0, 2]^3: (name, grid, nodes, h) -- plain, one -DBL_MAX coefficient, one NaN, +-1e308"""
    rng = np.random.default_rng(7)
    out = []
    for name, res, h, plant in (("plain", (4, 4, 4), 0.3, None), ("minus_dbl_max", (4, 4, 4), 0.3, -k2_fuzz.DBL_MAX),
                                ("nan", (4, 3, 5), 0.9, np.nan), ("huge", (3, 4, 4), 0.3, 1e308)):
        gd, r = orc.grid_desc([0.0, 0.0, 0.0], [2.0, 2.0, 2.0], res)
        cells = orc.build_cells(r)
        n = int(cells.max()) + 1
        x = orc.node_positions(gd, r, 0, n)
        v = np.linalg.norm(x - (1.0 + 0.1 * rng.standard_normal(3)), axis=1) - 0.6
        if plant is not None:
            v[int(rng.integers(n))] = plant
            if name == "huge":
                v[int(rng.integers(n))] = -1e308
        out.append((name, gd, r, v, cells, h))
    return out


def test_generate_density_map_equals_reference_tool(orc, tmp_path):
    """GenerateDensityMap (build/bin, the library's kernels) == the reference's own tool on small .cdf inputs with -DBL_MAX, NaN and
    +-1e308 coefficients, with and without --no-reduction"""
    if not (os.path.exists(REF_TOOL) and os.path.exists(OUR_TOOL)):
        pytest.skip("needs oracle/_ref/bin/GenerateDensityMap and build/bin/GenerateDensityMap")
    from make_reduce_golden import write_cdf
    from test_density_reduced_emulated import cdm_equal
    for name, gd, r, v, cells, h in _tool_inputs(orc):
        src = str(tmp_path / f"{name}.cdf")
        write_cdf(src, gd[0:3], gd[3:6], r, gd[6:9], gd[9:12], v, cells, np.arange(len(cells), dtype=np.uint32))
        for extra in ([], ["--no-reduction"]):
            outs = []
            for tag, tool in (("ref", REF_TOOL), ("ours", OUR_TOOL)):
                out = str(tmp_path / f"{name}_{tag}{len(extra)}.cdm")
                p = subprocess.run([tool, "-s", repr(h), "-r", "1000.0", "-o", out] + extra + [src], capture_output=True, text=True, timeout=600)
                assert p.returncode == 0, (name, tag, p.stdout + p.stderr)
                outs.append(out)
            assert cdm_equal(*outs), (name, extra)
