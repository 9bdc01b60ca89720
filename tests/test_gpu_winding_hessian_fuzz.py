"""K5 (winding numbers) and K2's Hessian mode fuzzed on the device.  Both kernels define their own bit-exact contract, restated in numpy
(tests/winding_ref.py, tests/hessian_ref.py); the CPU emulation gives K5's walk a static stack of K5_MAX_STACK entries and replaces K2's TMA
staging by a plain copy, so the fuzzers run here through the product's C-ABI too (tools/k5_fuzz.py, tools/k2_fuzz.py, backend `dg`):
  K5: tree sizes around powers of two up to 4097 and happy_buddha.obj (the device gets exactly stack_depth x 128 x 8 B of shared memory),
      tie-rich and degenerate meshes, scales 10^-300 .. 10^300, NaN / inf vertices and queries, every branch of k5_atan2, beta = 1, 2, 3.5,
      inf, point counts around the warp and block sizes, 2^20 points in one call; and the winding sign mode (dg_mesh_distance, dg_sample_sdf
      over ranges off the warp and block multiples, the band form, switching back) against the reference's unsigned distance.
  K2: the Hessian mode on every field kind and query pattern of k2_fuzz (+-1e308, +-inf, NaN, subnormal, -0.0 coefficients, no kept cell or
      one, warps of mostly dummy copies, prefix counts), 4 M queries in one call, and interpolate(..., hessian=True) on CUDA tensors.
Bar: bit-exact, any NaN equal to any NaN."""
import math
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools")); sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import k2_fuzz  # noqa: E402
import k5_fuzz  # noqa: E402
import winding_ref as wr  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def k5(dg):
    return k5_fuzz.DgK5()


def _run(result, msgs):
    meshes, total, bad = result
    assert bad == 0 and total > 0, "\n".join(msgs[:10])
    return meshes, total


def test_k5_tree_sizes_on_device(k5):
    """T = 1, 2, 3, 2^k - 1, 2^k, 2^k + 1 (k <= 12): a perfect tree fills the walk's stack to exactly stack_depth entries; beta = 2 and inf,
    every prefix count"""
    msgs = []
    _run(k5_fuzz.run_cases(k5, k5_fuzz.tree_cases(0), betas=(2.0, math.inf), counts=k5_fuzz.COUNTS, log=msgs.append, max_points=60), msgs)


def test_k5_many_triangles_happy_buddha_on_device(k5):
    """happy_buddha.obj (855,196 triangles, the deepest real tree) where it is staged, beta = inf and 2"""
    msgs = []
    buddha = wr.ref_resource(ROOT, "happy_buddha.obj")
    if buddha:
        V, F = wr.read_obj(buddha)
        case = [("happy_buddha", V, F, wr.query_points(V, 200, seed=3, near=100))]
        _run(k5_fuzz.run_cases(k5, case, betas=(math.inf, 2.0), log=msgs.append, max_points=60), msgs)


def test_k5_tie_rich_meshes_on_device(k5):
    """coplanar grids, cubes / octahedra with points on faces, edges, vertices and symmetry planes, duplicated triangles, slivers, soups,
    zero-area subtrees; beta = 1, 2, 3.5, inf"""
    msgs = []
    _run(k5_fuzz.run_cases(k5, k5_fuzz.tie_cases(21, 1), log=msgs.append, max_points=300), msgs)


def test_k5_scales_on_device(k5):
    """k1_fuzz's scale sweep 10^-24 .. 10^17 and 10^+-150, 10^+-300, centred and offset: overflow and subnormals in r2, |r|^5, det, den"""
    msgs = []
    _run(k5_fuzz.run_cases(k5, k5_fuzz.scale_cases(0), betas=(2.0, math.inf), log=msgs.append, max_points=60), msgs)


def test_k5_nonfinite_and_atan2_branches_on_device(k5):
    """NaN / inf vertices, NaN, +-inf and huge queries; one-triangle meshes whose points take every branch of k5_atan2"""
    assert k5_fuzz.ATAN2_BRANCHES <= k5_fuzz.atan2_coverage(k5_fuzz.atan2_cases())
    msgs = []
    _run(k5_fuzz.run_cases(k5, k5_fuzz.nonfinite_cases(), betas=k5_fuzz.BETAS, counts=(33, 129), log=msgs.append), msgs)
    _run(k5_fuzz.run_cases(k5, k5_fuzz.atan2_cases(), betas=k5_fuzz.BETAS, log=msgs.append), msgs)


def test_k5_many_points_on_device(k5):
    """2^20 points in one call, beta = inf"""
    msgs = []
    n, bad = k5_fuzz.run_large(k5, 1 << 20, seed=4, log=msgs.append)
    assert n == 1 << 20 and bad == 0, "\n".join(msgs)


def test_winding_sign_mode_on_device(k5):
    """dg_mesh_set_sign_mode(DG_SIGN_WINDING, beta) on the tie-rich meshes: signed dg_mesh_distance == (w > 0.5 ? -d_u : d_u) with the
    unsigned query's nearest point, entity and triangle (DBL_MAX / -1 where no triangle is accepted); dg_sample_sdf with sign +-1 over the
    lattice and over ranges off multiples of 32 and 128; dg_add_function_sdf_band; the pseudonormal bits after switching back"""
    msgs = []
    _run(k5_fuzz.run_sign(k5, 14, seed=2, log=msgs.append), msgs)


def test_k2_hessian_fuzz_on_device(capsys, dg):
    """tools/k2_fuzz.py's Hessian mode on the device: every field kind and query pattern, prefix counts"""
    rc = k2_fuzz.main(["k2_fuzz", "36", "5", "dg", "hessian"])
    out = capsys.readouterr().out
    assert rc == 0 and "36 fields" in out and " 0 mismatches" in out, out[-3000:]


def test_k2_hessian_many_queries_on_device(dg):
    """4 M queries in one call in the Hessian mode on a reduced field with NaN / inf / DBL_MAX coefficients"""
    msgs = []
    n, bad = k2_fuzz.run_many(k2_fuzz.DgK2(), 4 << 20, seed=2, log=msgs.append, mode="hessian")
    assert n == 4 << 20 and bad == 0, "\n".join(msgs)


@pytest.mark.parametrize("k", [1, 2, 3, 5, 7, 11])
def test_hessian_tensor_route_on_extreme_fields(dg, orc, tmp_path, k):
    """interpolate(..., hessian=True) on float64 CUDA tensors (also a view at an odd element offset) == the host route == the restatement,
    bit for bit, on k2_fuzz's fields: huge / non-finite / tiny coefficients, sentinels, a reduced field, no kept cell"""
    import torch
    from make_reduce_golden import write_cdf
    rng = np.random.default_rng(300 + k)
    case = k2_fuzz.make_field(orc, rng, k, str(tmp_path))
    gd, r, nodes, cells, cmap = case[:5]
    x = k2_fuzz.queries(rng, gd, r, nodes, cells, cmap)
    path = str(tmp_path / "f.cdf")
    write_cdf(path, gd[0:3], gd[3:6], r, gd[6:9], gd[9:12], nodes, cells, cmap)
    grid = dg.CubicLagrangeDiscreteGrid(path)
    host = grid.interpolate(0, x, hessian=True)
    phi_g, grad_g = grid.interpolate(0, x, gradient=True)
    assert k2_fuzz.hessian_ok(*host, phi_g, grad_g, k2_fuzz.restate(gd, r, nodes, cells, cmap, x)).all()
    xt = torch.from_numpy(np.concatenate([np.full((1, 3), 7.0), x])).to("cuda").reshape(-1)
    view = xt.reshape(-1, 3)[1:]                                             # starts 3 elements (24 bytes) into its storage
    assert view.storage_offset() == 3
    for xd in (view, view.clone()):
        got = grid.interpolate(0, xd, hessian=True)
        assert all(t.is_cuda for t in got)
        assert all(k2_fuzz.same(t.cpu().numpy(), h).all() for t, h in zip(got, host))
