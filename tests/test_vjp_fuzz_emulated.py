"""K11 and K12 fuzzed on the CPU emulation: the families of tools/k11_fuzz.py and tools/k12_fuzz.py on build/bin/libdgemu.so (the whole C-ABI
with its kernels compiled by g++), against the numpy restatements, with smaller budgets than tests/test_gpu_vjp_fuzz.py; and the two
restatement helpers the fuzzers rest on: closed_form_cells against the oracle's cell table, and interpolate_vjp_touched against
interpolate_vjp."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT
import interpolate_vjp_ref as ref

sys.path.insert(0, os.path.join(ROOT, "tools"))
import k11_fuzz  # noqa: E402
import k12_fuzz  # noqa: E402

EMU = k11_fuzz.EMU
SMALL_HUB = ((8, 8, 4), 1500)                    # 2^8 cells: the hub folds 256 + 31 * 32 incidences, a quarter of the device run's


@pytest.fixture(scope="module")
def k11():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    return k11_fuzz.Lib(EMU)


@pytest.fixture(scope="module")
def k12():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    return k12_fuzz.TrainLib(EMU)


def _run(result, msgs):
    cases, total, bad = result
    assert bad == 0 and total > 0, "\n".join(msgs[:10])


# ------------------------------------------------------------------------------------------------------------------------------- restatements
def test_closed_form_cells_equal_the_oracle_table(orc):
    """the numpy cell_node_id equals the oracle's build_cells (the reference's addFunction table) on small anisotropic grids"""
    for res in ((1, 1, 1), (1, 1, 5), (6, 1, 1), (1, 4, 1), (3, 2, 5), (7, 5, 3), (2, 9, 4)):
        want = orc.build_cells(res).astype(np.int64)
        got = ref.closed_form_cells(res, np.arange(len(want)))
        assert np.array_equal(got, want), res


def test_touched_restatement_equals_the_full_one(k11, orc, tmp_path):
    """interpolate_vjp_touched (rows of the touched cells only, a callable table) gives the bits of interpolate_vjp on every small family"""
    rng = np.random.default_rng(3)
    flds = []
    for k in range(8):
        gd, r, nodes, cells, cmap, label = k11_fuzz.k2_fuzz.make_field(orc, rng, k, str(tmp_path))
        flds.append((k11_fuzz.Field(k11.desc(gd[0:3], gd[3:6], r, gd[6:9], gd[9:12]), nodes, np.ascontiguousarray(cells, np.uint32),
                                    cmap, label), k11_fuzz.k2_fuzz.queries(rng, gd, r, nodes, cells, cmap)))
    flds += [(f, x) for f, x in k11_fuzz.table_fields(k11, 0, id_bits=(8,), hub=SMALL_HUB)]
    flds += [(f, f.points(rng, 400)) for f in k11_fuzz.pass_fields(k11, 0, dense=((8, 8, 4),), reduced=False)]
    for res in k11_fuzz.CLOSED:
        d = k11.desc([-1.0, 0.0, 0.5], [1.0, 0.7, 2.0], res)
        f = k11_fuzz.Field(d, rng.standard_normal(k11.num_nodes(res)), None, None, f"closed {res}")
        flds.append((f, f.points(rng, 300)))
    for f, x in flds:
        cells = f.cells if f.cells is not None else ref.closed_form_cells(f.res, np.arange(f.n_cells_kept))
        d = f.d
        args = (d.domain_min[:], d.domain_max[:], d.cell_size[:], d.inv_cell_size[:], d.resolution[:], f.nodes)
        for which in k11_fuzz.UPSTREAMS:
            gp, gg = k11_fuzz.upstreams(rng, len(x), which, special=(which == "both"))
            with np.errstate(all="ignore"):
                want = ref.interpolate_vjp(*args, cells, f.cmap, x, gp, gg)
                got = ref.interpolate_vjp_touched(*args, f.rows() if f.cells is None else f.cells, f.cmap, x, gp, gg, chunk=97)
            assert k11_fuzz.same(got, want).all(), (f.label, which)


# ------------------------------------------------------------------------------------------------------------------------------- K11
def test_k11_fields(k11):
    """six k2_fuzz.make_field rounds made trainable (plain, DBL_MAX, reduced, huge / non-finite / tiny coefficients; grids of 1 .. 6 cells
    per axis, so n_cells_kept <= 216: keys of up to 8 bits, one sort pass); upstreams phi, grad, both and special at n = 0 (zeros written,
    no pass runs), 1, 32 (one full group of the first level), 127 and 129 (either side of K11_THREADS = 128) and all ~1300 queries"""
    msgs = []
    _run(k11_fuzz.run_fields(k11, 6, 0, msgs.append, counts=(0, 1, 32, 127, 129)), msgs)


def test_k11_tables_passes_closed_form(k11):
    """permuted ids; 5 n + 1000 nodes, most unreferenced; a hub node in every one of 2^8 cells (256 + 31 * 32 incidences in one node's
    fold); largest node id 2^8 with n_nodes = 2^8 + 1 (9 key bits, the second pass of the incidence sort for that id alone).
    n_cells_kept = 2^8 (8 x 8 x 4) with queries in the last cell among sentinels (key 2^8: 9 bits, 2 passes).  cells == NULL against the
    uploaded table on 1 x 1 x 1, 1 x 1 x 9, 9 x 1 x 1, 7 x 5 x 3"""
    msgs = []
    _run(k11_fuzz.run_tables(k11, 0, msgs.append, id_bits=(8,), hub=SMALL_HUB), msgs)
    _run(k11_fuzz.run_passes(k11, 0, msgs.append, n=800, dense=((8, 8, 4),), reduced=False), msgs)
    _run(k11_fuzz.run_closed(k11, 0, msgs.append), msgs)


def test_k11_depths_and_values(k11):
    """cells of 31, 32, 33, 1023, 1025 queries in one call (levels S = 1 and 32); special upstreams; set_nodes_device then the VJP"""
    msgs = []
    _run(k11_fuzz.run_depth(k11, 0, msgs.append, depths=(31, 32, 33, 1023, 1025)), msgs)
    _run(k11_fuzz.run_values(k11, 0, msgs.append), msgs)


# ------------------------------------------------------------------------------------------------------------------------------- K12
def test_k12_mesh(k12):
    """k12_fuzz on meshes, every output combination: the forward outputs of two k9_fuzz tie rounds and its slack, scale (10^-3, 1, 10^150),
    cull, nonfinite and bound cases; refits, the VJP at the positions cast against once the mesh holds the next step's; synthetic outputs
    on 257-triangle soups at 10^-160, 10^-81, 10^-77, 1, 10^77, 10^80, 10^160 (n . n underflows to 0 below ~10^-81 and overflows to inf
    above ~10^77), with n = 1, 127, 128, 129, 257 rays (one to three blocks of K12_THREADS = 128)"""
    msgs = []
    _run(k12_fuzz.run_mesh_cases(k12, k12_fuzz.mesh_cases(0, 2, (-3, 0, 150), n=30), 0, msgs.append), msgs)
    _run(k12_fuzz.run_mesh_refits(k12, 0, msgs.append, n=30), msgs)
    _run(k12_fuzz.run_mesh_synthetic(k12, 0, msgs.append), msgs)


def test_k12_field(k12):
    """k12_fuzz on fields, with grad_nodes: every third k7_fuzz case (k2_fuzz fields, special, thin, tangent, grid, density, cursor, ulp,
    scale, hole and bound cases) on trainable copies; synthetic crossings clamped from outside, on a max face, in removed and DBL_MAX
    cells, NaN, statuses outside the enum, n = 1 .. 257; and the crossing where phi is exactly DBL_MAX with a finite den"""
    msgs = []
    cases = list(k12_fuzz.field_cases(0, 2))[1::3]
    _run(k12_fuzz.run_field_cases(k12, cases, 0, msgs.append), msgs)
    _run(k12_fuzz.run_field_synthetic(k12, 0, msgs.append), msgs)
