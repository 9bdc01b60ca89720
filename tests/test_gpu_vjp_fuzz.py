"""K11 (the VJP of interpolate in the node values) and K12 (the ray-cast VJPs) fuzzed on the device against their numpy restatements
(tests/interpolate_vjp_ref.py, tests/raycast_grad_ref.py), through the product's C-ABI (tools/k11_fuzz.py and tools/k12_fuzz.py, backend `dg`).
Every VJP runs twice through the host form and once through the _device form on a side stream, with the same bits.  The CPU emulation
compiles the same sources with g++; these runs add nvcc's fp64 code, the hardware warp shuffles of K11's first level and the sort, and the
launch geometry at the sizes where K11's grid-stride loops repeat (4096 blocks of 128 threads) and its deepest levels run.
Bar: bit-exact, any NaN equal to any NaN; +0.0 exactly for invalid rays and untouched nodes or vertices.
On the emulated library (the rehearsal) the budgets are smaller and the `large` tests are left out: the logic is what is checked there."""
import os
import sys

import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import k11_fuzz  # noqa: E402
import k12_fuzz  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def emulated(dg):
    return dg._capi.EMULATED


@pytest.fixture(scope="module")
def k11(dg):
    return k11_fuzz.Lib("dg", side=True)


@pytest.fixture(scope="module")
def k12(dg):
    return k12_fuzz.TrainLib("dg", side=True)


def _run(result, msgs):
    cases, total, bad = result
    assert bad == 0 and total > 0, "\n".join(msgs[:10])
    print(f"{cases} cases, {total} values")
    return cases, total


# ------------------------------------------------------------------------------------------------------------------------------- K11
def test_k11_fields_on_device(k11, emulated):
    """k2_fuzz.make_field rounds made trainable (plain, DBL_MAX, reduced, extreme coefficients, no kept cell, exactly one); upstreams phi,
    grad, both and special at n = 0, 1, 31, 32, 33, 127, 129 (around K11_THREADS = 128) and ~1300 k2_fuzz.queries points"""
    msgs = []
    _run(k11_fuzz.run_fields(k11, 4 if emulated else 24, 1, msgs.append, counts=(0, 1, 33, 129) if emulated else k11_fuzz.COUNTS), msgs)


def test_k11_tables_no_grid_makes_on_device(k11, emulated):
    """permuted node ids; 5 n + 1000 nodes, most unreferenced (runs of the inc_begin pass); a hub node in every one of 2^12 cells, so that
    one node folds about 4096 + 31 * 32 incidences; largest node id 2^8, 2^16, 2^24 with n_nodes = 2^k + 1: bit_width(n_nodes - 1) = k + 1 key
    bits of the incidence sort, 2, 3 and 4 passes of 8 bits, the last one for the top id's bit k alone"""
    msgs = []
    if emulated:                                  # tests/test_vjp_fuzz_emulated.py runs this family on the emulation: the logic only here
        _run(k11_fuzz.run_tables(k11, 2, msgs.append, id_bits=(), hub=((4, 4, 2), 200)), msgs)
    else:
        _run(k11_fuzz.run_tables(k11, 2, msgs.append), msgs)


def test_k11_sort_pass_boundaries_on_device(k11, emulated):
    """n_cells_kept = 2^8 (8 x 8 x 4: keys up to 2^8 need 9 bits, 2 passes) and 2^16 (64 x 64 x 16: 17 bits, 3 passes), and reduced fields
    of 2^16 - 1 and 2^16 + 1 kept cells, each with a query in the last kept cell (key n_cells_kept, the one key with the top bit)"""
    msgs = []
    if emulated:
        _run(k11_fuzz.run_passes(k11, 3, msgs.append, n=500, dense=((8, 8, 4),), reduced=False), msgs)
    else:
        _run(k11_fuzz.run_passes(k11, 3, msgs.append), msgs)


def test_k11_closed_form_table_on_device(k11):
    """cells == NULL (k11_inc_key_kernel's cell_node_id branch) against the uploaded table on 1 x 1 x 1, 1 x 1 x 9, 9 x 1 x 1, 7 x 5 x 3: the
    VJP (both against the restatement), interpolate and set_nodes with planted DBL_MAX coefficients give the same bits"""
    msgs = []
    _run(k11_fuzz.run_closed(k11, 4, msgs.append), msgs)


def test_k11_level_depths_on_device(k11, emulated):
    """cells of 31, 32, 33, 1023, 1025, 32767, 32769 queries in one call: 1, 1, 2, 32, 33, 1024 and 1025 groups, i.e. the levels S = 1, 32
    and 1024 with full and partial last blocks"""
    msgs = []
    _run(k11_fuzz.run_depth(k11, 5, msgs.append, depths=(31, 33, 1025) if emulated else k11_fuzz.DEPTHS), msgs)


def test_k11_special_upstreams_and_set_nodes_device_on_device(k11):
    """+-0, subnormal, +-1e308, +-inf, NaN upstreams on a dense and a reduced field; dg_field_set_nodes_device planting DBL_MAX coefficients,
    then dg_interpolate_vjp_device on the same stream (no synchronisation between them) sees them"""
    msgs = []
    _run(k11_fuzz.run_values(k11, 6, msgs.append), msgs)


def test_k11_one_cell_of_2_20_queries_large(k11):
    """one cell holding 2^20 + 1 queries among 5000 others: 32769 groups, levels S = 1, 32, 1024 and 32768 (deep[3], the fourth level)"""
    msgs = []
    _run(k11_fuzz.run_depth(k11, 7, msgs.append, huge=True), msgs)


def test_k11_grid_strides_large(k11):
    """128^3 through the closed-form table.  2^20 random queries: ~10^6 groups, far more than the 16384 warps of k11_first_level_kernel's
    launch (4096 blocks x 128 threads), so its grid-stride loop repeats.  2^19 + 2^16 singleton cells at the lowest cell ids and cells of
    1025, 100, 33, 32769, 64 queries at the five highest: more than the 2^19 threads of k11_level_kernel's launch, the deep cells' groups
    all past them"""
    msgs = []
    _run(k11_fuzz.run_strides(k11, 8, msgs.append), msgs)


def test_k11_256_cubed_large(k11):
    """256^3 through the closed-form table and through the uploaded table: n_cells_kept = 2^24 (25 key bits, 4 passes of the query sort; the
    last cell touched), node ids up to 118 M (27 bits, 4 passes of the incidence sort); VJP, interpolate and set_nodes with the same bits in
    both, and against the restatement.  Reports each creation's time and device memory"""
    msgs = []
    r = k11_fuzz.run_256(k11, 9, msgs.append)
    for m in msgs:
        if m.startswith("MEASURE") or "created" in m:
            print(m)
    _run(r, [m for m in msgs if m.startswith("MISMATCH")])


# ------------------------------------------------------------------------------------------------------------------------------- K12
def test_k12_mesh_cases_on_device(k12, emulated):
    """the forward outputs of k9_fuzz's tie, slack, scale, cull, nonfinite and bound cases, every output combination, upstreams t, bary,
    both and special"""
    msgs = []
    cases = k12_fuzz.mesh_cases(0, 2 if emulated else 16, (-3, 0, 150) if emulated else (-24, -3, 0, 5, 17, -150, -100, 100, 150))
    _run(k12_fuzz.run_mesh_cases(k12, cases, 0, msgs.append), msgs)


def test_k12_mesh_refits_and_synthetic_on_device(k12):
    """casts after refits, the VJP at the positions cast against once the mesh holds others; synthetic outputs on soups with degenerate
    triangles at 10^-160 .. 10^160 (n . n = 0 or inf), in-plane and subnormal directions, n = 1, 127, 128, 129, 257 (K12_THREADS = 128)"""
    msgs = []
    _run(k12_fuzz.run_mesh_refits(k12, 1, msgs.append), msgs)
    _run(k12_fuzz.run_mesh_synthetic(k12, 1, msgs.append), msgs)


def test_k12_field_cases_on_device(k12, emulated):
    """the forward outputs of k7_fuzz's fields, special rays, thin feature, grid, density, cursor, ulp, scale, hole and bound cases on
    trainable copies of their fields, iso != 0 among them, and the iso-at-sample rays, with grad_nodes"""
    msgs = []
    cases = list(k12_fuzz.field_cases(2, 2 if emulated else 12))
    if emulated:
        cases = cases[::6]
    _run(k12_fuzz.run_field_cases(k12, cases, 2, msgs.append), msgs)
    _run(k12_fuzz.run_iso_at_samples(k12, 2, msgs.append), msgs)


def test_k12_field_synthetic_on_device(k12):
    """crossing points clamped from outside, on a max face, in removed and DBL_MAX cells, NaN; statuses 0, 1, 2 and outside the enum; a
    crossing where phi is exactly DBL_MAX from a coefficient below it, with a finite nonzero den"""
    msgs = []
    _run(k12_fuzz.run_field_synthetic(k12, 3, msgs.append), msgs)
