"""K9 (ray casts on a mesh) and K10 (the distance gradient, its radix sort and the forward with weights) fuzzed on the device against their
numpy restatements (tests/mesh_raycast_ref.py, tests/mesh_distance_grad_ref.py), through the product's C-ABI (tools/k9_fuzz.py and
tools/k10_fuzz.py, backend `dg`).  The CPU emulation compiles the same sources with g++; these runs add nvcc's fp64 code, the hardware warp
collectives the sort's stability rests on, K9's stack in local memory and the device's launch geometry at 10^6+ elements.
  K9:  tree sizes around powers of two and happy_buddha.obj; ties with shuffled ids, stacked duplicates, zero-area triangles, a flat grid
       cast from its own plane; meshes whose fp32 boxes sit inside a vertex by less than the culling slack; scales 10^-45 .. 10^150 with a
       floor on the hit count; the culling switch at 2^1020; non-finite vertices and rays; bounds; prefix counts; refits; 2^22 rays.
  K10: the forward on k1_fuzz's tie, scale and awkward meshes in both sign modes; the VJP on synthetic outputs at the sort's pass and tile
       boundaries, every id pattern, segment lengths at the level tree's 32^k boundaries, a fan of 10^4 triangles, non-finite values, one
       segment of 2^22 + 1 queries; every VJP twice and once on a side stream, with the same bits.
Bar: bit-exact, any NaN equal to any NaN, except where a header promises the bits (K9's miss weights, K10's +0.0 point gradients).
On the emulated library (the rehearsal) the budgets are smaller: the logic is what is checked there."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import k9_fuzz  # noqa: E402
import k10_fuzz  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def emulated(dg):
    return dg._capi.EMULATED


@pytest.fixture(scope="module")
def k9(dg):
    return k9_fuzz.DgK9()


@pytest.fixture(scope="module")
def k10(dg, emulated):
    return k10_fuzz.DgK10(side=not emulated)            # the side stream needs torch on a device


def _run(result, msgs):
    cases, total, bad = result
    assert bad == 0 and total > 0, "\n".join(msgs[:10])
    return cases, total


# ------------------------------------------------------------------------------------------------------------------------------- K9
def test_k9_tree_sizes_on_device(k9, emulated):
    """T = 1, 2, 3, 2^k - 1, 2^k, 2^k + 1 (k <= 12): a perfect tree fills the walk's stack; happy_buddha.obj where it is staged"""
    msgs = []
    sizes = k9_fuzz.k5_fuzz.TREE_SIZES[::3] if emulated else k9_fuzz.k5_fuzz.TREE_SIZES
    _run(k9_fuzz.run_cases(k9, k9_fuzz.tree_cases(0, sizes), log=msgs.append), msgs)
    if not emulated and k9_fuzz.wr.ref_resource(ROOT, "happy_buddha.obj"):
        _run(k9_fuzz.run_cases(k9, k9_fuzz.buddha_case(1), log=msgs.append), msgs)


def test_k9_ties_and_slack_on_device(k9, emulated):
    """tie-rich meshes with shuffled ids, stacked duplicates, zero-area triangles, the flat grid cast from its plane (every hit at t = 0);
    and the meshes whose fp32 child box lies inside a vertex by less than the slack"""
    msgs = []
    _run(k9_fuzz.run_cases(k9, k9_fuzz.tie_cases(7 if emulated else 40, 1), log=msgs.append), msgs)
    _run(k9_fuzz.run_cases(k9, k9_fuzz.slack_cases(), log=msgs.append), msgs)


def test_k9_scales_on_device(k9, emulated):
    """sphere.obj at 10^-45 .. 10^-38 (fp32 half extent subnormal or 0), 10^-24 .. 10^17, 10^+-100, 10^+-150, centred and offset, scaled
    and unit directions; the restatement hits in every case but 10^150 with unit directions, where T = U Az + ... overflows"""
    msgs, hits = [], []
    exps = k9_fuzz.SCALE_EXPONENTS[::4] + (-150, 150) if emulated else k9_fuzz.SCALE_EXPONENTS
    _run(k9_fuzz.run_cases(k9, k9_fuzz.scale_cases(0, exps), log=msgs.append, hits=hits), msgs)
    dry = [label for label, h in hits if h == 0 and not ("1e150 " in label and "unit" in label)]
    assert not dry, f"no hits at all: {dry[:5]}"


def test_k9_cull_switch_and_nonfinite_on_device(k9):
    """origins and meshes at 2^1019, 2^1020, 2^1021; subnormal directions (Sz = inf); NaN / inf vertices; special origins and directions"""
    msgs, hits = [], []
    _run(k9_fuzz.run_cases(k9, k9_fuzz.cull_cases(0), log=msgs.append, hits=hits), msgs)
    assert all(h > 0 for label, h in hits if label.startswith("origins at"))
    _run(k9_fuzz.run_cases(k9, k9_fuzz.nonfinite_cases(0), log=msgs.append), msgs)


def test_k9_bounds_and_counts_on_device(k9):
    """[0, inf), [-inf, inf), [0, 1], [-0.5, 2]; t_min = t_max at a hit's t; t_max below every hit; prefixes of 1, 127, 128, 129, 257 rays"""
    msgs = []
    _run(k9_fuzz.run_cases(k9, k9_fuzz.bound_cases(0), log=msgs.append), msgs)
    _run(k9_fuzz.run_exact_bounds(k9, 0, msgs.append), msgs)
    _run(k9_fuzz.run_counts(k9, 0, msgs.append), msgs)


def test_k9_refits_on_device(k9):
    """refit to scaled, mirrored (status flips), translated positions, half the triangles collapsed to a point, one vertex NaN, and back"""
    msgs = []
    _run(k9_fuzz.run_refits(k9, 0, msgs.append), msgs)


def test_k9_large_on_device(k9):
    """2^22 rays in one call on bunny.obj: first, last and 3000 random rays against the restatement"""
    msgs = []
    n, bad, hit = k9_fuzz.run_large(k9, 1 << 22, 0, msgs.append)
    assert bad == 0 and n > 3000 and hit > 500, "\n".join(msgs)


# ------------------------------------------------------------------------------------------------------------------------------- K10
def test_k10_forward_on_device(k10, emulated):
    """dg_mesh_distance_bary == dg_mesh_distance (fields 0-3) and the restated weights, on k1_fuzz's tie, scale and awkward meshes, both sign
    modes, signed and unsigned; the VJP of those outputs"""
    msgs = []
    exps = k10_fuzz.k1_fuzz.SCALE_EXPONENTS[::6] if emulated else k10_fuzz.k1_fuzz.SCALE_EXPONENTS
    _run(k10_fuzz.run_forward(k10, 7 if emulated else 40, 2, msgs.append, exps), msgs)


def test_k10_vjp_sort_boundaries_on_device(k10, emulated):
    """T = 1, 255, 256, 257, 65535, 65536, 65537 and happy_buddha.obj (1, 2, 3 passes); every id pattern at n = 0 .. 2^17 + 1"""
    msgs = []
    if emulated:
        _run(k10_fuzz.run_vjp(k10, 3, msgs.append, counts=(0, 1, 33, 1025), sizes=(1, 256, 257), per_mesh=4), msgs)
    else:
        _run(k10_fuzz.run_vjp(k10, 3, msgs.append), msgs)


def test_k10_vjp_segments_fan_values_on_device(k10, emulated):
    """one segment of 31 .. 32769 queries among others on a fan of 10^4 triangles; g, d and x - p at +-0, subnormals, +-1e308, +-inf, NaN"""
    msgs = []
    _run(k10_fuzz.run_segments(k10, 4, msgs.append, lengths=(31, 33, 1025) if emulated else k10_fuzz.SEGMENTS), msgs)
    _run(k10_fuzz.run_values(k10, 4, msgs.append), msgs)


def test_k10_large_segment_on_device(k10):
    """one segment of 2^22 + 1 queries: five levels of the tree"""
    msgs = []
    n, bad = k10_fuzz.run_large_segment(k10, (1 << 22) + 1, 5, msgs.append)
    assert bad == 0 and n > 0, "\n".join(msgs)
