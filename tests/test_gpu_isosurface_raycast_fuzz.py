"""K6 (level sets by marching tetrahedra) and K7 (first crossings along rays) fuzzed on the device against their numpy restatements
(tests/isosurface_ref.py, tests/raycast_ref.py), through the product's C-ABI (tools/k6_fuzz.py and tools/k7_fuzz.py, backend `dg`).  The
CPU emulation compiles the same sources with g++; these runs add nvcc's fp64 code, K7's per-lane shared-memory block cache and its descent
stack in local memory, K6's 64-bit edge ids on a lattice of 6.5 * 10^8 points, and the device's launch geometry.
  K6:  k2_fuzz fields at s = 1, 2, 3, 16 and iso from 0 to +-DBL_MAX; every case in even and odd tetrahedra; iso equal to lattice values;
       n_cells and 7 Np around the tile and chunk sizes, Np = 2^24 and 2^24 + 1; the lattice-coordinate clamp; a 54^3 grid at s = 16 whose
       edge ids pass 2^32 (restated on windows); the refusal of 2^31 lattice points.  Host and device copies give the same bits.
  K7:  k2_fuzz fields cast from face, corner, outside and non-finite origins; grid rays, special rays, iso at a sample, the thin feature,
       tangent rays, density maps; the breakpoint cursors far from the origin, on one-cell axes, along 512 cells, at three-axis ties and
       at bounds equal to a breakpoint; cells a few ulps of t wide; scales 10^+-100 and 10^+-150 with a floor on crossings; reduced
       fields with scattered holes; bounds; prefix counts; 2^20 +- 1 and 2^21 + 1 rays through the host route.  Host and device routes
       give the same bits.
Bar: bit-exact, any NaN equal to any NaN.  On the emulated library (the rehearsal) the budgets are smaller: the logic is what is checked
there."""
import os
import sys
import time

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import k6_fuzz  # noqa: E402
import k7_fuzz  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def emulated(dg):
    return dg._capi.EMULATED


@pytest.fixture(scope="module")
def lib(dg):
    return k7_fuzz.Lib("dg")


def _run(result, msgs):
    cases, total, bad = result[:3]
    assert bad == 0 and total > 0, "\n".join(msgs[:10])
    return result


# ------------------------------------------------------------------------------------------------------------------------------- K6
def test_k6_random_fields_on_device(lib, emulated):
    """k2_fuzz fields (sentinels, extreme and non-finite coefficients, reduced, no kept cell, one) at s = 1, 2, 3, 16"""
    msgs = []
    _run(k6_fuzz.run_fields(lib, 8 if emulated else 96, 0, msgs.append), msgs)


def test_k6_cases_and_exact_hits_on_device(lib):
    """every one of the 16 cases in even and odd tetrahedra; iso equal to lattice values and +-0.0 on exact zeros"""
    msgs = []
    counts = _run(k6_fuzz.run_cases(lib, 0, msgs.append), msgs)[3]
    assert (counts > 0).all(), counts.tolist()
    hits = _run(k6_fuzz.run_exact(lib, 0, msgs.append), msgs)[3]
    assert hits > 100


def test_k6_sizes_and_clamp_on_device(lib, emulated):
    """n_cells and 7 Np around the 1024-entry tiles and the 32-edge chunks; Np = 2^24 and 2^24 + 1 (the values pass); the clamp"""
    msgs, tris = [], []
    _run(k6_fuzz.run_sizes(lib, msgs.append, big=not emulated, tris=tris), msgs)
    assert {t[0] for t in tris} == {t[0] for t in tris if t[3] > 0}, tris          # every size emits at some iso
    _run(k6_fuzz.run_clamp(lib, 0, msgs.append, 8), msgs)


def test_k6_refuses_a_lattice_of_2_31_points_on_device(lib):
    msgs = []
    n, bad = k6_fuzz.run_refusal(lib, msgs.append)
    assert bad == 0, "\n".join(msgs)


def test_k6_large_lattice_edge_ids_past_2_32_on_device(lib):
    """a 54^3 grid at s = 16: 647,214,625 lattice points, 4,530,502,375 edge ids; the device's mesh equals the windows' restatement"""
    msgs = []
    t = time.time()
    r = k6_fuzz.run_large(lib, msgs.append)
    print("\n".join(msgs))
    if r is None:
        pytest.skip(msgs[-1])
    n, bad, emax, tris = r
    print(f"large lattice: largest edge id {emax} ({emax / 2**32:.4f} * 2^32), {tris} triangles, {time.time() - t:.1f} s")
    assert bad == 0 and emax > 1 << 32 and tris > 0, "\n".join(msgs)


# ------------------------------------------------------------------------------------------------------------------------------- K7
def test_k7_random_fields_on_device(lib, emulated):
    msgs = []
    _run(k7_fuzz.run_fields(lib, 8 if emulated else 160, 0, msgs.append, n=60 if emulated else 200), msgs)


def test_k7_grid_special_thin_tangent_density_on_device(lib):
    """grid rays and segments; zero / NaN / inf / subnormal rays; iso at a sample; the thin feature (reported); tangents; density maps"""
    msgs = []
    _run(k7_fuzz.run_cases(lib, k7_fuzz.grid_cases(), msgs.append), msgs)
    _run(k7_fuzz.run_special(lib, msgs.append), msgs)
    used = _run(k7_fuzz.run_iso_at_samples(lib, msgs.append), msgs)[0]
    assert used >= 20
    _run(k7_fuzz.run_thin_and_tangent(lib, msgs.append), msgs)
    _run(k7_fuzz.run_cases(lib, k7_fuzz.density_cases(), msgs.append), msgs)


def test_k7_cursors_on_device(lib):
    """far-offset domains cast from 2^52 cells away; one-cell axes; 1 x 1 x 512; three-axis ties; bounds equal to a breakpoint"""
    msgs = []
    _run(k7_fuzz.run_cases(lib, k7_fuzz.cursor_cases(0), msgs.append), msgs)
    _run(k7_fuzz.run_plane_bounds(lib, msgs.append), msgs)


def test_k7_ulps_and_scales_on_device(lib):
    """cells a few ulps of t wide and bounds a few ulps apart; 10^+-100 and 10^+-150, with crossings wherever the clip does not overflow"""
    msgs, hits = [], []
    _run(k7_fuzz.run_cases(lib, k7_fuzz.ulp_cases(), msgs.append), msgs)
    _run(k7_fuzz.run_ulp_bounds(lib, msgs.append), msgs)
    _run(k7_fuzz.run_cases(lib, k7_fuzz.scale_cases(), msgs.append, hits=hits), msgs)
    assert not k7_fuzz.dry(hits), k7_fuzz.dry(hits)


def test_k7_holes_bounds_counts_on_device(lib):
    msgs = []
    _run(k7_fuzz.run_cases(lib, k7_fuzz.hole_cases(0), msgs.append), msgs)
    _run(k7_fuzz.run_cases(lib, k7_fuzz.bound_cases(), msgs.append), msgs)
    _run(k7_fuzz.run_exact_bounds(lib, msgs.append), msgs)
    _run(k7_fuzz.run_counts(lib, msgs.append), msgs)


@pytest.mark.parametrize("n", [(1 << 20) - 1, (1 << 20) + 1, (1 << 21) + 1])
def test_k7_large_host_staging_on_device(lib, n):
    """n rays through the host route (chunks of 2^20) give the device route's bits; 3000 of them, the first and the last, and the rays on
    either side of each chunk boundary against the restatement"""
    msgs = []
    k, bad, crossings = k7_fuzz.run_staging(lib, n, msgs.append)
    assert bad == 0 and k > 3000 and crossings > 100, "\n".join(msgs)
