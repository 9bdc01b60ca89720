"""K6 and K7 fuzzed on the CPU emulation: the families of tools/k6_fuzz.py and tools/k7_fuzz.py on build/bin/libdgemu.so (the whole library,
its kernels compiled for the CPU) against the numpy restatements, with smaller budgets than tests/test_gpu_isosurface_raycast_fuzz.py and
without the large lattice, the lattices of 2^24 and 2^24 + 1 points and the 2^20-ray calls.  Also the restatement's own window form
(isosurface_ref.extract_windows), which the large lattice on the device rests on, against the whole-lattice restatement."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import isosurface_ref as ir  # noqa: E402
import k6_fuzz  # noqa: E402
import k7_fuzz  # noqa: E402

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    return k7_fuzz.Lib(EMU)


def _run(result, msgs):
    cases, total, bad = result[:3]
    assert bad == 0 and total > 0, "\n".join(msgs[:10])
    return result


def test_extract_windows_equals_the_whole_lattice():
    """three negative blobs in a positive field; windows around them (one at the lattice's corner, one inside, one at the far corner)
    give the whole-lattice restatement's vertices and triangles"""
    L = ir.Lattice([0.0, -1.0, 0.5], [2.0, 1.0, 2.0], [0.25, 0.25, 0.25], (8, 8, 6), 3)
    P = L.points()
    f = np.ones(L.n_points)
    blobs = ((0.1, -0.9, 0.6), (1.0, 0.1, 1.3), (1.95, 0.95, 1.95))
    for c in blobs:
        f = np.minimum(f, np.linalg.norm(P - c, axis=1) - 0.2)
    f[np.abs(P[:, 0] - 1.5) < 1e-9] = np.nan                              # an invalid plane outside every window
    I, J, K = L.unlin(np.arange(L.n_points))
    h = L.cell / L.s
    windows = []
    for c in blobs:                                                       # the blob's box and one lattice cell more
        lo = np.maximum(0, np.floor((np.array(c) - 0.2 - L.mn) / h).astype(np.int64) - 1)
        hi = np.minimum(L.np - 1, np.ceil((np.array(c) + 0.2 - L.mn) / h).astype(np.int64) + 1)
        inside = (I >= lo[0]) & (I <= hi[0]) & (J >= lo[1]) & (J <= hi[1]) & (K >= lo[2]) & (K <= hi[2])
        windows.append((lo, hi, f[inside]))
    V, T = ir.extract(L, f, 0.0)
    Vw, Tw, E = ir.extract_windows(L, windows, 0.0)
    assert len(T) > 100
    assert np.array_equal(V.view(np.uint64), Vw.view(np.uint64)) and np.array_equal(T, Tw)
    assert len(E) == len(Vw) and (np.diff(E) > 0).all() and 7 * L.lin(*windows[-1][0]) <= E[-1] < 7 * L.n_points


def test_k6_random_fields(lib):
    msgs = []
    _run(k6_fuzz.run_fields(lib, 12, 1, msgs.append), msgs)


def test_k6_cases_exact_sizes_clamp(lib):
    """all 16 cases in even and odd tetrahedra; iso at lattice values and +-0.0; n_cells and 7 Np around the tile and chunk sizes; the
    lattice-coordinate clamp, taken and (a -0.0 maximum) not taken"""
    msgs = []
    counts = _run(k6_fuzz.run_cases(lib, 1, msgs.append), msgs)[3]
    assert (counts > 0).all(), counts.tolist()
    assert _run(k6_fuzz.run_exact(lib, 1, msgs.append), msgs)[3] > 100
    _run(k6_fuzz.run_sizes(lib, msgs.append, big=False), msgs)                # Np = 2^24 and 2^24 + 1 run on the device
    _run(k6_fuzz.run_clamp(lib, 1, msgs.append), msgs)


def test_k6_refusal(lib):
    msgs = []
    assert k6_fuzz.run_refusal(lib, msgs.append)[1] == 0, msgs


def test_k7_random_fields(lib):
    msgs = []
    _run(k7_fuzz.run_fields(lib, 16, 1, msgs.append, n=100), msgs)


def test_k7_grid_special_thin_tangent_density(lib):
    msgs = []
    _run(k7_fuzz.run_cases(lib, k7_fuzz.grid_cases(), msgs.append), msgs)
    _run(k7_fuzz.run_special(lib, msgs.append), msgs)
    assert _run(k7_fuzz.run_iso_at_samples(lib, msgs.append), msgs)[0] >= 20
    _run(k7_fuzz.run_thin_and_tangent(lib, msgs.append), msgs)
    _run(k7_fuzz.run_cases(lib, k7_fuzz.density_cases(), msgs.append), msgs)


def test_k7_cursors_ulps_scales(lib):
    msgs, hits = [], []
    _run(k7_fuzz.run_cases(lib, k7_fuzz.cursor_cases(1), msgs.append), msgs)
    _run(k7_fuzz.run_plane_bounds(lib, msgs.append), msgs)
    _run(k7_fuzz.run_cases(lib, k7_fuzz.ulp_cases(), msgs.append), msgs)
    _run(k7_fuzz.run_ulp_bounds(lib, msgs.append), msgs)
    _run(k7_fuzz.run_cases(lib, k7_fuzz.scale_cases(), msgs.append, hits=hits), msgs)
    assert not k7_fuzz.dry(hits), k7_fuzz.dry(hits)


def test_k7_holes_bounds_counts(lib):
    msgs = []
    _run(k7_fuzz.run_cases(lib, k7_fuzz.hole_cases(1), msgs.append), msgs)
    _run(k7_fuzz.run_cases(lib, k7_fuzz.bound_cases(), msgs.append), msgs)
    _run(k7_fuzz.run_exact_bounds(lib, msgs.append), msgs)
    _run(k7_fuzz.run_counts(lib, msgs.append), msgs)
