"""K1 on the device across mesh scales.  The fp32 filters (sphere interval, box skip, leaf_lower_bound) may only drop or order work where the
fp64 answer is certain; their error budget holds for 2^-40 <= Mq < 1e18 and they are off outside it.  The CPU emulation of the kernels
(tests/test_k1_emulated.py) does not reproduce every detail of the device's fp32 arithmetic (the 2-ulp errors of sqrt.approx and
__fdividef), so the scale sweep, a short tie-rich fuzz run in both modes and the awkward meshes run here too: the product library through
its C-ABI (tools/k1_fuzz.py, backend `dg`: dg_mesh_create, dg_mesh_distance, dg_node_positions, dg_sample_sdf) against the reference's own
TriangleMeshDistance.h where build() compiled it (oracle/_ref), else against the oracle port pinned to it.  Bar: bit-exact."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import k1_fuzz  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be(dg):
    return k1_fuzz.DgK1()


@pytest.mark.parametrize("mode", ["points", "grid"])
def test_scale_sweep_on_device(be, mode):
    """soups, strips and coplanar grids at 10^k, k = -24 .. 17, centred and offset, plus soups at the 1e18 limit: arbitrary points (signed +
    unsigned: distance bits, nearest point, entity, triangle id) or the node loop on a (9, 7, 6) lattice == the reference, bit for bit"""
    msgs = []
    meshes, checked, bad = k1_fuzz.run_scales(be, seed=0, modes=(mode,), log=msgs.append)
    assert meshes == 2 * 3 * len(k1_fuzz.SCALE_EXPONENTS) + 2 and checked > 100000
    assert bad == 0, f"{bad} mismatches: " + "\n".join(msgs[:8])


@pytest.mark.parametrize("mode", ["points", "grid"])
def test_tie_rich_fuzz_on_device(mode, capsys, dg):
    """tools/k1_fuzz.py on the device: coplanar grids, cubes / octahedra on half-integer lattices, duplicated triangles, slivers, random
    soups at scales 1e-24 .. 1e17"""
    rc = k1_fuzz.main(["k1_fuzz", "42", "7", "dg", mode])
    out = capsys.readouterr().out
    assert rc == 0 and "0 mismatches" in out, out[-3000:]


@pytest.mark.parametrize("n_tri,scale,offset,degenerate", k1_fuzz.AWKWARD)
def test_awkward_meshes_on_device(be, n_tri, scale, offset, degenerate):
    """the corner cases of test_k1_emulated.py on the device: one- and two-triangle meshes, tiny and huge coordinates, far and non-finite
    queries, degenerate triangles -- same distance bits (NaN for NaN), nearest point, entity and triangle; DBL_MAX / -1 where the
    reference accepts no triangle"""
    V, F, x, lost = k1_fuzz.awkward_case(n_tri, scale, offset, degenerate)
    ref = k1_fuzz.reference(V, F)
    h = be.mesh(V, F)
    try:
        n, bad, msg = k1_fuzz.check_points(be, h, ref, x)
        assert bad == 0, msg
        for signed in (1, 0):
            d, _, _, t = be.distance(h, lost, signed, near=False)
            assert (d == np.finfo(np.float64).max).all() and (t == -1).all()
    finally:
        be.destroy(h)
