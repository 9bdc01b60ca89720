"""K9 and K10 fuzzed on the CPU emulation: the families of tools/k9_fuzz.py on build/bin/libk9emu.so and libk9emu_nocull.so (culling on and
compiled out), and those of tools/k10_fuzz.py on build/bin/libdgemu.so (the forward) and libk10emu.so (the VJP and its sort), against the
numpy restatements, with smaller budgets than tests/test_gpu_mesh_raycast_grad_fuzz.py.  The refits need K8 and run in the rehearsal of the
device file (tests/test_mesh_raycast_grad_fuzz_rehearsal.py)."""
import os
import sys

import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import k9_fuzz  # noqa: E402
import k10_fuzz  # noqa: E402

BIN = os.path.join(ROOT, "build", "bin")


def _need(*names):
    for nm in names:
        if not os.path.exists(os.path.join(BIN, nm)):
            pytest.skip(f"build/bin/{nm} not built (make cpp)")


@pytest.fixture(scope="module", params=["libk9emu.so", "libk9emu_nocull.so"])
def k9(request):
    _need(request.param)
    return k9_fuzz.EmuK9(os.path.join(BIN, request.param))


@pytest.fixture(scope="module")
def k10():
    _need("libdgemu.so", "libk10emu.so")
    return k10_fuzz.EmuK10()


def _run(result, msgs):
    cases, total, bad = result
    assert bad == 0 and total > 0, "\n".join(msgs[:10])


def test_k9_trees_ties_and_slack(k9):
    """tree sizes around powers of two; tie-rich meshes with shuffled ids, duplicates, zero-area triangles, the flat grid cast from its
    plane; the meshes whose fp32 box lies inside a vertex by less than the culling slack"""
    msgs = []
    _run(k9_fuzz.run_cases(k9, k9_fuzz.tree_cases(0, k9_fuzz.k5_fuzz.TREE_SIZES[::2], n=40), log=msgs.append), msgs)
    _run(k9_fuzz.run_cases(k9, k9_fuzz.tie_cases(7, 0, n=60), log=msgs.append), msgs)
    _run(k9_fuzz.run_cases(k9, k9_fuzz.slack_cases(), log=msgs.append), msgs)


def test_k9_scales_with_hits(k9):
    """10^-45 .. 10^-38, a stride of 10^-24 .. 10^17, 10^+-100, 10^+-150: the restatement hits in every case but 10^150 with unit
    directions"""
    msgs, hits = [], []
    exps = tuple(range(-45, -37)) + tuple(range(-24, 18, 5)) + (-150, -100, 100, 150)
    _run(k9_fuzz.run_cases(k9, k9_fuzz.scale_cases(0, exps, n=24), log=msgs.append, hits=hits), msgs)
    dry = [label for label, h in hits if h == 0 and not ("1e150 " in label and "unit" in label)]
    assert not dry, f"no hits at all: {dry[:5]}"


def test_k9_cull_switch_nonfinite_bounds_counts(k9):
    msgs = []
    _run(k9_fuzz.run_cases(k9, k9_fuzz.cull_cases(0), log=msgs.append), msgs)
    _run(k9_fuzz.run_cases(k9, k9_fuzz.nonfinite_cases(0, n=20), log=msgs.append), msgs)
    _run(k9_fuzz.run_cases(k9, k9_fuzz.bound_cases(0, n=40), log=msgs.append), msgs)
    _run(k9_fuzz.run_exact_bounds(k9, 0, msgs.append, n=30), msgs)
    _run(k9_fuzz.run_counts(k9, 0, msgs.append), msgs)


def test_k10_forward(k10):
    msgs = []
    _run(k10_fuzz.run_forward(k10, 14, 0, msgs.append, scale_exponents=(-24, -12, -3, 0, 4, 11, 17)), msgs)


def test_k10_vjp_sort_boundaries(k10):
    """T = 1 .. 65537 (1, 2, 3 passes), every id pattern, counts around the tile and scan-chunk sizes (a rotating subset per mesh)"""
    msgs = []
    _run(k10_fuzz.run_vjp(k10, 0, msgs.append, per_mesh=8), msgs)


def test_k10_vjp_segments_fan_values(k10):
    msgs = []
    _run(k10_fuzz.run_segments(k10, 0, msgs.append), msgs)
    _run(k10_fuzz.run_values(k10, 0, msgs.append), msgs)
