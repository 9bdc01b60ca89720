"""tests/test_gpu_isosurface_raycast_fuzz.py rehearsed on the CPU: the K6 and K7 device fuzz tests run against build/bin/libdgemu.so -- the
whole library with every kernel emulated (tests/emu) -- so that their Python- and tool-level logic (the `dg` backends of tools/k6_fuzz.py
and tools/k7_fuzz.py, dg_isosurface_copy_device, dg_field_raycast_device) is checked without a GPU, on the smaller budgets the file takes
on the emulated library.  The large lattice and the 2^20-ray calls are left to the GPU."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")


def test_gpu_isosurface_raycast_fuzz_tests_pass_on_the_emulated_library():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    env = dict(os.environ, DISCREGRID_B200_LIB=EMU, LD_PRELOAD=EMU, DG_ALLOW_EMULATED_LIBRARY="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-k", "not large", "-p", "no:cacheprovider",
                        "tests/test_gpu_isosurface_raycast_fuzz.py"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
