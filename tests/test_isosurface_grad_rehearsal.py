"""tests/test_gpu_isosurface_grad.py rehearsed on the CPU: the device tests of K13 run against build/bin/libdgemu.so -- the whole library with
every kernel emulated (tests/emu), where torch tensors take the device route as CPU tensors over the same memory -- so that their
Python-level logic (both C-ABI forms, the autograd Function, the token of the trainable field, the refusals) is checked without a GPU.  The
tensor route on CUDA streams, the Adam fit, the bunny, the large lattice and the C++ check are left to the GPU."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")


def test_gpu_isosurface_grad_tests_pass_on_the_emulated_library():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    env = dict(os.environ, DISCREGRID_B200_LIB=EMU, LD_PRELOAD=EMU, DG_ALLOW_EMULATED_LIBRARY="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-k", "not tensor and not bunny and not large and not cpp",
                        "-p", "no:cacheprovider", "tests/test_gpu_isosurface_grad.py"], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1500)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
