"""tests/test_gpu_device_function.py rehearsed on the CPU: the device-function GPU tests (Python types with torch callbacks, the C-ABI, the
fixtures, a callback that calls the library) run against build/bin/libdgemu.so -- the whole library with every kernel emulated (tests/emu),
where the callbacks get CPU tensors over the same memory -- so that their Python-level logic is checked without a GPU.  The full-size runs
and the C++ facade binary (which moves data with the real CUDA runtime) are left to the GPU."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")


def test_gpu_device_function_tests_pass_on_the_emulated_library():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    env = dict(os.environ, DISCREGRID_B200_LIB=EMU, LD_PRELOAD=EMU, DG_ALLOW_EMULATED_LIBRARY="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-k", "not full_size and not cpp_facade", "-p", "no:cacheprovider",
                        "tests/test_gpu_device_function.py"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
