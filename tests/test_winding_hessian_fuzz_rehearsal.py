"""tests/test_gpu_winding_hessian_fuzz.py rehearsed on the CPU: the K5 and K2-Hessian device fuzz tests run against build/bin/libdgemu.so --
the whole library with every kernel emulated (tests/emu) -- so that their Python- and tool-level logic (the `dg` backends of tools/k5_fuzz.py
and tools/k2_fuzz.py, the winding sign mode checks) is checked without a GPU.  The CUDA-tensor tests and the 2^20-point and 4 M-query runs
are left to the GPU."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")


def test_gpu_winding_hessian_fuzz_tests_pass_on_the_emulated_library():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    env = dict(os.environ, DISCREGRID_B200_LIB=EMU, LD_PRELOAD=EMU, DG_ALLOW_EMULATED_LIBRARY="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-k", "not tensor and not many", "-p", "no:cacheprovider",
                        "tests/test_gpu_winding_hessian_fuzz.py"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
