"""tests/test_gpu_vjp_fuzz.py rehearsed on the CPU: the K11 and K12 device fuzz tests run against build/bin/libdgemu.so -- the whole library
with every kernel emulated (tests/emu) -- so that their Python- and tool-level logic (the `dg` backends of tools/k11_fuzz.py and
tools/k12_fuzz.py, the device forms, set_nodes_device, the trainable copies of k7_fuzz's fields) is checked without a GPU, on the smaller
budgets the file takes on the emulated library.  The 2^20 + 1-query cell, the stride families, the 256^3 fields and the side stream are left
to the GPU (the device forms run on the default stream with host memory)."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "build", "bin", "libdgemu.so")


def test_gpu_vjp_fuzz_tests_pass_on_the_emulated_library():
    if not os.path.exists(EMU):
        pytest.skip("build/bin/libdgemu.so not built (make cpp)")
    env = dict(os.environ, DISCREGRID_B200_LIB=EMU, LD_PRELOAD=EMU, DG_ALLOW_EMULATED_LIBRARY="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-k", "not large", "-p", "no:cacheprovider",
                        "tests/test_gpu_vjp_fuzz.py"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail
