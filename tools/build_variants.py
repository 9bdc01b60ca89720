#!/usr/bin/env python
"""Builds tuning variants of libdiscregrid_b200.so (same sources, different -D knobs) into build/variants/<name>.so.
Usage: python tools/build_variants.py name1:-DK1_PKT_MIN_BLOCKS=12,-DK1_POP_TRIES=2 name2:...   (select one with DISCREGRID_B200_LIB)"""
import glob, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "discregrid_b200", "csrc")
NV = ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin", "/usr/bin/g++", "-std=c++17", "-O3", "-lineinfo",
      "-fmad=false", "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden"]
out_dir = os.path.join(ROOT, "build", "variants"); os.makedirs(out_dir, exist_ok=True)
procs = []
for spec in sys.argv[1:]:
    name, _, defs = spec.partition(":")
    defs = [d for d in defs.split(",") if d]
    srcs = sorted(glob.glob(os.path.join(SRC, "*.cu")) + glob.glob(os.path.join(SRC, "*.cpp")))      # the library's sources
    cmd = NV + defs + ["-shared", "-o", os.path.join(out_dir, name + ".so")] + srcs
    procs.append((name, subprocess.Popen(cmd)))
for name, p in procs:
    assert p.wait() == 0, name
    print("built", name)
