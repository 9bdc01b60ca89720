"""Reduced density-map fixtures from the reference's own GenerateDensityMap (oracle/_ref/bin/GenerateDensityMap, built by oracle/Makefile):
the tool runs with its default reduction (addFunction(density_func, true) + reduceField(0, p0) + reduceField(1, p1),
cmd/generate_density_map/main.cpp:117-147) on SDF fixtures that are already committed here, and its .cdm output is kept.  h is a number of
cell diagonals of each SDF's grid, rho0 = 1000.  For the anisotropic grid the script checks that the survivors of the SDF field's reduction
share Z-curve keys, so that the fixture pins the order std::sort leaves among equal keys (dg_reduce_field's tie flag, host passes).
Writes ref_density_*.cdm and ref_density_cases.json next to this file.

usage: python tests/golden/make_density_golden.py      (needs oracle/_ref, i.e. `make -C oracle ref` with the reference sources present)"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
TOOL = os.path.join(ROOT, "oracle", "_ref", "bin", "GenerateDensityMap")

# name -> SDF fixture, h in cell diagonals, rest density, whether the SDF field's survivors must share Z-curve keys
CASES = {
    "bunny_12": dict(sdf="ref_bunny_12.cdf", h_diag=1.0, rho0=1000.0, ties=False),
    "dragon_10_inverted": dict(sdf="ref_dragon_10_inverted.cdf", h_diag=0.75, rho0=1000.0, ties=False),
    # dense band field: DBL_MAX wherever the distance exceeds the band, so K3's predicate and both reductions meet the sentinel
    "band_dragon_12_inverted": dict(sdf="ref_band_dragon_12_inverted.cdf", h_diag=0.5, rho0=1000.0, ties=False),
    "aniso": dict(sdf="ref_aniso_field.cdf", h_diag=0.5, rho0=1000.0, ties=True),
    # a sphere SDF with one -DBL_MAX coefficient (made by make_inputs): d / h overflows to -inf near it, gamma = +inf, and the quadrature
    # points outside the kernel support add inf * 0 = NaN -- the reference's density is NaN there
    "minus_dbl_max": dict(sdf="ref_density_minus_dbl_max_sdf.cdf", h_diag=0.35, rho0=1000.0, ties=False),
}


def make_inputs():
    """the SDF inputs that are not made by another script: a sphere SDF on a 4^3 grid over [0, 2]^3 with node 126 (an x-edge node) set to -DBL_MAX"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from oracle_api import Oracle
    from make_reduce_golden import write_cdf
    orc = Oracle()
    gd, r = orc.grid_desc([0.0, 0.0, 0.0], [2.0, 2.0, 2.0], (4, 4, 4))
    cells = orc.build_cells(r)
    x = orc.node_positions(gd, r, 0, int(cells.max()) + 1)
    v = np.linalg.norm(x - np.array([1.0, 0.9, 1.1]), axis=1) - 0.6
    v[126] = -np.finfo(np.float64).max
    write_cdf(os.path.join(HERE, CASES["minus_dbl_max"]["sdf"]), gd[0:3], gd[3:6], r, gd[6:9], gd[9:12], v, cells,
              np.arange(len(cells), dtype=np.uint32))


def read_grid(path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_oracle_golden import read_cdf
    return read_cdf(path)


def h_of(g, h_diag):
    cell = np.asarray(g["cell"], np.float64)
    return float(h_diag * np.sqrt((cell[0] * cell[0] + cell[1] * cell[1]) + cell[2] * cell[2]))


def sdf_field_tie_flag(g, h):
    """dg_reduce_field (every pass on the host) on the SDF field with the tool's first predicate: 1.0 when its survivors share Z-curve keys"""
    sys.path.insert(0, ROOT)
    from discregrid_b200 import _capi as capi
    from discregrid_b200.grid import grid_desc
    d = grid_desc(g["mn"], g["mx"], g["res"], g["cell"], g["inv"])
    nodes = np.ascontiguousarray(g["nodes"][0], np.float64).copy()
    cells = np.ascontiguousarray(g["cells"][0], np.uint32).copy()
    cell = np.asarray(g["cell"], np.float64)
    diag = np.sqrt((cell[0] * cell[0] + cell[1] * cell[1]) + cell[2] * cell[2])
    keep = ((-6.0 * h < nodes + diag) & (nodes - diag < 2.0 * h) & (nodes != np.finfo(np.float64).max)).astype(np.uint8)
    cmap = np.empty(int(np.prod(np.asarray(g["res"], np.uint64))), np.uint32)
    n_out, c_out, tm = C.c_uint64(), C.c_uint64(), np.zeros(5)
    capi.check(capi.lib.dg_reduce_field(C.byref(d), capi.ptr(nodes, capi.F64P), len(nodes), keep.ctypes.data_as(C.POINTER(C.c_uint8)),
                                        capi.ptr(cells, capi.U32P), len(cells), capi.ptr(cmap, capi.U32P), 2, C.byref(n_out), C.byref(c_out),
                                        capi.ptr(tm, capi.F64P)))
    return tm[4]


def main():
    make_inputs()
    meta = {}
    for name, case in CASES.items():
        src = os.path.join(HERE, case["sdf"])
        g = read_grid(src)
        h = h_of(g, case["h_diag"])
        out = os.path.join(HERE, f"ref_density_{name}.cdm")
        r = subprocess.run([TOOL, "-s", repr(h), "-r", repr(case["rho0"]), "-o", out, src], capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit(f"{name}: {r.stdout}\n{r.stderr}")
        if case["ties"]:
            assert sdf_field_tie_flag(g, h) == 1.0, f"{name}: the SDF field's survivors do not share Z-curve keys at h = {h}"
        meta[name] = dict(case, h=h, h_hex=float.hex(h), file=os.path.basename(out))
        print(name, out, os.path.getsize(out), "bytes, h", h)
    with open(os.path.join(HERE, "ref_density_cases.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
