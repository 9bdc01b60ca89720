"""Volume-map fixtures from the reference-side generator (oracle/_ref/bin/RefGenerateVolumeMap, built by oracle/ref_volume.mk from
oracle/ref_volume_map.cpp and the reference's own sources): the volume map's contract as lambdas over the reference's
CubicLagrangeDiscreteGrid, GaussQuadrature::integrate and CubicKernel, then reduceField(0, p0) and reduceField(1, 0 <= v) unless
--no-reduction.  It runs on SDF fixtures that are already committed here; h is a number of cell diagonals of each SDF's grid.
Writes ref_volume_*.cdm and ref_volume_cases.json next to this file.

usage: python tests/golden/make_volume_golden.py      (needs oracle/_ref, i.e. `make cpp` with the reference sources present)"""
import json
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
TOOL = os.path.join(ROOT, "oracle", "_ref", "bin", "RefGenerateVolumeMap")

# name -> SDF fixture, h in cell diagonals, scale, --no-reduction
CASES = {
    # h small enough that both reductions drop nodes (at one cell diagonal every node of these 12^3 / 10^3 grids is kept)
    "bunny_12": dict(sdf="ref_bunny_12.cdf", h_diag=0.3, scale=0.8, no_reduction=False),
    "dragon_10_inverted": dict(sdf="ref_dragon_10_inverted.cdf", h_diag=0.05, scale=1.0, no_reduction=False),
    "dragon_10_inverted_dense": dict(sdf="ref_dragon_10_inverted.cdf", h_diag=2.5, scale=0.8, no_reduction=True),
    # dense band field: DBL_MAX wherever the distance exceeds the band, so the predicate, gamma and both reductions meet the sentinel
    "band_dragon_12_inverted": dict(sdf="ref_band_dragon_12_inverted.cdf", h_diag=0.5, scale=0.8, no_reduction=False),
    "band_dragon_12_inverted_dense": dict(sdf="ref_band_dragon_12_inverted.cdf", h_diag=0.5, scale=0.8, no_reduction=True),
    # the anisotropic grid whose SDF survivors share Z-curve keys (the tie order of reduceField's std::sort)
    "aniso": dict(sdf="ref_aniso_field.cdf", h_diag=0.5, scale=0.8, no_reduction=False),
    "aniso_dense": dict(sdf="ref_aniso_field.cdf", h_diag=0.5, scale=0.8, no_reduction=True),
}


def read_cdf(path):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_oracle_golden import read_cdf as read
    return read(path)


def h_of(path, h_diag):
    cell = np.asarray(read_cdf(path)["cell"], np.float64)
    return float(h_diag * np.sqrt((cell[0] * cell[0] + cell[1] * cell[1]) + cell[2] * cell[2]))


def main():
    meta = {}
    for name, case in CASES.items():
        src = os.path.join(HERE, case["sdf"])
        h = h_of(src, case["h_diag"])
        out = os.path.join(HERE, f"ref_volume_{name}.cdm")
        cmd = [TOOL, "-s", repr(h), "--scale", repr(case["scale"]), "-o", out] + (["--no-reduction"] if case["no_reduction"] else []) + [src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit(f"{name}: {r.stdout}\n{r.stderr}")
        meta[name] = dict(case, h=h, h_hex=float.hex(h), file=os.path.basename(out))
        print(name, out, os.path.getsize(out), "bytes, h", h)
        if not case["no_reduction"]:                  # a reduced fixture must exercise both reductions
            g = read_cdf(out)
            n_grid = len(read_cdf(src)["nodes"][0])
            assert len(g["nodes"][0]) < n_grid and len(g["nodes"][1]) < n_grid, f"{name}: a reduction keeps every node at h = {h}"
    with open(os.path.join(HERE, "ref_volume_cases.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
