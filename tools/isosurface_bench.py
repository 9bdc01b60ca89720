#!/usr/bin/env python
"""Level-set extraction (K6, csrc/k6_isosurface.cu) on one GPU.

  dense s=1, s=2 : CubicLagrangeDiscreteGrid.isosurface on the bunny.obj 256^3 dense SDF, iso = 0.
  band s=1       : the 512^3 reduced narrow band of 2 cell diagonals (addReducedBandField), extracted from the device field built from the
                   kept handle (no host round trip).
  K2 rate        : value-only interpolate on CUDA tensors of as many uniform points as the dense s=1 lattice has, timed with CUDA events.
Cases are alternated and run `--runs` times; medians of the host clock around the call (which ends with a device synchronise) and of the
per-stage times (timings_ms: values, classify, scans, emit, total).  Device memory is computed from the shapes (DESIGN section 4), not
measured.  The HBM share counts algorithmic bytes only -- each kept cell's 256-byte block read once, the values written once and read by
classify and emit, the edge flags written, scanned and read, the counts, and the output -- over the 3.35 TB/s data sheet.  The card's name,
power limit and max SM clock are read in the same run.  Needs oracle/_ref/resources (make -C oracle ref).

usage: python tools/isosurface_bench.py [--runs 5] [--out result.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def lattice(g, s):
    n = [s * int(r) + 1 for r in g.resolution()]
    return int(np.prod(n)), int(np.prod([k - 1 for k in n]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    import winding_ref as wr
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    obj = os.path.join(ROOT, "oracle", "_ref", "resources", "bunny.obj")
    if not os.path.exists(obj):
        raise SystemExit(f"{obj} is not staged (make -C oracle ref)")
    result = {"card": card(), "runs": a.runs}
    print("card:", result["card"], flush=True)
    dg.selftest()
    V, F = wr.read_obj(obj)
    md = dg.TriangleMeshDistance(V, F)
    mn, mx = dg.generate_sdf_domain(V)
    dense = dg.CubicLagrangeDiscreteGrid(mn, mx, (256, 256, 256))
    dense.addFunction(dg.MeshSignedDistance(md))
    band = dg.CubicLagrangeDiscreteGrid(mn, mx, (512, 512, 512))
    band.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, 2.0 * float(np.linalg.norm(band.cellSize()))))
    kept_cells = len(band.m_cells[0])
    cases = {"dense256_s1": (dense, 1, 256 ** 3), "dense256_s2": (dense, 2, 256 ** 3), "band512_s1": (band, 1, kept_cells)}
    for g, s, _ in cases.values():                     # device fields (the band's from its kept handle) and a warm-up
        g.isosurface(0, 0.0, s)
    wall = {k: [] for k in cases}
    stages = {k: [] for k in cases}
    sizes = {}
    for _ in range(a.runs):
        for k, (g, s, _) in cases.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            Vx, T = g.isosurface(0, 0.0, s)
            wall[k].append((time.perf_counter() - t0) * 1e3)
            stages[k].append(g.last_isosurface_ms.copy())
            sizes[k] = (len(Vx), len(T))
    # K2 value-only on as many uniform points as the dense s=1 lattice
    n_q = lattice(dense, 1)[0]
    gen = torch.Generator(device="cuda").manual_seed(0)
    lo, hi = torch.tensor(mn, device="cuda"), torch.tensor(mx, device="cuda")
    xq = lo + torch.rand((n_q, 3), dtype=torch.float64, device="cuda", generator=gen) * (hi - lo)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    k2 = []
    dense.interpolate(0, xq)
    for _ in range(a.runs):
        e0.record(); dense.interpolate(0, xq); e1.record(); torch.cuda.synchronize()
        k2.append(e0.elapsed_time(e1))
    k2_ms = statistics.median(k2)
    result["k2_value_only"] = {"queries": n_q, "ms": k2_ms, "gq_per_s": n_q / k2_ms / 1e6}
    print(f"K2 value-only, {n_q} uniform queries: {k2_ms:.2f} ms = {n_q / k2_ms / 1e6:.2f} Gq/s", flush=True)
    for k, (g, s, cells_read) in cases.items():
        npts, ncells = lattice(g, s)
        st = np.median(np.array(stages[k]), axis=0)
        nv, nt = sizes[k]
        mem = 8 * npts + 7 * npts + ncells + (7 * npts + 31) // 32 * 4 + 24 * min(npts, 1 << 24) + 24 * nv + 12 * nt
        algo = (256 * cells_read + 8 * npts * 3 + 7 * npts * 3 + ncells * 2 + 24 * nv + 12 * nt)
        r = {"lattice_points": npts, "vertices": nv, "triangles": nt, "wall_ms": statistics.median(wall[k]),
             "stages_ms": dict(zip(["values", "classify", "scans", "emit", "total"], st.round(3).tolist())),
             "lattice_points_per_s": npts / (st[4] * 1e-3), "values_pass_gq_per_s": npts / st[0] / 1e6,
             "device_bytes_computed": mem, "algorithmic_bytes": algo, "hbm_share": algo / (st[4] * 1e-3) / HBM}
        result[k] = r
        print(f"{k}: {npts} lattice points, {nv} vertices, {nt} triangles; median {r['wall_ms']:.1f} ms wall; stages {r['stages_ms']}; "
              f"{r['lattice_points_per_s'] / 1e9:.3f} G lattice points/s; values pass {r['values_pass_gq_per_s']:.2f} Gq/s "
              f"(K2 value-only {result['k2_value_only']['gq_per_s']:.2f}); device memory {mem / 1e9:.2f} GB computed; "
              f"HBM share {100 * r['hbm_share']:.1f} %", flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
