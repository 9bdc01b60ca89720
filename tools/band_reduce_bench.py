#!/usr/bin/env python
"""Reduced narrow band: the one-call route (CubicLagrangeDiscreteGrid.addReducedBandField -> dg_reduced_band_create) against the two-step
route (addFunction(MeshSignedDistance, pred=MeshDistanceBand) -> dg_add_function_sdf_band, then reduceField(always true) -> node positions,
keep flags, dg_reduce_field), with w = `--cells` cell diagonals.

Every run is a fresh subprocess, so that its peak host RSS (getrusage ru_maxrss) belongs to one route: it first runs the route once on a
32^3 grid (module loading), then times the full-size call with a host clock (the call is synchronous).  Routes alternate, repeat after
repeat; the medians are reported.  The two-step route is skipped, and the skip reported, when MemAvailable is below an estimate of its host
allocations.  Where both routes ran, their outputs (nodes, cells, cell map) are compared through SHA-256 digests of the raw bytes.  The
card's name and power limit are read in the same run with a query-only nvidia-smi.  Prints one JSON line; writes nothing.

Workloads: the reference's bunny.obj (oracle/_ref/resources, staged by `make -C oracle ref`) at 256^3 and 512^3, and the 100,000-triangle
bumpy torus at 256^3.

usage: tools/band_reduce_bench.py [--repeats 3] [--cells 2.0] [--cases bunny:256,bunny:512,torus:256]"""
import argparse
import hashlib
import json
import os
import resource
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load(dg, name):
    if name == "torus":
        return dg.bumpy_torus()                                  # 250 x 200 quads = 100,000 triangles
    p = os.path.join(ROOT, "oracle", "_ref", "resources", name + ".obj")
    if not os.path.exists(p):
        raise SystemExit(f"{p} is not staged (make -C oracle ref)")
    return dg.TriangleMesh(p)


def child(route, name, res, cells):
    import discregrid_b200 as dg
    mesh = load(dg, name)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)

    def run(r):
        sdf = dg.CubicLagrangeDiscreteGrid(mn, mx, [r, r, r])
        cell = sdf.cellSize()
        w = cells * float(np.sqrt((cell * cell).sum()))
        t0 = time.perf_counter()
        if route == "new":
            sdf.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, w))
        else:
            sdf.addFunction(dg.MeshSignedDistance(md), False, dg.MeshDistanceBand(md, w))
            sdf.reduceField(0, lambda x, v: np.ones(len(v), bool))
        return sdf, w, (time.perf_counter() - t0) * 1e3

    run(32)
    sdf, w, ms = run(res)
    digest = hashlib.sha256()
    for a in (sdf.m_nodes[0], sdf.m_cells[0], sdf.m_cell_map[0]):
        digest.update(np.ascontiguousarray(a).tobytes())
    out = {"ms": ms, "peak_rss_bytes": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024, "band": w, "n_nodes_grid": sdf.nNodes(),
           "n_nodes_kept": len(sdf.m_nodes[0]), "n_cells_kept": len(sdf.m_cells[0]), "n_cells_grid": sdf.nCells(), "sha256": digest.hexdigest()}
    if route == "new":
        out["tie_path"] = bool(sdf.last_reduced_band_ms[5])
        out["stage_ms"] = dict(zip(("sample", "cells", "nodes", "sort", "write", "total"), [float(v) for v in np.delete(sdf.last_reduced_band_ms, 5)]))
    print(json.dumps(out))


def mem_available():
    with open("/proc/meminfo") as fh:
        for line in fh:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def old_route_bytes(res):
    """host allocations of the two-step route: dense nodes, cells and cell map; node positions; reduceField's copies of nodes and cells,
    keep flags and their temporaries; dg_reduce_field's marks, swap-walk permutation and new ids"""
    n = (res + 1) ** 3 + 6 * res * (res + 1) ** 2
    nc = res ** 3
    return n * (8 + 24 + 8 + 4 + 1 + 4 + 4) + nc * (2 * 128 + 4 + 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cells", type=float, default=2.0, help="band width in cell diagonals")
    ap.add_argument("--cases", default="bunny:256,bunny:512,torus:256")
    ap.add_argument("--child", nargs=3, metavar=("ROUTE", "MESH", "RES"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child[0], args.child[1], int(args.child[2]), args.cells)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    card, power = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    result = {"metric": "reduced narrow band: one call vs addFunction(band) + reduceField (host clock, synchronous, fresh process per run)",
              "gpu": card, "power_limit": power, "band_cell_diagonals": args.cells, "cases": []}
    for case in args.cases.split(","):
        name, res = case.split(":")
        res = int(res)
        need, avail = old_route_bytes(res), mem_available()
        routes = ["new", "old"] if avail >= need else ["new"]
        runs = {r: [] for r in routes}
        for _ in range(args.repeats):
            for r in routes:
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--cells", str(args.cells), "--child", r, name, str(res)],
                                   capture_output=True, text=True)
                if p.returncode != 0:
                    raise SystemExit(f"{r} {name} {res}^3 failed:\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
                runs[r].append(json.loads(p.stdout.strip().splitlines()[-1]))
        entry = {"mesh": name, "resolution": res}
        for r, rs in runs.items():
            entry[r] = {"ms_median": float(np.median([x["ms"] for x in rs])), "ms": [x["ms"] for x in rs],
                        "peak_rss_bytes": max(x["peak_rss_bytes"] for x in rs)}
            if r == "new":
                entry[r]["stage_ms_last"] = rs[-1]["stage_ms"]
                entry["tie_path"] = rs[-1]["tie_path"]
        first = runs["new"][0]
        entry.update({k: first[k] for k in ("band", "n_nodes_grid", "n_nodes_kept", "n_cells_grid", "n_cells_kept")})
        if "old" in runs:
            digests = {x["sha256"] for r in runs for x in runs[r]}
            entry["outputs_bit_identical"] = len(digests) == 1
            entry["speedup_median"] = entry["old"]["ms_median"] / entry["new"]["ms_median"]
        else:
            entry["old"] = f"skipped: MemAvailable {avail / 2**30:.1f} GiB < {need / 2**30:.1f} GiB estimated for the two-step route"
        result["cases"].append(entry)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
