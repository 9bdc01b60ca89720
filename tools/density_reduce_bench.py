#!/usr/bin/env python
"""Reduced density map: the one-call route (CubicLagrangeDiscreteGrid.addReducedDensityMap -> dg_reduced_density_map_create) against the
two-step route (addFunction(DensityMapFunction) -> dg_density_map, then reduceField(0, p0) and reduceField(1, p1) -> node positions, keep
flags in numpy, dg_reduce_field), with GenerateDensityMap's predicates, rho0 = 1000 and h = `--h-cells` cell diagonals of the SDF's grid.

The SDFs are made first, by GenerateSDF on the GPU, into a temporary directory.  Every run is a fresh subprocess, so that its peak host RSS
(getrusage ru_maxrss) belongs to one route: it loads the SDF, runs the route once on a 32^3 SDF (module loading), then times the full-size
calls with a host clock (the calls are synchronous; loading the file is not timed).  Routes alternate, repeat after repeat; the medians are
reported, with the per-stage timings_ms of the last one-call run, the survivor counts and SHA-256 digests of both output fields.
GenerateDensityMap (which takes the one-call route) is timed start to exit on the same SDFs, with its peak RSS.  The card's name and power
limit are read in the same run with a query-only nvidia-smi.  Prints one JSON line; writes nothing outside the temporary directory.

Workloads: the reference's bunny.obj at 128^3 and 256^3 and dragon.obj at 256^3 (oracle/_ref/resources, staged by `make -C oracle ref`).

usage: tools/density_reduce_bench.py [--repeats 3] [--h-cells 1.0] [--cases bunny:128,bunny:256,dragon:256]"""
import argparse
import hashlib
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BIN = os.path.join(ROOT, "build", "bin")
RHO0 = 1000.0
STAGES = ("upload_pack", "density", "f0_cells", "f0_nodes", "f0_sort", "f0_write", "f1_cells", "f1_nodes", "f1_sort", "f1_write")


def h_of(sdf, h_cells):
    c = sdf.cellSize()
    return h_cells * float(np.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]))


def run_route(dg, route, path, h_cells):
    """(grid, h, ms of the route, ms per step: loading the file, then the route's calls)"""
    t0 = time.perf_counter()
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    steps = {"load": (time.perf_counter() - t0) * 1e3}
    h = h_of(sdf, h_cells)
    c = sdf.cellSize()
    diag = float(np.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]))
    t0 = time.perf_counter()
    t = t0

    def step(key):
        nonlocal t
        now = time.perf_counter()
        steps[key] = (now - t) * 1e3
        t = now
    if route == "new":
        sdf.addReducedDensityMap(dg.DensityMapFunction(0, h, RHO0))
        step("addReducedDensityMap")
    else:
        sdf.addFunction(dg.DensityMapFunction(0, h, RHO0))          # dg_field_create (upload + host checks of the rows), K3, cell table
        step("addFunction")
        sdf.reduceField(0, lambda x, v: (-6.0 * h < v + diag) & (v - diag < 2.0 * h))
        step("reduceField0")
        sdf.reduceField(1, lambda x, v: (0.0 <= v) & (v <= 3.0 * RHO0))
        step("reduceField1")
    return sdf, h, (time.perf_counter() - t0) * 1e3, steps


def child(route, path, warm, h_cells):
    import discregrid_b200 as dg
    run_route(dg, route, warm, h_cells)
    sdf, h, ms, steps = run_route(dg, route, path, h_cells)
    digest = hashlib.sha256()
    for f in range(2):
        for a in (sdf.m_nodes[f], sdf.m_cells[f], sdf.m_cell_map[f]):
            digest.update(np.ascontiguousarray(a).tobytes())
    out = {"ms": ms, "peak_rss_bytes": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024, "h": h, "n_nodes_grid": sdf.nNodes(),
           "n_cells_grid": sdf.nCells(), "sdf_nodes_kept": len(sdf.m_nodes[0]), "sdf_cells_kept": len(sdf.m_cells[0]),
           "density_nodes_kept": len(sdf.m_nodes[1]), "density_cells_kept": len(sdf.m_cells[1]), "sha256": digest.hexdigest(), "step_ms": steps}
    if route == "new":
        t = [float(v) for v in sdf.last_reduced_density_ms]
        out["stage_ms"] = dict(zip(STAGES + ("total",), t[:10] + [t[12]]))
        out["tie_path"] = [bool(t[10]), bool(t[11])]
    print(json.dumps(out))


def timed_tool(args):
    """wall time start to exit and peak RSS of one tool run (a fresh probe process, so RUSAGE_CHILDREN is that run alone)"""
    probe = ("import resource, subprocess, sys, time; t = time.perf_counter(); r = subprocess.run(sys.argv[1:], capture_output=True); "
             "print(r.returncode, (time.perf_counter() - t) * 1e3, resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss * 1024)")
    p = subprocess.run([sys.executable, "-c", probe] + args, capture_output=True, text=True, check=True)
    rc, ms, rss = p.stdout.split()
    if int(rc) != 0:
        raise SystemExit(f"{args} failed with {rc}")
    return float(ms), int(rss)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--h-cells", type=float, default=1.0, help="smoothing length in cell diagonals")
    ap.add_argument("--cases", default="bunny:128,bunny:256,dragon:256")
    ap.add_argument("--child", nargs=3, metavar=("ROUTE", "SDF", "WARM"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child[0], args.child[1], args.child[2], args.h_cells)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    card, power = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    result = {"metric": "reduced density map: one call vs addFunction(DensityMapFunction) + reduceField x 2 (host clock, synchronous, fresh "
                        "process per run); GenerateDensityMap start to exit", "gpu": card, "power_limit": power, "h_cell_diagonals": args.h_cells,
              "rho0": RHO0, "cases": []}
    with tempfile.TemporaryDirectory() as tmp:
        def make_sdf(name, res):
            mesh = os.path.join(ROOT, "oracle", "_ref", "resources", name + ".obj")
            if not os.path.exists(mesh):
                raise SystemExit(f"{mesh} is not staged (make -C oracle ref)")
            out = os.path.join(tmp, f"{name}_{res}.cdf")
            if not os.path.exists(out):
                subprocess.run([os.path.join(BIN, "GenerateSDF"), "-r", f"{res} {res} {res}", "-o", out]
                               + (["-i"] if name == "dragon" else []) + [mesh], capture_output=True, check=True)
            return out
        for case in args.cases.split(","):
            name, res = case.split(":")
            res = int(res)
            path, warm = make_sdf(name, res), make_sdf(name, 32)
            runs = {"new": [], "old": []}
            tool = []
            for _ in range(args.repeats):
                for r in runs:
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--h-cells", str(args.h_cells), "--child", r, path, warm],
                                       capture_output=True, text=True)
                    if p.returncode != 0:
                        raise SystemExit(f"{r} {name} {res}^3 failed:\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
                    runs[r].append(json.loads(p.stdout.strip().splitlines()[-1]))
                h = runs["new"][-1]["h"]
                tool.append(timed_tool([os.path.join(BIN, "GenerateDensityMap"), "-s", repr(h), "-r", repr(RHO0), "-o",
                                        os.path.join(tmp, "out.cdm"), path]))
            entry = {"mesh": name, "resolution": res}
            for r, rs in runs.items():
                entry[r] = {"ms_median": float(np.median([x["ms"] for x in rs])), "ms": [x["ms"] for x in rs],
                            "peak_rss_bytes": max(x["peak_rss_bytes"] for x in rs)}
            for r, rs in runs.items():
                entry[r]["step_ms_last"] = rs[-1]["step_ms"]
            entry["new"]["stage_ms_last"] = runs["new"][-1]["stage_ms"]
            entry["tie_path"] = runs["new"][-1]["tie_path"]
            first = runs["new"][0]
            entry.update({k: first[k] for k in ("h", "n_nodes_grid", "n_cells_grid", "sdf_nodes_kept", "sdf_cells_kept", "density_nodes_kept",
                                                "density_cells_kept")})
            digests = {x["sha256"] for r in runs for x in runs[r]}
            entry["outputs_bit_identical"] = len(digests) == 1
            entry["sha256"] = sorted(digests)
            entry["speedup_median"] = entry["old"]["ms_median"] / entry["new"]["ms_median"]
            entry["generate_density_map"] = {"ms_median": float(np.median([t[0] for t in tool])), "ms": [t[0] for t in tool],
                                             "peak_rss_bytes": max(t[1] for t in tool)}
            result["cases"].append(entry)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
