#!/usr/bin/env python
"""Volume map (K3's volume-map kernel) against K3's density map, and the one-call reduced volume map against its two-step route.

1. Kernels: dg_volume_map_device and dg_density_map_device (sample predicate on, as the tools run them) alternate on the same device field
   and into the same CUDA tensor, h = `--h-cells` cell diagonals of the SDF's grid, scale 0.8, rho0 = 1000.  Each call is timed with CUDA
   events after a warm-up call; medians over `--repeats` pairs are reported, with the share of nodes that take the 16^3 branch.
2. Reduced route: CubicLagrangeDiscreteGrid.addReducedVolumeMap (dg_reduced_volume_map_create) against addFunction(VolumeMapFunction) +
   reduceField(0, p0) + reduceField(1, 0 <= v), each in a fresh process (host clock around synchronous calls, after a 32^3 warm-up run;
   peak RSS from getrusage), alternating.  These children are started before this process imports torch or the library or loads a grid,
   so that their peak RSS is their own (ru_maxrss carries the parent's high-water mark across fork + exec).  SHA-256 digests of both output fields show that the routes agree.

The SDFs are the reference's bunny.obj at 128^3 and 256^3 (oracle/_ref/resources), made by GenerateSDF on the GPU into a temporary
directory.  The card's name, power limit and max SM clock are read in the same run with a query-only nvidia-smi.  Prints one JSON line;
writes nothing outside the temporary directory.

usage: tools/volume_map_bench.py [--repeats 5] [--h-cells 1.0] [--res 128,256]"""
import argparse
import ctypes as C
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
SCALE, RHO0 = 0.8, 1000.0


def h_of(sdf, h_cells):
    c = sdf.cellSize()
    return h_cells * float(np.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]))


def kernels(dg, path, h_cells, repeats):
    import torch
    from discregrid_b200 import _capi as capi
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    h = h_of(sdf, h_cells)
    f = sdf._device_field(0)
    n = sdf.nNodes()
    out = torch.empty(n, dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream()
    calls = {"volume": lambda: capi.lib.dg_volume_map_device(f, h, SCALE, 0, 0, n, C.c_void_p(out.data_ptr()), C.c_void_p(stream.cuda_stream)),
             "density": lambda: capi.lib.dg_density_map_device(f, h, RHO0, 0, 0, n, C.c_void_p(out.data_ptr()), C.c_void_p(stream.cuda_stream))}
    ms = {k: [] for k in calls}
    branch = {}
    for k, call in calls.items():                     # warm-up, and the share of nodes that integrate (neither DBL_MAX nor beyond 2h)
        capi.check(call())
        torch.cuda.synchronize()
        v = out.cpu().numpy()
        branch[k] = float(((v != np.finfo(np.float64).max) & (v != 0.0)).mean())
    for _ in range(repeats):
        for k, call in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            capi.check(call())
            b.record(stream)
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    entry = {"n_nodes": n, "h": h}
    for k in calls:
        entry[k] = {"ms_median": float(np.median(ms[k])), "ms": ms[k], "nodes_integrated_share": branch[k]}
    entry["volume_over_density"] = entry["volume"]["ms_median"] / entry["density"]["ms_median"]
    return entry


def run_route(dg, route, path, h_cells):
    t0 = time.perf_counter()
    sdf = dg.CubicLagrangeDiscreteGrid(path)
    load = (time.perf_counter() - t0) * 1e3
    h = h_of(sdf, h_cells)
    c = sdf.cellSize()
    diag = float(np.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]))
    t0 = time.perf_counter()
    if route == "new":
        sdf.addReducedVolumeMap(dg.VolumeMapFunction(0, h, SCALE))
    else:
        sdf.addFunction(dg.VolumeMapFunction(0, h, SCALE))
        sdf.reduceField(0, lambda x, v: (-6.0 * h < v + diag) & (v - diag < 2.0 * h))
        sdf.reduceField(1, lambda x, v: 0.0 <= v)
    return sdf, (time.perf_counter() - t0) * 1e3, load


def child(route, path, warm, h_cells):
    import discregrid_b200 as dg
    run_route(dg, route, warm, h_cells)
    sdf, ms, load = run_route(dg, route, path, h_cells)
    digest = hashlib.sha256()
    for f in range(2):
        for a in (sdf.m_nodes[f], sdf.m_cells[f], sdf.m_cell_map[f]):
            digest.update(np.ascontiguousarray(a).tobytes())
    out = {"ms": ms, "load_ms": load, "peak_rss_bytes": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024,
           "sdf_nodes_kept": len(sdf.m_nodes[0]), "volume_nodes_kept": len(sdf.m_nodes[1]), "sha256": digest.hexdigest()}
    if route == "new":
        out["stage_ms"] = [float(v) for v in sdf.last_reduced_volume_ms]
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--h-cells", type=float, default=1.0, help="smoothing length in cell diagonals")
    ap.add_argument("--res", default="128,256")
    ap.add_argument("--child", nargs=3, metavar=("ROUTE", "SDF", "WARM"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child[0], args.child[1], args.child[2], args.h_cells)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       check=True)
    card, power, clock = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    result = {"metric": "volume map vs K3 density map (CUDA events, medians); reduced volume map one call vs addFunction + reduceField x 2 "
                        "(host clock, fresh process per run)", "gpu": card, "power_limit": power, "max_sm_clock": clock,
              "h_cell_diagonals": args.h_cells, "scale": SCALE, "rho0": RHO0, "cases": []}
    mesh = os.path.join(ROOT, "oracle", "_ref", "resources", "bunny.obj")
    if not os.path.exists(mesh):
        raise SystemExit(f"{mesh} is not staged (make -C oracle ref)")
    resolutions = [int(r) for r in args.res.split(",")]
    with tempfile.TemporaryDirectory() as tmp:
        def make_sdf(res):
            out = os.path.join(tmp, f"bunny_{res}.cdf")
            if not os.path.exists(out):
                subprocess.run([os.path.join(BIN, "GenerateSDF"), "-r", f"{res} {res} {res}", "-o", out, mesh], capture_output=True, check=True)
            return out
        warm = make_sdf(32)
        paths = {res: make_sdf(res) for res in resolutions}
        # The route children run first, while this process has loaded neither torch, the library nor any grid: a child's ru_maxrss starts
        # from the high-water mark it inherits across fork + exec, so a parent that had touched gigabytes would set a floor under both routes.
        parent_rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
        for res in resolutions:
            runs = {"new": [], "old": []}
            for _ in range(max(1, args.repeats // 2)):
                for r in runs:
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--h-cells", str(args.h_cells), "--child", r, paths[res], warm],
                                       capture_output=True, text=True)
                    if p.returncode != 0:
                        raise SystemExit(f"{r} {res}^3 failed:\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
                    runs[r].append(json.loads(p.stdout.strip().splitlines()[-1]))
            entry = {"resolution": res, "parent_peak_rss_bytes_before_children": parent_rss}
            for r, rs in runs.items():
                entry["reduced_" + r] = {"ms_median": float(np.median([x["ms"] for x in rs])), "ms": [x["ms"] for x in rs],
                                         "peak_rss_bytes": max(x["peak_rss_bytes"] for x in rs), "sdf_nodes_kept": rs[0]["sdf_nodes_kept"],
                                         "volume_nodes_kept": rs[0]["volume_nodes_kept"]}
            entry["reduced_new"]["stage_ms_last"] = runs["new"][-1]["stage_ms"]
            entry["reduced_outputs_bit_identical"] = len({x["sha256"] for r in runs for x in runs[r]}) == 1
            result["cases"].append(entry)
        import discregrid_b200 as dg
        for entry in result["cases"]:
            entry.update(kernels(dg, paths[entry["resolution"]], args.h_cells, args.repeats))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
