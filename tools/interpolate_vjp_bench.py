#!/usr/bin/env python
"""Trainable fields on the GPU (K11): the vector-Jacobian product of interpolate in the node values next to K2 itself, on a 256^3 bunny SDF.

  k2          : interpolate with gradient, 10 M random points in the domain (dg_interpolate_batch_device on the trainable field)
  vjp_phi     : dg_interpolate_vjp_device with the upstream gradient of phi only
  vjp_both    : dg_interpolate_vjp_device with the upstream gradients of phi and of grad
  set_nodes   : dg_field_set_nodes_device (K2's pack of all cells and the DBL_MAX flags)
  step        : one forward + backward of interpolate(0, x, gradient=True, coefficients=c) with a loss on phi and grad
  create      : dg_field_create_trainable, including the upload and the incidence table's sort (host clock; the call synchronises)

Each device timing is CUDA events around one call, after a 256 MiB L2 flush outside the event pair; the components alternate within one
process, and the medians of `--runs` runs are reported.  Every run's node gradient must have the same bits.  The card's name and power
limit are read in the same run.  Needs oracle/_ref/resources/bunny.obj (make -C oracle ref).

usage: python tools/interpolate_vjp_bench.py [--runs 5] [--queries 10000000] [--field-res 256] [--out result.json]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--queries", type=int, default=10_000_000)
    ap.add_argument("--field-res", type=int, default=256)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    path = os.path.join(ROOT, "oracle", "_ref", "resources", "bunny.obj")
    if not os.path.exists(path):
        raise SystemExit(f"{path} is not staged (make -C oracle ref)")
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    result = {"card": card(), "runs": a.runs, "queries": a.queries, "field_res": a.field_res}
    print("card:", result["card"], flush=True)
    dev = torch.device("cuda", 0)
    torch.zeros(1, device=dev)
    dg.selftest()
    mesh = dg.TriangleMesh(path)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    r = a.field_res
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, (r, r, r))
    g.addFunction(dg.MeshSignedDistance(md))
    nodes, cells, cmap = g.m_nodes[0], np.ascontiguousarray(g.m_cells[0]), g.m_cell_map[0]
    rng = np.random.default_rng(0)
    x = torch.from_numpy(mn + rng.random((a.queries, 3)) * (mx - mn)).to(dev)
    gphi = torch.from_numpy(rng.standard_normal(a.queries)).to(dev)
    ggrad = torch.from_numpy(rng.standard_normal((a.queries, 3))).to(dev)
    c = torch.from_numpy(nodes).to(dev)
    n, nn = a.queries, len(nodes)
    phi = torch.empty(n, dtype=torch.float64, device=dev)
    grad = torch.empty((n, 3), dtype=torch.float64, device=dev)
    out = torch.empty(nn, dtype=torch.float64, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def create():
        h = C.c_void_p()
        t0 = time.perf_counter()
        capi.check(capi.lib.dg_field_create_trainable(C.byref(g._desc), capi.ptr(nodes, capi.F64P), nn, capi.ptr(cells, capi.U32P), len(cells),
                                                      capi.ptr(cmap, capi.U32P), C.byref(h)))
        return (time.perf_counter() - t0) * 1e3, h

    t_create, h = create()
    st = lambda: torch.cuda.current_stream().cuda_stream                  # noqa: E731

    def timed(fn):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        return e0.elapsed_time(e1)

    cg = c.clone().requires_grad_(True)
    gp2, gg2 = gphi.clone(), ggrad.clone()

    def step():
        p, gr = g.interpolate(0, x, gradient=True, coefficients=cg)
        ((p * gp2).sum() + (gr * gg2).sum()).backward()

    comps = {
        "k2": lambda: capi.check(capi.lib.dg_interpolate_batch_device(h, x.data_ptr(), n, phi.data_ptr(), grad.data_ptr(), st())),
        "vjp_phi": lambda: capi.check(capi.lib.dg_interpolate_vjp_device(h, x.data_ptr(), n, gphi.data_ptr(), None, out.data_ptr(), st())),
        "vjp_both": lambda: capi.check(capi.lib.dg_interpolate_vjp_device(h, x.data_ptr(), n, gphi.data_ptr(), ggrad.data_ptr(), out.data_ptr(), st())),
        "set_nodes": lambda: capi.check(capi.lib.dg_field_set_nodes_device(h, c.data_ptr(), nn, st())),
        "step": step,
    }
    for fn in comps.values():                                                 # warm-up of every shape
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in comps}
    times["create"] = [t_create]
    grads = []
    for _ in range(a.runs):
        for k, fn in comps.items():
            times[k].append(timed(fn))
            if k == "vjp_both":
                grads.append(out.cpu().numpy().view(np.uint64).copy())
        capi.lib.dg_field_destroy(h)
        t, h = create()
        times["create"].append(t)
    capi.lib.dg_field_destroy(h)
    result["median_ms"] = {k: statistics.median(v) for k, v in times.items()}
    result["same_bits_every_run"] = all(np.array_equal(grads[0], q) for q in grads[1:])
    result["nodes"], result["cells"] = nn, len(cells)
    print(json.dumps(result), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)
    if not result["same_bits_every_run"]:
        raise SystemExit("the node gradient changed between runs")


if __name__ == "__main__":
    main()
