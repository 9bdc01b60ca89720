#!/usr/bin/env python
"""K2's Hessian mode against its gradient mode, on the device entry points.

  kernels  : 10 M uniform points in the domain of a 256^3 bunny SDF, CUDA tensors in and out: dg_interpolate_batch_device with a gradient
             against dg_interpolate_hessian_batch_device, alternated, each launch timed with CUDA events after a 256 MB write that flushes
             the 50 MB L2.  Reported: Gq/s and algorithmic GB/s of each mode (312 B/query for value + gradient: x 24 + block 256 + phi 8 +
             grad 24; 384 B/query with the Hessian's 72) and their share of the H100 SXM data-sheet 3.35 TB/s.
  autograd : interpolate(0, x, hessian=True) on x that requires grad, then torch.autograd.grad(phi.sum(), x, create_graph=True) and a
             backward of a loss on that gradient (the Eikonal-style use), timed with CUDA events around the Python calls; next to the
             first-order route it extends (gradient=True forward + backward).

Medians of `--runs` runs; the Hessian mode's phi and grad are compared bit for bit with the gradient mode's.  The card's name, power limit
and max SM clock are read in the same run.  Needs oracle/_ref/resources/bunny.obj (make -C oracle ref).

usage: python tools/hessian_bench.py [--runs 7] [--queries 10000000] [--field-res 256] [--out result.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TB_S = 3.35                 # H100 SXM data sheet
BYTES_GRAD, BYTES_HESS = 24 + 256 + 8 + 24, 24 + 256 + 8 + 24 + 72


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
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
    dg.selftest()
    mesh = dg.TriangleMesh(path)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    r = a.field_res
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, (r, r, r))
    g.addFunction(dg.MeshSignedDistance(md))
    n = a.queries
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.from_numpy(mn).cuda() + torch.rand((n, 3), dtype=torch.float64, device="cuda", generator=gen) * torch.from_numpy(mx - mn).cuda()
    f = g._device_field(0)
    phi_g, grad_g = torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty((n, 3), dtype=torch.float64, device="cuda")
    phi_h, grad_h = torch.empty_like(phi_g), torch.empty_like(grad_g)
    hess = torch.empty((n, 3, 3), dtype=torch.float64, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def launch_grad():
        capi.check(capi.lib.dg_interpolate_batch_device(f, x.data_ptr(), n, phi_g.data_ptr(), grad_g.data_ptr(), stream))

    def launch_hess():
        capi.check(capi.lib.dg_interpolate_hessian_batch_device(f, x.data_ptr(), n, phi_h.data_ptr(), grad_h.data_ptr(), hess.data_ptr(), stream))

    def timed(fn):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    for fn in (launch_grad, launch_hess):
        timed(fn)
    t_grad, t_hess = [], []
    for _ in range(a.runs):
        t_grad.append(timed(launch_grad))
        t_hess.append(timed(launch_hess))
    torch.cuda.synchronize()
    same = bool(torch.equal(phi_g.view(torch.int64), phi_h.view(torch.int64)) and torch.equal(grad_g.view(torch.int64), grad_h.view(torch.int64)))
    modes = {}
    for name, ts, b in (("gradient", t_grad, BYTES_GRAD), ("hessian", t_hess, BYTES_HESS)):
        ms = statistics.median(ts)
        gbs = n * b / ms / 1e6
        modes[name] = {"ms": ms, "min_ms": min(ts), "max_ms": max(ts), "gq_s": n / ms / 1e6, "bytes_per_query": b, "gb_s": gbs,
                       "share_of_3_35_tb_s": gbs / (HBM_TB_S * 1e3)}
    modes["hessian_over_gradient_time"] = modes["hessian"]["ms"] / modes["gradient"]["ms"]
    modes["phi_grad_identical"] = same
    result["kernels"] = modes
    print(json.dumps(modes), flush=True)
    del phi_h, grad_h, hess

    # ---- the Python route with autograd: second order (hessian=True) next to first order (gradient=True)
    def second_order():
        xr = x.detach().requires_grad_(True)
        phi = g.interpolate(0, xr, hessian=True)[0]
        (gx,) = torch.autograd.grad(phi.sum(), xr, create_graph=True)
        ((gx * gx).sum(dim=1) - 1.0).square().sum().backward()
        return xr.grad

    def first_order():
        xr = x.detach().requires_grad_(True)
        g.interpolate(0, xr, gradient=True)[0].sum().backward()
        return xr.grad

    def fwd_create_graph():
        xr = x.detach().requires_grad_(True)
        phi = g.interpolate(0, xr, hessian=True)[0]
        return torch.autograd.grad(phi.sum(), xr, create_graph=True)[0]

    timings = {"first_order_fwd_bwd": [], "hessian_fwd_create_graph_bwd": [], "hessian_fwd_create_graph_bwd_then_eikonal_bwd": []}
    fns = {"first_order_fwd_bwd": first_order, "hessian_fwd_create_graph_bwd": fwd_create_graph,
           "hessian_fwd_create_graph_bwd_then_eikonal_bwd": second_order}
    for fn in fns.values():
        timed(fn)
    for _ in range(a.runs):
        for k, fn in fns.items():
            timings[k].append(timed(fn))
    result["autograd"] = {k: {"ms": statistics.median(v), "gq_s": n / statistics.median(v) / 1e6} for k, v in timings.items()}
    print(json.dumps(result["autograd"]), flush=True)
    result["card_after"] = card()
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
