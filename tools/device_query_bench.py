#!/usr/bin/env python
"""Queries that stay on the GPU against the numpy route, and the first interpolate of a reduced field from its kept handle against the
copy and re-upload it replaces.

  interpolate : 10 M random points in the domain of a 256^3 bunny SDF, with gradient.  CUDA tensors in and out (dg_interpolate_batch_device
                on torch's current stream, timed with CUDA events) against numpy arrays in and out (dg_interpolate_batch, pageable memory,
                host clock around the synchronous call).
  distance    : signed_distance of the bunny on 1 M random points, the same two routes (dg_mesh_distance_device / dg_mesh_distance).
  first use   : addReducedBandField on the 512^3 bunny (w = 2 cell diagonals, the band of tools/band_reduce_bench.py), then the first
                interpolate (1,000 points): from the kept handle (dg_field_create_reduced) against after dropping the handle (dg_field_create
                of the host copy: the route every reduced field took before).  Host clock, both calls synchronous.

The routes alternate within one process; the medians of `--runs` runs are reported, and the results of the two routes are compared bit for
bit.  The card's name and power limit are read in the same run.  Needs oracle/_ref/resources/bunny.obj (make -C oracle ref).

usage: python tools/device_query_bench.py [--runs 5] [--queries 10000000] [--points 1000000] [--band-res 512] [--out result.json]"""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def cuda_ms(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def host_ms(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def alternate(runs, device_fn, host_fn):
    """medians of alternated runs (one warm-up of each first) and the last outputs of both"""
    device_fn(); host_fn()
    dev, hst = [], []
    for _ in range(runs):
        ms, d_out = device_fn(); dev.append(ms)
        ms, h_out = host_fn(); hst.append(ms)
    return statistics.median(dev), statistics.median(hst), d_out, h_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--queries", type=int, default=10_000_000)
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--field-res", type=int, default=256)
    ap.add_argument("--band-res", type=int, default=512)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    path = os.path.join(ROOT, "oracle", "_ref", "resources", "bunny.obj")
    if not os.path.exists(path):
        raise SystemExit(f"{path} is not staged (make -C oracle ref)")
    result = {"card": card(), "runs": a.runs}
    print("card:", result["card"], flush=True)
    torch.zeros(1, device="cuda")
    dg.selftest()
    mesh = dg.TriangleMesh(path)
    md = dg.TriangleMeshDistance(mesh)
    mn, mx = dg.generate_sdf_domain(mesh.vertices)
    rng = np.random.default_rng(0)

    # ---- interpolate with gradient, 10 M points on a 256^3 field
    r = a.field_res
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, (r, r, r))
    g.addFunction(dg.MeshSignedDistance(md))
    x = mn + rng.random((a.queries, 3)) * (mx - mn)
    xt = torch.from_numpy(x).cuda()
    dev, hst, d_out, h_out = alternate(a.runs, lambda: cuda_ms(lambda: g.interpolate(0, xt, gradient=True)),
                                       lambda: host_ms(lambda: g.interpolate(0, x, gradient=True)))
    same = bool(np.array_equal(bits(d_out[0].cpu().numpy()), bits(h_out[0])) and np.array_equal(bits(d_out[1].cpu().numpy()), bits(h_out[1])))
    result["interpolate"] = {"res": r, "queries": a.queries, "tensor_ms": dev, "numpy_ms": hst, "tensor_gq_s": a.queries / dev / 1e6,
                             "numpy_gq_s": a.queries / hst / 1e6, "speedup": hst / dev, "identical": same}
    print(json.dumps(result["interpolate"]), flush=True)
    del g, xt, d_out, h_out

    # ---- signed distance, 1 M points
    p = mn + rng.random((a.points, 3)) * (mx - mn)
    pt = torch.from_numpy(p).cuda()
    dev, hst, d_out, h_out = alternate(a.runs, lambda: cuda_ms(lambda: md.signed_distance(pt)), lambda: host_ms(lambda: md.signed_distance(p)))
    same = all(np.array_equal(np.ascontiguousarray(t.cpu().numpy()).view(np.uint8), np.ascontiguousarray(h).view(np.uint8)) for t, h in zip(d_out, h_out))
    result["signed_distance"] = {"points": a.points, "tensor_ms": dev, "numpy_ms": hst, "tensor_mq_s": a.points / dev / 1e3,
                                 "numpy_mq_s": a.points / hst / 1e3, "speedup": hst / dev, "identical": same}
    print(json.dumps(result["signed_distance"]), flush=True)
    del pt, d_out, h_out

    # ---- the first interpolate after addReducedBandField: kept handle against copy + re-upload
    r = a.band_res
    q = mn + rng.random((1000, 3)) * (mx - mn)
    kept, upload, same = [], [], True
    for _ in range(a.runs):
        b = dg.CubicLagrangeDiscreteGrid(mn, mx, (r, r, r))
        cell = b.cellSize()
        b.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, 2.0 * float(np.sqrt((cell * cell).sum()))))
        ms, phi_kept = host_ms(lambda: b.interpolate(0, q, gradient=True))
        kept.append(ms)
        b._invalidate()                                # drops the device field: the next one is uploaded from the host members
        ms, phi_up = host_ms(lambda: b.interpolate(0, q, gradient=True))
        upload.append(ms)
        same = same and all(np.array_equal(bits(u), bits(v)) for u, v in zip(phi_kept, phi_up))
        n_nodes, n_cells = len(b.m_nodes[0]), len(b.m_cells[0])
        del b
    result["first_interpolate"] = {"res": r, "nodes_kept": n_nodes, "cells_kept": n_cells, "kept_handle_ms": statistics.median(kept),
                                   "copy_upload_ms": statistics.median(upload), "speedup": statistics.median(upload) / statistics.median(kept),
                                   "identical": same}
    print(json.dumps(result["first_interpolate"]), flush=True)
    result["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
