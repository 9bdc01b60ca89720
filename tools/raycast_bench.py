#!/usr/bin/env python
"""Ray casts (K7, csrc/k7_raycast.cu) on one GPU: dg_field_raycast_device on CUDA tensors, timed with CUDA events.

  ccd      : 10 M segments x0 -> x1 (t in [0, 1]) of half a cell diagonal, x0 within two cell diagonals of the bunny.obj 256^3 dense SDF's
             zero level set: continuous collision detection of a particle step.
  camera   : a 2048^2 pinhole image of the same field, t_max = inf.
  band512  : the same camera against the 512^3 reduced narrow band of 2 cell diagonals, cast on the device field built from its kept handle.
The workloads are alternated and run `--runs` times; each timed call is preceded by a write of 256 MiB, which flushes the 50 MB L2.  Medians.
Segments, nodes and evaluations per ray are counted by the restatement (tests/raycast_ref.py) on a sample of rays; the fp64 rate is
FP64_PER_EVAL (the fp64 operations of one evaluation, counted from the source: position, clamp, cell location and K2's value sum) times the
sample's mean evaluations per ray times rays, over the kernel time -- against dg_fp64_rate_probe in the same run.  The card's name, power
limit and max SM clock are read in the same run.  Needs oracle/_ref/resources (make -C oracle ref).

usage: python tools/raycast_bench.py [--runs 5] [--sample 300] [--out result.json]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
FP64_PER_EVAL = 172


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def camera(torch, mn, mx, res):
    c = 0.5 * (mn + mx)
    ext = float(np.linalg.norm(mx - mn))
    eye = c + np.array([0.3, 0.2, 1.0]) * ext
    fwd = (c - eye) / np.linalg.norm(c - eye)
    right = np.cross(fwd, [0.0, 1.0, 0.0]); right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    s = (torch.arange(res, dtype=torch.float64, device="cuda") + 0.5) / res * 2 - 1
    v, u = torch.meshgrid(s, s, indexing="ij")
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda")
    D = t(fwd)[None] + 0.35 * (u.reshape(-1, 1) * t(right)[None] + v.reshape(-1, 1) * t(up)[None])
    return t(eye)[None].expand(res * res, 3).contiguous(), D.contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--sample", type=int, default=300)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    import raycast_ref as rr
    import winding_ref as wr
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    obj = os.path.join(ROOT, "oracle", "_ref", "resources", "bunny.obj")
    if not os.path.exists(obj):
        raise SystemExit(f"{obj} is not staged (make -C oracle ref)")
    result = {"card": card(), "runs": a.runs}
    print("card:", result["card"], flush=True)
    dg.selftest()
    rate = C.c_double()
    capi.check(capi.lib.dg_fp64_rate_probe(C.byref(rate)))
    result["fp64_probe_tflops"] = rate.value
    V, F = wr.read_obj(obj)
    md = dg.TriangleMeshDistance(V, F)
    mn, mx = dg.generate_sdf_domain(V)
    dense = dg.CubicLagrangeDiscreteGrid(mn, mx, (256, 256, 256))
    dense.addFunction(dg.MeshSignedDistance(md))
    band = dg.CubicLagrangeDiscreteGrid(mn, mx, (512, 512, 512))
    band.addReducedBandField(dg.MeshSignedDistance(md), dg.MeshDistanceBand(md, 2.0 * float(np.linalg.norm(band.cellSize()))))
    band._device_field(0)                                    # built from the kept handle
    # CCD steps near the surface
    h = float(np.linalg.norm(dense.cellSize()))
    gen = torch.Generator(device="cuda").manual_seed(0)
    lo_t, hi_t = torch.tensor(mn, device="cuda"), torch.tensor(mx, device="cuda")
    X0 = []
    n_ccd = 10_000_000
    while sum(len(x) for x in X0) < n_ccd:
        x = lo_t + torch.rand((1 << 24, 3), dtype=torch.float64, device="cuda", generator=gen) * (hi_t - lo_t)
        X0.append(x[dense.interpolate(0, x).abs() < 2 * h])
    X0 = torch.cat(X0)[:n_ccd].contiguous()
    step = torch.randn((n_ccd, 3), dtype=torch.float64, device="cuda", generator=gen)
    step = (0.5 * h) * step / torch.linalg.norm(step, dim=1, keepdim=True)
    Oc, Dc = camera(torch, mn, mx, 2048)
    cases = {"ccd": (dense, X0, step, 0.0, 1.0), "camera": (dense, Oc, Dc, 0.0, float("inf")), "band512": (band, Oc, Dc, 0.0, float("inf"))}
    flush = torch.empty(1 << 25, dtype=torch.float64, device="cuda")
    times = {k: [] for k in cases}
    status = {}
    for g, O, D, t0, t1 in cases.values():
        g.raycast(0, O, D, 0.0, t0, t1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.runs):
        for k, (g, O, D, t0, t1) in cases.items():
            flush.zero_()
            e0.record()
            r = g.raycast(0, O, D, 0.0, t0, t1)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            status[k] = r[2]
    for k, (g, O, D, t0, t1) in cases.items():
        ms = statistics.median(times[k])
        n = len(O)
        idx = torch.randint(0, n, (a.sample,), device="cuda", generator=gen).cpu().numpy()
        _, _, _, st = rr.raycast(rr.Grid.of_grid(g), lambda x: g.interpolate(0, x), O[idx].cpu().numpy(), D[idx].cpu().numpy(), 0.0, t0, t1,
                                 with_stats=True)
        ev = float(st["evaluations"].mean())
        flops = FP64_PER_EVAL * ev * n / (ms * 1e-3)
        hits = int((status[k] != 0).sum())
        r = {"rays": n, "median_ms": ms, "spread_ms": [min(times[k]), max(times[k])], "rays_per_s": n / (ms * 1e-3), "hits": hits,
             "segments_per_ray": float(st["segments"].mean()), "nodes_per_ray": float(st["nodes"].mean()), "evaluations_per_ray": ev,
             "fp64_tflops": flops / 1e12, "fp64_share_of_probe": flops / 1e12 / rate.value}
        result[k] = r
        print(f"{k}: {n} rays, {hits} crossings, median {ms:.2f} ms ({min(times[k]):.2f}..{max(times[k]):.2f}) = {r['rays_per_s'] / 1e6:.1f} M rays/s; "
              f"per ray {r['segments_per_ray']:.1f} segments, {r['nodes_per_ray']:.1f} nodes, {ev:.1f} evaluations (sample of {a.sample}); "
              f"{r['fp64_tflops']:.2f} fp64 TFLOP/s = {100 * r['fp64_share_of_probe']:.1f} % of the probe's {rate.value:.1f}", flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
