#!/usr/bin/env python
"""Differentiable mesh distances (K10, csrc/k10_distance_grad.cu and radix_sort.cu, with K1's mesh_distance_bary_kernel) on one GPU, on CUDA
tensors, timed with CUDA events.

  fwd_bunny_distance : dg_mesh_distance_device, signed, every output, on 10 M points near bunny.obj (the reference for the next row).
  fwd_bunny_bary     : dg_mesh_distance_bary_device on the same points: the same outputs and the barycentric weights.
  vjp_bunny          : dg_mesh_distance_vjp_device with grad_points and grad_vertices for those 10 M queries.
  vjp_buddha         : the same on 10 M points near happy_buddha.obj (855,196 triangles: three digit passes of the sort, as for the bunny).
  vjp_box            : the same on 10 M points near box.obj (12 triangles: segments of ~0.8 M queries, the longest the sum meets).
Points: a uniform triangle, a uniform point on it, then a normal offset of sigma = 2 % of the bounding-box diagonal.  The workloads are
alternated and run `--runs` times; each timed call is preceded by a write of 256 MiB, which flushes the 50 MB L2.  Medians.  Every run's
gradients are compared bit for bit with the first run's.  The card's name, power limit and max SM clock are read in the same run.  Needs
oracle/_ref/resources (make -C oracle ref).

usage: python tools/mesh_distance_grad_bench.py [--runs 5] [--n 10000000] [--out result.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def near_surface(torch, V, F, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Vt = torch.from_numpy(V).cuda(); Ft = torch.from_numpy(F.astype(np.int64)).cuda()
    t = torch.randint(0, len(F), (n,), device="cuda", generator=g)
    u = torch.rand((n, 2), dtype=torch.float64, device="cuda", generator=g)
    flip = u.sum(1, keepdim=True) > 1
    u = torch.where(flip, 1 - u, u)
    a, b, c = Vt[Ft[t, 0]], Vt[Ft[t, 1]], Vt[Ft[t, 2]]
    nrm = torch.linalg.cross(b - a, c - a)
    nrm = nrm / nrm.norm(dim=1, keepdim=True).clamp_min(1e-300)
    sigma = 0.02 * float(np.linalg.norm(V.max(0) - V.min(0)))
    x = a + u[:, :1] * (b - a) + u[:, 1:] * (c - a) + sigma * torch.randn((n, 1), dtype=torch.float64, device="cuda", generator=g) * nrm
    return x.contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    import winding_ref as wr

    res_dir = os.path.join(ROOT, "oracle", "_ref", "resources")
    result = {"card": card(), "n": a.n}
    print("card:", result["card"], flush=True)
    meshes = {"bunny": wr.read_obj(os.path.join(res_dir, "bunny.obj")), "buddha": wr.read_obj(os.path.join(res_dir, "happy_buddha.obj")),
              "box": wr.read_obj(os.path.join(ROOT, "tests", "golden", "box.obj"))}
    st = lambda: torch.cuda.current_stream().cuda_stream      # noqa: E731
    state = {}
    for name, (V, F) in meshes.items():
        md = dg.TriangleMeshDistance(V, F)
        x = near_surface(torch, V, F, a.n, 1)
        n = len(x)
        out = dict(dist=torch.empty(n, dtype=torch.float64, device="cuda"), near=torch.empty((n, 3), dtype=torch.float64, device="cuda"),
                   ent=torch.empty(n, dtype=torch.int32, device="cuda"), tri=torch.empty(n, dtype=torch.int32, device="cuda"),
                   bary=torch.empty((n, 3), dtype=torch.float64, device="cuda"))
        capi.check(capi.lib.dg_mesh_distance_bary_device(md.handle, x.data_ptr(), n, 1, out["dist"].data_ptr(), out["near"].data_ptr(),
                                                         out["ent"].data_ptr(), out["tri"].data_ptr(), out["bary"].data_ptr(), st()))
        g = torch.randn(n, dtype=torch.float64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        gp = torch.empty((n, 3), dtype=torch.float64, device="cuda")
        gv = torch.empty((md.n_vertices, 3), dtype=torch.float64, device="cuda")
        state[name] = (md, x, out, g, gp, gv)
        result[f"{name}_triangles"] = len(F)

    def fwd(bary):
        md, x, o, _, _, _ = state["bunny"]
        n = len(x)
        if bary:
            capi.check(capi.lib.dg_mesh_distance_bary_device(md.handle, x.data_ptr(), n, 1, o["dist"].data_ptr(), o["near"].data_ptr(),
                                                             o["ent"].data_ptr(), o["tri"].data_ptr(), o["bary"].data_ptr(), st()))
        else:
            capi.check(capi.lib.dg_mesh_distance_device(md.handle, x.data_ptr(), n, 1, o["dist"].data_ptr(), o["near"].data_ptr(),
                                                        o["ent"].data_ptr(), o["tri"].data_ptr(), st()))

    def vjp(name):
        md, x, o, g, gp, gv = state[name]
        capi.check(capi.lib.dg_mesh_distance_vjp_device(md.handle, len(x), x.data_ptr(), o["dist"].data_ptr(), o["near"].data_ptr(),
                                                        o["tri"].data_ptr(), o["bary"].data_ptr(), g.data_ptr(), gp.data_ptr(), gv.data_ptr(), st()))

    cases = {"fwd_bunny_distance": lambda: fwd(False), "fwd_bunny_bary": lambda: fwd(True),
             "vjp_bunny": lambda: vjp("bunny"), "vjp_buddha": lambda: vjp("buddha"), "vjp_box": lambda: vjp("box")}
    flush = torch.empty(1 << 25, dtype=torch.float64, device="cuda")
    for fn in cases.values():
        fn()
    torch.cuda.synchronize()
    first = {k: (s[4].clone(), s[5].clone()) for k, s in state.items()}
    same = {k: True for k in state}
    times = {k: [] for k in cases}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.runs):
        for k, fn in cases.items():
            flush.zero_()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            if k.startswith("vjp_"):
                name = k[4:]
                s = state[name]
                same[name] &= bool(torch.equal(s[4].view(torch.int64), first[name][0].view(torch.int64)) and
                                   torch.equal(s[5].view(torch.int64), first[name][1].view(torch.int64)))
    for k in cases:
        ms = statistics.median(times[k])
        r = {"median_ms": ms, "spread_ms": [min(times[k]), max(times[k])], "queries_per_s": a.n / (ms * 1e-3)}
        if k.startswith("vjp_"):
            r["same_bits_every_run"] = same[k[4:]]
        result[k] = r
        extra = f", same bits every run: {r['same_bits_every_run']}" if "same_bits_every_run" in r else ""
        print(f"{k}: median {ms:.3f} ms ({min(times[k]):.3f}..{max(times[k]):.3f}) = {r['queries_per_s'] / 1e6:.1f} M queries/s{extra}", flush=True)
    result["bary_over_distance"] = result["fwd_bunny_bary"]["median_ms"] / result["fwd_bunny_distance"]["median_ms"]
    print(f"forward with weights / dg_mesh_distance_device: {result['bary_over_distance']:.3f}", flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
