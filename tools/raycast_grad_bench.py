#!/usr/bin/env python
"""Differentiable ray casts (K12, csrc/k12_raycast_grad.cu, with K10's vertex sums and K2 + K11 for fields) on one GPU, on CUDA tensors,
timed with CUDA events.

Mesh (bunny.obj, happy_buddha.obj; the rays of tools/mesh_raycast_bench.py):
  <w>_k9            : the forward, dg_mesh_raycast_device.
  <w>_vjp_t_o       : dg_mesh_raycast_vjp_device with grad_t, grad_origins only: the per-ray kernel alone.
  <w>_vjp_t_od      : grad_t, grad_origins and grad_directions (the per-ray kernel writes both).
  <w>_vjp_tb_od     : grad_t and grad_barycentric, the same two outputs.
  <w>_vjp_tb_odv    : grad_t and grad_barycentric, all three outputs: the per-ray kernel and K10's sort and sums.
  Workloads w: bunny_camera and buddha_camera (2048^2 pinhole images), bunny_ccd (10 M segments of half a cell diagonal of the bunny's
  256^3 SDF, starting within two cell diagonals of its surface).
Field (the bunny's 256^3 SDF as a trainable field, the same camera and segments):
  <w>_k7            : the forward, dg_field_raycast_device on the trainable field.
  <w>_k2            : K2's gradient mode alone at the crossing points (what the VJP evaluates).
  <w>_vjp_od        : dg_field_raycast_vjp_device to grad_origins and grad_directions: the two per-ray kernels and K2.
  <w>_vjp_odn       : the same with grad_nodes: K11 on top.
The workloads are alternated and run `--runs` times; each timed call is preceded by a write of 256 MiB, which flushes the 50 MB L2.  Medians
and spreads.  Every run's gradients are compared bit for bit with the first run's.  The card's name, power limit and max SM clock are read
in the same run.  Needs oracle/_ref/resources (make -C oracle ref).

usage: python tools/raycast_grad_bench.py [--runs 5] [--res 2048] [--n 10000000] [--out result.json]"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mesh_distance_grad_bench import card, near_surface      # noqa: E402


def camera(torch, V, res):
    """a res x res pinhole image looking at the mesh's box centre from outside"""
    lo, hi = V.min(0), V.max(0)
    c, ext = (lo + hi) / 2, float(np.linalg.norm(hi - lo))
    eye = torch.tensor(c + np.array([0.35, 0.25, 1.2]) * ext, dtype=torch.float64, device="cuda")
    fwd = torch.tensor(c, dtype=torch.float64, device="cuda") - eye
    fwd = fwd / fwd.norm()
    up = torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64, device="cuda")
    right = torch.linalg.cross(fwd, up); right = right / right.norm()
    up = torch.linalg.cross(right, fwd)
    s = (torch.arange(res, dtype=torch.float64, device="cuda") + 0.5) / res * 2 - 1
    u, v = torch.meshgrid(s, s, indexing="ij")
    d = fwd + 0.45 * (u.reshape(-1, 1) * right + v.reshape(-1, 1) * up)
    return eye.expand_as(d).contiguous(), d.contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--res", type=int, default=2048)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    import winding_ref as wr
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res_dir = os.path.join(ROOT, "oracle", "_ref", "resources")
    for f in ("bunny.obj", "happy_buddha.obj"):
        if not os.path.exists(os.path.join(res_dir, f)):
            raise SystemExit(f"{f} is not staged (make -C oracle ref)")
    result = {"card": card(), "runs": a.runs, "camera": a.res, "ccd_n": a.n, "grid": a.grid}
    print("card:", result["card"], flush=True)
    dg.selftest()
    st = lambda: torch.cuda.current_stream().cuda_stream      # noqa: E731
    f64 = dict(dtype=torch.float64, device="cuda")
    V, F = wr.read_obj(os.path.join(res_dir, "bunny.obj"))
    Vb, Fb = wr.read_obj(os.path.join(res_dir, "happy_buddha.obj"))
    md, mdb = dg.TriangleMeshDistance(V, F), dg.TriangleMeshDistance(Vb, Fb)
    mn, mx = dg.generate_sdf_domain(V)
    grid = dg.CubicLagrangeDiscreteGrid(mn, mx, (a.grid,) * 3)
    fid = grid.addFunction(dg.MeshSignedDistance(md))
    tf = grid._trainable_field(fid)
    h = float(np.linalg.norm(grid.cellSize()))
    gen = torch.Generator(device="cuda").manual_seed(5)
    x0 = near_surface(torch, V, F, a.n, 1)
    step = torch.randn((a.n, 3), generator=gen, **f64)
    step = (0.5 * h * step / step.norm(dim=1, keepdim=True)).contiguous()
    rays = {"bunny_camera": camera(torch, V, a.res), "bunny_ccd": (x0, step), "buddha_camera": camera(torch, Vb, a.res)}
    tmax = {"bunny_camera": float("inf"), "bunny_ccd": 1.0, "buddha_camera": float("inf")}
    meshes = {"bunny_camera": (md, V), "bunny_ccd": (md, V), "buddha_camera": (mdb, Vb)}
    ms = {}
    for w, (o, d) in rays.items():
        m, Vw = meshes[w]
        n = len(o)
        s = dict(t=torch.empty(n, **f64), tid=torch.empty(n, dtype=torch.int32, device="cuda"), b=torch.empty((n, 3), **f64),
                 st=torch.empty(n, dtype=torch.int32, device="cuda"), V=torch.tensor(np.asarray(Vw), **f64),
                 gt=torch.randn(n, generator=gen, **f64), gb=torch.randn((n, 3), generator=gen, **f64),
                 go=torch.empty((n, 3), **f64), gd=torch.empty((n, 3), **f64), gv=torch.empty((len(Vw), 3), **f64))
        ms[w] = s
    fs = {}
    for w in ("bunny_camera", "bunny_ccd"):
        o, d = rays[w]
        n = len(o)
        fs[w] = dict(tl=torch.empty(n, **f64), th=torch.empty(n, **f64), st=torch.empty(n, dtype=torch.int32, device="cuda"),
                     g=torch.randn(n, generator=gen, **f64), go=torch.empty((n, 3), **f64), gd=torch.empty((n, 3), **f64),
                     gn=torch.empty(tf.n_nodes, **f64), phi=torch.empty(n, **f64), grad=torch.empty((n, 3), **f64))

    def k9(w):
        o, d = rays[w]; s = ms[w]
        capi.check(capi.lib.dg_mesh_raycast_device(meshes[w][0].handle, o.data_ptr(), d.data_ptr(), len(o), 0.0, tmax[w], s["t"].data_ptr(),
                                                   s["tid"].data_ptr(), s["b"].data_ptr(), s["st"].data_ptr(), st()))

    def mvjp(w, bary, want):
        o, d = rays[w]; s = ms[w]
        p = lambda k: s[k].data_ptr() if k in want else None      # noqa: E731
        capi.check(capi.lib.dg_mesh_raycast_vjp_device(meshes[w][0].handle, len(o), d.data_ptr(), s["t"].data_ptr(), s["tid"].data_ptr(),
                                                       s["b"].data_ptr(), s["V"].data_ptr(), s["gt"].data_ptr(),
                                                       s["gb"].data_ptr() if bary else None, p("go"), p("gd"), p("gv"), st()))

    def k7(w):
        o, d = rays[w]; s = fs[w]
        capi.check(capi.lib.dg_field_raycast_device(tf.handle, o.data_ptr(), d.data_ptr(), len(o), 0.0, 0.0, tmax[w], s["tl"].data_ptr(),
                                                    s["th"].data_ptr(), s["st"].data_ptr(), st()))

    xc = {}
    for w in fs:
        k7(w)
        o, d = rays[w]; s = fs[w]
        x = o + s["tl"][:, None] * d
        lo, hi = torch.tensor(grid._desc.domain_min[:], **f64), torch.tensor(grid._desc.domain_max[:], **f64)
        x = torch.where(x < lo, lo, torch.where(x > hi, hi, x))
        xc[w] = torch.where((s["st"] != 0)[:, None], x, torch.full_like(x, float("inf"))).contiguous()

    def k2(w):
        s = fs[w]
        capi.check(capi.lib.dg_interpolate_batch_device(tf.handle, xc[w].data_ptr(), len(xc[w]), s["phi"].data_ptr(), s["grad"].data_ptr(), st()))

    def fvjp(w, nodes):
        o, d = rays[w]; s = fs[w]
        capi.check(capi.lib.dg_field_raycast_vjp_device(tf.handle, len(o), o.data_ptr(), d.data_ptr(), s["tl"].data_ptr(), s["st"].data_ptr(),
                                                        s["g"].data_ptr(), None, s["go"].data_ptr(), s["gd"].data_ptr(),
                                                        s["gn"].data_ptr() if nodes else None, st()))

    cases = {}
    for w in ms:
        cases[f"{w}_k9"] = (lambda w=w: k9(w), None)
        cases[f"{w}_vjp_t_o"] = (lambda w=w: mvjp(w, False, ("go",)), (ms[w], ("go",)))
        cases[f"{w}_vjp_t_od"] = (lambda w=w: mvjp(w, False, ("go", "gd")), (ms[w], ("go", "gd")))
        cases[f"{w}_vjp_tb_od"] = (lambda w=w: mvjp(w, True, ("go", "gd")), (ms[w], ("go", "gd")))
        cases[f"{w}_vjp_tb_odv"] = (lambda w=w: mvjp(w, True, ("go", "gd", "gv")), (ms[w], ("go", "gd", "gv")))
    for w in fs:
        cases[f"field_{w}_k7"] = (lambda w=w: k7(w), None)
        cases[f"field_{w}_k2"] = (lambda w=w: k2(w), None)
        cases[f"field_{w}_vjp_od"] = (lambda w=w: fvjp(w, False), (fs[w], ("go", "gd")))
        cases[f"field_{w}_vjp_odn"] = (lambda w=w: fvjp(w, True), (fs[w], ("go", "gd", "gn")))
    flush = torch.empty(1 << 25, **f64)
    for w in ms:
        k9(w)
    first = {}
    for k, (fn, chk) in cases.items():
        fn()
        torch.cuda.synchronize()
        if chk:
            first[k] = [chk[0][x].clone() for x in chk[1]]
    same = {k: True for k in first}
    times = {k: [] for k in cases}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.runs):
        for k, (fn, chk) in cases.items():
            flush.zero_()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            if chk:
                same[k] &= all(bool(torch.equal(chk[0][x].view(torch.int64), f.view(torch.int64))) for x, f in zip(chk[1], first[k]))
    for w in ms:
        result[f"{w}_hits"] = int((ms[w]["tid"] >= 0).sum().item())
    for w in fs:
        result[f"field_{w}_hits"] = int((fs[w]["st"] != 0).sum().item())
    for k in cases:
        med = statistics.median(times[k])
        r = {"median_ms": med, "spread_ms": [min(times[k]), max(times[k])]}
        if k in same:
            r["same_bits_every_run"] = same[k]
        result[k] = r
        extra = f", same bits every run: {r['same_bits_every_run']}" if k in same else ""
        print(f"{k}: median {med:.3f} ms ({min(times[k]):.3f}..{max(times[k]):.3f}){extra}", flush=True)
    for w in ms:
        tot, ray = result[f"{w}_vjp_tb_odv"]["median_ms"], result[f"{w}_vjp_tb_od"]["median_ms"]
        print(f"{w}: per-ray kernel {ray:.3f} ms, K10's sort and sums about {tot - ray:.3f} ms of {tot:.3f} ms", flush=True)
    for w in fs:
        od, odn, k2t = result[f"field_{w}_vjp_od"]["median_ms"], result[f"field_{w}_vjp_odn"]["median_ms"], result[f"field_{w}_k2"]["median_ms"]
        print(f"field {w}: K2 {k2t:.3f} ms, per-ray kernels about {od - k2t:.3f} ms, K11 about {odn - od:.3f} ms of {odn:.3f} ms", flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
