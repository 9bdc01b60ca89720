#!/usr/bin/env python
"""Ray casts on a mesh (K9, csrc/k9_mesh_raycast.cu) on one GPU: dg_mesh_raycast_device on CUDA tensors, timed with CUDA events, next to K7
(dg_field_raycast_device) on the same rays in the same run.

  bunny_camera   : a 2048^2 pinhole image of bunny.obj (t_max = inf); K7 on the bunny's 256^3 dense SDF along the same rays.
  bunny_ccd      : 10 M segments x0 -> x1 (t in [0, 1]) of half a cell diagonal of that SDF, x0 within two cell diagonals of its zero level
                   set (the generator of tools/raycast_bench.py); K7 on the same segments.
  buddha_camera  : a 2048^2 pinhole image of happy_buddha.obj (K9 only).
  deform         : the bunny twisted by 0.3 rad: dg_mesh_refit_device + the 10 M segments cast on the mesh, against dg_mesh_refit_device +
                   K1 at 128^3 (dg_sample_sdf_device) + dg_field_create_device + K7 on the same segments.
The workloads are alternated and run `--runs` times; each timed call is preceded by a write of 256 MiB, which flushes the 50 MB L2.  Medians.
Boxes visited and triangles tested per ray are counted on a sample of rays by the emulated kernel (build/bin/libk9emu.so, the product's TU
compiled for the CPU with counters); the outputs of the sample are checked against the device's bit for bit.  The card's name, power limit
and max SM clock are read in the same run.  Needs oracle/_ref/resources (make -C oracle ref).

usage: python tools/mesh_raycast_bench.py [--runs 5] [--sample 300] [--out result.json]"""
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
EMU = os.path.join(ROOT, "build", "bin", "libk9emu.so")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def twist(V, angle):
    lo, hi = V[:, 1].min(), V[:, 1].max()
    t = angle * (V[:, 1] - lo) / (hi - lo)
    c, s = np.cos(t), np.sin(t)
    return np.stack([c * V[:, 0] + s * V[:, 2], V[:, 1], -s * V[:, 0] + c * V[:, 2]], 1)


def emu_counts(V, F, O, D, t0, t1):
    """(boxes, triangles) per ray and the outputs of the emulated kernel on the rays O, D"""
    DP, U32P, I32P = C.POINTER(C.c_double), C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
    lib = C.CDLL(EMU)
    lib.emu_k9_create.restype = C.c_void_p
    lib.emu_k9_create.argtypes = [DP, C.c_uint64, U32P, C.c_uint64]
    lib.emu_k9_destroy.argtypes = [C.c_void_p]
    lib.emu_k9_raycast.argtypes = [C.c_void_p, DP, DP, C.c_uint64, C.c_double, C.c_double, DP, I32P, DP, I32P]
    lib.emu_k9_counters.argtypes = [C.POINTER(C.c_ulonglong)]
    V = np.ascontiguousarray(V, np.float64); F = np.ascontiguousarray(F, np.uint32)
    O = np.ascontiguousarray(O, np.float64); D = np.ascontiguousarray(D, np.float64)
    h = lib.emu_k9_create(V.ctypes.data_as(DP), len(V), F.ctypes.data_as(U32P), len(F))
    n = len(O)
    t, tid, b, st = np.empty(n), np.empty(n, np.int32), np.empty((n, 3)), np.empty(n, np.int32)
    lib.emu_k9_counters_reset()
    lib.emu_k9_raycast(h, O.ctypes.data_as(DP), D.ctypes.data_as(DP), n, t0, t1, t.ctypes.data_as(DP), tid.ctypes.data_as(I32P),
                       b.ctypes.data_as(DP), st.ctypes.data_as(I32P))
    c = (C.c_ulonglong * 3)()
    lib.emu_k9_counters(c)
    lib.emu_k9_destroy(h)
    return c[0] / n, c[1] / n, (t, tid, b, st)


def camera(torch, lo, hi, res):
    c = 0.5 * (lo + hi)
    ext = float(np.linalg.norm(hi - lo))
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
    import winding_ref as wr
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res_dir = os.path.join(ROOT, "oracle", "_ref", "resources")
    for f in ("bunny.obj", "happy_buddha.obj"):
        if not os.path.exists(os.path.join(res_dir, f)):
            raise SystemExit(f"{f} is not staged (make -C oracle ref)")
    result = {"card": card(), "runs": a.runs}
    print("card:", result["card"], flush=True)
    dg.selftest()
    st_ptr = lambda: torch.cuda.current_stream().cuda_stream
    V, F = wr.read_obj(os.path.join(res_dir, "bunny.obj"))
    Vb, Fb = wr.read_obj(os.path.join(res_dir, "happy_buddha.obj"))
    md = dg.TriangleMeshDistance(V, F)
    mdb = dg.TriangleMeshDistance(Vb, Fb)
    mn, mx = dg.generate_sdf_domain(V)
    dense = dg.CubicLagrangeDiscreteGrid(mn, mx, (256, 256, 256))
    dense.addFunction(dg.MeshSignedDistance(md))
    fh = dense._device_field(0)
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
    step = ((0.5 * h) * step / torch.linalg.norm(step, dim=1, keepdim=True)).contiguous()
    Oc, Dc = camera(torch, V.min(0), V.max(0), 2048)
    Ob, Db = camera(torch, Vb.min(0), Vb.max(0), 2048)

    def k9(m, O, D, t0, t1):
        n = len(O)
        out = (torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"),
               torch.empty((n, 3), dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"))
        return lambda: (capi.check(capi.lib.dg_mesh_raycast_device(m.handle, O.data_ptr(), D.data_ptr(), n, t0, t1, out[0].data_ptr(),
                                                                   out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), st_ptr())), out)[1]

    def k7(field, O, D, t0, t1):
        n = len(O)
        out = (torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.float64, device="cuda"),
               torch.empty(n, dtype=torch.int32, device="cuda"))
        return lambda: (capi.check(capi.lib.dg_field_raycast_device(field, O.data_ptr(), D.data_ptr(), n, 0.0, t0, t1, out[0].data_ptr(),
                                                                    out[1].data_ptr(), out[2].data_ptr(), st_ptr())), out)[1]

    # the deforming case: refit + cast on the mesh, against refit + K1 resample at 128^3 + field + K7
    mdd = dg.TriangleMeshDistance(V, F)
    V1 = torch.from_numpy(np.ascontiguousarray(twist(V, 0.3))).cuda()
    mn1, mx1 = dg.generate_sdf_domain(twist(V, 0.3))
    desc = dg.CubicLagrangeDiscreteGrid(mn1, mx1, (128, 128, 128))._desc
    nn = C.c_uint64()
    capi.check(capi.lib.dg_grid_num_nodes(desc.resolution, C.byref(nn)))
    nodes = torch.empty(nn.value, dtype=torch.float64, device="cuda")
    cast_d = k9(mdd, X0, step, 0.0, 1.0)

    def deform_mesh():
        capi.check(capi.lib.dg_mesh_refit_device(mdd.handle, V1.data_ptr(), len(V1), st_ptr()))
        return cast_d()

    def deform_field():
        capi.check(capi.lib.dg_mesh_refit_device(mdd.handle, V1.data_ptr(), len(V1), st_ptr()))
        capi.check(capi.lib.dg_sample_sdf_device(mdd.handle, C.byref(desc), 1.0, 0, nn.value, nodes.data_ptr(), st_ptr()))
        f = C.c_void_p()
        capi.check(capi.lib.dg_field_create_device(C.byref(desc), nodes.data_ptr(), nn.value, st_ptr(), C.byref(f)))
        r = k7(f, X0, step, 0.0, 1.0)()
        torch.cuda.synchronize()
        capi.lib.dg_field_destroy(f)
        return r

    cases = {
        "bunny_camera_k9": k9(md, Oc, Dc, 0.0, float("inf")), "bunny_camera_k7_256": k7(fh, Oc, Dc, 0.0, float("inf")),
        "bunny_ccd_k9": k9(md, X0, step, 0.0, 1.0), "bunny_ccd_k7_256": k7(fh, X0, step, 0.0, 1.0),
        "buddha_camera_k9": k9(mdb, Ob, Db, 0.0, float("inf")),
        "deform_refit_k9": deform_mesh, "deform_refit_k1_128_k7": deform_field,
    }
    flush = torch.empty(1 << 25, dtype=torch.float64, device="cuda")
    times = {k: [] for k in cases}
    outs = {}
    for k, fn in cases.items():
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.runs):
        for k, fn in cases.items():
            flush.zero_()
            e0.record()
            outs[k] = fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    rays = {"bunny_camera": (md, V, F, Oc, Dc, float("inf")), "bunny_ccd": (md, V, F, X0, step, 1.0), "buddha_camera": (mdb, Vb, Fb, Ob, Db, float("inf"))}
    for k in cases:
        ms = statistics.median(times[k])
        r = {"median_ms": ms, "spread_ms": [min(times[k]), max(times[k])]}
        base = k.rsplit("_k", 1)[0] if not k.startswith("deform") else None
        if k.endswith("_k9") and base in rays:
            m, Vm, Fm, O, D, t1 = rays[base]
            n = len(O)
            t, tid, b, st = outs[k]
            r.update({"rays": n, "rays_per_s": n / (ms * 1e-3), "hits": int((st != 0).sum())})
            if os.path.exists(EMU):
                idx = torch.randint(0, n, (a.sample,), device="cuda", generator=gen)
                boxes, tris, emu = emu_counts(Vm, Fm, O[idx].cpu().numpy(), D[idx].cpu().numpy(), 0.0, t1)
                same = all(np.array_equal(np.ascontiguousarray(x[idx].cpu().numpy()).view(np.uint8), np.ascontiguousarray(y).view(np.uint8))
                           for x, y in zip((t, tid, b, st), emu))
                r.update({"boxes_per_ray": boxes, "triangles_per_ray": tris, "sample": a.sample, "sample_equals_emulation": bool(same)})
        elif k.endswith("_k7_256"):
            n = len(outs[k][0])
            r.update({"rays": n, "rays_per_s": n / (ms * 1e-3), "hits": int((outs[k][2] != 0).sum())})
        result[k] = r
        extra = "".join(f", {key} {r[key]:.1f}" for key in ("boxes_per_ray", "triangles_per_ray") if key in r)
        rate = f" = {r['rays_per_s'] / 1e6:.1f} M rays/s, {r['hits']} hits" if "rays_per_s" in r else ""
        same = f", sample == emulation: {r['sample_equals_emulation']}" if "sample_equals_emulation" in r else ""
        print(f"{k}: median {ms:.3f} ms ({min(times[k]):.3f}..{max(times[k]):.3f}){rate}{extra}{same}", flush=True)
    if a.out:
        with open(a.out, "w") as fh_:
            json.dump(result, fh_, indent=1)


if __name__ == "__main__":
    main()
