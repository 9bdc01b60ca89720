#!/usr/bin/env python
"""Times the refit (dg_mesh_refit_device, K8) against a rebuild (dg_mesh_create: host build + upload) on the reference meshes twisted about y,
and what the refit's looser tree costs afterwards: the K1 node loop at 128^3 and 10 M near-surface signed_distance queries on the refit mesh
vs the freshly built one.  CUDA events with warm-up and medians; the card name and power limit are read in the same run.  Outputs at the
timed sizes are checked against the reference's rule over the exported refit tree (build/bin/liborctree.so) on a strided sample, and one
torch.profiler run counts the host<->device copies of the device form.  usage: tools/refit_bench.py [--reps 7] [--queries 10000000]"""
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
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def twist(V, angle):
    lo, hi = V[:, 1].min(), V[:, 1].max()
    t = angle * (V[:, 1] - lo) / (hi - lo)
    c, s = np.cos(t), np.sin(t)
    return np.stack([c * V[:, 0] + s * V[:, 2], V[:, 1], -s * V[:, 0] + c * V[:, 2]], 1)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def events_ms(fn, reps, warm=2):
    import torch
    for _ in range(warm):
        fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--queries", type=int, default=10_000_000)
    ap.add_argument("--meshes", default="bunny.obj,dragon.obj,happy_buddha.obj")
    args = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    import winding_ref as wr
    from test_gpu_refit import TreeOracle
    from oracle_api import Oracle
    orc = Oracle()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit_w": pl}))
    for mesh in args.meshes.split(","):
        V, F = wr.read_obj(os.path.join(ROOT, "oracle", "_ref", "resources", mesh))
        for angle in (0.0, 0.1, 0.5, 1.5):
            V1 = twist(V, angle)
            Vt = torch.from_numpy(V1).cuda()
            md = dg.TriangleMeshDistance(V, F)
            st = torch.cuda.current_stream().cuda_stream
            refit = lambda: capi.check(capi.lib.dg_mesh_refit_device(md.handle, Vt.data_ptr(), len(V1), st))
            t_refit, t_build = [], []
            for _ in range(args.reps):                         # alternated
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); refit(); b.record(); b.synchronize(); t_refit.append(a.elapsed_time(b))
                t0 = time.perf_counter(); fresh = dg.TriangleMeshDistance(V1, F); torch.cuda.synchronize()
                t_build.append(1e3 * (time.perf_counter() - t0))
            mn, mx = dg.generate_sdf_domain(V1)
            gd, res = orc.grid_desc(mn, mx, (128, 128, 128))
            nn = orc.num_nodes(res)
            desc = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))._desc
            out = torch.empty(nn, dtype=torch.float64, device="cuda")
            k1 = {}
            for tag, m in (("refit", md), ("fresh", fresh)):
                k1[tag] = events_ms(lambda: capi.check(capi.lib.dg_sample_sdf_device(m.handle, C.byref(desc), 1.0, 0, nn, out.data_ptr(), st)),
                                    max(3, args.reps // 2))
            ids = np.arange(0, nn, 997, dtype=np.uint64)
            ref = TreeOracle(md, V1, F)
            want = ref.distance(orc.node_positions_at(gd, res, ids), True)[0]
            capi.check(capi.lib.dg_sample_sdf_device(md.handle, C.byref(desc), 1.0, 0, nn, out.data_ptr(), st))
            ok_grid = bool(np.array_equal(out.cpu().numpy()[ids.astype(np.int64)].view(np.uint64), want.view(np.uint64)))
            rng = np.random.default_rng(0)
            x = V1[rng.integers(0, len(V1), args.queries)] + rng.normal(0, 1e-3 * float(np.ptp(V1)), (args.queries, 3))
            xt = torch.from_numpy(x).cuda()
            q = {}
            for tag, m in (("refit", md), ("fresh", fresh)):
                q[tag] = events_ms(lambda: m.signed_distance(xt), max(3, args.reps // 2))
            d = md.signed_distance(xt).distance.cpu().numpy()
            s = np.arange(0, args.queries, 4999)
            ok_q = bool(np.array_equal(d[s].view(np.uint64), ref.distance(x[s], True)[0].view(np.uint64)))
            ref.close()
            print(json.dumps({"mesh": mesh, "triangles": len(F), "twist_rad": angle, "refit_ms": statistics.median(t_refit),
                              "dg_mesh_create_ms": statistics.median(t_build), "k1_128_ms": k1, "queries": args.queries,
                              "signed_distance_ms": q, "grid_equals_reference_rule_over_refit_tree": ok_grid,
                              "queries_equal_reference_rule_over_refit_tree": ok_q}), flush=True)
            del fresh
    # host<->device copies of one device-form refit
    V, F = wr.read_obj(os.path.join(ROOT, "oracle", "_ref", "resources", "bunny.obj"))
    md = dg.TriangleMeshDistance(V, F)
    Vt = torch.from_numpy(twist(V, 0.5)).cuda()
    md.refit(Vt)
    torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        md.refit(Vt)
        torch.cuda.synchronize()
    copies = [(e.name, e.device_type.name) for e in prof.events() if "Memcpy" in e.name and ("HtoD" in e.name or "DtoH" in e.name)]
    print(json.dumps({"profiler_host_device_copies_of_one_refit": len(copies), "names": sorted(set(n for n, _ in copies))}))


if __name__ == "__main__":
    main()
