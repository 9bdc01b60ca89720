#!/usr/bin/env python
"""User functions on the GPU: the host route against the one-call route, for an analytic function written in eager torch.

  host   : nodePositions() -> numpy function and sample predicate -> addSampledFunction -> reduceField(numpy predicate)
  device : addReducedFunction(DeviceFunction, DeviceSamplePredicate, DeviceNodePredicate) with the same function in torch

The function is the distance to an off-centre sphere minus its radius, the sample predicate a half-space, the reduce predicate a value
window and a position bound (tests/test_gpu_device_function.py ANALYTIC).  Every run is a fresh process (peak RSS is the process's own);
the routes alternate, and the medians of `--runs` runs are reported with the output digests, which must agree.  The device route's callbacks
synchronise the library's stream before they return, so the time spent in them (the function's GPU work included) is separated from the
library's own stages.  The card's name and power limit are read in the same run.

usage: python tools/device_function_bench.py [--res 256 512] [--runs 3] [--out result.json]"""
import argparse
import hashlib
import json
import os
import resource
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANALYTIC = dict(mn=(-1.0, -1.0, -1.0), mx=(1.0, 1.0, 1.0), centre=(0.13, -0.07, 0.21), r=0.55, c=0.6, vmax=0.02, z0=-0.5)


def digest(g):
    h = hashlib.sha256()
    for a in (g.m_nodes[0], g.m_cells[0], g.m_cell_map[0]):
        h.update(a.tobytes())
    return h.hexdigest()[:16]


def child(route, res):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import discregrid_b200 as dg
    p = ANALYTIC
    torch.zeros(1, device="cuda")
    dg.selftest()
    g = dg.CubicLagrangeDiscreteGrid(p["mn"], p["mx"], (res, res, res))
    out = {"route": route, "res": res}
    t0 = time.perf_counter()
    if route == "host":
        x = g.nodePositions()
        v = np.empty(len(x))
        for b in range(0, len(x), 1 << 24):                      # numpy temporaries of one slice at a time
            xs = x[b:b + (1 << 24)]
            dx, dy, dz = xs[:, 0] - p["centre"][0], xs[:, 1] - p["centre"][1], xs[:, 2] - p["centre"][2]
            v[b:b + len(xs)] = np.where(xs[:, 0] + 0.5 * xs[:, 1] < p["c"], np.sqrt((dx * dx + dy * dy) + dz * dz) - p["r"], dg.DBL_MAX)
        del x
        t1 = time.perf_counter()
        g.addSampledFunction(v)
        del v
        t2 = time.perf_counter()
        g.reduceField(0, lambda x, v: (v <= p["vmax"]) & (x[:, 2] > p["z0"]))
        t3 = time.perf_counter()
        out.update(positions_numpy_s=t1 - t0, add_sampled_s=t2 - t1, reduce_field_s=t3 - t2)
    else:
        def synced(fn):
            def f(*a):
                r = fn(*a)
                torch.cuda.current_stream().synchronize()      # the library's stream (ExternalStream): the callback's own work ends here
                return r
            return f

        def func(x, keep):
            dx, dy, dz = x[:, 0] - p["centre"][0], x[:, 1] - p["centre"][1], x[:, 2] - p["centre"][2]
            return torch.sqrt((dx * dx + dy * dy) + dz * dz) - p["r"]
        g.addReducedFunction(dg.DeviceFunction(synced(func)), dg.DeviceSamplePredicate(synced(lambda x: x[:, 0] + 0.5 * x[:, 1] < p["c"])),
                             dg.DeviceNodePredicate(synced(lambda x, v: (v <= p["vmax"]) & (x[:, 2] > p["z0"]))))
        tm = g.last_reduced_function_ms
        out.update(positions_and_callbacks_s=tm[0] / 1e3, in_callbacks_s=tm[7] / 1e3, cells_s=tm[1] / 1e3, node_compaction_s=tm[2] / 1e3,
                   sort_s=tm[3] / 1e3, write_back_s=tm[4] / 1e3, ties=bool(tm[5]), library_total_s=tm[6] / 1e3)
    out["wall_s"] = time.perf_counter() - t0
    out["survivors"] = len(g.m_nodes[0])
    out["nodes"] = g.nNodes()
    out["digest"] = digest(g)
    out["peak_rss_gb"] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20
    print(json.dumps(out))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out")
    ap.add_argument("--child", nargs=2, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.child[0], int(a.child[1]))
        return
    result = {"card": card(), "cases": []}
    print("card:", result["card"], flush=True)
    for res in a.res:
        runs = {"host": [], "device": []}
        for _ in range(a.runs):
            for route in ("host", "device"):
                r = subprocess.run([sys.executable, __file__, "--child", route, str(res)], capture_output=True, text=True, timeout=3600)
                if r.returncode != 0:
                    raise SystemExit(f"{route} {res}^3 failed:\n{r.stderr[-3000:]}")
                runs[route].append(json.loads(r.stdout.strip().splitlines()[-1]))
        digests = {r["digest"] for rs in runs.values() for r in rs}
        case = {"res": res, "identical": len(digests) == 1}
        for route, rs in runs.items():
            keys = [k for k, v in rs[0].items() if isinstance(v, float)]
            case[route] = {k: statistics.median(r[k] for r in rs) for k in keys}
            case[route]["survivors"] = rs[0]["survivors"]
        case["speedup"] = case["host"]["wall_s"] / case["device"]["wall_s"]
        result["cases"].append(case)
        print(json.dumps(case), flush=True)
    result["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
