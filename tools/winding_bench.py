#!/usr/bin/env python
"""The winding sign mode (K5, csrc/k5_winding.cu) against the pseudonormal mode, on the device entry points.

  winding  : dg_mesh_winding_number_device on 10 M uniform points in the 10 %-padded bounding box of bunny.obj and happy_buddha.obj (beta = 2),
             CUDA tensors in and out; plus the one-time host build + upload of the records (first use).
  nodes    : the bunny 128^3 node loop, dg_sample_sdf_device in the pseudonormal mode (K1) and in the winding mode (K1 with sign = +1, then the
             node pass), alternated.
  reduced  : dg_reduced_band_create on the 512^3 bunny with a band of 2 cell diagonals, both modes alternated (host clock around the call,
             which ends with a device synchronise).
  accuracy : max |w(beta=2) - w(inf)| and sign disagreements (w > 0.5) on 20,000 points (15,000 uniform in the padded box, 5,000 within 1e-3
             of the diagonal from a vertex) of bunny, the open bunny (top 15 % of its y-extent cut away) and happy_buddha; and how many of the
             uniform points the pseudonormal sign gets wrong against w(inf) > 0.5 where |w(inf) - 0.5| > 0.15.
Device work is timed with CUDA events around each launch after a 256 MB write that flushes the 50 MB L2; medians of `--runs`.  The card's
name, power limit and max SM clock are read in the same run.  Needs oracle/_ref/resources (make -C oracle ref).

usage: python tools/winding_bench.py [--runs 5] [--points 10000000] [--out result.json]"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--out")
    a = ap.parse_args()
    import ctypes as C
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    import winding_ref as wr
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res_dir = os.path.join(ROOT, "oracle", "_ref", "resources")
    if not os.path.exists(os.path.join(res_dir, "bunny.obj")):
        raise SystemExit(f"{res_dir} is not staged (make -C oracle ref)")
    result = {"card": card(), "runs": a.runs}
    print("card:", result["card"], flush=True)
    dg.selftest()
    stream = torch.cuda.current_stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def timed(fn):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream); fn(); e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    meshes = {n: wr.read_obj(os.path.join(res_dir, n + ".obj")) for n in ("bunny", "happy_buddha")}
    meshes["open_bunny"] = wr.cut_top(*meshes["bunny"])

    # ---- winding-number throughput
    for name in ("bunny", "happy_buddha"):
        V, F = meshes[name]
        md = dg.TriangleMeshDistance(V, F)
        x = torch.from_numpy(wr.query_points(V, a.points, seed=1)).cuda()
        w = torch.empty(a.points, dtype=torch.float64, device="cuda")
        t0 = time.perf_counter()
        md.winding_number(np.zeros((1, 3)))                       # first use: host build + upload of the records
        first_ms = (time.perf_counter() - t0) * 1e3

        def run():
            capi.check(capi.lib.dg_mesh_winding_number_device(md.handle, x.data_ptr(), a.points, 2.0, w.data_ptr(), stream.cuda_stream))
        run(); torch.cuda.synchronize()
        ms = statistics.median(timed(run) for _ in range(a.runs))
        result[f"winding_{name}"] = {"triangles": len(F), "points": a.points, "ms": ms, "Gq_s": a.points / ms / 1e6, "first_use_ms": first_ms}
        print(f"winding_number {name} ({len(F)} tri): {ms:.2f} ms for {a.points} points = {a.points / ms / 1e6:.3f} Gq/s; "
              f"records built + uploaded at first use in {first_ms:.0f} ms", flush=True)
        del x, w

    # ---- the 128^3 node loop, both modes
    V, F = meshes["bunny"]
    md = dg.TriangleMeshDistance(V, F)
    mn, mx = dg.generate_sdf_domain(V)
    g = dg.CubicLagrangeDiscreteGrid(mn, mx, (128, 128, 128))
    n = g.nNodes()
    out = {m: torch.empty(n, dtype=torch.float64, device="cuda") for m in ("pseudonormal", "winding")}

    def sample(mode):
        def run():
            capi.check(capi.lib.dg_sample_sdf_device(md.handle, C.byref(g._desc), 1.0, 0, n, C.c_void_p(out[mode].data_ptr()), stream.cuda_stream))
        return run
    times = {"pseudonormal": [], "winding": []}
    for mode in ("pseudonormal", "winding"):
        md.set_sign_mode(mode); sample(mode)(); torch.cuda.synchronize()
    for _ in range(a.runs):
        for mode in ("pseudonormal", "winding"):
            md.set_sign_mode(mode)
            times[mode].append(timed(sample(mode)))
    md.set_sign_mode("pseudonormal")
    a_p, a_w = out["pseudonormal"].cpu().numpy(), out["winding"].cpu().numpy()
    nz = a_p != 0.0
    same = bool(np.array_equal(a_p.view(np.uint64)[nz], a_w.view(np.uint64)[nz]))
    tp, tw = statistics.median(times["pseudonormal"]), statistics.median(times["winding"])
    result["nodes_bunny_128"] = {"nodes": n, "pseudonormal_ms": tp, "winding_ms": tw, "node_pass_ms": tw - tp, "equal_bits_nonzero": same}
    print(f"bunny 128^3 node loop ({n} nodes): pseudonormal {tp:.2f} ms, winding {tw:.2f} ms (node pass ~{tw - tp:.2f} ms); "
          f"equal bits at nonzero nodes: {same}", flush=True)
    del out

    # ---- the 512^3 reduced band, both modes
    g5 = dg.CubicLagrangeDiscreteGrid(mn, mx, (512, 512, 512))
    band = 2.0 * float(np.linalg.norm(g5.m_cell_size))
    times = {"pseudonormal": [], "winding": []}
    sizes = {}
    for rep in range(max(2, a.runs // 2) + 1):
        for mode in ("pseudonormal", "winding"):
            md.set_sign_mode(mode)
            h = C.c_void_p()
            tm = np.zeros(7)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            capi.check(capi.lib.dg_reduced_band_create(md.handle, C.byref(g5._desc), 1.0, band, 0, C.byref(h), capi.ptr(tm, capi.F64P)))
            t = (time.perf_counter() - t0) * 1e3
            nn, nc = C.c_uint64(), C.c_uint64()
            capi.check(capi.lib.dg_reduced_band_sizes(h, C.byref(nn), C.byref(nc)))
            sizes[mode] = (nn.value, nc.value)
            capi.lib.dg_reduced_band_destroy(h)
            if rep > 0:
                times[mode].append((t, tm[0]))
    md.set_sign_mode("pseudonormal")
    rp = statistics.median(t for t, _ in times["pseudonormal"]); rw = statistics.median(t for t, _ in times["winding"])
    sp = statistics.median(s for _, s in times["pseudonormal"]); sw = statistics.median(s for _, s in times["winding"])
    result["reduced_bunny_512"] = {"pseudonormal_ms": rp, "winding_ms": rw, "sampling_pseudonormal_ms": sp, "sampling_winding_ms": sw,
                                   "kept_nodes": sizes["pseudonormal"][0], "same_sizes": sizes["pseudonormal"] == sizes["winding"]}
    print(f"bunny 512^3 reduced band: pseudonormal {rp:.0f} ms (sampling {sp:.0f}), winding {rw:.0f} ms (sampling {sw:.0f}); "
          f"{sizes['pseudonormal'][0]} nodes kept, same sizes: {sizes['pseudonormal'] == sizes['winding']}", flush=True)

    # ---- accuracy of the far field at beta = 2
    for name in ("bunny", "open_bunny", "happy_buddha"):
        V, F = meshes[name]
        md = dg.TriangleMeshDistance(V, F)
        p = wr.query_points(V, 15000, seed=2, near=5000)
        w_inf, w2 = md.winding_number(p, math.inf), md.winding_number(p, 2.0)
        err = float(np.max(np.abs(w2 - w_inf)))
        flips = int(np.sum((w2 > 0.5) != (w_inf > 0.5)))
        d_pn = md.signed_distance(p[:15000]).distance
        clear = np.abs(w_inf[:15000] - 0.5) > 0.15
        pn_wrong = int(np.sum(((d_pn < 0) != (w_inf[:15000] > 0.5)) & clear))
        result[f"accuracy_{name}"] = {"max_err_beta2": err, "sign_flips_beta2": flips, "pseudonormal_wrong_of_15000": pn_wrong,
                                      "borderline": int(np.sum(~clear))}
        print(f"{name}: max |w(2) - w(inf)| = {err:.4g}, sign flips at beta 2: {flips} / 20000; pseudonormal sign wrong at {pn_wrong} of 15000 "
              f"uniform points ({int(np.sum(~clear))} borderline)", flush=True)

    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
