#!/usr/bin/env python
"""Narrow-band K1 against the full node loop on one GPU: dg_sample_sdf_band_device (classifier passes + band node loop, w = `--cells` cell
diagonals) alternated with dg_sample_sdf_device on the same grid, each launch timed with CUDA events after a 256 MiB L2 flush (the policy of
bench.py's headline).  Workloads: bench.py's headline mesh and grid (bunny.obj 128^3 when staged) and its 256^3 target torus (100,000
triangles).  Parity of the same run, at no extra cost: every in-band node equals the full output bit for bit and the nodes set to DBL_MAX are
exactly those with |full| > w.  Reports median and mean over the launches with every launch time (the GPUs are shared: single launches
can be delayed by other work).  Prints one JSON line; writes nothing.

usage: tools/band_bench.py [--steps 12] [--cells 2.0] [--resolution 128] [--target-resolution 256]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12, help="timed launches of each form (alternated)")
    ap.add_argument("--cells", type=float, default=2.0, help="band width in cell diagonals")
    ap.add_argument("--resolution", type=int, default=0, help="headline grid resolution (default: bench.py's)")
    ap.add_argument("--target-resolution", type=int, default=256)
    args = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    import bench
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream()
    sp = C.c_void_p(stream.cuda_stream)

    def timed(fn):
        flush.fill_(1)                                          # L2 flush, outside the event pair
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    def leg(mesh, text, res):
        md = dg.TriangleMeshDistance(mesh)
        mn, mx = dg.generate_sdf_domain(mesh.vertices)
        desc = dg.grid_desc(mn, mx, res)
        n = C.c_uint64(); capi.check(capi.lib.dg_grid_num_nodes(desc.resolution, C.byref(n))); n = n.value
        cell = np.array(desc.cell_size[:])
        w = args.cells * float(np.sqrt((cell * cell).sum()))
        full = torch.empty(n, dtype=torch.float64, device=dev)
        band = torch.empty(n, dtype=torch.float64, device=dev)

        def run_full():
            capi.check(capi.lib.dg_sample_sdf_device(md.handle, C.byref(desc), 1.0, 0, n, C.c_void_p(full.data_ptr()), sp))

        def run_band():
            capi.check(capi.lib.dg_sample_sdf_band_device(md.handle, C.byref(desc), 1.0, w, 0, n, C.c_void_p(band.data_ptr()), sp))
        run_full(); run_band(); torch.cuda.synchronize()
        f_ms, b_ms = [], []
        for _ in range(args.steps):
            f_ms.append(timed(run_full))
            b_ms.append(timed(run_band))
        inb = full.abs() <= w
        out = {"workload": f"{text}, {res[0]}^3 grid ({n} nodes)", "band": w, "band_cell_diagonals": args.cells,
               "band_ms_median": float(np.median(b_ms)), "full_ms_median": float(np.median(f_ms)), "band_ms_mean": float(np.mean(b_ms)),
               "full_ms_mean": float(np.mean(f_ms)), "band_per_launch_ms": b_ms, "full_per_launch_ms": f_ms,
               "speedup_vs_full_median": float(np.median(f_ms)) / float(np.median(b_ms)), "fraction_nodes_in_band": float(inb.double().mean().item()),
               "parity_in_band_bit_exact": bool(torch.equal(band[inb].view(torch.int64), full[inb].view(torch.int64))),
               "parity_dbl_max_outside": bool((band[~inb] == capi.DBL_MAX).all())}
        del full, band, inb
        torch.cuda.empty_cache()
        return out

    hmesh, htext, _ = bench.workload_mesh(dg, bench.WORKLOAD["source"])
    hres = [args.resolution] * 3 if args.resolution else bench.WORKLOAD["resolution"]
    tmesh, ttext, _ = bench.workload_mesh(dg, "target")
    result = {"metric": "narrow-band K1 vs full node loop (CUDA events, L2 flushed, alternated)", "gpu": torch.cuda.get_device_name(0),
              "headline": leg(hmesh, htext, hres), "target": leg(tmesh, ttext, [args.target_resolution] * 3)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
