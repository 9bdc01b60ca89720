#!/usr/bin/env python
"""Differentiable level sets (K13, csrc/k13_isosurface_grad.cu) on one GPU: the forward with edge ids against the forward without them, and
the VJP, on the bunny's 256^3 SDF.

Forward (dg_isosurface_create at s = 1 and 2): this library, which also writes the edge id of every vertex, against a second library built
  from the parent commit (--parent-lib), which does not.  Each round runs one process per library, alternated; a process makes the same
  field through the library's C-ABI, extracts once to warm up and then `--reps` times, and reports the stage times of dg_isosurface_create (host clocks around synchronised
  stages): emit (vertices, edge ids, triangles) and total.  Medians and spreads over rounds x reps.
VJP (the bunny's 256^3 SDF as a trainable field, its vertices at s = 1 and 2, a random upstream):
  s<s>_vjp     : dg_isosurface_vjp_device: the edge-id check (one synchronise), the point and vertex kernels, K2 value-only, K11.
  s<s>_k2      : K2's value-only launch alone at the 2n edge endpoints.
  s<s>_k11     : K11's VJP alone over the same 2n points (dg_interpolate_vjp_device with an upstream of the same size).
  The rest of s<s>_vjp is the check and the two per-vertex kernels.  CUDA events; each timed call is preceded by a write of 256 MiB, which
  flushes the 50 MB L2; the cases are alternated, `--runs` times, and every run's grad_nodes is compared bit for bit with the first run's.
The card's name, power limit and max SM clock are read in the same run.  Needs oracle/_ref/resources (make -C oracle ref).

usage: python tools/isosurface_grad_bench.py --parent-lib <parent libdiscregrid_b200.so> [--runs 5] [--reps 3] [--out result.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

# one library's forward, through its C-ABI alone (the parent's library lacks the symbols the package now declares)
FORWARD = r"""
import ctypes as C, json, sys
import numpy as np
lib = C.CDLL(sys.argv[1])
class GridDesc(C.Structure):
    _fields_ = [("domain_min", C.c_double * 3), ("domain_max", C.c_double * 3), ("resolution", C.c_uint32 * 3), ("_pad", C.c_uint32),
                ("cell_size", C.c_double * 3), ("inv_cell_size", C.c_double * 3)]
vp, dp, up = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_uint32)
lib.dg_grid_init.argtypes = [dp, dp, up, C.POINTER(GridDesc)]
lib.dg_field_create.argtypes = [C.POINTER(GridDesc), dp, C.c_uint64, up, C.c_uint64, up, C.POINTER(vp)]
lib.dg_isosurface_create.argtypes = [vp, C.c_double, C.c_uint32, C.POINTER(vp), dp]
lib.dg_isosurface_destroy.argtypes = [vp]
lib.dg_field_destroy.argtypes = [vp]
z = np.load(sys.argv[2])
mn, mx, res = (np.ascontiguousarray(z[k]) for k in ("mn", "mx", "res"))
nodes, cells, cmap = (np.ascontiguousarray(z[k]) for k in ("nodes", "cells", "cmap"))
desc = GridDesc()
assert lib.dg_grid_init(mn.ctypes.data_as(dp), mx.ctypes.data_as(dp), res.ctypes.data_as(up), C.byref(desc)) == 0
h = vp()
assert lib.dg_field_create(C.byref(desc), nodes.ctypes.data_as(dp), len(nodes), cells.ctypes.data_as(up), len(cells),
                           cmap.ctypes.data_as(up), C.byref(h)) == 0
out = {}
for s in (1, 2):
    ms = []
    for k in range(int(sys.argv[3]) + 1):
        t = np.zeros(5)
        r = vp()
        assert lib.dg_isosurface_create(h, 0.0, s, C.byref(r), t.ctypes.data_as(dp)) == 0
        lib.dg_isosurface_destroy(r)
        if k:
            ms.append([float(t[3]), float(t[4])])
    out[s] = ms
lib.dg_field_destroy(h)
print(json.dumps(out))
"""


def forward_round(lib, npz, reps):
    r = subprocess.run([sys.executable, "-c", FORWARD, lib, npz, str(reps)], capture_output=True, text=True, timeout=1200)
    if r.returncode != 0:
        raise SystemExit(r.stdout + r.stderr)
    return {int(k): v for k, v in json.loads(r.stdout.strip().splitlines()[-1]).items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--grid", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import discregrid_b200 as dg
    from discregrid_b200 import _capi as capi
    import winding_ref as wr
    from mesh_distance_grad_bench import card
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    if not os.path.exists(a.parent_lib):
        raise SystemExit(f"{a.parent_lib} does not exist")
    p = os.path.join(ROOT, "oracle", "_ref", "resources", "bunny.obj")
    if not os.path.exists(p):
        raise SystemExit("bunny.obj is not staged (make -C oracle ref)")
    result = {"card": card(), "runs": a.runs, "reps": a.reps, "grid": a.grid}
    print("card:", result["card"], flush=True)
    dg.selftest()
    V, F = wr.read_obj(p)
    md = dg.TriangleMeshDistance(V, F)
    mn, mx = dg.generate_sdf_domain(V)
    grid = dg.CubicLagrangeDiscreteGrid(mn, mx, (a.grid,) * 3)
    fid = grid.addFunction(dg.MeshSignedDistance(md))

    # ---- forward: this library against the parent's, one process each, alternated
    fw = {(who, s): [] for who in ("new", "parent") for s in (1, 2)}
    with tempfile.TemporaryDirectory() as tmp:
        npz = os.path.join(tmp, "bunny.npz")
        d = grid._desc
        np.savez(npz, mn=np.array(d.domain_min[:]), mx=np.array(d.domain_max[:]), res=np.array(d.resolution[:], np.uint32),
                 nodes=np.asarray(grid.m_nodes[fid], np.float64), cells=np.asarray(grid.m_cells[fid], np.uint32).reshape(-1, 32),
                 cmap=np.asarray(grid.m_cell_map[fid], np.uint32))
        for _ in range(a.runs):
            for who, lib in (("new", capi.LIB_PATH), ("parent", a.parent_lib)):
                for s, ms in forward_round(lib, npz, a.reps).items():
                    fw[(who, s)] += ms
    for (who, s), ms in fw.items():
        emit, tot = [m[0] for m in ms], [m[1] for m in ms]
        r = {"emit_median_ms": statistics.median(emit), "emit_spread_ms": [min(emit), max(emit)],
             "total_median_ms": statistics.median(tot), "total_spread_ms": [min(tot), max(tot)]}
        result[f"forward_{who}_s{s}"] = r
        print(f"forward {who} s={s}: emit median {r['emit_median_ms']:.2f} ms ({min(emit):.2f}..{max(emit):.2f}), total median "
              f"{r['total_median_ms']:.2f} ms ({min(tot):.2f}..{max(tot):.2f})", flush=True)

    # ---- VJP on the trainable field
    f64 = dict(dtype=torch.float64, device="cuda")
    st = lambda: torch.cuda.current_stream().cuda_stream      # noqa: E731
    tf = grid._trainable_field(fid)
    gen = torch.Generator(device="cuda").manual_seed(3)
    d = grid._desc
    lo, hi = torch.tensor(d.domain_min[:], **f64), torch.tensor(d.domain_max[:], **f64)
    cell = torch.tensor(d.cell_size[:], **f64)
    mask = torch.tensor([1, 2, 4, 3, 5, 6, 7], dtype=torch.int64, device="cuda")
    cases, state = {}, {}
    for s in (1, 2):
        Vs, _, E = grid.isosurface(fid, 0.0, s, device=True, coefficients=torch.tensor(grid.m_nodes[fid], **f64), edges=True)
        n = len(E)
        npt = [s * int(r) + 1 for r in d.resolution[:]]
        lp, m = E // 7, mask[E % 7]
        ijk = torch.stack([lp % npt[0], (lp // npt[0]) % npt[1], lp // (npt[0] * npt[1])], 1)
        off = torch.stack([m & 1, (m >> 1) & 1, m >> 2], 1)
        xp = lo + cell * (ijk.double() / s); xq = lo + cell * ((ijk + off).double() / s)
        x = torch.stack([torch.minimum(xp, hi), torch.minimum(xq, hi)], 1).reshape(-1, 3).contiguous()
        state[s] = dict(E=E, gV=torch.randn((n, 3), generator=gen, **f64), gn=torch.empty(tf.n_nodes, **f64), x=x,
                        phi=torch.empty(2 * n, **f64), gphi=torch.randn(2 * n, generator=gen, **f64), gk=torch.empty(tf.n_nodes, **f64))
        result[f"s{s}_vertices"] = n
        print(f"s={s}: {n} vertices", flush=True)

        def vjp(s=s):
            z = state[s]
            capi.check(capi.lib.dg_isosurface_vjp_device(tf.handle, 0.0, s, len(z["E"]), z["E"].data_ptr(), z["gV"].data_ptr(), z["gn"].data_ptr(), st()))

        def k2(s=s):
            z = state[s]
            capi.check(capi.lib.dg_interpolate_batch_device(tf.handle, z["x"].data_ptr(), len(z["x"]), z["phi"].data_ptr(), None, st()))

        def k11(s=s):
            z = state[s]
            capi.check(capi.lib.dg_interpolate_vjp_device(tf.handle, z["x"].data_ptr(), len(z["x"]), z["gphi"].data_ptr(), None, z["gk"].data_ptr(), st()))
        cases[f"s{s}_vjp"] = (vjp, "gn", s)
        cases[f"s{s}_k2"] = (k2, None, s)
        cases[f"s{s}_k11"] = (k11, None, s)
    flush = torch.empty(1 << 25, **f64)
    first = {}
    for k, (fn, chk, s) in cases.items():
        fn()
        torch.cuda.synchronize()
        if chk:
            first[k] = state[s][chk].clone()
    same = {k: True for k in first}
    times = {k: [] for k in cases}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.runs):
        for k, (fn, chk, s) in cases.items():
            flush.zero_()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
            if chk:
                same[k] &= bool(torch.equal(state[s][chk].view(torch.int64), first[k].view(torch.int64)))
    for k in cases:
        med = statistics.median(times[k])
        r = {"median_ms": med, "spread_ms": [min(times[k]), max(times[k])]}
        if k in same:
            r["same_bits_every_run"] = same[k]
        result[k] = r
        extra = f", same bits every run: {r['same_bits_every_run']}" if k in same else ""
        print(f"{k}: median {med:.3f} ms ({min(times[k]):.3f}..{max(times[k]):.3f}){extra}", flush=True)
    for s in (1, 2):
        tot, k2t, k11t = (result[f"s{s}_{c}"]["median_ms"] for c in ("vjp", "k2", "k11"))
        print(f"s={s}: K2 {k2t:.3f} ms, K11 {k11t:.3f} ms, check and per-vertex kernels about {tot - k2t - k11t:.3f} ms of {tot:.3f} ms", flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
