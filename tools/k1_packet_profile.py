#!/usr/bin/env python
"""Event counts of the PACKET walk (nearest_triangle_packet) as tests/emu runs it (build/bin/libk1emu.so; `make cpp`), per brick of 32
queries: node steps, leaf visits, exact fp64 blocks, re-tests of deferred children, how the reference's choice was replayed (no order needed /
tie shortcut / sort), comparator calls, and which check sent lanes to the per-lane fallback -- plus a bit-for-bit comparison of the output with
the per-lane emulated build (libk1emu_perlane.so) over the same node range.  The event figures quoted in DESIGN.md section 4 come from here.
A node range should cover whole brick layers (multiples of 4 planes of the vertex array): bricks cut by the range run half empty and the
"per brick" figures (events / (nodes / 32)) double.
usage: tools/k1_packet_profile.py resolution [mesh.obj|torus] [l_begin l_end]"""
import ctypes as C, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import discregrid_b200 as dg
import bench
from oracle_api import Oracle
res = int(sys.argv[1]); 
mesh = dg.TriangleMesh(sys.argv[2]) if len(sys.argv) > 2 and sys.argv[2] != "torus" else dg.bumpy_torus(*bench.WORKLOAD["torus"])
lib = C.CDLL(os.path.join(ROOT, "build", "bin", "libk1emu.so"))
ref = C.CDLL(os.path.join(ROOT, "build", "bin", "libk1emu_perlane.so"))       # the per-lane walk: an independent implementation
dp, u32p = C.POINTER(C.c_double), C.POINTER(C.c_uint32)
orc = Oracle()
V = np.ascontiguousarray(mesh.vertices, np.float64); F = np.ascontiguousarray(mesh.faces, np.uint32)
mn, mx = orc.generate_sdf_domain(V)
gd, r = orc.grid_desc(mn, mx, (res,) * 3)
nn = (res + 1) ** 3 + 2 * 3 * res * (res + 1) ** 2
L0 = int(sys.argv[3]) if len(sys.argv) > 3 else 0; L1 = int(sys.argv[4]) if len(sys.argv) > 4 else nn
nn = L1 - L0
outs=[]
for L in (lib, ref):
    L.emu_mesh_create.restype = C.c_void_p
    L.emu_mesh_create.argtypes = [dp, C.c_uint64, u32p, C.c_uint64]
    L.emu_sample_sdf.argtypes = [C.c_void_p, dp, u32p, C.c_double, C.c_uint64, C.c_uint64, dp]
    h = L.emu_mesh_create(V.ctypes.data_as(dp), len(V), F.ctypes.data_as(u32p), len(F))
    out = np.empty(nn)
    cnt = (C.c_ulonglong * 32)()
    L.emu_counters(cnt, 1)
    t=time.time()
    assert L.emu_sample_sdf(h, gd.ctypes.data_as(dp), r.ctypes.data_as(u32p), 1.0, L0, L1, out.ctypes.data_as(dp)) == 0
    dt=time.time()-t
    L.emu_counters(cnt, 1)
    c = [int(x) for x in cnt]
    outs.append(out)
    if L is lib:
        B = nn/32.0
        # counters are incremented per lane (each fiber executes the statement) -> divide by 32 for warp-level events
        print(f"{len(F)} tri, {res}^3, {nn} nodes, {dt:.1f}s")
        print(f"per brick: pops {c[16]/32/B:.1f} (hit {c[17]/32/B:.1f})  leaf filter steps {c[18]/32/B:.1f}  exact blocks {c[19]/32/B:.1f}  exact lanes {c[20]/B:.1f}  node steps {c[21]/32/B:.1f}")
        print(f"tie-shortcut lanes {c[26]/nn*100:.2f} % ({c[27]/max(1,c[26]):.2f} compares each); sorted lanes {c[22]/nn*100:.2f} % of queries, swaps {c[23]}; fallback warps {c[24]/32/B*100:.2f} %  fallback lanes {c[25]/nn*100:.3f} %")
        print(f"comparator calls per brick (max over lanes): {c[28]/B:.2f}"); print(f"fallback reasons (lanes): on-surface {c[15]}  dropped-in-closure {c[29]}  wide closure {c[30]}  certificate {c[31]}"); print("per-lane counters inside fallback: iterations", c[0]/32/B, "per brick")
print("bit-identical:", np.array_equal(outs[0].view(np.uint64), outs[1].view(np.uint64)), "mismatches", int((outs[0].view(np.uint64)!=outs[1].view(np.uint64)).sum()))
