#!/usr/bin/env python
"""Parity fuzzer for the density map: the product's K3 kernel code against the oracle's restatement of GenerateDensityMap's node function
(itself pinned to the reference tool's .cdm output) on random small grids.  Kinds, round k % 10 (each within the first 10 rounds):
  0 smooth sphere SDF   1 rough SDF   2 DBL_MAX sentinels   3 reduced SDF input (removed cells, renumbered nodes)
  4 -DBL_MAX coefficients   5 +-1e308 / +-1e306 (64 M / h overflows on fine grids)   6 NaN   7 +-inf, subnormals, -0.0
  8 grid scaled so that h lies just below / above 2^300 or 2^-300, the limits of the fast division
  9 h = +inf or a subnormal h
rho0 cycles through 1000, 0, -1, NaN, +inf, 1, 100; both predicate modes every round; node sub-ranges every third round.  Bit for bit,
any NaN equal to any NaN.

usage: tools/k3_fuzz.py [rounds=40] [seed=0] [lib=build/bin/libk23emu.so]
  lib  a build of tests/emu (libk23emu*.so), or `dg`: the product library through its C-ABI (dg_field_create, dg_density_map) -- needs a GPU
The functions are shared with tests/test_k23_emulated.py and tests/test_gpu_k23_fuzz.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle_api import Oracle  # noqa: E402
from k2_fuzz import DBL_MAX, backend, plant, reduce_layout, same  # noqa: E402,F401

RHO0 = (1000.0, 0.0, -1.0, np.nan, np.inf, 1.0, 100.0)
KINDS = ("smooth", "rough", "sentinel", "reduced", "-DBL_MAX", "huge", "NaN", "inf/subnormal/-0", "h near 2^+-300", "h inf/subnormal")


def make_case(orc, rng, k):
    """round k -> dict(gd, r, nodes, cells, cmap, h, rho0, l0, l1, label)"""
    kind = k % 10
    res = tuple(int(v) for v in (rng.integers(4, 7, 3) if kind in (4, 6) else rng.integers(1, 5, 3)))
    mn = rng.standard_normal(3); mx = mn + 0.5 + rng.random(3) * 2.0
    scale = 1.0
    if kind == 5:                                                                # fine cells: 64 M / h overflows for M = 1e306
        scale = 1e-3
    if kind == 8:                                                                # h = 2^(+-300) (1 -+ 2^-20): scale the grid to it
        e = 300 if (k // 10) % 2 == 0 else -300
        scale = 2.0 ** e
    mn, mx = mn * scale, mx * scale
    gd, r = orc.grid_desc(mn, mx, res)
    cells = orc.build_cells(r)
    n = int(cells.max()) + 1
    x = orc.node_positions(gd, r, 0, n)
    ctr = 0.5 * (mn + mx) + 0.2 * scale * rng.standard_normal(3)
    v = np.linalg.norm(x - ctr, axis=1) - (0.3 + 0.5 * rng.random()) * scale   # signed distance to a sphere
    h = float((0.15 + rng.random() * 2.0) * gd[6:9].min())
    if kind in (4, 6):                                                           # a support over a cell wide on a larger grid: points outside
        h = float((1.2 + rng.random()) * gd[6:9].max())                         # it reach the planted coefficient's cells while points inside do not
    if kind == 1: v += 0.05 * scale * rng.standard_normal(n)
    if kind == 2: v[rng.random(n) < 0.03] = DBL_MAX
    if kind == 4: v[rng.choice(n, size=int(rng.integers(2, 6)), replace=False)] = -DBL_MAX
    if kind == 5:
        at = rng.choice(n, size=4, replace=False)
        v[at] = (1e308, -1e308, 1e306, -1e306)
    if kind == 6: v[rng.choice(n, size=int(rng.integers(1, 4)), replace=False)] = np.nan
    if kind == 7: v = plant(rng, plant(rng, v, "nonfinite", 2), "tiny")
    if kind == 8:
        h = float(np.ldexp(1.0 - 2.0 ** -20 if (k // 20) % 2 == 0 else 1.0 + 2.0 ** -20, 300 if (k // 10) % 2 == 0 else -300))
    if kind == 9:
        h = np.inf if (k // 10) % 2 == 0 else 1e-310
    cmap = np.arange(len(cells), dtype=np.uint32)
    if kind == 3 or (kind in (4, 6) and (k // 10) % 2 == 1):
        v, cells, cmap = reduce_layout(rng, cells, v, 0.7)
    rho0 = RHO0[k % len(RHO0)]
    l0 = int(rng.integers(0, n // 2)) if k % 3 == 0 else 0
    l1 = int(rng.integers(l0 + 1, n + 1)) if k % 3 == 0 else n
    return dict(gd=gd, r=r, nodes=np.ascontiguousarray(v), cells=np.ascontiguousarray(cells), cmap=cmap, h=h, rho0=rho0, l0=l0, l1=l1,
                label=f"case {k} ({KINDS[kind]}) res {res} h {h!r} rho0 {rho0!r}")


def check_case(be, orc, c):
    """both predicate modes -> (nodes checked, mismatches, first mismatch)"""
    f = be.field(c["gd"], c["r"], c["nodes"], c["cells"], c["cmap"])
    total = bad = 0
    first = None
    try:
        for no_red in (0, 1):
            want = orc.density_map(c["gd"], c["r"], c["nodes"], c["h"], c["rho0"], bool(no_red), c["l0"], c["l1"], cells=c["cells"],
                                   cell_map=c["cmap"])
            got = be.density(f, c["h"], c["rho0"], no_red, c["l0"], c["l1"])
            ok = same(got, want)
            total += len(got)
            if not ok.all():
                i = int(np.nonzero(~ok)[0][0]); bad += int((~ok).sum())
                first = first or f"MISMATCH {c['label']} no_reduction {no_red} node {c['l0'] + i}: {got[i]!r} vs {want[i]!r}"
    finally:
        be.destroy(f)
    return total, bad, first


def run(be, rounds, seed, log=print):
    """-> (fields, nodes checked, mismatches)"""
    rng = np.random.default_rng(seed)
    orc = Oracle()
    total = bad = 0
    for k in range(rounds):
        n, b, msg = check_case(be, orc, make_case(orc, rng, k))
        total += n; bad += b
        if msg: log(msg)
    return rounds, total, bad


def main(argv):
    rounds = int(argv[1]) if len(argv) > 1 else 40
    seed = int(argv[2]) if len(argv) > 2 else 0
    lib = argv[3] if len(argv) > 3 else os.path.join(ROOT, "build", "bin", "libk23emu.so")
    fields, total, bad = run(backend(lib), rounds, seed)
    print(f"{fields} fields, {total} nodes, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
