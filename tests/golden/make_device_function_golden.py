"""Fixtures for user functions on the GPU (dg_add_function_device, dg_reduced_function_create, dg_reduce_field_device), made by the
reference's own grid class: a small program (written to a temporary directory, compiled against the reference's unmodified library sources
with the flags of oracle/Makefile) runs

    g.addFunction(func, false, pred);  g.reduceField(0, pred2);  g.save(out);

with analytic lambdas that numpy and eager torch reproduce operation for operation:

    func(x)     = std::sqrt((dx*dx + dy*dy) + dz*dz) - r,   d = x - centre     (an off-centre sphere's distance)
    pred(x)     = x[0] + 0.5*x[1] < c                                          (a sample predicate that depends on the position)
    pred2(x, v) = v <= vmax && x[2] > z0                                       (a reduce predicate on the value and the position)

Every parameter is written as a hex float, so the tests use the same doubles.  Writes ref_devfn_*.cdf and ref_devfn_cases.json next to
this file.

The program is compiled with the compiler, flags, include paths and reference library sources that oracle/Makefile uses for the reference's
grid class (read from that Makefile), so the two builds cannot drift apart.

usage: python tests/golden/make_device_function_golden.py      (after `make -C oracle ref`, which needs the reference's sources)"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

# name -> grid, function parameters, whether pred / pred2 are used
CASES = {
    # anisotropic cells (the Z-curve key quantises with the largest cell, so survivors share keys) with both predicates
    "aniso_reduced": dict(mn=(-1.0, -0.7, -0.4), mx=(1.2, 0.9, 0.5), res=(19, 6, 11), centre=(0.15, 0.05, 0.02), r=0.6, c=0.7, vmax=0.2, z0=-0.25,
                          sample=True, reduce=True),
    # the dense field of addFunction(func, false, pred): DBL_MAX where x0 + 0.5 x1 >= c
    "dense_sampled": dict(mn=(-1.0, -1.0, -1.0), mx=(1.0, 1.0, 1.0), res=(7, 5, 6), centre=(0.1, -0.2, 0.05), r=0.5, c=0.3, vmax=0.0, z0=0.0,
                          sample=True, reduce=False),
    # no sample predicate, reduced
    "box_reduced": dict(mn=(0.0, 0.0, 0.0), mx=(1.0, 2.0, 1.5), res=(6, 9, 7), centre=(0.4, 1.1, 0.7), r=0.45, c=0.0, vmax=0.05, z0=0.3,
                        sample=False, reduce=True),
}

PROGRAM = r"""
#include <cmath>
#include <cstdlib>
#include <string>
#include <Eigen/Dense>
#include <Discregrid/All>
using Eigen::Vector3d;
int main(int argc, char** argv)
{
    if (argc != 20) return 2;
    double a[16];
    for (int i = 0; i < 16; i++) a[i] = std::strtod(argv[2 + i], nullptr);    // mn[3] mx[3] res[3] centre[3] r c vmax z0
    const bool sample = argv[18][0] == '1', reduce = argv[19][0] == '1';
    Eigen::AlignedBox3d domain(Vector3d(a[0], a[1], a[2]), Vector3d(a[3], a[4], a[5]));
    std::array<unsigned int, 3> res = {{(unsigned)a[6], (unsigned)a[7], (unsigned)a[8]}};
    const double cx = a[9], cy = a[10], cz = a[11], r = a[12], c = a[13], vmax = a[14], z0 = a[15];
    Discregrid::CubicLagrangeDiscreteGrid g(domain, res);
    auto func = [&](Vector3d const& x) {
        const double dx = x[0] - cx, dy = x[1] - cy, dz = x[2] - cz;
        return std::sqrt((dx * dx + dy * dy) + dz * dz) - r;
    };
    Discregrid::DiscreteGrid::SamplePredicate pred = nullptr;
    if (sample) pred = [&](Vector3d const& x) { return x[0] + 0.5 * x[1] < c; };
    g.addFunction(func, false, pred);
    if (reduce) g.reduceField(0, [&](Vector3d const& x, double v) { return v <= vmax && x[2] > z0; });
    g.save(std::string(argv[1]));
    return 0;
}
"""


def oracle_make_var(name):
    """a variable of oracle/Makefile as that Makefile defines it, so that this program is built exactly as the reference's library there"""
    r = subprocess.run(["make", "-s", "--no-print-directory", "-f", os.path.join(ROOT, "oracle", "Makefile"), "--eval", "print-%: ; @echo $($*)",
                        f"print-{name}"], capture_output=True, text=True, check=True)
    return r.stdout.split()


def build(tmp):
    src = os.path.join(tmp, "devfn_golden.cpp")
    with open(src, "w") as f:
        f.write(PROGRAM)
    exe = os.path.join(tmp, "devfn_golden")
    # compiler, flags, include paths (the Eigen stand-in, the reference's headers, oracle/_ref/gen) and library sources of oracle/Makefile
    cmd = oracle_make_var("CXX") + oracle_make_var("REFFLAGS") + oracle_make_var("REFINC") + ["-o", exe, src] + oracle_make_var("REFLIBSRC")
    subprocess.run(cmd, check=True)
    return exe


def main():
    meta = {}
    with tempfile.TemporaryDirectory() as tmp:
        exe = build(tmp)
        for name, case in CASES.items():
            out = os.path.join(HERE, f"ref_devfn_{name}.cdf")
            vals = [*case["mn"], *case["mx"], *case["res"], *case["centre"], case["r"], case["c"], case["vmax"], case["z0"]]
            args = [float.hex(float(v)) for v in vals] + ["1" if case["sample"] else "0", "1" if case["reduce"] else "0"]
            subprocess.run([exe, out] + args, check=True)
            meta[name] = dict(case, file=os.path.basename(out))
            print(name, out, os.path.getsize(out), "bytes", file=sys.stderr)
    with open(os.path.join(HERE, "ref_devfn_cases.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
