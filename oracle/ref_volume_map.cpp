// oracle/ref_volume_map.cpp -- TEST INFRASTRUCTURE: a reference-side volume-map generator.  The reference has no volume map; this tool
// states the library's volume-map contract (DESIGN section 3, "Volume map") as lambdas over the reference's OWN building blocks, compiled
// from its unmodified sources by oracle/ref_volume.mk: its CubicLagrangeDiscreteGrid (loaded from the .cdf, interpolate, addFunction,
// reduceField, save), GenerateDensityMap's GaussQuadrature::integrate and CubicKernel.  Its .cdm output is what GenerateVolumeMap must
// write byte for byte (tests/golden/make_volume_golden.py).
//   RefGenerateVolumeMap [-s h] [--scale s] [-o out.cdm] [--no-reduction] field.cdf
#include <Discregrid/All>
#include <Eigen/Dense>

#include <cstdlib>
#include <fstream>
#include <iostream>
#include <limits>
#include <memory>
#include <string>

#include "sph_kernel.hpp"
#include "gauss_quadrature.hpp"

using namespace Eigen;

int main(int argc, char* argv[])
{
    double h = 0.1, scale = 0.8;
    bool no_reduction = false;
    std::string output_file, filename;
    for (int a = 1; a < argc; a++) {
        const std::string s = argv[a];
        if ((s == "-s" || s == "--scale" || s == "-o") && a + 1 >= argc) { std::cerr << "missing value for " << s << std::endl; return 1; }
        if (s == "-s") h = std::stod(argv[++a]);
        else if (s == "--scale") scale = std::stod(argv[++a]);
        else if (s == "-o") output_file = argv[++a];
        else if (s == "--no-reduction") no_reduction = true;
        else filename = s;
    }
    if (filename.empty() || !std::ifstream(filename).good()) { std::cerr << "ERROR: no input SDF" << std::endl; return 1; }

    auto sdf = std::unique_ptr<Discregrid::CubicLagrangeDiscreteGrid>(new Discregrid::CubicLagrangeDiscreteGrid(filename));

    CubicKernel kernel;
    kernel.setRadius(h);
    const double w_zero = kernel.W(Vector3d::Zero());
    // gamma: 1 inside, the kernel ramp over the first smoothing length outside, 0 beyond (and for DBL_MAX / NaN)
    auto gamma = [&](double d) -> double {
        if (d <= 0.0) return 1.0;
        if (d < h) return kernel.W(Vector3d(d, 0.0, 0.0)) / w_zero;
        return 0.0;
    };
    const AlignedBox3d int_domain(Vector3d::Constant(-h), Vector3d::Constant(h));
    auto volume_func = [&](Vector3d const& x) -> double {
        const double dist = sdf->interpolate(0u, x);
        if (dist > (1.0 + 1.0) * h) return 0.0;
        auto integrand = [&](Vector3d const& xi) -> double {
            if (xi.squaredNorm() > h * h) return 0.0;
            return gamma(sdf->interpolate(0u, x + xi));
        };
        return scale * GaussQuadrature::integrate(integrand, int_domain, 30);
    };

    const double cell_diag = sdf->cellSize().norm();
    sdf->addFunction(volume_func, false, [&](Vector3d const& x_) {
        if (no_reduction) return true;
        const Vector3d x = x_.cwiseMax(sdf->domain().min()).cwiseMin(sdf->domain().max());
        const double dist = sdf->interpolate(0u, x);
        if (dist == std::numeric_limits<double>::max()) return false;
        return -6.0 * h < dist + cell_diag && dist - cell_diag < 2.0 * h;
    });
    if (!no_reduction) {
        sdf->reduceField(0u, [&](Vector3d const&, double v) { return -6.0 * h < v + cell_diag && v - cell_diag < 2.0 * h; });
        sdf->reduceField(1u, [&](Vector3d const&, double v) { return 0.0 <= v; });
    }
    if (output_file.empty()) {
        output_file = filename.substr(0, filename.find_last_of('.')) + ".cdm";
    }
    sdf->save(output_file);
    return 0;
}
