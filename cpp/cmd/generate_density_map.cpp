// GenerateDensityMap -- same command line and output as the reference tool (cmd/generate_density_map/main.cpp:29-171):
//   GenerateDensityMap [-r rho0] [-s h] [-o out.cdm] [--no-reduction] field.cdf
// density_func / gamma / predicate / 16^3 Gauss quadrature run in the K3 kernel; with reduction, K3 and both reduceField calls run in one
// library call (addReducedDensityMap -> dg_reduced_density_map_create), without --no-reduction's dense fields on the host.
#include <Discregrid/All>
#include <cstdlib>
#include <iostream>
#include <string>

using namespace Eigen;

int main(int argc, char* argv[])
{
    double rho0 = 1000.0, h = 0.1;
    bool no_reduction = false;
    std::string output_file, filename;
    for (int a = 1; a < argc; a++) {
        const std::string s = argv[a];
        auto next = [&]() -> std::string { if (a + 1 >= argc) { std::cerr << "missing value for " << s << std::endl; std::exit(1); } return argv[++a]; };
        if (s == "-r" || s == "--rest_density") rho0 = std::stod(next());
        else if (s == "-s" || s == "--smoothing_length") h = std::stod(next());
        else if (s == "-o" || s == "--output") output_file = next();
        else if (s == "--no-reduction") no_reduction = true;
        else if (s == "-i" || s == "--invert") {}                           // declared but never read in the reference (main.cpp:37)
        else if (s == "-h" || s == "--help") { std::cout << "GenerateDensityMap [-r rho0] [-s h] [-o out.cdm] [--no-reduction] field.cdf" << std::endl; return 0; }
        else filename = s;
    }
    if (filename.empty()) { std::cout << "ERROR: No input SDF given." << std::endl; return 1; }
    if (!std::ifstream(filename).good()) { std::cerr << "ERROR: Input file does not exist!" << std::endl; return 1; }
    try {
        std::cout << "Load SDF...";
        Discregrid::CubicLagrangeDiscreteGrid sdf(filename);
        std::cout << "DONE" << std::endl;
        std::cout << "Generate density map..." << std::endl;
        const Discregrid::DensityMapFunction density{&sdf, 0u, h, rho0, no_reduction};
        if (no_reduction) {
            Discregrid::DiscreteGrid::ContinuousFunction func = density;
            sdf.addFunction(func, true);
        } else {
            // addFunction(func, true) + reduceField(0u, -6h < v + cell_diag && v - cell_diag < 2h) + reduceField(1u, 0 <= v && v <= 3 rho0),
            // with cell_diag = sdf.cellSize().norm(), in one library call: the dense density field stays on the GPU
            std::cout << "Reduce discrete fields..." << std::endl;
            sdf.addReducedDensityMap(density, true);
            std::cout << "DONE" << std::endl;
        }
        std::cout << "Serialize discretization...";
        if (output_file.empty()) {
            output_file = filename;
            if (output_file.find(".") != std::string::npos) output_file = output_file.substr(0, output_file.find_last_of("."));
            output_file += ".cdm";
        }
        sdf.save(output_file);
        std::cout << "DONE" << std::endl;
    } catch (std::exception const& e) {
        std::cerr << "error: " << e.what() << std::endl;
        return 1;
    }
    return 0;
}
