// GenerateVolumeMap -- the volume map of Bender et al. 2019 (SPlisHSPlasH's SPH boundary representation) of an SDF, with the command line
// and the structure of GenerateDensityMap:
//   GenerateVolumeMap [-s h] [--scale s] [-o out.cdm] [--no-reduction] field.cdf
// The volume function, GenerateDensityMap's sample predicate and the 16^3 Gauss quadrature run in K3's volume-map kernel.  With reduction,
// the volume map and reduceField(0, p0) + reduceField(1, 0 <= v) run in one library call (addReducedVolumeMap ->
// dg_reduced_volume_map_create), without the dense fields on the host.
#include <Discregrid/All>
#include <cstdlib>
#include <iostream>
#include <string>

using namespace Eigen;

int main(int argc, char* argv[])
{
    double h = 0.1, scale = 0.8;
    bool no_reduction = false;
    std::string output_file, filename;
    for (int a = 1; a < argc; a++) {
        const std::string s = argv[a];
        auto next = [&]() -> std::string { if (a + 1 >= argc) { std::cerr << "missing value for " << s << std::endl; std::exit(1); } return argv[++a]; };
        if (s == "-s" || s == "--smoothing_length") h = std::stod(next());
        else if (s == "--scale") scale = std::stod(next());
        else if (s == "-o" || s == "--output") output_file = next();
        else if (s == "--no-reduction") no_reduction = true;
        else if (s == "-h" || s == "--help") { std::cout << "GenerateVolumeMap [-s h] [--scale s] [-o out.cdm] [--no-reduction] field.cdf" << std::endl; return 0; }
        else filename = s;
    }
    if (filename.empty()) { std::cout << "ERROR: No input SDF given." << std::endl; return 1; }
    if (!std::ifstream(filename).good()) { std::cerr << "ERROR: Input file does not exist!" << std::endl; return 1; }
    try {
        std::cout << "Load SDF...";
        Discregrid::CubicLagrangeDiscreteGrid sdf(filename);
        std::cout << "DONE" << std::endl;
        std::cout << "Generate volume map..." << std::endl;
        const Discregrid::VolumeMapFunction volume(&sdf, 0u, h, scale, no_reduction);
        if (no_reduction) {
            Discregrid::DiscreteGrid::ContinuousFunction func = volume;
            sdf.addFunction(func, true);
        } else {
            // addFunction(func, true) + reduceField(0u, -6h < v + cell_diag && v - cell_diag < 2h) + reduceField(1u, 0 <= v), with
            // cell_diag = sdf.cellSize().norm(), in one library call: the dense volume field stays on the GPU
            std::cout << "Reduce discrete fields..." << std::endl;
            sdf.addReducedVolumeMap(volume, true);
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
