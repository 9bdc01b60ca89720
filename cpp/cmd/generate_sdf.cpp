// GenerateSDF -- same command line and output as the reference tool (cmd/generate_sdf/main.cpp:28-130), sampling on the GPU.
//   GenerateSDF [-r "nx ny nz"] [-d "minx miny minz maxx maxy maxz"] [-i] [-o out.cdf] [--gpus N] [--band W [--no-reduction]]
//               [--sign pseudonormal|winding] input.obj
// --gpus N (new, SURVEY 5 "same flags + --gpus N"): the node loop is dealt to N GPUs of this node (dg_add_function_sdf_multi); same file.
// --band W (new): a narrow-band field -- addFunction(func, verbose, pred) with pred(x) = |distance(x)| <= W (world units), DBL_MAX
//   elsewhere, then reduceField with an always-true predicate (drops the DBL_MAX nodes and the cells without a kept node), as
//   GenerateDensityMap does (cmd/generate_density_map/main.cpp:119-147) -- both in one call (addReducedBandField), so that only the reduced
//   field reaches the host.  --no-reduction keeps the dense field (addFunction with the band predicate).  One GPU only.
// --sign pseudonormal|winding (new): where the distances take their sign from.  pseudonormal (default) is the reference's rule, right for
//   closed manifold meshes; winding uses the generalized winding number (inside iff w > 0.5) for open or non-manifold meshes.  One GPU only.
// The one functional change against the reference source: the functor handed to addFunction is the recognisable
// MeshSignedDistanceFunction instead of an anonymous lambda (main.cpp:94-102).
#include <Discregrid/All>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

using namespace Eigen;

int main(int argc, char* argv[])
{
    std::array<unsigned int, 3> resolution = {{10, 10, 10}};               // reference default "10 10 10"
    std::string domain_str, output_file, filename;
    bool invert = false;
    int n_gpus = 1;
    bool use_band = false, no_reduction = false;
    std::string sign_mode = "pseudonormal";
    double band = 0.0;
    for (int a = 1; a < argc; a++) {
        const std::string s = argv[a];
        auto next = [&]() -> std::string { if (a + 1 >= argc) { std::cerr << "missing value for " << s << std::endl; std::exit(1); } return argv[++a]; };
        if (s == "-h" || s == "--help") {
            std::cout << "Generates a signed distance field from a closed two-manifold triangle mesh.\n"
                         "  -r, --resolution \"nx ny nz\"   -d, --domain \"minx miny minz maxx maxy maxz\"   -i, --invert   -o, --output file.cdf   --gpus N\n"
                         "  --band W   keep only nodes within distance W of the surface (others DBL_MAX), then reduce the field\n"
                         "  --no-reduction   with --band: keep the dense field (no reduceField)\n"
                         "  --sign pseudonormal|winding   sign from the pseudonormal (default; closed meshes) or the generalized winding number\n"
                         "Example: GenerateSDF -r \"50 50 50\" dragon.obj" << std::endl;
            return 0;
        } else if (s == "-r" || s == "--resolution") { std::istringstream is(next()); is >> resolution[0] >> resolution[1] >> resolution[2]; }
        else if (s == "-d" || s == "--domain") domain_str = next();
        else if (s == "-i" || s == "--invert") invert = true;
        else if (s == "-o" || s == "--output") output_file = next();
        else if (s == "--gpus") n_gpus = std::atoi(next().c_str());
        else if (s == "--band") { use_band = true; band = std::strtod(next().c_str(), nullptr); }
        else if (s == "--no-reduction") no_reduction = true;
        else if (s == "--sign") sign_mode = next();
        else filename = s;
    }
    if (filename.empty()) { std::cout << "ERROR: No input mesh given." << std::endl; return 1; }
    if (!std::ifstream(filename).good()) { std::cerr << "ERROR: Input file does not exist!" << std::endl; return 1; }
    if (use_band && n_gpus > 1) { std::cerr << "ERROR: --band runs on one GPU; it cannot be combined with --gpus " << n_gpus << std::endl; return 1; }
    if (sign_mode != "pseudonormal" && sign_mode != "winding") { std::cerr << "ERROR: --sign must be pseudonormal or winding" << std::endl; return 1; }
    if (sign_mode == "winding" && n_gpus > 1) { std::cerr << "ERROR: --sign winding runs on one GPU; it cannot be combined with --gpus " << n_gpus << std::endl; return 1; }
    if (use_band && !(band >= 0.0)) { std::cerr << "ERROR: --band needs a width >= 0" << std::endl; return 1; }
    try {
        std::cout << "Load mesh...";
        Discregrid::TriangleMesh mesh(filename);
        std::cout << "DONE" << std::endl;
        std::cout << "Set up data structures...";
        Discregrid::TriangleMeshDistance md(mesh);
        if (n_gpus > 1) md.useGpus(n_gpus);
        if (sign_mode == "winding") md.setSignMode(Discregrid::SignMode::Winding);
        std::cout << "DONE" << std::endl;

        AlignedBox3d domain;
        domain.setEmpty();
        if (!domain_str.empty()) { std::istringstream is(domain_str); Vector3d a, b; is >> a.x() >> a.y() >> a.z() >> b.x() >> b.y() >> b.z(); domain = AlignedBox3d(a, b); }
        if (domain.isEmpty()) {
            double mn[3], mx[3];                                           // main.cpp:83-91 (asymmetric padding), done by the library
            std::vector<double> V(3 * mesh.nVertices());
            for (std::size_t i = 0; i < mesh.nVertices(); i++) for (int d = 0; d < 3; d++) V[3 * i + d] = mesh.vertex((unsigned)i)[d];
            if (dg_generate_sdf_domain(V.data(), mesh.nVertices(), mn, mx) != DG_OK) { std::cerr << dg_last_error() << std::endl; return 1; }
            domain = AlignedBox3d(Vector3d(mn[0], mn[1], mn[2]), Vector3d(mx[0], mx[1], mx[2]));
        }
        Discregrid::CubicLagrangeDiscreteGrid sdf(domain, resolution);
        Discregrid::DiscreteGrid::ContinuousFunction func = Discregrid::MeshSignedDistanceFunction(md, invert);
        std::cout << "Generate discretization..." << std::endl;
        if (use_band && no_reduction) sdf.addFunction(func, true, Discregrid::MeshDistanceBandPredicate(md, band));
        else if (use_band) {
            // addFunction(func, pred) + reduceField(always true) in one call: only the reduced field reaches the host
            std::cout << "Reduce discretization...";
            sdf.addReducedBandField(Discregrid::MeshSignedDistanceFunction(md, invert), Discregrid::MeshDistanceBandPredicate(md, band), true);
            std::cout << "DONE" << std::endl;
        } else sdf.addFunction(func, true);
        std::cout << "DONE" << std::endl;
        std::cout << "Serialize discretization...";
        if (output_file.empty()) {
            output_file = filename;
            if (output_file.find(".") != std::string::npos) output_file = output_file.substr(0, output_file.find_last_of("."));
            output_file += ".cdf";
        }
        sdf.save(output_file);
        std::cout << "DONE" << std::endl;
    } catch (std::exception const& e) {
        std::cerr << "error: " << e.what() << std::endl;
        return 1;
    }
    return 0;
}
