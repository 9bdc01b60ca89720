// tests/cpp/winding_check.cpp -- the C++ facade's sign mode: TriangleMeshDistance::setSignMode(SignMode::Winding, beta), winding_number (both
// forms) and signed_distance in the winding mode, on a mesh file.  Writes w (n) then the winding-signed distances (n) as raw doubles for
// comparison with the Python route, and checks that useGpus(2) throws in the winding mode.
// usage: winding_check <mesh.obj> <points.f64> <beta> <out.f64>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>
#include <Discregrid/All>

using namespace Discregrid;

int main(int argc, char** argv)
{
    if (argc != 5) { std::fprintf(stderr, "usage: %s mesh.obj points.f64 beta out.f64\n", argv[0]); return 2; }
    std::ifstream pf(argv[2], std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(pf)), std::istreambuf_iterator<char>());
    std::vector<double> x(raw.size() / sizeof(double));
    std::memcpy(x.data(), raw.data(), x.size() * sizeof(double));
    const std::size_t n = x.size() / 3;
    const double beta = std::strtod(argv[3], nullptr);
    std::vector<double> out(2 * n);
    try {
        TriangleMesh mesh(argv[1]);
        TriangleMeshDistance md(mesh);
        md.setSignMode(SignMode::Winding, beta);
        if (md.signMode() != SignMode::Winding) { std::fprintf(stderr, "signMode() did not change\n"); return 1; }
        md.winding_number(x.data(), n, out.data(), beta);
        const std::vector<Result> r = md.signed_distance_batch(x.data(), n);
        for (std::size_t i = 0; i < n; i++) out[n + i] = r[i].distance;
        if (n > 0) {
            const double w0 = md.winding_number(std::array<double, 3>{{x[0], x[1], x[2]}}, beta);
            if (std::memcmp(&w0, &out[0], sizeof w0) != 0) { std::fprintf(stderr, "single-point winding_number differs from the batch\n"); return 1; }
        }
        bool threw = false;
        try { md.useGpus(2); } catch (std::exception const&) { threw = true; }
        if (!threw) { std::fprintf(stderr, "useGpus(2) did not throw in the winding mode\n"); return 1; }
        bool refused = false;
        try { md.setSignMode(SignMode::Winding, 0.5); } catch (std::exception const&) { refused = true; }
        if (!refused) { std::fprintf(stderr, "beta = 0.5 was accepted\n"); return 1; }
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[4], std::ios::binary);
    f.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(double)));
    std::printf("winding_check OK: %zu points\n", n);
    return 0;
}
