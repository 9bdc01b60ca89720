// tests/cpp/device_query_check.cpp -- the C++ facade's reduced fields reach interpolate without the host: addReducedBandField and
// addReducedDensityMap keep the library's handle, and the first interpolate builds the device field from it (dg_field_create_reduced).
// This program defines its own dg_field_create, which refuses and counts: the facade's calls bind to it, so any interpolate that went
// through an upload fails.  Writes phi (n) followed by grad (n x 3) as raw doubles for each field:
//   <out>_band.f64 (the reduced band), <out>_sdf.f64 and <out>_density.f64 (the two fields of addReducedDensityMap on <sdf.cdf>).
// usage: device_query_check <out prefix> <mesh.obj> mn[3] mx[3] res band <sdf.cdf> h rho0 <points.f64>   (numbers as hex floats)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>
#include <Discregrid/All>

using namespace Discregrid;

static int g_field_create_calls = 0;

extern "C" int dg_field_create(const dg_grid_desc*, const double*, uint64_t, const uint32_t*, uint64_t, const uint32_t*, dg_field** out)
{
    g_field_create_calls++;
    if (out) *out = nullptr;
    return DG_ERR_INVALID;
}

static void write_query(CubicLagrangeDiscreteGrid const& g, unsigned field, std::vector<double> const& x, std::string const& path)
{
    const std::size_t n = x.size() / 3;
    std::vector<double> out(4 * n);
    g.interpolate(field, n, x.data(), out.data(), out.data() + n);
    std::ofstream f(path, std::ios::binary);
    f.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(double)));
}

int main(int argc, char** argv)
{
    if (argc != 15) { std::fprintf(stderr, "usage: %s out mesh.obj mn[3] mx[3] res band sdf.cdf h rho0 points.f64\n", argv[0]); return 2; }
    const std::string out = argv[1], mesh_path = argv[2];
    double a[7];
    for (int i = 0; i < 7; i++) a[i] = std::strtod(argv[3 + i], nullptr);
    const unsigned res = (unsigned)std::strtoul(argv[9], nullptr, 10);
    const double band = std::strtod(argv[10], nullptr);
    const std::string sdf_path = argv[11];
    const double h = std::strtod(argv[12], nullptr), rho0 = std::strtod(argv[13], nullptr);
    std::ifstream pf(argv[14], std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(pf)), std::istreambuf_iterator<char>());
    std::vector<double> x(raw.size() / sizeof(double));
    std::memcpy(x.data(), raw.data(), x.size() * sizeof(double));
    try {
        {
            TriangleMesh mesh(mesh_path);
            TriangleMeshDistance md(mesh);
            CubicLagrangeDiscreteGrid g(Eigen::AlignedBox3d(Eigen::Vector3d(a[0], a[1], a[2]), Eigen::Vector3d(a[3], a[4], a[5])), {{res, res, res}});
            const unsigned id = g.addReducedBandField(MeshSignedDistanceFunction(md), MeshDistanceBandPredicate(md, band));
            write_query(g, id, x, out + "_band.f64");
        }
        {
            CubicLagrangeDiscreteGrid g(sdf_path);
            DensityMapFunction f{&g, 0u, h, rho0, false};
            const unsigned id = g.addReducedDensityMap(f);
            write_query(g, 0, x, out + "_sdf.f64");
            write_query(g, id, x, out + "_density.f64");
        }
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s (dg_field_create calls: %d)\n", e.what(), g_field_create_calls);
        return 1;
    }
    if (g_field_create_calls) { std::fprintf(stderr, "dg_field_create was called %d times\n", g_field_create_calls); return 1; }
    std::printf("device_query_check OK\n");
    return 0;
}
