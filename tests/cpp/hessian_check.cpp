// tests/cpp/hessian_check.cpp -- the C++ facade's batched Hessian overload, interpolate(field, n, x, phi, grad, hess), on a grid loaded from
// a .cdf / .cdm file.  Writes phi (n), grad (n x 3) and hess (n x 3 x 3) as raw doubles, one after the other, for comparison with the
// Python route.
// usage: hessian_check <grid file> <field id> <points.f64> <out.f64>
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
    if (argc != 5) { std::fprintf(stderr, "usage: %s grid.cdf field points.f64 out.f64\n", argv[0]); return 2; }
    const unsigned field = (unsigned)std::strtoul(argv[2], nullptr, 10);
    std::ifstream pf(argv[3], std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(pf)), std::istreambuf_iterator<char>());
    std::vector<double> x(raw.size() / sizeof(double));
    std::memcpy(x.data(), raw.data(), x.size() * sizeof(double));
    const std::size_t n = x.size() / 3;
    std::vector<double> out(13 * n);
    try {
        CubicLagrangeDiscreteGrid g(argv[1]);
        g.interpolate(field, n, x.data(), out.data(), out.data() + n, out.data() + 4 * n);
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[4], std::ios::binary);
    f.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(double)));
    std::printf("hessian_check OK: %zu points\n", n);
    return 0;
}
