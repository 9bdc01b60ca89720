// tests/cpp/raycast_check.cpp -- the C++ facade's batched raycast(field, n, origins, directions, iso, t_min, t_max, t_lo, t_hi, status) on a
// grid loaded from a .cdf / .cdm file.  Writes t_lo (n doubles), t_hi (n doubles) and status (n int32), one after the other, for comparison
// with the Python route.
// usage: raycast_check <grid file> <field id> <rays.f64: n x 6, origin then direction> <iso> <t_min> <t_max> <out.bin>
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
    if (argc != 8) { std::fprintf(stderr, "usage: %s grid.cdf field rays.f64 iso t_min t_max out.bin\n", argv[0]); return 2; }
    const unsigned field = (unsigned)std::strtoul(argv[2], nullptr, 10);
    std::ifstream rf(argv[3], std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(rf)), std::istreambuf_iterator<char>());
    const std::size_t n = raw.size() / (6 * sizeof(double));
    std::vector<double> o(3 * n), d(3 * n);
    for (std::size_t i = 0; i < n; i++) {
        std::memcpy(&o[3 * i], raw.data() + (6 * i) * sizeof(double), 3 * sizeof(double));
        std::memcpy(&d[3 * i], raw.data() + (6 * i + 3) * sizeof(double), 3 * sizeof(double));
    }
    std::vector<double> t(2 * n);
    std::vector<std::int32_t> st(n);
    try {
        CubicLagrangeDiscreteGrid g(argv[1]);
        g.raycast(field, n, o.data(), d.data(), std::strtod(argv[4], nullptr), std::strtod(argv[5], nullptr), std::strtod(argv[6], nullptr),
                  t.data(), t.data() + n, st.data());
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[7], std::ios::binary);
    f.write(reinterpret_cast<const char*>(t.data()), (std::streamsize)(t.size() * sizeof(double)));
    f.write(reinterpret_cast<const char*>(st.data()), (std::streamsize)(st.size() * sizeof(std::int32_t)));
    std::printf("raycast_check OK: %zu rays\n", n);
    return 0;
}
