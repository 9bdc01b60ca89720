// tests/cpp/refit_check.cpp -- the C++ facade's refit: TriangleMeshDistance::refit from a std::vector of vertices and from a device pointer, on
// a mesh file.  Both routes must give the same signed distances bit for bit; writes them (n doubles) for comparison with the Python route.
// usage: refit_check <mesh.obj> <vertices.f64> <points.f64> <out.f64>
#include <array>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>
#include <cuda_runtime.h>
#include <Discregrid/All>

using namespace Discregrid;

static std::vector<double> read_f64(const char* path)
{
    std::ifstream f(path, std::ios::binary);
    std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    std::vector<double> v(raw.size() / sizeof(double));
    std::memcpy(v.data(), raw.data(), v.size() * sizeof(double));
    return v;
}

int main(int argc, char** argv)
{
    if (argc != 5) { std::fprintf(stderr, "usage: %s mesh.obj vertices.f64 points.f64 out.f64\n", argv[0]); return 2; }
    const std::vector<double> V = read_f64(argv[2]), x = read_f64(argv[3]);
    const std::size_t nV = V.size() / 3, n = x.size() / 3;
    std::vector<std::array<double, 3>> Vv(nV);
    for (std::size_t i = 0; i < nV; i++) Vv[i] = {{V[3 * i], V[3 * i + 1], V[3 * i + 2]}};
    std::vector<double> out(n);
    try {
        TriangleMesh mesh(argv[1]);
        TriangleMeshDistance a(mesh), b(mesh);
        a.refit(Vv);
        double* d_V = nullptr;
        if (cudaMalloc(reinterpret_cast<void**>(&d_V), V.size() * sizeof(double)) != cudaSuccess) { std::fprintf(stderr, "cudaMalloc failed\n"); return 1; }
        cudaMemcpy(d_V, V.data(), V.size() * sizeof(double), cudaMemcpyHostToDevice);
        b.refit(d_V, nV);
        cudaFree(d_V);
        const std::vector<Result> ra = a.signed_distance_batch(x.data(), n), rb = b.signed_distance_batch(x.data(), n);
        for (std::size_t i = 0; i < n; i++) {
            if (std::memcmp(&ra[i].distance, &rb[i].distance, sizeof(double)) != 0 || ra[i].triangle_id != rb[i].triangle_id) {
                std::fprintf(stderr, "point %zu: the host-vector and device-pointer refits differ\n", i);
                return 1;
            }
            out[i] = ra[i].distance;
        }
        bool refused = false;
        try { a.refit(std::vector<std::array<double, 3>>(Vv.begin(), Vv.end() - 1)); } catch (std::exception const&) { refused = true; }
        if (!refused) { std::fprintf(stderr, "a refit with one vertex missing was accepted\n"); return 1; }
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[4], std::ios::binary);
    f.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(double)));
    std::printf("refit_check OK: %zu points\n", n);
    return 0;
}
