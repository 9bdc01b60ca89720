// tests/cpp/mesh_raycast_check.cpp -- the C++ facade's mesh raycast: TriangleMeshDistance::raycast on host arrays and on device pointers, on a
// mesh file.  Both routes must give the same results bit for bit; writes t (n doubles), barycentric (3n doubles), triangle_id (n int32) and
// status (n int32) for comparison with the Python route.
// usage: mesh_raycast_check <mesh.obj> <rays.f64: n x (origin, direction)> <t_min> <t_max> <out.bin>
#include <cstdio>
#include <cstdlib>
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

template <class T> static T* to_device(const std::vector<T>& h)
{
    T* p = nullptr;
    if (cudaMalloc(reinterpret_cast<void**>(&p), (h.empty() ? 1 : h.size()) * sizeof(T)) != cudaSuccess) return nullptr;
    cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
    return p;
}

int main(int argc, char** argv)
{
    if (argc != 6) { std::fprintf(stderr, "usage: %s mesh.obj rays.f64 t_min t_max out.bin\n", argv[0]); return 2; }
    const std::vector<double> R = read_f64(argv[2]);
    const std::size_t n = R.size() / 6;
    const double t0 = std::strtod(argv[3], nullptr), t1 = std::strtod(argv[4], nullptr);
    std::vector<double> O(3 * n), D(3 * n);
    for (std::size_t i = 0; i < n; i++)
        for (int k = 0; k < 3; k++) { O[3 * i + k] = R[6 * i + k]; D[3 * i + k] = R[6 * i + 3 + k]; }
    std::vector<double> t(n), b(3 * n), t2(n), b2(3 * n);
    std::vector<int32_t> id(n), st(n), id2(n), st2(n);
    try {
        TriangleMesh mesh(argv[1]);
        TriangleMeshDistance md(mesh);
        md.raycast(n, O.data(), D.data(), t0, t1, t.data(), id.data(), b.data(), st.data());
        double *dO = to_device(O), *dD = to_device(D), *dt = to_device(t2), *db = to_device(b2);
        int32_t *did = to_device(id2), *dst = to_device(st2);
        if (!dO || !dD || !dt || !db || !did || !dst) { std::fprintf(stderr, "cudaMalloc failed\n"); return 1; }
        md.raycast(n, dO, dD, t0, t1, dt, did, db, dst, nullptr);
        cudaMemcpy(t2.data(), dt, n * sizeof(double), cudaMemcpyDeviceToHost);
        cudaMemcpy(b2.data(), db, 3 * n * sizeof(double), cudaMemcpyDeviceToHost);
        cudaMemcpy(id2.data(), did, n * sizeof(int32_t), cudaMemcpyDeviceToHost);
        cudaMemcpy(st2.data(), dst, n * sizeof(int32_t), cudaMemcpyDeviceToHost);
        cudaFree(dO); cudaFree(dD); cudaFree(dt); cudaFree(db); cudaFree(did); cudaFree(dst);
        if (std::memcmp(t.data(), t2.data(), n * sizeof(double)) != 0 || std::memcmp(b.data(), b2.data(), 3 * n * sizeof(double)) != 0 ||
            id != id2 || st != st2) {
            std::fprintf(stderr, "the host-array and device-pointer casts differ\n");
            return 1;
        }
        bool refused = false;
        try { md.raycast(n, O.data(), D.data(), 1.0, 0.0, t.data(), id.data(), b.data(), st.data()); } catch (std::exception const&) { refused = true; }
        if (!refused) { std::fprintf(stderr, "t_min > t_max was accepted\n"); return 1; }
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[5], std::ios::binary);
    f.write(reinterpret_cast<const char*>(t.data()), (std::streamsize)(n * sizeof(double)));
    f.write(reinterpret_cast<const char*>(b.data()), (std::streamsize)(3 * n * sizeof(double)));
    f.write(reinterpret_cast<const char*>(id.data()), (std::streamsize)(n * sizeof(int32_t)));
    f.write(reinterpret_cast<const char*>(st.data()), (std::streamsize)(n * sizeof(int32_t)));
    std::printf("mesh_raycast_check OK: %zu rays\n", n);
    return 0;
}
