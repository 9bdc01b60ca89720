// tests/cpp/isosurface_grad_check.cpp -- the C++ facade's level-set gradient on device pointers: CubicLagrangeDiscreteGrid::isosurface with
// edge ids on a grid file, then isosurface_vjp on the trainable field (which holds the file's values) for a given upstream gradient of the
// vertices.  It must give the same bits on a side stream and on the legacy stream.  Writes, for comparison with the Python route, the
// vertices (3 n_vertices), the edge ids as doubles (n_vertices) and grad_nodes (nodes), as doubles.
// usage: isosurface_grad_check <grid.cdf> <iso> <subdivisions> <grad_vertices.f64> <out.f64>
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

template <class T> static T* upload(const std::vector<T>& h)
{
    T* d = nullptr;
    if (cudaMalloc(reinterpret_cast<void**>(&d), (h.size() ? h.size() : 1) * sizeof(T)) != cudaSuccess) return nullptr;
    cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
    return d;
}

int main(int argc, char** argv)
{
    if (argc != 6) {
        std::fprintf(stderr, "usage: %s grid.cdf iso subdivisions grad_vertices.f64 out.f64\n", argv[0]);
        return 2;
    }
    const double iso = std::atof(argv[2]);
    const unsigned s = (unsigned)std::atoi(argv[3]);
    const std::vector<double> gV = read_f64(argv[4]);
    std::vector<double> out;
    try {
        CubicLagrangeDiscreteGrid grid(argv[1]);
        const std::size_t nn = grid.nodeData(0).size();
        std::vector<std::uint64_t> edges;
        TriangleMesh mesh = grid.isosurface(0, iso, s, &edges);
        const std::size_t nv = edges.size();
        if (mesh.nVertices() != nv) { std::fprintf(stderr, "%zu vertices, %zu edge ids\n", (std::size_t)mesh.nVertices(), nv); return 1; }
        if (gV.size() != 3 * nv) { std::fprintf(stderr, "grad_vertices: %zu values for %zu vertices\n", gV.size(), nv); return 1; }
        for (std::size_t i = 0; i < nv; i++) {
            const Eigen::Vector3d& p = mesh.vertex((unsigned int)i);
            out.push_back(p[0]); out.push_back(p[1]); out.push_back(p[2]);
        }
        for (std::size_t i = 0; i < nv; i++) out.push_back((double)edges[i]);
        cudaStream_t side;
        cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
        std::uint64_t* de = upload(edges);
        double* dg = upload(gV);
        std::vector<double> first;
        for (int pass = 0; pass < 2; pass++) {
            double* gn = upload(std::vector<double>(nn ? nn : 1, 7.0));
            cudaDeviceSynchronize();
            grid.isosurface_vjp(0, iso, s, nv, de, dg, gn, pass == 0 ? (void*)side : nullptr);
            if (cudaDeviceSynchronize() != cudaSuccess) { std::fprintf(stderr, "CUDA error\n"); return 1; }
            std::vector<double> r(nn);
            cudaMemcpy(r.data(), gn, nn * sizeof(double), cudaMemcpyDeviceToHost);
            if (pass == 0) first = r;
            else if (std::memcmp(first.data(), r.data(), nn * sizeof(double)) != 0) { std::fprintf(stderr, "the node gradient depends on the stream\n"); return 1; }
            cudaFree(gn);
        }
        out.insert(out.end(), first.begin(), first.end());
        bool refused = false;
        try { grid.isosurface_vjp(0, iso, 17, nv, de, dg, nullptr); }
        catch (std::exception const&) { refused = true; }
        if (!refused) { std::fprintf(stderr, "isosurface_vjp with 17 subdivisions was accepted\n"); return 1; }
        cudaFree(de); cudaFree(dg);
        cudaStreamDestroy(side);
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[5], std::ios::binary);
    f.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(double)));
    std::printf("isosurface_grad_check OK: %zu vertices\n", out.size());
    return 0;
}
