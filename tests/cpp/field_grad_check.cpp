// tests/cpp/field_grad_check.cpp -- the C++ facade's trainable field: setNodesDevice and interpolate_vjp on device pointers, on a grid file.
// The node gradient must not depend on the stream, and after setNodesDevice(v) interpolate on the trainable field must give the bits of
// dg_field_create of v.  Writes the node gradient (nodes doubles) of field 0 for comparison with the Python route.
// usage: field_grad_check <grid.cdf> <points.f64> <grad_phi.f64> <grad_grad.f64> <values.f64> <out.f64>
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

template <class T> static T* upload(const std::vector<T>& h)
{
    T* d = nullptr;
    if (cudaMalloc(reinterpret_cast<void**>(&d), (h.size() ? h.size() : 1) * sizeof(T)) != cudaSuccess) return nullptr;
    cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
    return d;
}

int main(int argc, char** argv)
{
    if (argc != 7) { std::fprintf(stderr, "usage: %s grid.cdf points.f64 grad_phi.f64 grad_grad.f64 values.f64 out.f64\n", argv[0]); return 2; }
    const std::vector<double> x = read_f64(argv[2]), gp = read_f64(argv[3]), gg = read_f64(argv[4]), v = read_f64(argv[5]);
    const std::size_t n = x.size() / 3;
    std::vector<double> out;
    try {
        CubicLagrangeDiscreteGrid grid(argv[1]), plain(argv[1]);
        const std::size_t nn = grid.nodeData(0).size();
        if (v.size() != nn) { std::fprintf(stderr, "values: %zu, field: %zu nodes\n", v.size(), nn); return 1; }
        double *d_x = upload(x), *d_gp = upload(gp), *d_gg = upload(gg), *d_v = upload(v), *d_out = nullptr, *d_out2 = nullptr;
        double *d_phi = nullptr, *d_grad = nullptr;
        cudaMalloc(reinterpret_cast<void**>(&d_out), nn * sizeof(double));
        cudaMalloc(reinterpret_cast<void**>(&d_out2), nn * sizeof(double));
        cudaMalloc(reinterpret_cast<void**>(&d_phi), (n ? n : 1) * sizeof(double));
        cudaMalloc(reinterpret_cast<void**>(&d_grad), (n ? 3 * n : 1) * sizeof(double));
        cudaStream_t side;
        cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
        grid.setNodesDevice(0, d_v, nn, side);
        grid.interpolate_vjp(0, n, d_x, d_gp, d_gg, d_out, side);
        cudaStreamSynchronize(side);
        grid.interpolate_vjp(0, n, d_x, d_gp, d_gg, d_out2, nullptr);
        if (cudaDeviceSynchronize() != cudaSuccess) { std::fprintf(stderr, "CUDA error\n"); return 1; }
        out.resize(nn);
        std::vector<double> out2(nn);
        cudaMemcpy(out.data(), d_out, nn * sizeof(double), cudaMemcpyDeviceToHost);
        cudaMemcpy(out2.data(), d_out2, nn * sizeof(double), cudaMemcpyDeviceToHost);
        if (std::memcmp(out.data(), out2.data(), nn * sizeof(double)) != 0) { std::fprintf(stderr, "the node gradient depends on the stream\n"); return 1; }
        // after setNodesDevice(v) the trainable field interpolates like a grid whose members are v
        if (dg_interpolate_batch_device(grid.trainableField(0), d_x, n, d_phi, d_grad, nullptr) != DG_OK) { std::fprintf(stderr, "%s\n", dg_last_error()); return 1; }
        std::vector<double> phi(n), grad(3 * n), phi2(n), grad2(3 * n);
        cudaMemcpy(phi.data(), d_phi, n * sizeof(double), cudaMemcpyDeviceToHost);
        cudaMemcpy(grad.data(), d_grad, 3 * n * sizeof(double), cudaMemcpyDeviceToHost);
        const dg_grid_desc d = plain.desc();
        dg_field* pf = nullptr;
        if (dg_field_create(&d, v.data(), nn, reinterpret_cast<const std::uint32_t*>(plain.cellData(0).data()), plain.cellData(0).size(),
                            plain.cellMap(0).data(), &pf) != DG_OK ||
            dg_interpolate_batch(pf, x.data(), n, phi2.data(), grad2.data()) != DG_OK) { std::fprintf(stderr, "%s\n", dg_last_error()); return 1; }
        dg_field_destroy(pf);
        if (std::memcmp(phi.data(), phi2.data(), n * sizeof(double)) != 0 || std::memcmp(grad.data(), grad2.data(), 3 * n * sizeof(double)) != 0) {
            std::fprintf(stderr, "the trainable field after setNodesDevice differs from a grid with those values\n");
            return 1;
        }
        bool refused = false;
        try { grid.setNodesDevice(0, d_v, nn - 1); } catch (std::exception const&) { refused = true; }
        if (!refused) { std::fprintf(stderr, "setNodesDevice with one value missing was accepted\n"); return 1; }
        for (double* p : {d_x, d_gp, d_gg, d_v, d_out, d_out2, d_phi, d_grad}) cudaFree(p);
        cudaStreamDestroy(side);
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[6], std::ios::binary);
    f.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(double)));
    std::printf("field_grad_check OK: %zu points\n", n);
    return 0;
}
