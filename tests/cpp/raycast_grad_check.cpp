// tests/cpp/raycast_grad_check.cpp -- the C++ facade's ray-cast gradients on device pointers: TriangleMeshDistance::raycast_vjp on a mesh
// file and CubicLagrangeDiscreteGrid::raycast_vjp on a grid file (the trainable field after setNodesDevice, with the node gradient).  Each
// must give the same bits on a side stream and on the legacy stream.  Writes, for comparison with the Python route, the mesh's
// grad_origins (3n), grad_directions (3n), grad_vertices (3 n_vertices), then the field's grad_origins (3n), grad_directions (3n) and
// grad_nodes (nodes), as doubles.
// usage: raycast_grad_check <mesh.obj> <vertices.f64> <grid.cdf> <values.f64> <origins.f64> <directions.f64> <grad_t.f64> <grad_bary.f64>
//        <out.f64>
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

static std::vector<double> download(const double* d, std::size_t n)
{
    std::vector<double> h(n);
    cudaMemcpy(h.data(), d, n * sizeof(double), cudaMemcpyDeviceToHost);
    return h;
}

static double* zeros(std::size_t n) { return upload(std::vector<double>(n ? n : 1, 0.0)); }

int main(int argc, char** argv)
{
    if (argc != 10) {
        std::fprintf(stderr, "usage: %s mesh.obj vertices.f64 grid.cdf values.f64 origins.f64 directions.f64 grad_t.f64 grad_bary.f64 out.f64\n", argv[0]);
        return 2;
    }
    const std::vector<double> V = read_f64(argv[2]), v = read_f64(argv[4]), O = read_f64(argv[5]), D = read_f64(argv[6]);
    const std::vector<double> gt = read_f64(argv[7]), gb = read_f64(argv[8]);
    const std::size_t n = O.size() / 3, nV = V.size() / 3;
    std::vector<double> out;
    try {
        cudaStream_t side;
        cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
        double *dO = upload(O), *dD = upload(D), *dV = upload(V), *dgt = upload(gt), *dgb = upload(gb), *dv = upload(v);
        // mesh: cast, then the three gradients on the side stream and on the legacy stream
        TriangleMesh mesh(argv[1]);
        TriangleMeshDistance md(mesh);
        double *dt = zeros(n), *db = zeros(3 * n);
        int32_t *did = upload(std::vector<int32_t>(n ? n : 1)), *dst = upload(std::vector<int32_t>(n ? n : 1));
        md.raycast(n, dO, dD, 0.0, 1e300, dt, did, db, dst, nullptr);
        std::vector<double> first;
        for (int pass = 0; pass < 2; pass++) {
            double *go = zeros(3 * n), *gd = zeros(3 * n), *gv = zeros(3 * nV);
            cudaDeviceSynchronize();
            md.raycast_vjp(n, dD, dt, did, db, dV, dgt, dgb, go, gd, gv, pass == 0 ? (void*)side : nullptr);
            if (cudaDeviceSynchronize() != cudaSuccess) { std::fprintf(stderr, "CUDA error\n"); return 1; }
            std::vector<double> r = download(go, 3 * n), a = download(gd, 3 * n), c = download(gv, 3 * nV);
            r.insert(r.end(), a.begin(), a.end()); r.insert(r.end(), c.begin(), c.end());
            if (pass == 0) first = r;
            else if (std::memcmp(first.data(), r.data(), r.size() * sizeof(double)) != 0) { std::fprintf(stderr, "the mesh gradient depends on the stream\n"); return 1; }
            cudaFree(go); cudaFree(gd); cudaFree(gv);
        }
        out = first;
        // field: the trainable field holding v, cast on it, then the gradients with the node gradient
        CubicLagrangeDiscreteGrid grid(argv[3]);
        const std::size_t nn = grid.nodeData(0).size();
        if (v.size() != nn) { std::fprintf(stderr, "values: %zu, field: %zu nodes\n", v.size(), nn); return 1; }
        grid.setNodesDevice(0, dv, nn, nullptr);
        double *tl = zeros(n), *th = zeros(n);
        if (dg_field_raycast_device(grid.trainableField(0), dO, dD, n, 0.0, 0.0, 1e300, tl, th, dst, nullptr) != DG_OK) {
            std::fprintf(stderr, "%s\n", dg_last_error());
            return 1;
        }
        for (int pass = 0; pass < 2; pass++) {
            double *go = zeros(3 * n), *gd = zeros(3 * n), *gn = zeros(nn);
            cudaDeviceSynchronize();
            grid.raycast_vjp(0, n, dO, dD, tl, dst, dgt, nullptr, go, gd, gn, pass == 0 ? (void*)side : nullptr);
            if (cudaDeviceSynchronize() != cudaSuccess) { std::fprintf(stderr, "CUDA error\n"); return 1; }
            std::vector<double> r = download(go, 3 * n), a = download(gd, 3 * n), c = download(gn, nn);
            r.insert(r.end(), a.begin(), a.end()); r.insert(r.end(), c.begin(), c.end());
            if (pass == 0) out.insert(out.end(), r.begin(), r.end());
            else if (std::memcmp(out.data() + (out.size() - r.size()), r.data(), r.size() * sizeof(double)) != 0) {
                std::fprintf(stderr, "the field gradient depends on the stream\n");
                return 1;
            }
            cudaFree(go); cudaFree(gd); cudaFree(gn);
        }
        bool refused = false;
        try { md.raycast_vjp(n, dD, dt, did, db, dV, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr); }
        catch (std::exception const&) { refused = true; }
        if (!refused) { std::fprintf(stderr, "raycast_vjp without an upstream gradient was accepted\n"); return 1; }
        for (double* p : {dO, dD, dV, dgt, dgb, dv, dt, db, tl, th}) cudaFree(p);
        cudaFree(did); cudaFree(dst);
        cudaStreamDestroy(side);
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::ofstream f(argv[9], std::ios::binary);
    f.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(double)));
    std::printf("raycast_grad_check OK: %zu rays\n", n);
    return 0;
}
