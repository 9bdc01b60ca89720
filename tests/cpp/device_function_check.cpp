// tests/cpp/device_function_check.cpp -- the C++ facade's device callbacks (DeviceFunction, DeviceSamplePredicate, DeviceNodePredicate) on
// the analytic case of tests/golden/make_device_function_golden.py.  The callbacks move each chunk to the host with cudaMemcpyAsync on the
// stream they are given, evaluate the reference's lambdas there and copy the result back, so the fields must be byte-identical to the
// reference's own files.  Writes <out>_one.cdf (addReducedFunction), <out>_two.cdf (addFunction + reduceField(DeviceNodePredicate)) and
// <out>_dense.cdf (addFunction alone).
// usage: device_function_check <out prefix> mn[3] mx[3] res[3] centre[3] r c vmax z0 sample(0|1) reduce(0|1)   (numbers as hex floats)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include <Discregrid/All>

using namespace Discregrid;

static void cuda_check(cudaError_t e)
{
    if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
}

int main(int argc, char** argv)
{
    if (argc != 20) { std::fprintf(stderr, "usage: %s out mn[3] mx[3] res[3] centre[3] r c vmax z0 sample reduce\n", argv[0]); return 2; }
    double a[16];
    for (int i = 0; i < 16; i++) a[i] = std::strtod(argv[2 + i], nullptr);
    const bool sample = argv[18][0] == '1', reduce = argv[19][0] == '1';
    const Eigen::AlignedBox3d domain(Eigen::Vector3d(a[0], a[1], a[2]), Eigen::Vector3d(a[3], a[4], a[5]));
    const std::array<unsigned int, 3> res = {{(unsigned)a[6], (unsigned)a[7], (unsigned)a[8]}};
    const double cx = a[9], cy = a[10], cz = a[11], r = a[12], c = a[13], vmax = a[14], z0 = a[15];
    const std::string out = argv[1];

    auto to_host = [](const void* d, std::size_t bytes, void* stream) {
        std::vector<char> h(bytes);
        cuda_check(cudaMemcpyAsync(h.data(), d, bytes, cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)));
        cuda_check(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
        return h;
    };
    auto to_device = [](void* d, const void* h, std::size_t bytes, void* stream) {
        cuda_check(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)));
        cuda_check(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
    };
    DeviceFunction func;
    func.f = [&](const double* d_x, const std::uint8_t*, std::uint64_t n, double* d_values, void* stream) {
        const std::vector<char> hx = to_host(d_x, 24 * n, stream);
        const double* x = reinterpret_cast<const double*>(hx.data());
        std::vector<double> v(n);
        for (std::uint64_t i = 0; i < n; i++) {
            const double dx = x[3 * i] - cx, dy = x[3 * i + 1] - cy, dz = x[3 * i + 2] - cz;
            v[i] = std::sqrt((dx * dx + dy * dy) + dz * dz) - r;
        }
        to_device(d_values, v.data(), 8 * n, stream);
        return 0;
    };
    DeviceSamplePredicate spred;
    spred.f = [&](const double* d_x, std::uint64_t n, std::uint8_t* d_keep, void* stream) {
        const std::vector<char> hx = to_host(d_x, 24 * n, stream);
        const double* x = reinterpret_cast<const double*>(hx.data());
        std::vector<std::uint8_t> k(n);
        for (std::uint64_t i = 0; i < n; i++) k[i] = (x[3 * i] + 0.5 * x[3 * i + 1] < c) ? 1 : 0;
        to_device(d_keep, k.data(), n, stream);
        return 0;
    };
    DeviceNodePredicate rpred;
    rpred.f = [&](const double* d_x, const double* d_values, std::uint64_t n, std::uint8_t* d_keep, void* stream) {
        const std::vector<char> hx = to_host(d_x, 24 * n, stream), hv = to_host(d_values, 8 * n, stream);
        const double* x = reinterpret_cast<const double*>(hx.data());
        const double* v = reinterpret_cast<const double*>(hv.data());
        std::vector<std::uint8_t> k(n);
        for (std::uint64_t i = 0; i < n; i++) k[i] = (v[i] <= vmax && x[3 * i + 2] > z0) ? 1 : 0;
        to_device(d_keep, k.data(), n, stream);
        return 0;
    };
    try {
        {
            CubicLagrangeDiscreteGrid g(domain, res);
            g.addReducedFunction(func, sample ? &spred : nullptr, reduce ? &rpred : nullptr);
            g.save(out + "_one.cdf");
        }
        {
            CubicLagrangeDiscreteGrid g(domain, res);
            const unsigned id = sample ? g.addFunction(func, false, spred) : g.addFunction(func);
            g.save(out + "_dense.cdf");
            if (reduce) g.reduceField(id, rpred);
            g.save(out + "_two.cdf");
        }
        // the rules: a device function with a host predicate, a device predicate with a host function, and a throwing callback
        CubicLagrangeDiscreteGrid g(domain, res);
        int refused = 0;
        try { g.addFunction(func, false, [](Eigen::Vector3d const&) { return true; }); } catch (std::invalid_argument const&) { refused++; }
        try { g.addFunction([](Eigen::Vector3d const&) { return 0.0; }, false, spred); } catch (std::invalid_argument const&) { refused++; }
        DeviceFunction bad;
        bad.f = [](const double*, const std::uint8_t*, std::uint64_t, double*, void*) -> int { throw std::out_of_range("thrown by the callback"); };
        try { g.addReducedFunction(bad); } catch (std::out_of_range const&) { refused++; }
        if (refused != 3 || g.nFields() != 0) { std::fprintf(stderr, "facade rules: %d of 3 refusals\n", refused); return 1; }
    } catch (std::exception const& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    std::printf("device_function_check OK\n");
    return 0;
}
