// C-ABI of libdiscregrid_b200.so (include/discregrid_b200.h): handles, error reporting, host<->device plumbing.
// All numerics live in the kernels (k1_sdf.cu, k2_interp.cu, k3_density.cu) and in bvh_build.cpp.
#include "../../include/discregrid_b200.h"

#include <atomic>
#include <cassert>
#include <condition_variable>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <limits>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>
#if defined(__linux__)
#include <sys/mman.h>
#endif

// NCCL is used through dlopen (multi-GPU section): only its types are needed at build time
#if __has_include(<nccl.h>) && !defined(DG_EMU)
#include <nccl.h>
#include <dlfcn.h>
#define DG_HAVE_NCCL 1
#else
#define DG_HAVE_NCCL 0
#endif

#include "bvh_build.h"
#include "dg_device.cuh"
#include "k1_sdf.h"
#include "k2_interp.h"
#include "k3_density.h"
#include "k4_reduce.h"
#include "k5_winding.h"
#include "k6_isosurface.h"
#include "k7_raycast.h"
#include "k8_refit.h"
#include "k9_mesh_raycast.h"
#include "reduce_field.h"
#include "obj_reader.h"

using namespace dgb;

// ------------------------------------------------------------------------------------------------ state
namespace {

thread_local std::string g_err;
std::atomic<uint64_t> g_launches{0};

int fail(int code, const char* fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

// C++ exceptions (allocation failures in the host-side containers and threads) must not cross the C boundary
template <class F>
int guarded(const char* who, F&& body)
{
    try { return body(); }
    catch (const std::bad_alloc&) { return fail(DG_ERR_NOMEM, "%s: out of host memory", who); }
    catch (const std::exception& ex) { return fail(DG_ERR_INVALID, "%s: %s", who, ex.what()); }
}

// the status code of a failed CUDA call
int cuda_code(cudaError_t e)
{
    if (e == cudaErrorMemoryAllocation) return DG_ERR_NOMEM;
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) return DG_ERR_NO_DEVICE;
    return DG_ERR_CUDA;
}

#define DG_CUDA(call)                                                                                          \
    do {                                                                                                       \
        const cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess) return fail(cuda_code(e_), "%s failed: %s", #call, cudaGetErrorString(e_));     \
    } while (0)

#define DG_LAUNCH(call)          \
    do {                         \
        DG_CUDA(call);           \
        g_launches.fetch_add(1); \
    } while (0)

int require_device()
{
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        cudaGetLastError();
        return fail(DG_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    return DG_OK;
}

// a handle's device arrays (and K1's dynamic shared-memory attribute) belong to the device it was created on
int check_handle_device(int handle_device, const char* who)
{
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return fail(DG_ERR_NO_DEVICE, "%s: no current CUDA device", who); }
    if (dev != handle_device) return fail(DG_ERR_INVALID, "%s: the handle lives on device %d but the current device is %d (dg_set_device)", who, handle_device, dev);
    return DG_OK;
}

// page-locked host memory (cudaMallocHost / cudaHostRegister, by any CUDA runtime instance of the process) can be DMA'd directly
bool is_pinned_host(const void* p)
{
    if (!p) return true;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// simple owning device buffer
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    cudaError_t alloc(size_t count)
    {
        release();
        n = count;
        return cudaMalloc(reinterpret_cast<void**>(&p), (count ? count : 1) * sizeof(T));
    }
    void release()
    {
        if (p) cudaFree(p);
        p = nullptr; n = 0;
    }
    size_t bytes() const { return n * sizeof(T); }
};

// the device copy of a grid descriptor; refuses the grids dg_grid_num_nodes refuses (2^31 nodes or more among them)
int grid_checked(const dg_grid_desc* d, GridDev& g, const char* who)
{
    if (!d) return fail(DG_ERR_INVALID, "%s: grid descriptor is NULL", who);
    for (int k = 0; k < 3; k++) {
        if (d->resolution[k] == 0) return fail(DG_ERR_INVALID, "%s: resolution must be >= 1 in every dimension", who);
        g.mn[k] = d->domain_min[k]; g.mx[k] = d->domain_max[k];
        g.cell[k] = d->cell_size[k]; g.inv[k] = d->inv_cell_size[k];
        g.n[k] = d->resolution[k];
    }
    uint64_t nn = 0;
    if (dg_grid_num_nodes(d->resolution, &nn) != DG_OK)
        return fail(DG_ERR_INVALID, "%s: grid too large: node ids must fit uint32 (reference file format)", who);
    const unsigned nx = g.n[0], ny = g.n[1], nz = g.n[2];
    g.nv = (nx + 1) * (ny + 1) * (nz + 1);
    g.ne_x = nx * (ny + 1) * (nz + 1);
    g.ne_y = (nx + 1) * ny * (nz + 1);
    g.ne_z = (nx + 1) * (ny + 1) * nz;
    return DG_OK;
}

uint64_t grid_nodes(const GridDev& g) { return (uint64_t)g.nv + 2ull * ((uint64_t)g.ne_x + g.ne_y + g.ne_z); }
uint64_t grid_cells(const GridDev& g) { return (uint64_t)g.n[0] * g.n[1] * g.n[2]; }

int check_reduce_flags(uint32_t flags, const char* who)
{
    if (flags & ~DG_REDUCE_REFERENCE_SORT) return fail(DG_ERR_INVALID, "%s: unknown flags 0x%x (only DG_REDUCE_REFERENCE_SORT)", who, flags);
    return DG_OK;
}

// The host-array form of a query: device buffers for `chunk` points of every input and of every non-NULL output (bytes: per point), then
// upload -> launch -> download chunk by chunk on the legacy default stream, and a device synchronise.  launch(d_in, d_out, b, c) runs the
// query on points [b, b + c) in the buffers (NULL for a NULL output); n == 0 makes one launch of no points.
struct HostIn { const void* p; size_t bytes; };
struct HostOut { void* p; size_t bytes; };

template <class Launch>
int stage_on_device(uint64_t n, uint64_t chunk, std::initializer_list<HostIn> in, std::initializer_list<HostOut> out, Launch&& launch)
{
    constexpr size_t kMax = 4;
    assert(in.size() <= kMax && out.size() <= kMax);
    const HostIn* ins = in.begin();
    const HostOut* outs = out.begin();
    DevBuf<char> d_in[kMax], d_out[kMax];
    void* p_in[kMax] = {};
    void* p_out[kMax] = {};
    for (size_t k = 0; k < in.size(); k++) { DG_CUDA(d_in[k].alloc(chunk * ins[k].bytes)); p_in[k] = d_in[k].p; }
    for (size_t k = 0; k < out.size(); k++)
        if (outs[k].p) { DG_CUDA(d_out[k].alloc(chunk * outs[k].bytes)); p_out[k] = d_out[k].p; }
    uint64_t b = 0;
    do {
        const uint64_t c = std::min(chunk, n - b);
        for (size_t k = 0; k < in.size() && c; k++)
            DG_CUDA(cudaMemcpy(p_in[k], static_cast<const char*>(ins[k].p) + b * ins[k].bytes, c * ins[k].bytes, cudaMemcpyHostToDevice));
        if (int rc = launch(p_in, p_out, b, c)) return rc;
        for (size_t k = 0; k < out.size() && c; k++)
            if (p_out[k]) DG_CUDA(cudaMemcpy(static_cast<char*>(outs[k].p) + b * outs[k].bytes, p_out[k], c * outs[k].bytes, cudaMemcpyDeviceToHost));
        b += c;
    } while (b < n);
    DG_CUDA(cudaDeviceSynchronize());
    return DG_OK;
}

std::atomic<int> g_selftest_state{0};   // 0 = not run, 1 = ok, -1 = failed

}  // namespace

// ------------------------------------------------------------------------------------------------ handles
struct dg_mesh {
    HostBvh host;
    DevBuf<SpherePair> d_spheres;
    DevBuf<LeafRecord> d_leaves;
    DevBuf<PseudoNormals> d_normals;
    DevBuf<float4> d_nodes_f;
    DevBuf<LeafF> d_leaves_f;
    DeviceBvh dev;
    int device = 0;
    uint64_t build_us = 0, upload_us = 0;
    // sign mode (dg_mesh_set_sign_mode) and the winding-number records of K5, built and uploaded at their first use
    int sign_mode = DG_SIGN_PSEUDONORMAL;
    double beta = 2.0;
    mutable std::mutex wind_mu;
    mutable bool wind_ready = false;
    mutable DevBuf<WindLeaf> d_wind_leaves;
    mutable DevBuf<WindClusterPair> d_wind_clusters;
    mutable WindDev wind;
    // dg_mesh_refit (k8_refit.cu): topology tables and scratch, allocated at the first refit and kept
    std::atomic<int> borrows{0};            // live dg_mesh_group's whose replicas copy this mesh's records
    bool failed = false;                    // a refit stopped after it had started to write records
    bool refit_ready = false;               // the tables below are allocated and uploaded
    bool refit_done = false;                // the records are those of a refit: d_V holds the positions, host V and pseudonormals are stale
    std::vector<uint32_t> refit_levels;     // RefitTopoHost::level_begin
    DevBuf<double> d_V;                     // [nV][3] the positions of the last refit
    DevBuf<uint32_t> d_F, d_f_leaf, d_inc_begin, d_inc;
    DevBuf<int32_t> d_order;
    DevBuf<RefitNodeRef> d_nodes;
    DevBuf<RefitSums> d_sums;
    DevBuf<RefitBounds> d_part;
    DevBuf<double> d_bounds, d_pn_tri, d_angle, d_pn_vert, d_pn_edge;
    size_t refit_bytes() const
    {
        return d_V.bytes() + d_F.bytes() + d_f_leaf.bytes() + d_inc_begin.bytes() + d_inc.bytes() + d_order.bytes() + d_nodes.bytes() +
               d_sums.bytes() + d_part.bytes() + d_bounds.bytes() + d_pn_tri.bytes() + d_angle.bytes() + d_pn_vert.bytes() + d_pn_edge.bytes();
    }
};

// every call on a mesh refuses NULL, and a mesh whose refit failed half way (its records are a mix of two vertex sets)
static int mesh_usable(const dg_mesh* m, const char* who)
{
    if (!m) return fail(DG_ERR_INVALID, "%s: mesh is NULL (not constructed)", who);
    if (m->failed)
        return fail(DG_ERR_INVALID, "%s: a refit of this mesh failed after it had started to write the records; the mesh is unusable "
                    "(dg_mesh_destroy it and create it again)", who);
    return DG_OK;
}

struct dg_field {
    dg_grid_desc desc;
    FieldDev dev;
    DevBuf<double> d_packed;
    DevBuf<unsigned> d_cell_map;
    DevBuf<double2> d_tab;
    uint64_t n_nodes = 0, n_cells_kept = 0;
    double coeff_max = 0.0;      // k3_coeff_max of the packed coefficients: whether K3 may skip points outside the kernel support
    int device = 0;
};

// ------------------------------------------------------------------------------------------------ library
extern "C" {

int dg_abi_version(void) { return DG_ABI_VERSION; }
const char* dg_last_error(void) { return g_err.c_str(); }
uint64_t dg_kernel_launch_count(void) { return g_launches.load(); }
void dg_kernel_launch_count_reset(void) { g_launches.store(0); }

int dg_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int dg_set_device(int device)
{
    if (int rc = require_device()) return rc;
    DG_CUDA(cudaSetDevice(device));
    return DG_OK;
}

int dg_selftest(void)
{
    if (int rc = require_device()) return rc;
    // a*b + c where the unfused result (two roundings) differs from the fused one:
    // a = b = 1 + 2^-27  ->  a*b = 1 + 2^-26 + 2^-54 (rounds to 1 + 2^-26); c = -(1 + 2^-26).
    const double a = 1.0 + std::ldexp(1.0, -27), c = -(1.0 + std::ldexp(1.0, -26));
    DevBuf<double> out;
    DG_CUDA(out.alloc(1));
    DG_LAUNCH(k1_launch_fma_probe(a, a, c, out.p, nullptr));
    double r = -1.0;
    DG_CUDA(cudaMemcpy(&r, out.p, sizeof r, cudaMemcpyDeviceToHost));
    if (r != 0.0) {
        g_selftest_state = -1;
        return fail(DG_ERR_SELFTEST, "device code was compiled with FMA contraction (a*b+c probe returned %.17g, expected 0): "
                    "build with -fmad=false", r);
    }
    g_selftest_state = 1;
    return DG_OK;
}

// Measured fp64 issue rate of the current device for the library's own instruction mix (DMUL + DADD, no FMA): Tflop/s.
int dg_fp64_rate_probe(double* tflops)
{
    if (int rc = require_device()) return rc;
    if (!tflops) return fail(DG_ERR_INVALID, "dg_fp64_rate_probe: NULL argument");
    int dev = 0, n_sm = 0;
    DG_CUDA(cudaGetDevice(&dev));
    DG_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    const int blocks = n_sm * 8, iters = 1 << 14;
    DevBuf<double> out;
    DG_CUDA(out.alloc(1));
    cudaEvent_t e0, e1;
    DG_CUDA(cudaEventCreate(&e0)); DG_CUDA(cudaEventCreate(&e1));
    float best = 0.f;
    for (int rep = 0; rep < 4; rep++) {                       // first repetition warms up
        DG_CUDA(cudaEventRecord(e0, nullptr));
        DG_LAUNCH(k1_launch_fp64_rate_probe(blocks, iters, out.p, nullptr));
        DG_CUDA(cudaEventRecord(e1, nullptr));
        DG_CUDA(cudaEventSynchronize(e1));
        float ms = 0.f;
        DG_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && (best == 0.f || ms < best)) best = ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    const double flops = (double)blocks * 256.0 * 8.0 * 2.0 * (double)iters;
    *tflops = best > 0.f ? flops / (best * 1e-3) / 1e12 : 0.0;
    return DG_OK;
}

static int ensure_selftest()
{
    const int s = g_selftest_state.load();
    if (s == 1) return DG_OK;
    if (s == -1) return fail(DG_ERR_SELFTEST, "device self-test failed earlier (FMA contraction on)");
    return dg_selftest();
}

// ------------------------------------------------------------------------------------------------ grid helpers
int dg_grid_init(const double mn[3], const double mx[3], const uint32_t res[3], dg_grid_desc* out)
{
    if (!mn || !mx || !res || !out) return fail(DG_ERR_INVALID, "dg_grid_init: NULL argument");
    uint64_t nn;
    if (int rc = dg_grid_num_nodes(res, &nn)) return rc;
    std::memset(out, 0, sizeof *out);
    for (int d = 0; d < 3; d++) {
        out->domain_min[d] = mn[d]; out->domain_max[d] = mx[d]; out->resolution[d] = res[d];
        out->cell_size[d] = (mx[d] - mn[d]) / (double)res[d];      // diagonal().cwiseQuotient(n.cast<double>())
        out->inv_cell_size[d] = 1.0 / out->cell_size[d];           // cwiseInverse()
    }
    return DG_OK;
}

int dg_grid_num_nodes(const uint32_t res[3], uint64_t* n_nodes)
{
    if (!res || !n_nodes) return fail(DG_ERR_INVALID, "dg_grid_num_nodes: NULL argument");
    if (res[0] == 0 || res[1] == 0 || res[2] == 0) return fail(DG_ERR_INVALID, "resolution must be >= 1 in every dimension");
    const uint64_t nx = res[0], ny = res[1], nz = res[2];
    const uint64_t nv = (nx + 1) * (ny + 1) * (nz + 1);
    const uint64_t ne = nx * (ny + 1) * (nz + 1) + (nx + 1) * ny * (nz + 1) + (nx + 1) * (ny + 1) * nz;
    const uint64_t total = nv + 2 * ne;
    // the reference indexes nodes with `int l` (cubic_lagrange_discrete_grid.cpp:809) and stores uint32 ids
    if (nx > 65535 || ny > 65535 || nz > 65535 || total > 0x7fffffffull || nx * ny * nz > 0x7fffffffull)
        return fail(DG_ERR_INVALID, "grid too large: %llu nodes exceed the reference's int/uint32 node ids", (unsigned long long)total);
    *n_nodes = total;
    return DG_OK;
}

int dg_generate_sdf_domain(const double* V, uint64_t nV, double mn[3], double mx[3])
{
    if (!V || !mn || !mx || nV == 0) return fail(DG_ERR_INVALID, "dg_generate_sdf_domain: NULL / empty argument");
    for (int d = 0; d < 3; d++) { mn[d] = DBL_MAX; mx[d] = -DBL_MAX; }     // AlignedBox::setEmpty + extend
    for (uint64_t i = 0; i < nV; i++)
        for (int d = 0; d < 3; d++) { mn[d] = std::fmin(mn[d], V[3 * i + d]); mx[d] = std::fmax(mx[d], V[3 * i + d]); }
    // cmd/generate_sdf/main.cpp:89-90: max is padded first, then min with the grown diagonal.  Eigen >= 3.3 reduces a
    // Vector3d as (a0 + a1) + a2.
    for (int pass = 0; pass < 2; pass++) {
        const double dx = mx[0] - mn[0], dy = mx[1] - mn[1], dz = mx[2] - mn[2];
        const double nrm = std::sqrt((dx * dx + dy * dy) + dz * dz);
        const double pad = 1.0e-3 * nrm * 1.0;
        for (int d = 0; d < 3; d++) { if (pass == 0) mx[d] += pad; else mn[d] -= pad; }
    }
    return DG_OK;
}

// ------------------------------------------------------------------------------------------------ mesh
int dg_mesh_create(const double* V, uint64_t nV, const uint32_t* F, uint64_t nT, dg_mesh** out)
{
    if (!out) return fail(DG_ERR_INVALID, "dg_mesh_create: out is NULL");
    *out = nullptr;
    if (!V || !F || nT == 0 || nV == 0) return fail(DG_ERR_INVALID, "dg_mesh_create: empty triangle list");   // ref: exit(-1)
    if (int rc = require_device()) return rc;
    if (int rc = ensure_selftest()) return rc;
    std::unique_ptr<dg_mesh> m(new (std::nothrow) dg_mesh());
    if (!m) return fail(DG_ERR_NOMEM, "dg_mesh_create: out of host memory");
    const auto t0 = std::chrono::steady_clock::now();
    const char* why = "";
    try {
        if (!build_host_bvh(V, nV, F, nT, m->host, &why, true)) return fail(DG_ERR_INVALID, "dg_mesh_create: %s", why);
    } catch (const std::bad_alloc&) { return fail(DG_ERR_NOMEM, "dg_mesh_create: out of host memory"); }
    const auto t1 = std::chrono::steady_clock::now();
    m->build_us = (uint64_t)std::chrono::duration_cast<std::chrono::microseconds>(t1 - t0).count();

    DG_CUDA(cudaGetDevice(&m->device));
    DG_CUDA(m->d_spheres.alloc(nT));
    DG_CUDA(m->d_leaves.alloc(nT));
    DG_CUDA(m->d_normals.alloc(nT));
    DG_CUDA(m->d_nodes_f.alloc(nT * K1_NODEF_STRIDE));
    DG_CUDA(m->d_leaves_f.alloc(nT));
    DG_CUDA(cudaMemcpy(m->d_leaves_f.p, m->host.leaves_f.data(), nT * sizeof(LeafF), cudaMemcpyHostToDevice));
    m->dev.leaves_f = m->d_leaves_f.p;
    DG_CUDA(cudaMemcpy(m->d_spheres.p, m->host.spheres.data(), nT * sizeof(SpherePair), cudaMemcpyHostToDevice));
    DG_CUDA(cudaMemcpy(m->d_leaves.p, m->host.leaves.data(), nT * sizeof(LeafRecord), cudaMemcpyHostToDevice));
    DG_CUDA(cudaMemcpy(m->d_normals.p, m->host.normals.data(), nT * sizeof(PseudoNormals), cudaMemcpyHostToDevice));
    {   // the fp32 record of every internal node: sphere pair + child boxes, bvh_build.h
        static_assert(K1_NODEF_STRIDE * sizeof(float4) >= sizeof(SpherePairF) + sizeof(BoxPairF), "node record too small");
        RawVec<float4> rec(nT * K1_NODEF_STRIDE);
        pack_node_records(m->host, K1_NODEF_STRIDE, reinterpret_cast<float*>(rec.data()));
        DG_CUDA(cudaMemcpy(m->d_nodes_f.p, rec.data(), rec.size() * sizeof(float4), cudaMemcpyHostToDevice));
    }
    m->dev.nodes_f = m->d_nodes_f.p;
    for (int d = 0; d < 3; d++) m->dev.ctr[d] = m->host.center[d];
    m->dev.half_extent = (float)m->host.half_extent * 1.0000002f;   // rounded up
    m->dev.spheres = m->d_spheres.p; m->dev.leaves = m->d_leaves.p; m->dev.normals = m->d_normals.p;
    m->dev.n_tri = (int)nT;
    m->dev.stack_depth = m->host.max_depth > 1 ? m->host.max_depth - 1 : 1;
    DG_CUDA(k1_configure(m->dev.stack_depth));
    const auto t2 = std::chrono::steady_clock::now();
    m->upload_us = (uint64_t)std::chrono::duration_cast<std::chrono::microseconds>(t2 - t1).count();
    // the device records are the product; the host copies of the big arrays are no longer needed
    RawVec<SpherePair>().swap(m->host.spheres);
    RawVec<SpherePairF>().swap(m->host.spheres_f);
    RawVec<BoxPairF>().swap(m->host.boxes_f);
    RawVec<LeafF>().swap(m->host.leaves_f);        // keep `order`, V, F, pseudonormals for diagnostics
    RawVec<LeafRecord>().swap(m->host.leaves);
    RawVec<PseudoNormals>().swap(m->host.normals);
    *out = m.release();
    return DG_OK;
}

int dg_mesh_destroy(dg_mesh* m)
{
    if (!m) return DG_OK;
    delete m;
    return DG_OK;
}

int dg_mesh_info(const dg_mesh* m, uint64_t info[8])
{
    if (int rc = mesh_usable(m, "dg_mesh_info")) return rc;
    if (!info) return fail(DG_ERR_INVALID, "dg_mesh_info: NULL argument");
    info[0] = m->host.n_vertices; info[1] = m->host.n_triangles; info[2] = (uint64_t)m->dev.stack_depth;
    info[3] = (uint64_t)m->host.flags;
    info[4] = m->d_spheres.bytes() + m->d_leaves.bytes() + m->d_normals.bytes() + m->d_nodes_f.bytes() + m->d_leaves_f.bytes();
    info[4] += m->refit_bytes();                                            // 0 until the first dg_mesh_refit
    {
        std::lock_guard<std::mutex> lock(m->wind_mu);
        info[4] += m->d_wind_leaves.bytes() + m->d_wind_clusters.bytes();      // 0 until the winding records are first used
    }
    info[5] = m->build_us; info[6] = m->upload_us; info[7] = (uint64_t)m->device;
    return DG_OK;
}

int dg_mesh_tree(const dg_mesh* m, double* spheres, int32_t* kids)
{
    if (int rc = mesh_usable(m, "dg_mesh_tree")) return rc;
    // the sphere pairs were released after upload: read them back from the device
    HostBvh tmp;
    tmp.n_triangles = m->host.n_triangles;
    tmp.order = m->host.order;
    tmp.spheres.resize(m->host.n_triangles);
    DG_CUDA(cudaMemcpy(tmp.spheres.data(), m->d_spheres.p, m->host.n_triangles * sizeof(SpherePair), cudaMemcpyDeviceToHost));
    export_reference_tree(tmp, spheres, kids);
    return DG_OK;
}

int dg_mesh_pseudonormals(const dg_mesh* m, double* tri, double* edge, double* vert)
{
    if (int rc = mesh_usable(m, "dg_mesh_pseudonormals")) return rc;
    if (m->refit_done) {        // the reference's arrays rebuilt from the device's per-leaf blocks (V0 V1 V2 E01 E12 E02 F)
        const uint64_t nT = m->host.n_triangles;
        RawVec<PseudoNormals> blk(nT);
        DG_CUDA(cudaMemcpy(blk.data(), m->d_normals.p, nT * sizeof(PseudoNormals), cudaMemcpyDeviceToHost));
        if (vert) std::fill(vert, vert + 3 * m->host.n_vertices, std::numeric_limits<double>::quiet_NaN());     // no triangle uses it
        for (uint64_t pos = 0; pos < nT; pos++) {
            const size_t id = (size_t)m->host.order[pos];
            const PseudoNormals& N = blk[pos];
            for (int d = 0; d < 3; d++) {
                if (tri) tri[3 * id + d] = N.n[6][d];
                if (edge) for (int k = 0; k < 3; k++) edge[9 * id + 3 * k + d] = N.n[3 + k][d];
                if (vert) for (int k = 0; k < 3; k++) vert[3 * (size_t)m->host.F[3 * id + k] + d] = N.n[k][d];
            }
        }
        return DG_OK;
    }
    if (tri) std::memcpy(tri, m->host.pn_tri.data(), m->host.pn_tri.size() * sizeof(double));
    if (edge) std::memcpy(edge, m->host.pn_edge.data(), m->host.pn_edge.size() * sizeof(double));
    if (vert) std::memcpy(vert, m->host.pn_vert.data(), m->host.pn_vert.size() * sizeof(double));
    return DG_OK;
}

// ------------------------------------------------------------------------------------------------ refit (k8_refit.cu)
// the scratch and tables of the refit as K8 reads them; output pointers are set by the caller
static RefitDev refit_dev(const dg_mesh* m)
{
    RefitDev r;
    r.V = m->d_V.p; r.n_vertices = m->host.n_vertices;
    r.n_tri = (int)m->host.n_triangles; r.levels = m->host.max_depth;
    r.F = m->d_F.p; r.f_leaf = m->d_f_leaf.p; r.order = m->d_order.p; r.inc_begin = m->d_inc_begin.p; r.inc = m->d_inc.p; r.nodes = m->d_nodes.p;
    r.sums = m->d_sums.p; r.part = m->d_part.p; r.bounds = m->d_bounds.p;
    r.pn_tri = m->d_pn_tri.p; r.angle = m->d_angle.p; r.pn_vert = m->d_pn_vert.p; r.pn_edge = m->d_pn_edge.p;
    r.nodef_stride = K1_NODEF_STRIDE;
    static_assert(K1_NODEF_STRIDE <= K8_MAX_NODEF_STRIDE, "k8_pack_kernel stages at most K8_MAX_NODEF_STRIDE float4s");
    return r;
}

// ------------------------------------------------------------------------------------------------ K5: winding numbers, the winding sign mode
static int check_beta(double beta, const char* who)
{
    if (!(beta >= 1.0)) return fail(DG_ERR_INVALID, "%s: beta must be >= 1 or +inf (got %g)", who, beta);     // below 1 or NaN
    return DG_OK;
}

// the mesh's K5 records on its device, built (host threads) and uploaded at the first call; later calls only read them
static int winding_dev(const dg_mesh* m, const WindDev*& out, const char* who)
{
    std::lock_guard<std::mutex> lock(m->wind_mu);
    if (!m->wind_ready && m->refit_done) {      // the host copy of V is stale: the records of the refit positions, built by K8's kernels
        const uint64_t nT = m->host.n_triangles;
        if (m->dev.stack_depth > K5_MAX_STACK) return fail(DG_ERR_INVALID, "%s: tree too deep for the winding walk", who);
        DevBuf<WindLeaf> dl;
        DevBuf<WindClusterPair> dc;
        DG_CUDA(dl.alloc(nT));
        DG_CUDA(dc.alloc(nT));
        RefitDev r = refit_dev(m);
        r.wind_leaves = dl.p; r.wind_clusters = dc.p;
        DG_LAUNCH(k8_launch_refit(r, m->refit_levels, false, nullptr));
        DG_CUDA(cudaStreamSynchronize(nullptr));
        std::swap(m->d_wind_leaves.p, dl.p); std::swap(m->d_wind_leaves.n, dl.n);
        std::swap(m->d_wind_clusters.p, dc.p); std::swap(m->d_wind_clusters.n, dc.n);
        m->wind.leaves = m->d_wind_leaves.p; m->wind.clusters = m->d_wind_clusters.p;
        m->wind.n_tri = (int)nT; m->wind.stack_depth = m->dev.stack_depth;
        m->wind_ready = true;
    }
    if (!m->wind_ready) {
        const uint64_t nT = m->host.n_triangles;
        if (m->dev.stack_depth > K5_MAX_STACK) return fail(DG_ERR_INVALID, "%s: tree too deep for the winding walk", who);
        RawVec<WindLeaf> leaves;
        RawVec<WindClusterPair> clusters;
        try { build_winding_records(m->host, leaves, clusters); }
        catch (const std::bad_alloc&) { return fail(DG_ERR_NOMEM, "%s: out of host memory", who); }
        DevBuf<WindLeaf> dl;
        DevBuf<WindClusterPair> dc;
        DG_CUDA(dl.alloc(nT));
        DG_CUDA(dc.alloc(nT));
        DG_CUDA(cudaMemcpy(dl.p, leaves.data(), nT * sizeof(WindLeaf), cudaMemcpyHostToDevice));
        DG_CUDA(cudaMemcpy(dc.p, clusters.data(), nT * sizeof(WindClusterPair), cudaMemcpyHostToDevice));
        std::swap(m->d_wind_leaves.p, dl.p); std::swap(m->d_wind_leaves.n, dl.n);
        std::swap(m->d_wind_clusters.p, dc.p); std::swap(m->d_wind_clusters.n, dc.n);
        m->wind.leaves = m->d_wind_leaves.p; m->wind.clusters = m->d_wind_clusters.p;
        m->wind.n_tri = (int)nT; m->wind.stack_depth = m->dev.stack_depth;
        m->wind_ready = true;
    }
    out = &m->wind;
    return DG_OK;
}

static int refuse_winding(const dg_mesh* m, const char* who)
{
    if (m && m->sign_mode == DG_SIGN_WINDING)
        return fail(DG_ERR_INVALID, "%s: the mesh is in the winding sign mode, which runs on one GPU only (dg_sample_sdf_device, dg_add_function_sdf, "
                    "dg_reduced_band_create ...); set DG_SIGN_PSEUDONORMAL for the multi-GPU and sharded entry points", who);
    return DG_OK;
}

int dg_mesh_set_sign_mode(dg_mesh* m, int mode, double beta)
{
    if (int rc = mesh_usable(m, "dg_mesh_set_sign_mode")) return rc;
    if (mode != DG_SIGN_PSEUDONORMAL && mode != DG_SIGN_WINDING) return fail(DG_ERR_INVALID, "dg_mesh_set_sign_mode: unknown mode %d", mode);
    if (int rc = check_beta(beta, "dg_mesh_set_sign_mode")) return rc;
    m->sign_mode = mode;
    m->beta = beta;
    return DG_OK;
}

// topology tables (from F and the leaf order, once) and every scratch buffer: all allocated before any record is written
static int refit_prepare(dg_mesh* m)
{
    if (m->refit_ready) return DG_OK;
    const uint64_t nT = m->host.n_triangles, nV = m->host.n_vertices;
    RefitTopoHost topo;
    k8_build_topology(m->host, topo);
    DG_CUDA(m->d_V.alloc(3 * nV));
    DG_CUDA(m->d_F.alloc(3 * nT)); DG_CUDA(m->d_f_leaf.alloc(3 * nT)); DG_CUDA(m->d_order.alloc(nT));
    DG_CUDA(m->d_inc_begin.alloc(nV + 1)); DG_CUDA(m->d_inc.alloc(3 * nT));
    DG_CUDA(m->d_nodes.alloc(topo.nodes.size()));
    DG_CUDA(m->d_sums.alloc(nT)); DG_CUDA(m->d_part.alloc(k8_bounds_entries(nV))); DG_CUDA(m->d_bounds.alloc(5));
    DG_CUDA(m->d_pn_tri.alloc(3 * nT)); DG_CUDA(m->d_angle.alloc(3 * nT)); DG_CUDA(m->d_pn_vert.alloc(3 * nV)); DG_CUDA(m->d_pn_edge.alloc(9 * nT));
    DG_CUDA(cudaMemcpy(m->d_F.p, m->host.F.data(), 3 * nT * sizeof(uint32_t), cudaMemcpyHostToDevice));
    DG_CUDA(cudaMemcpy(m->d_f_leaf.p, topo.f_leaf.data(), 3 * nT * sizeof(uint32_t), cudaMemcpyHostToDevice));
    DG_CUDA(cudaMemcpy(m->d_order.p, m->host.order.data(), nT * sizeof(int32_t), cudaMemcpyHostToDevice));
    DG_CUDA(cudaMemcpy(m->d_inc_begin.p, topo.inc_begin.data(), (nV + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice));
    DG_CUDA(cudaMemcpy(m->d_inc.p, topo.inc.data(), 3 * nT * sizeof(uint32_t), cudaMemcpyHostToDevice));
    if (!topo.nodes.empty()) DG_CUDA(cudaMemcpy(m->d_nodes.p, topo.nodes.data(), topo.nodes.size() * sizeof(RefitNodeRef), cudaMemcpyHostToDevice));
    m->refit_levels = topo.level_begin;
    m->refit_ready = true;
    return DG_OK;
}

static int refit_checks(dg_mesh* m, const void* v, uint64_t nV, const char* who)
{
    if (int rc = mesh_usable(m, who)) return rc;
    if (nV && !v) return fail(DG_ERR_INVALID, "%s: vertices is NULL", who);
    if (nV != m->host.n_vertices)
        return fail(DG_ERR_INVALID, "%s: %llu vertices, but the mesh was built with %llu (a refit keeps the triangles; dg_mesh_create for a new topology)",
                    who, (unsigned long long)nV, (unsigned long long)m->host.n_vertices);
    if (int rc = check_handle_device(m->device, who)) return rc;
    if (m->borrows.load() > 0)
        return fail(DG_ERR_INVALID, "%s: a live dg_mesh_group replicates this mesh on other GPUs; its replicas would go stale (destroy the group first)", who);
    return DG_OK;
}

int dg_mesh_refit_device(dg_mesh* m, const double* d_vertices, uint64_t n_vertices, void* stream)
{
    if (int rc = refit_checks(m, d_vertices, n_vertices, "dg_mesh_refit_device")) return rc;
    if (d_vertices != m->d_V.p) {             // device (or managed) memory of the mesh's device: refused before anything is written
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, d_vertices) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
#ifndef DG_EMU
        if ((a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != m->device)
            return fail(DG_ERR_INVALID, "dg_mesh_refit_device: vertices is not device memory of the mesh's device %d (dg_mesh_refit takes a host array)",
                        m->device);
#endif
    }
    if (int rc = refit_prepare(m)) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    const uint64_t nV = n_vertices;
    // from here on records are written: a CUDA error leaves the mesh failed
    auto broken = [&](cudaError_t e, const char* what) {
        m->failed = true;
        return fail(cuda_code(e), "dg_mesh_refit_device: %s failed: %s; the mesh is left unusable "
                    "(dg_mesh_destroy it)", what, cudaGetErrorString(e));
    };
    cudaError_t e;
    if (d_vertices != m->d_V.p && (e = cudaMemcpyAsync(m->d_V.p, d_vertices, 3 * nV * sizeof(double), cudaMemcpyDeviceToDevice, st)) != cudaSuccess)
        return broken(e, "cudaMemcpyAsync of the vertices");
    std::lock_guard<std::mutex> lock(m->wind_mu);
    RefitDev r = refit_dev(m);
    r.spheres = m->d_spheres.p; r.leaves = m->d_leaves.p; r.leaves_f = m->d_leaves_f.p; r.normals = m->d_normals.p; r.nodes_f = m->d_nodes_f.p;
    if (m->wind_ready) { r.wind_leaves = m->d_wind_leaves.p; r.wind_clusters = m->d_wind_clusters.p; }     // else built at their first use
    if ((e = k8_launch_refit(r, m->refit_levels, true, st)) != cudaSuccess) return broken(e, "k8_launch_refit");
    g_launches.fetch_add(1);
    double b[5];
    if ((e = cudaMemcpyAsync(b, m->d_bounds.p, sizeof b, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return broken(e, "cudaMemcpyAsync of the bounds");
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return broken(e, "cudaStreamSynchronize");
    for (int d = 0; d < 3; d++) { m->host.center[d] = b[d]; m->dev.ctr[d] = b[d]; }
    m->host.half_extent = b[3];
    m->dev.half_extent = (float)m->host.half_extent * 1.0000002f;   // rounded up, as dg_mesh_create
    m->refit_done = true;
    return DG_OK;
}

int dg_mesh_refit(dg_mesh* m, const double* vertices, uint64_t n_vertices)
{
    if (int rc = refit_checks(m, vertices, n_vertices, "dg_mesh_refit")) return rc;
    if (int rc = refit_prepare(m)) return rc;
    const cudaError_t e = cudaMemcpy(m->d_V.p, vertices, 3 * n_vertices * sizeof(double), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {                   // d_V may now hold part of the new positions: out of step with the records
        m->failed = true;
        return fail(cuda_code(e), "dg_mesh_refit: upload of the vertices failed: %s; the mesh "
                    "is left unusable (dg_mesh_destroy it)", cudaGetErrorString(e));
    }
    return dg_mesh_refit_device(m, m->d_V.p, n_vertices, nullptr);
}

// the argument checks of the winding-number and distance queries; the device check is the caller's, since the host forms return at n == 0
// before it
static int winding_check(const dg_mesh* m, const void* x, uint64_t n, double beta, const void* w, const char* who)
{
    if (int rc = mesh_usable(m, who)) return rc;
    if (int rc = check_beta(beta, who)) return rc;
    if (n && (!x || !w)) return fail(DG_ERR_INVALID, "%s: points or output is NULL", who);
    return DG_OK;
}

static int winding_launch(const dg_mesh* m, const double* d_x, uint64_t n, double beta, double* d_w, cudaStream_t st, const char* who)
{
    const WindDev* wd = nullptr;
    if (int rc = winding_dev(m, wd, who)) return rc;
    DG_LAUNCH(k5_launch_winding(*wd, d_x, n, beta, d_w, st));
    return DG_OK;
}

int dg_mesh_winding_number_device(const dg_mesh* m, const double* d_x, uint64_t n, double beta, double* d_w, void* stream)
{
    static const char* who = "dg_mesh_winding_number_device";
    if (int rc = winding_check(m, d_x, n, beta, d_w, who)) return rc;
    if (int rc = check_handle_device(m->device, who)) return rc;
    if (n == 0) return DG_OK;
    return winding_launch(m, d_x, n, beta, d_w, (cudaStream_t)stream, who);
}

int dg_mesh_winding_number(const dg_mesh* m, const double* x, uint64_t n, double beta, double* w)
{
    static const char* who = "dg_mesh_winding_number";
    if (int rc = winding_check(m, x, n, beta, w, who)) return rc;
    if (n == 0) return DG_OK;
    if (int rc = check_handle_device(m->device, who)) return rc;
    return stage_on_device(n, n, {{x, 3 * sizeof(double)}}, {{w, sizeof(double)}}, [&](void* const* in, void* const* out, uint64_t, uint64_t c) {
        return winding_launch(m, (const double*)in[0], c, beta, (double*)out[0], nullptr, who);
    });
}

static int distance_check(const dg_mesh* m, const void* pts, uint64_t n, const char* who)
{
    if (int rc = mesh_usable(m, who)) return rc;
    if (n && !pts) return fail(DG_ERR_INVALID, "%s: points is NULL", who);
    return DG_OK;
}

static int distance_launch(const dg_mesh* m, const double* d_pts, uint64_t n, int is_signed, double* d_dist, double* d_near, int32_t* d_ent,
                           int32_t* d_tri, cudaStream_t st, const char* who)
{
    if (is_signed && m->sign_mode == DG_SIGN_WINDING) {       // the unsigned query, then the sign from w (k5_winding.cu)
        const WindDev* wd = nullptr;
        if (int rc = winding_dev(m, wd, who)) return rc;
        DG_LAUNCH(k1_launch_distance(m->dev, d_pts, n, 0, d_dist, d_near, d_ent, d_tri, st));
        if (d_dist) DG_LAUNCH(k5_launch_sign_points(*wd, d_pts, n, m->beta, d_dist, st));
        return DG_OK;
    }
    DG_LAUNCH(k1_launch_distance(m->dev, d_pts, n, is_signed, d_dist, d_near, d_ent, d_tri, st));
    return DG_OK;
}

int dg_mesh_distance_device(const dg_mesh* m, const double* d_pts, uint64_t n, int is_signed, double* d_dist, double* d_near,
                            int32_t* d_ent, int32_t* d_tri, void* stream)
{
    static const char* who = "dg_mesh_distance_device";
    if (int rc = distance_check(m, d_pts, n, who)) return rc;
    if (int rc = check_handle_device(m->device, who)) return rc;
    return distance_launch(m, d_pts, n, is_signed, d_dist, d_near, d_ent, d_tri, (cudaStream_t)stream, who);
}

int dg_mesh_distance(const dg_mesh* m, const double* pts, uint64_t n, int is_signed, double* dist, double* nearp, int32_t* ent,
                     int32_t* tri)
{
    static const char* who = "dg_mesh_distance";
    if (int rc = distance_check(m, pts, n, who)) return rc;
    if (n == 0) return DG_OK;
    if (int rc = check_handle_device(m->device, who)) return rc;
    return stage_on_device(n, n, {{pts, 3 * sizeof(double)}},
                           {{dist, sizeof(double)}, {nearp, 3 * sizeof(double)}, {ent, sizeof(int32_t)}, {tri, sizeof(int32_t)}},
                           [&](void* const* in, void* const* out, uint64_t, uint64_t c) {
                               return distance_launch(m, (const double*)in[0], c, is_signed, (double*)out[0], (double*)out[1], (int32_t*)out[2],
                                                      (int32_t*)out[3], nullptr, who);
                           });
}

// ------------------------------------------------------------------------------------------------ K1
static int check_range(const dg_grid_desc* grid, uint64_t b, uint64_t e, GridDev& g, const char* who)
{
    if (int rc = grid_checked(grid, g, who)) return rc;
    const uint64_t nn = grid_nodes(g);
    if (b > e || e > nn) return fail(DG_ERR_INVALID, "%s: node range [%llu, %llu) outside [0, %llu]", who, (unsigned long long)b,
                                      (unsigned long long)e, (unsigned long long)nn);
    return DG_OK;
}

int dg_sample_sdf_device(const dg_mesh* m, const dg_grid_desc* grid, double sign, uint64_t l_begin, uint64_t l_end, double* d_out,
                         void* stream)
{
    static const char* who = "dg_sample_sdf_device";
    if (int rc = mesh_usable(m, who)) return rc;
    GridDev g;
    if (int rc = check_range(grid, l_begin, l_end, g, who)) return rc;
    if (l_end > l_begin && !d_out) return fail(DG_ERR_INVALID, "%s: output is NULL", who);
    if (int rc = check_handle_device(m->device, who)) return rc;
    if (m->sign_mode == DG_SIGN_WINDING) {      // K1 with sign = +1, then the node pass of k5_winding.cu
        const WindDev* wd = nullptr;
        if (int rc = winding_dev(m, wd, who)) return rc;
        DG_LAUNCH(k1_launch_sample_nodes(m->dev, g, 1.0, l_begin, l_end - l_begin, d_out, (cudaStream_t)stream));
        DG_LAUNCH(k5_launch_sign_nodes(*wd, g, sign, INFINITY, m->beta, l_begin, l_end - l_begin, d_out, (cudaStream_t)stream));
        return DG_OK;
    }
    DG_LAUNCH(k1_launch_sample_nodes(m->dev, g, sign, l_begin, l_end - l_begin, d_out, (cudaStream_t)stream));
    return DG_OK;
}

static int check_band(double band, const char* who)
{
    if (!(band >= 0.0)) return fail(DG_ERR_INVALID, "%s: band must be >= 0 (got %g)", who, band);     // negative or NaN
    return DG_OK;
}

// addFunction(func, verbose, pred) with pred(x) = |md.signed_distance(x).distance| <= band (cubic_lagrange_discrete_grid.cpp:806-817): the
// classifier passes and the band form of the node loop, in stream order; the scratch is allocated and released on the same stream.
int dg_sample_sdf_band_device(const dg_mesh* m, const dg_grid_desc* grid, double sign, double band, uint64_t l_begin, uint64_t l_end, double* d_out,
                              void* stream)
{
    static const char* who = "dg_sample_sdf_band_device";
    if (int rc = mesh_usable(m, who)) return rc;
    GridDev g;
    if (int rc = check_range(grid, l_begin, l_end, g, who)) return rc;
    if (int rc = check_band(band, who)) return rc;
    if (l_end > l_begin && !d_out) return fail(DG_ERR_INVALID, "%s: output is NULL", who);
    if (int rc = check_handle_device(m->device, who)) return rc;
    if (l_end == l_begin) return DG_OK;
    const cudaStream_t st = (cudaStream_t)stream;
    const WindDev* wd = nullptr;
    if (m->sign_mode == DG_SIGN_WINDING) { if (int rc = winding_dev(m, wd, who)) return rc; }
    const double k1_sign = wd ? 1.0 : sign;     // winding mode: K1 with sign = +1, then the node pass
    const size_t bytes = k1_band_scratch_bytes(g, l_begin, l_end - l_begin);
    void* scratch = nullptr;
#ifdef DG_EMU
    DG_CUDA(cudaMalloc(&scratch, bytes));
    const cudaError_t e = k1_launch_sample_nodes_band(m->dev, g, k1_sign, band, l_begin, l_end - l_begin, d_out, scratch, st);
    cudaFree(scratch);
#else
    DG_CUDA(cudaMallocAsync(&scratch, bytes, st));
    const cudaError_t e = k1_launch_sample_nodes_band(m->dev, g, k1_sign, band, l_begin, l_end - l_begin, d_out, scratch, st);
    cudaFreeAsync(scratch, st);
#endif
    DG_LAUNCH(e);
    if (wd) DG_LAUNCH(k5_launch_sign_nodes(*wd, g, sign, band, m->beta, l_begin, l_end - l_begin, d_out, st));
    return DG_OK;
}

// Host-buffer path of K1.  Resources that are expensive to create per call (device scratch, two pinned staging buffers,
// streams, events) live in a per-process pool.  The range is cut into a few kernel launches dealt to two streams (a K1
// launch ends with a tail of long-running warps; the next launch fills the machine meanwhile); a third stream DMAs
// finished chunks into the pinned double buffer while the CPU copies the previous piece into the caller's (pageable) memory.
namespace {
struct HostPathPool {
    std::mutex mu;
    int device = -1;
    double* d_out = nullptr; size_t d_cap = 0;
    double* stage[2] = {nullptr, nullptr};
    cudaStream_t s_k[2] = {nullptr, nullptr}, s_c = nullptr;
    cudaEvent_t dma_ev[2] = {nullptr, nullptr};
    std::vector<cudaEvent_t> chunk_ev;
    void* band_scratch[2] = {nullptr, nullptr}; size_t band_cap = 0;   // scratch of the narrow-band classifier, one per kernel stream
    static constexpr size_t kPiece = 4u << 20;          // doubles per staging buffer (32 MiB)
    cudaError_t prepare(size_t n, size_t n_chunks, size_t band_bytes = 0)
    {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev != device) { release(); device = dev; }
        if (!s_c) {
            for (int i = 0; i < 2 && e == cudaSuccess; i++) e = cudaStreamCreateWithFlags(&s_k[i], cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s_c, cudaStreamNonBlocking);
            for (int i = 0; i < 2 && e == cudaSuccess; i++) e = cudaEventCreateWithFlags(&dma_ev[i], cudaEventDisableTiming);
            for (int i = 0; i < 2 && e == cudaSuccess; i++) e = cudaMallocHost(reinterpret_cast<void**>(&stage[i]), kPiece * sizeof(double));
            if (e != cudaSuccess) { release(); return e; }          // never leave a half-built pool behind
        }
        if (n > d_cap) {
            if (d_out) cudaFree(d_out);
            d_out = nullptr; d_cap = 0;
            e = cudaMalloc(reinterpret_cast<void**>(&d_out), n * sizeof(double));
            if (e != cudaSuccess) return e;
            d_cap = n;
        }
        if (band_bytes > band_cap) {
            for (int i = 0; i < 2; i++) { if (band_scratch[i]) cudaFree(band_scratch[i]); band_scratch[i] = nullptr; }
            band_cap = 0;
            for (int i = 0; i < 2; i++) { e = cudaMalloc(&band_scratch[i], band_bytes); if (e != cudaSuccess) return e; }
            band_cap = band_bytes;
        }
        while (chunk_ev.size() < n_chunks) {
            cudaEvent_t ev;
            e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
            if (e != cudaSuccess) return e;
            chunk_ev.push_back(ev);
        }
        return cudaSuccess;
    }
    void release()
    {
        if (d_out) cudaFree(d_out);
        d_out = nullptr; d_cap = 0;
        for (int i = 0; i < 2; i++) { if (band_scratch[i]) cudaFree(band_scratch[i]); band_scratch[i] = nullptr; }
        band_cap = 0;
        for (int i = 0; i < 2; i++) { if (stage[i]) cudaFreeHost(stage[i]); stage[i] = nullptr; if (s_k[i]) cudaStreamDestroy(s_k[i]); s_k[i] = nullptr;
                                      if (dma_ev[i]) cudaEventDestroy(dma_ev[i]); dma_ev[i] = nullptr; }
        if (s_c) cudaStreamDestroy(s_c);
        s_c = nullptr;
        for (auto ev : chunk_ev) cudaEventDestroy(ev);
        chunk_ev.clear();
    }
};
HostPathPool g_pool;
}  // namespace

// the pipeline of the host-buffer path; the caller holds g_pool.mu.  copier: the table workers of dg_add_function_sdf, which share the copies
// from the pinned piece into the caller's memory with this thread (fresh pageable memory: page faults and remote NUMA nodes make a single
// thread's copy the bottleneck on a loaded host); NULL: this thread copies alone.  band: NULL = the plain node loop (exactly the kernels it
// always launched); else every chunk is the narrow-band form (classifier + band node loop, k1_launch_sample_nodes_band)
namespace { struct HostTablesJob; }
static void tables_job_copy(HostTablesJob* job, void* dst, const void* src, size_t bytes);
// the D2H half of the pipeline: d_src[0, n) -> out_host, one staging piece at a time; piece i first waits for g_pool.chunk_ev[off / chunk], so
// a piece must not straddle two chunks that complete on different streams.  The caller holds g_pool.mu.
static int drain_to_host_locked(const double* d_src, uint64_t n, uint64_t chunk, double* out_host, HostTablesJob* copier)
{
    const uint64_t piece = HostPathPool::kPiece;
    const uint64_t n_pieces = (n + piece - 1) / piece;
    for (uint64_t i = 0; i <= n_pieces; i++) {
        if (i < n_pieces) {
            const uint64_t off = i * piece, cnt = (off + piece <= n) ? piece : n - off;
            DG_CUDA(cudaStreamWaitEvent(g_pool.s_c, g_pool.chunk_ev[off / chunk], 0));
            DG_CUDA(cudaMemcpyAsync(g_pool.stage[i & 1], d_src + off, cnt * sizeof(double), cudaMemcpyDeviceToHost, g_pool.s_c));
            DG_CUDA(cudaEventRecord(g_pool.dma_ev[i & 1], g_pool.s_c));
        }
        if (i >= 1) {
            const uint64_t off = (i - 1) * piece, cnt = (off + piece <= n) ? piece : n - off;
            DG_CUDA(cudaEventSynchronize(g_pool.dma_ev[(i - 1) & 1]));
            const double* src = g_pool.stage[(i - 1) & 1];
            if (copier) tables_job_copy(copier, out_host + off, src, cnt * sizeof(double));
            else std::memcpy(out_host + off, src, cnt * sizeof(double));
        }
    }
    return DG_OK;
}

static int sample_sdf_host_locked(const dg_mesh* m, const GridDev& g, double sign, uint64_t l_begin, uint64_t n, double* out_host, HostTablesJob* copier = nullptr,
                                  const double* band = nullptr)
{
    // kernel chunks: a handful, each a multiple of the staging piece so that pieces never straddle chunks
    const uint64_t piece = HostPathPool::kPiece;
    const uint64_t n_pieces = (n + piece - 1) / piece;
    const uint64_t pieces_per_chunk = n_pieces <= 4 ? 1 : (n_pieces + 7) / 8;
    const uint64_t chunk = pieces_per_chunk * piece;
    const uint64_t n_chunks = (n + chunk - 1) / chunk;
    size_t band_bytes = 0;
    if (band)
        for (uint64_t c = 0; c < n_chunks; c++) {
            const uint64_t b = c * chunk, cnt = (b + chunk <= n) ? chunk : n - b;
            band_bytes = std::max(band_bytes, k1_band_scratch_bytes(g, l_begin + b, cnt));
        }
    const WindDev* wd = nullptr;             // winding mode: every chunk is K1 with sign = +1, then the node pass of k5_winding.cu
    if (m->sign_mode == DG_SIGN_WINDING) { if (int rc = winding_dev(m, wd, "dg_sample_sdf")) return rc; }
    const double k1_sign = wd ? 1.0 : sign;
    DG_CUDA(g_pool.prepare(n, n_chunks, band_bytes));
    for (uint64_t c = 0; c < n_chunks; c++) {
        const uint64_t b = c * chunk, cnt = (b + chunk <= n) ? chunk : n - b;
        if (band) DG_LAUNCH(k1_launch_sample_nodes_band(m->dev, g, k1_sign, *band, l_begin + b, cnt, g_pool.d_out + b, g_pool.band_scratch[c & 1], g_pool.s_k[c & 1]));
        else DG_LAUNCH(k1_launch_sample_nodes(m->dev, g, k1_sign, l_begin + b, cnt, g_pool.d_out + b, g_pool.s_k[c & 1]));
        if (wd) DG_LAUNCH(k5_launch_sign_nodes(*wd, g, sign, band ? *band : INFINITY, m->beta, l_begin + b, cnt, g_pool.d_out + b, g_pool.s_k[c & 1]));
        DG_CUDA(cudaEventRecord(g_pool.chunk_ev[c], g_pool.s_k[c & 1]));
    }
    return drain_to_host_locked(g_pool.d_out, n, chunk, out_host, copier);
}

// Makes the pages of [p, p + bytes) present and writable WITHOUT changing their content (safe against a concurrent writer).
static void prefault_preserving(char* p, uint64_t bytes)
{
    if (bytes == 0) return;
#if defined(__linux__) && !defined(DG_EMU)
    const uintptr_t a = reinterpret_cast<uintptr_t>(p) & ~uintptr_t(4095), z = (reinterpret_cast<uintptr_t>(p) + bytes + 4095) & ~uintptr_t(4095);
#ifndef MADV_POPULATE_WRITE
#define MADV_POPULATE_WRITE 23
#endif
    if (madvise(reinterpret_cast<void*>(a), z - a, MADV_POPULATE_WRITE) == 0) return;
#endif
    for (uint64_t o = 0; o < bytes; o += 4096) __atomic_fetch_or(reinterpret_cast<unsigned char*>(p + o), 0, __ATOMIC_RELAXED);
    __atomic_fetch_or(reinterpret_cast<unsigned char*>(p + bytes - 1), 0, __ATOMIC_RELAXED);
}

// closed-form connectivity of cells [c0, c1) (cubic_lagrange_discrete_grid.cpp:833-886), host side: plain index algebra
static void fill_cells_host(const GridDev& g, uint64_t c0, uint64_t c1, uint32_t* out /* (c1 - c0) x 32 */)
{
    const unsigned nx = g.n[0], ny = g.n[1], nz = g.n[2];
    const unsigned nv = g.nv, off_x = nv, off_y = nv + 2u * g.ne_x, off_z = off_y + 2u * g.ne_y;
    unsigned k = (unsigned)(c0 / ((uint64_t)nx * ny)), rem = (unsigned)(c0 % ((uint64_t)nx * ny)), j = rem / nx, i = rem % nx;
    for (uint64_t c = c0; c < c1; c++) {
        uint32_t* cell = out + 32 * (c - c0);
        const unsigned v00 = (nx + 1) * (ny + 1) * k + (nx + 1) * j + i, v10 = v00 + (nx + 1), v01 = v00 + (nx + 1) * (ny + 1), v11 = v01 + (nx + 1);
        cell[0] = v00; cell[1] = v00 + 1; cell[2] = v10; cell[3] = v10 + 1; cell[4] = v01; cell[5] = v01 + 1; cell[6] = v11; cell[7] = v11 + 1;
        const unsigned x0 = off_x + 2 * (nx * (ny + 1) * k + nx * j + i), x1 = off_x + 2 * (nx * (ny + 1) * (k + 1) + nx * j + i);
        const unsigned x2 = off_x + 2 * (nx * (ny + 1) * k + nx * (j + 1) + i), x3 = off_x + 2 * (nx * (ny + 1) * (k + 1) + nx * (j + 1) + i);
        cell[8] = x0; cell[9] = x0 + 1; cell[10] = x1; cell[11] = x1 + 1; cell[12] = x2; cell[13] = x2 + 1; cell[14] = x3; cell[15] = x3 + 1;
        const unsigned y0 = off_y + 2 * (ny * (nz + 1) * i + ny * k + j), y1 = off_y + 2 * (ny * (nz + 1) * (i + 1) + ny * k + j);
        const unsigned y2 = off_y + 2 * (ny * (nz + 1) * i + ny * (k + 1) + j), y3 = off_y + 2 * (ny * (nz + 1) * (i + 1) + ny * (k + 1) + j);
        cell[16] = y0; cell[17] = y0 + 1; cell[18] = y1; cell[19] = y1 + 1; cell[20] = y2; cell[21] = y2 + 1; cell[22] = y3; cell[23] = y3 + 1;
        const unsigned z0 = off_z + 2 * (nz * (nx + 1) * j + nz * i + k), z1 = off_z + 2 * (nz * (nx + 1) * (j + 1) + nz * i + k);
        const unsigned z2 = off_z + 2 * (nz * (nx + 1) * j + nz * (i + 1) + k), z3 = off_z + 2 * (nz * (nx + 1) * (j + 1) + nz * (i + 1) + k);
        cell[24] = z0; cell[25] = z0 + 1; cell[26] = z1; cell[27] = z1 + 1; cell[28] = z2; cell[29] = z2 + 1; cell[30] = z3; cell[31] = z3 + 1;
        if (++i == nx) { i = 0; if (++j == ny) { j = 0; ++k; } }
    }
}

// Host side of addFunction while the GPU samples the nodes: worker threads pre-fault the coefficient array (content-preserving: the
// D2H pipeline may already be writing there), then write the connectivity table (:833-886) and the identity cell map (:888-891)
// straight into the caller's memory -- 4 MiB blocks dealt dynamically.
namespace {
struct HostTablesJob {
    GridDev g; uint64_t n_nodes = 0, n_cells = 0;
    double* nodes = nullptr; uint32_t* cells = nullptr; uint32_t* cell_map = nullptr;
    std::atomic<uint64_t> next_task{0};
    std::atomic<int> prefault_left{0};
    uint64_t nb_nodes = 0, nb_cells = 0, nb_map = 0, n_tasks = 0;
    static constexpr uint64_t blk = 4u << 20;
    std::chrono::steady_clock::time_point t0;
    double ms_prefault = 0.0;
    unsigned n_workers = 0;
    std::vector<std::thread> th;
    // copy service: once the tables are written the workers wait here and share the copies staging buffer -> caller memory with the
    // thread that drives the pipeline (one thread copies ~2-4 GB/s into pages another thread faulted in; the pipeline needs a 32 MiB
    // piece every few milliseconds, which a loaded host does not sustain single-threaded)
    struct CopyJob { char* dst; const char* src; size_t bytes; std::atomic<size_t> next{0}, done{0}; };
    std::mutex c_mu; std::condition_variable c_cv;
    std::shared_ptr<CopyJob> c_job;                              // guarded by c_mu; a late worker only ever touches the job it picked up
    uint64_t c_gen = 0; bool c_quit = false;
    static constexpr size_t c_blk = 1u << 20;
    static void copy_blocks(CopyJob& j)
    {
        for (;;) {
            const size_t b = j.next.fetch_add(c_blk);
            if (b >= j.bytes) break;
            const size_t n = std::min(c_blk, j.bytes - b);
            std::memcpy(j.dst + b, j.src + b, n);
            j.done.fetch_add(n);
        }
    }
    void copy(void* dst, const void* src, size_t bytes)          // called by the pipeline's thread
    {
        if (bytes < 4 * c_blk || th.empty()) { std::memcpy(dst, src, bytes); return; }
        auto job = std::make_shared<CopyJob>();
        job->dst = static_cast<char*>(dst); job->src = static_cast<const char*>(src); job->bytes = bytes;
        { std::lock_guard<std::mutex> lk(c_mu); c_job = job; c_gen++; }
        c_cv.notify_all();
        copy_blocks(*job);
        while (job->done.load() < bytes) std::this_thread::yield();
    }
    void serve_copies()
    {
        uint64_t seen = 0;
        for (;;) {
            std::shared_ptr<CopyJob> job;
            {
                std::unique_lock<std::mutex> lk(c_mu);
                c_cv.wait(lk, [&] { return c_quit || c_gen != seen; });
                if (c_quit) return;
                seen = c_gen; job = c_job;
            }
            if (job) copy_blocks(*job);
        }
    }
    void work()
    {
        for (;;) {
            const uint64_t t = next_task.fetch_add(1);
            if (t >= n_tasks) break;
            if (t < nb_nodes) {
                char* p = reinterpret_cast<char*>(nodes);
                const uint64_t b = t * blk, e = std::min<uint64_t>(n_nodes * 8, b + blk);
                prefault_preserving(p + b, e - b);
                if (prefault_left.fetch_sub(1) == 1) ms_prefault = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            } else if (t < nb_nodes + nb_cells) {
                const uint64_t per = blk / 128, c0 = (t - nb_nodes) * per, c1 = std::min<uint64_t>(n_cells, c0 + per);
                fill_cells_host(g, c0, c1, cells + 32 * c0);
            } else {
                const uint64_t per = blk / 4, c0 = (t - nb_nodes - nb_cells) * per, c1 = std::min<uint64_t>(n_cells, c0 + per);
                for (uint64_t c = c0; c < c1; c++) cell_map[c] = (uint32_t)c;
            }
        }
    }
    void start(const GridDev& g_, uint64_t n_nodes_, double* nodes_, uint32_t* cells_, uint32_t* cell_map_)
    {
        g = g_; n_nodes = n_nodes_; n_cells = (uint64_t)g.n[0] * g.n[1] * g.n[2];
        nodes = nodes_; cells = cells_; cell_map = cell_map_;
        nb_nodes = (n_nodes * 8 + blk - 1) / blk;
        nb_cells = cells ? (n_cells * 128 + blk - 1) / blk : 0;
        nb_map = cell_map ? (n_cells * 4 + blk - 1) / blk : 0;
        n_tasks = nb_nodes + nb_cells + nb_map;
        prefault_left = (int)std::min<uint64_t>(nb_nodes, 0x7fffffff);
        t0 = std::chrono::steady_clock::now();
        // a quarter of the usable CPUs, at most 24: under a cgroup CPU quota, workers that keep every CPU of the quota busy get the thread
        // that drives the GPU pipeline throttled along with them.
        const unsigned hw = host_threads();
        n_workers = std::max(1u, std::min(hw / 4u, 24u));
        try { for (unsigned k = 0; k < n_workers; k++) th.emplace_back([this]() { work(); serve_copies(); }); } catch (...) { /* fewer workers: finish() does the rest */ }
    }
    void finish()
    {
        work();                                         // whatever is left
        { std::lock_guard<std::mutex> lk(c_mu); c_quit = true; }
        c_cv.notify_all();
        for (auto& t : th) t.join();
        th.clear();
    }
    ~HostTablesJob() { if (!th.empty()) finish(); }      // an early return of the caller must not leave joinable threads behind
};
}  // namespace

static void tables_job_copy(HostTablesJob* job, void* dst, const void* src, size_t bytes) { job->copy(dst, src, bytes); }

int dg_sample_sdf(const dg_mesh* m, const dg_grid_desc* grid, double sign, uint64_t l_begin, uint64_t l_end, double* out_host)
{
    if (int rc = mesh_usable(m, "dg_sample_sdf")) return rc;
    GridDev g;
    if (int rc = check_range(grid, l_begin, l_end, g, "dg_sample_sdf")) return rc;
    const uint64_t n = l_end - l_begin;
    if (n == 0) return DG_OK;
    if (!out_host) return fail(DG_ERR_INVALID, "dg_sample_sdf: output is NULL");
    if (int rc = check_handle_device(m->device, "dg_sample_sdf")) return rc;
    // A large range into pageable memory: one thread copying staging buffer -> caller memory (2 - 4 GB/s into pages it has to fault in itself)
    // is slower than the packet walk produces coefficients, so a few workers pre-fault the range and share the copies, exactly as in
    // dg_add_function_sdf.
    static const uint64_t helpers_min_bytes = []() -> uint64_t {
        const char* e = std::getenv("DG_HOST_HELPERS_MIN_BYTES");
        return (e && *e) ? (uint64_t)std::strtoull(e, nullptr, 10) : (uint64_t)(32u << 20);
    }();
    if (n * sizeof(double) >= helpers_min_bytes) {
        HostTablesJob job;
        job.start(g, n, out_host, nullptr, nullptr);
        int rc;
        {
            std::lock_guard<std::mutex> lock(g_pool.mu);
            rc = sample_sdf_host_locked(m, g, sign, l_begin, n, out_host, &job);
        }
        job.finish();
        return rc;
    }
    std::lock_guard<std::mutex> lock(g_pool.mu);
    return sample_sdf_host_locked(m, g, sign, l_begin, n, out_host);
}


// The whole of CubicLagrangeDiscreteGrid::addFunction(GenerateSDF functor) into the caller's three arrays
// (cubic_lagrange_discrete_grid.cpp:780-899): node loop on the GPU (K1 chunks on two streams, D2H through the pinned double
// buffer), and -- while the GPU works -- the host threads write the 32-index connectivity table (:833-886) and the identity cell
// map (:888-891) straight into the caller's memory and pre-fault the coefficient array, so that the call ends one D2H piece after
// the last kernel chunk.
static int dg_add_function_sdf_impl(const dg_mesh* m, const dg_grid_desc* grid, double sign, double* nodes_host, uint32_t* cells_host, uint32_t* cell_map_host,
                        double* timings_ms, const double* band = nullptr)
{
    const char* who = band ? "dg_add_function_sdf_band" : "dg_add_function_sdf";
    if (int rc = mesh_usable(m, who)) return rc;
    if (band) { if (int rc = check_band(*band, who)) return rc; }
    GridDev g;
    if (int rc = grid_checked(grid, g, who)) return rc;
    const uint64_t n_nodes = grid_nodes(g);
    if (!nodes_host) return fail(DG_ERR_INVALID, "%s: nodes output is NULL", who);
    if (int rc = check_handle_device(m->device, who)) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    auto ms_since = [&](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count(); };
    HostTablesJob job;
    job.start(g, n_nodes, nodes_host, cells_host, cell_map_host);
    int rc;
    {
        std::lock_guard<std::mutex> lock(g_pool.mu);
        rc = sample_sdf_host_locked(m, g, sign, 0, n_nodes, nodes_host, &job, band);
    }
    const double ms_nodes = ms_since(t0);
    job.finish();
    if (timings_ms) { timings_ms[0] = ms_since(t0); timings_ms[1] = ms_nodes; timings_ms[2] = timings_ms[0]; timings_ms[3] = job.ms_prefault; timings_ms[4] = (double)job.n_workers; timings_ms[5] = 1.0; }
    return rc;
}

int dg_add_function_sdf(const dg_mesh* m, const dg_grid_desc* grid, double sign, double* nodes_host, uint32_t* cells_host, uint32_t* cell_map_host,
                        double* timings_ms)
{
    return guarded("dg_add_function_sdf", [&]() { return dg_add_function_sdf_impl(m, grid, sign, nodes_host, cells_host, cell_map_host, timings_ms); });
}

// addFunction(func, verbose, pred) with pred(x) = |md.signed_distance(x).distance| <= band (cubic_lagrange_discrete_grid.cpp:780-899, node
// loop :806-817): the same pipeline as dg_add_function_sdf, every kernel chunk in its narrow-band form
int dg_add_function_sdf_band(const dg_mesh* m, const dg_grid_desc* grid, double sign, double band, double* nodes_host, uint32_t* cells_host,
                             uint32_t* cell_map_host, double* timings_ms)
{
    return guarded("dg_add_function_sdf_band", [&]() { return dg_add_function_sdf_impl(m, grid, sign, nodes_host, cells_host, cell_map_host, timings_ms, &band); });
}

// ------------------------------------------------------------------------------------------------ multi-GPU from ONE process
// SURVEY 8(b)/(e): `dg_sample_sdf(..., n_gpus, ...)`.  A dg_mesh_group replicates a mesh's device records on further GPUs (peer
// copies over NVLink from the first device, no second host build) and keeps per-device streams, buffers and -- for the device-resident
// form -- one NCCL communicator per device (ncclCommInitAll; libnccl is loaded at first use, the library does not link it).
// Work split: plane pairs of the four node arrays dealt round-robin (the interleaved layout of k1_sdf.cu), every part one launch.

struct dg_mesh_group {
    struct PerDev {
        cudaStream_t st[2] = {nullptr, nullptr};
        cudaEvent_t ev[16] = {};                            // one per part of this device (at most 16 parts in all)
        double* d_buf = nullptr; size_t d_cap = 0;          // host form: 2 slots; device form: n exchange slots
        double* h_stage = nullptr; size_t h_cap = 0;        // pinned staging (pageable destinations only)
        void* comm = nullptr;                               // ncclComm_t
    };
    int n = 0;
    std::vector<int> devices;
    std::vector<dg_mesh*> parts;                            // parts[0] is the caller's mesh (not owned); the others are replicas
    std::vector<PerDev> dev;
    bool comms_ready = false;
    bool borrowed = false;                                  // counted in parts[0]->borrows (dg_mesh_refit refuses while > 0)
    std::mutex mu;
};

namespace {
#if DG_HAVE_NCCL
struct NcclApi {
    void* so = nullptr;
    ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool load()
    {
        if (so) return true;
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) { so = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if (so) break; }
        if (!so) return false;
        CommInitAll = reinterpret_cast<decltype(CommInitAll)>(dlsym(so, "ncclCommInitAll"));
        CommDestroy = reinterpret_cast<decltype(CommDestroy)>(dlsym(so, "ncclCommDestroy"));
        AllGather = reinterpret_cast<decltype(AllGather)>(dlsym(so, "ncclAllGather"));
        GroupStart = reinterpret_cast<decltype(GroupStart)>(dlsym(so, "ncclGroupStart"));
        GroupEnd = reinterpret_cast<decltype(GroupEnd)>(dlsym(so, "ncclGroupEnd"));
        GetErrorString = reinterpret_cast<decltype(GetErrorString)>(dlsym(so, "ncclGetErrorString"));
        return CommInitAll && CommDestroy && AllGather && GroupStart && GroupEnd && GetErrorString;
    }
};
NcclApi g_nccl;
#endif

struct DeviceGuard {                                  // restores the caller's current device
    int prev = -1;
    DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

int group_grow(dg_mesh_group::PerDev& d, size_t dev_elems, size_t host_elems)
{
    if (dev_elems > d.d_cap) {
        if (d.d_buf) cudaFree(d.d_buf);
        d.d_buf = nullptr; d.d_cap = 0;
        DG_CUDA(cudaMalloc(reinterpret_cast<void**>(&d.d_buf), dev_elems * sizeof(double)));
        d.d_cap = dev_elems;
    }
    if (host_elems > d.h_cap) {
        if (d.h_stage) cudaFreeHost(d.h_stage);
        d.h_stage = nullptr; d.h_cap = 0;
        DG_CUDA(cudaMallocHost(reinterpret_cast<void**>(&d.h_stage), host_elems * sizeof(double)));
        d.h_cap = host_elems;
    }
    return DG_OK;
}
}  // namespace

int dg_mesh_group_destroy(dg_mesh_group* grp)
{
    if (!grp) return DG_OK;
    DeviceGuard guard;
    for (int i = 0; i < grp->n; i++) {
        if (cudaSetDevice(grp->devices[i]) != cudaSuccess) { cudaGetLastError(); continue; }
        auto& d = grp->dev[i];
#if DG_HAVE_NCCL
        if (d.comm && g_nccl.CommDestroy) g_nccl.CommDestroy(static_cast<ncclComm_t>(d.comm));
#endif
        for (int k = 0; k < 2; k++) if (d.st[k]) cudaStreamDestroy(d.st[k]);
        for (int k = 0; k < 16; k++) if (d.ev[k]) cudaEventDestroy(d.ev[k]);
        if (d.d_buf) cudaFree(d.d_buf);
        if (d.h_stage) cudaFreeHost(d.h_stage);
        if (i > 0 && (size_t)i < grp->parts.size()) delete grp->parts[i];
    }
    if (grp->borrowed) grp->parts[0]->borrows.fetch_sub(1);
    delete grp;
    return DG_OK;
}

int dg_mesh_group_create(const dg_mesh* mesh, int n_gpus, const int* devices, dg_mesh_group** out)
{
    if (!out) return fail(DG_ERR_INVALID, "dg_mesh_group_create: out is NULL");
    *out = nullptr;
    if (int rc = mesh_usable(mesh, "dg_mesh_group_create")) return rc;
    if (int rc = refuse_winding(mesh, "dg_mesh_group_create")) return rc;
    if (int rc = require_device()) return rc;
    const int have = dg_device_count();
    if (n_gpus < 1 || n_gpus > 16 || n_gpus > have) return fail(DG_ERR_INVALID, "dg_mesh_group_create: n_gpus = %d, but 1..min(16, %d visible devices) are possible", n_gpus, have);
    std::unique_ptr<dg_mesh_group, int (*)(dg_mesh_group*)> grp(new (std::nothrow) dg_mesh_group(), dg_mesh_group_destroy);
    if (!grp) return fail(DG_ERR_NOMEM, "dg_mesh_group_create: out of host memory");
    grp->devices.push_back(mesh->device);
    for (int k = 0, next = 0; k < n_gpus - 1; k++) {
        int dv;
        if (devices) { dv = devices[k + 1]; if (devices[0] != mesh->device) return fail(DG_ERR_INVALID, "dg_mesh_group_create: devices[0] must be the mesh's device (%d)", mesh->device); }
        else { while (next == mesh->device) next++; dv = next++; }
        if (dv < 0 || dv >= have || std::find(grp->devices.begin(), grp->devices.end(), dv) != grp->devices.end())
            return fail(DG_ERR_INVALID, "dg_mesh_group_create: bad or repeated device id %d", dv);
        grp->devices.push_back(dv);
    }
    grp->dev.resize(n_gpus);
    grp->parts.push_back(const_cast<dg_mesh*>(mesh));
    DeviceGuard guard;
    const size_t nT = mesh->host.n_triangles;
    for (int i = 0; i < n_gpus; i++) {
        DG_CUDA(cudaSetDevice(grp->devices[i]));
        grp->n = i + 1;                                             // destroy() only visits initialised entries
        auto& d = grp->dev[i];
        for (int k = 0; k < 2; k++) DG_CUDA(cudaStreamCreateWithFlags(&d.st[k], cudaStreamNonBlocking));
        for (int k = 0; k < 16; k++) DG_CUDA(cudaEventCreateWithFlags(&d.ev[k], cudaEventDisableTiming));
        if (i == 0) continue;
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, grp->devices[i], mesh->device) == cudaSuccess && can) { if (cudaDeviceEnablePeerAccess(mesh->device, 0) != cudaSuccess) cudaGetLastError(); }
        dg_mesh* r = new (std::nothrow) dg_mesh();
        if (!r) return fail(DG_ERR_NOMEM, "dg_mesh_group_create: out of host memory");
        grp->parts.push_back(r);
        r->device = grp->devices[i];
        r->host.n_triangles = mesh->host.n_triangles; r->host.n_vertices = mesh->host.n_vertices; r->host.flags = mesh->host.flags;
        DG_CUDA(r->d_spheres.alloc(nT)); DG_CUDA(r->d_leaves.alloc(nT)); DG_CUDA(r->d_normals.alloc(nT)); DG_CUDA(r->d_nodes_f.alloc(nT * K1_NODEF_STRIDE));
        DG_CUDA(cudaMemcpyPeer(r->d_spheres.p, r->device, mesh->d_spheres.p, mesh->device, nT * sizeof(SpherePair)));
        DG_CUDA(cudaMemcpyPeer(r->d_leaves.p, r->device, mesh->d_leaves.p, mesh->device, nT * sizeof(LeafRecord)));
        DG_CUDA(cudaMemcpyPeer(r->d_normals.p, r->device, mesh->d_normals.p, mesh->device, nT * sizeof(PseudoNormals)));
        DG_CUDA(cudaMemcpyPeer(r->d_nodes_f.p, r->device, mesh->d_nodes_f.p, mesh->device, nT * K1_NODEF_STRIDE * sizeof(float4)));
        r->dev = mesh->dev;
        r->dev.spheres = r->d_spheres.p; r->dev.leaves = r->d_leaves.p; r->dev.normals = r->d_normals.p; r->dev.nodes_f = r->d_nodes_f.p;
        DG_CUDA(r->d_leaves_f.alloc(nT));
        DG_CUDA(cudaMemcpyPeer(r->d_leaves_f.p, r->device, mesh->d_leaves_f.p, mesh->device, nT * sizeof(LeafF)));
        r->dev.leaves_f = r->d_leaves_f.p;
        DG_CUDA(k1_configure(r->dev.stack_depth));
        DG_CUDA(cudaDeviceSynchronize());
    }
    grp->parts[0]->borrows.fetch_add(1);
    grp->borrowed = true;
    *out = grp.release();
    return DG_OK;
}

int dg_mesh_group_size(const dg_mesh_group* grp) { return grp ? grp->n : 0; }

// addFunction across the group's GPUs, host arrays out.  n x 2 parts (two launches per GPU on two streams, so that the D2H of a
// GPU's first part runs under its second launch); each GPU is driven by its own host thread and DMAs the contiguous plane-pair runs
// of its parts to their final positions (directly when nodes_host is page-locked, else through pinned staging).  No collective is
// needed: the exchange target is host memory.  cells_host / cell_map_host as in dg_add_function_sdf (nullable).
int dg_add_function_sdf_multi(dg_mesh_group* grp, const dg_grid_desc* grid, double sign, double* nodes_host, uint32_t* cells_host,
                              uint32_t* cell_map_host, double* timings_ms)
{
    return guarded("dg_add_function_sdf_multi", [&]() -> int {
        if (!grp) return fail(DG_ERR_INVALID, "dg_add_function_sdf_multi: group is NULL");
        if (int rc = refuse_winding(grp->parts[0], "dg_add_function_sdf_multi")) return rc;
        GridDev g;
        if (int rc = grid_checked(grid, g, "dg_add_function_sdf_multi")) return rc;
        const uint64_t n_nodes = grid_nodes(g);
        if (!nodes_host) return fail(DG_ERR_INVALID, "dg_add_function_sdf_multi: nodes output is NULL");
        std::lock_guard<std::mutex> lock(grp->mu);
        const int n = grp->n;
        // parts per GPU: at least two (the D2H and the host copy of one part run under the next launch), more when the grid is large -- what
        // stays exposed at the end is the copy of ONE part into the caller's memory -- but never below ~4 M
        // nodes per launch (every launch ends with a tail of long-running warps) and never more than 16 parts in all
        unsigned splits = (2 * n <= 16) ? 2u : 1u;
        {
            const uint64_t by_size = n_nodes / (4000000ull * (uint64_t)n);
            const unsigned cap = 16u / (unsigned)n;
            if (by_size > splits) splits = (unsigned)std::min<uint64_t>(by_size, cap);
        }
        InterleavedLayout L;
        if (!k1_interleaved_layout(g, (unsigned)n * splits, L)) return fail(DG_ERR_INVALID, "dg_add_function_sdf_multi: grid too large for the exchange layout");
        const auto t0 = std::chrono::steady_clock::now();
        auto ms_since = [&](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count(); };
        const bool direct = is_pinned_host(nodes_host);
        HostTablesJob job;
        job.start(g, n_nodes, nodes_host, cells_host, cell_map_host);
        std::vector<int> rcs(n, DG_OK);
        std::vector<std::string> errs(n);
        std::vector<uint64_t> launches(n, 0);
        auto drive = [&](int i) -> int {
            DG_CUDA(cudaSetDevice(grp->devices[i]));
            auto& d = grp->dev[i];
            if (int rc = group_grow(d, (size_t)splits * L.slot_elems, direct ? 0 : (size_t)splits * L.slot_elems)) return rc;
            std::vector<K1Run> runs[16];
            for (unsigned sp = 0; sp < splits; sp++) {
                const unsigned part = (unsigned)i + sp * (unsigned)n;
                double* d_slot = d.d_buf + (size_t)sp * L.slot_elems;
                cudaStream_t stream = d.st[sp & 1u];
                DG_CUDA(k1_launch_sample_interleaved(grp->parts[i]->dev, g, sign, L, part, d_slot, stream));
                launches[i]++;
                k1_interleaved_runs(g, L, part, runs[sp]);
                uint64_t used = 0;
                for (const auto& r : runs[sp]) used = std::max<uint64_t>(used, r.slot_pos + r.count);
                if (direct) { for (const auto& r : runs[sp]) DG_CUDA(cudaMemcpyAsync(nodes_host + r.node_begin, d_slot + r.slot_pos, r.count * sizeof(double), cudaMemcpyDeviceToHost, stream)); }
                else if (used) DG_CUDA(cudaMemcpyAsync(d.h_stage + (size_t)sp * L.slot_elems, d_slot, used * sizeof(double), cudaMemcpyDeviceToHost, stream));
                DG_CUDA(cudaEventRecord(d.ev[sp], stream));
            }
            for (unsigned sp = 0; sp < splits; sp++) {
                DG_CUDA(cudaEventSynchronize(d.ev[sp]));
                if (!direct) for (const auto& r : runs[sp]) std::memcpy(nodes_host + r.node_begin, d.h_stage + (size_t)sp * L.slot_elems + r.slot_pos, r.count * sizeof(double));
            }
            return DG_OK;
        };
        {
            DeviceGuard guard;
            std::vector<std::thread> th;
            auto guarded = [&](int i) {
                try { rcs[i] = drive(i); if (rcs[i] != DG_OK) errs[i] = g_err; }
                catch (const std::exception& ex) { rcs[i] = DG_ERR_NOMEM; errs[i] = ex.what(); }
            };
            for (int i = 1; i < n; i++) th.emplace_back([&, i]() { DeviceGuard tg; guarded(i); });
            guarded(0);
            for (auto& t : th) t.join();
        }
        const double ms_nodes = ms_since(t0);
        job.finish();
        for (int i = 0; i < n; i++) g_launches.fetch_add(launches[i]);
        if (timings_ms) { timings_ms[0] = ms_since(t0); timings_ms[1] = ms_nodes; timings_ms[2] = timings_ms[0]; timings_ms[3] = job.ms_prefault; timings_ms[4] = (double)job.n_workers; timings_ms[5] = (double)n; }
        for (int i = 0; i < n; i++) if (rcs[i] != DG_OK) return fail(rcs[i], "dg_add_function_sdf_multi (device %d): %s", grp->devices[i], errs[i].c_str());
        return DG_OK;
    });
}

// Device-resident form (the coefficient array is needed on every GPU, e.g. for K2/K3 replicas): GPU i samples part i of n into its
// slot of an n x slot_elems exchange buffer, ONE in-place ncclAllGather per device (grouped) moves the slots over NVLink, and an
// unpack kernel scatters them into the reference's node order in d_out[i] (device i's memory, n_nodes doubles each).
int dg_sample_sdf_multi_device(dg_mesh_group* grp, const dg_grid_desc* grid, double sign, double* const* d_out)
{
    if (!grp || !d_out) return fail(DG_ERR_INVALID, "dg_sample_sdf_multi_device: NULL argument");
    if (int rc = refuse_winding(grp->parts[0], "dg_sample_sdf_multi_device")) return rc;
    GridDev g;
    if (int rc = grid_checked(grid, g, "dg_sample_sdf_multi_device")) return rc;
    std::lock_guard<std::mutex> lock(grp->mu);
    const int n = grp->n;
    for (int i = 0; i < n; i++) if (!d_out[i]) return fail(DG_ERR_INVALID, "dg_sample_sdf_multi_device: d_out[%d] is NULL", i);
    InterleavedLayout L;
    if (!k1_interleaved_layout(g, (unsigned)n, L)) return fail(DG_ERR_INVALID, "dg_sample_sdf_multi_device: grid too large for the exchange layout");
    DeviceGuard guard;
#if DG_HAVE_NCCL
    if (n > 1 && !grp->comms_ready) {
        if (!g_nccl.load()) return fail(DG_ERR_CUDA, "dg_sample_sdf_multi_device: libnccl.so.2 could not be loaded (%s)", dlerror() ? dlerror() : "missing symbol");
        std::vector<ncclComm_t> comms(n);
        const ncclResult_t r = g_nccl.CommInitAll(comms.data(), n, grp->devices.data());
        if (r != ncclSuccess) return fail(DG_ERR_CUDA, "ncclCommInitAll failed: %s", g_nccl.GetErrorString(r));
        for (int i = 0; i < n; i++) grp->dev[i].comm = comms[i];
        grp->comms_ready = true;
    }
#else
    if (n > 1) return fail(DG_ERR_CUDA, "dg_sample_sdf_multi_device: built without NCCL");
#endif
    for (int i = 0; i < n; i++) {
        DG_CUDA(cudaSetDevice(grp->devices[i]));
        if (int rc = group_grow(grp->dev[i], (size_t)n * L.slot_elems, 0)) return rc;
        DG_LAUNCH(k1_launch_sample_interleaved(grp->parts[i]->dev, g, sign, L, (unsigned)i, grp->dev[i].d_buf + (size_t)i * L.slot_elems, grp->dev[i].st[0]));
    }
#if DG_HAVE_NCCL
    if (n > 1) {
        ncclResult_t r = g_nccl.GroupStart();
        for (int i = 0; i < n && r == ncclSuccess; i++)
            r = g_nccl.AllGather(grp->dev[i].d_buf + (size_t)i * L.slot_elems, grp->dev[i].d_buf, L.slot_elems, ncclDouble, static_cast<ncclComm_t>(grp->dev[i].comm), grp->dev[i].st[0]);
        const ncclResult_t r2 = g_nccl.GroupEnd();
        if (r != ncclSuccess || r2 != ncclSuccess) return fail(DG_ERR_CUDA, "ncclAllGather failed: %s", g_nccl.GetErrorString(r != ncclSuccess ? r : r2));
    }
#endif
    for (int i = 0; i < n; i++) {
        DG_CUDA(cudaSetDevice(grp->devices[i]));
        DG_LAUNCH(k1_launch_unpack_interleaved(g, L, grp->dev[i].d_buf, d_out[i], grp->dev[i].st[0]));
    }
    for (int i = 0; i < n; i++) {
        DG_CUDA(cudaSetDevice(grp->devices[i]));
        DG_CUDA(cudaStreamSynchronize(grp->dev[i].st[0]));
    }
    return DG_OK;
}

// plane ranges of part `part` of `n_parts`: whole plane pairs, so boundaries fall on even plane indices
static void slab_planes(const GridDev& g, uint32_t part, uint32_t n_parts, unsigned pb[4], unsigned pe[4])
{
    const unsigned Ds[4] = {g.n[2] + 1, g.n[2] + 1, g.n[0] + 1, g.n[1] + 1};
    for (int a = 0; a < 4; a++) {
        const uint64_t groups = (Ds[a] + 1) / 2;
        const uint64_t q0 = groups * part / n_parts, q1 = groups * (part + 1) / n_parts;
        pb[a] = (unsigned)std::min<uint64_t>(q0 * 2, Ds[a]);
        pe[a] = (unsigned)std::min<uint64_t>(q1 * 2, Ds[a]);
    }
}

int dg_slab_ranges(const dg_grid_desc* grid, uint32_t part, uint32_t n_parts, uint64_t ranges[8])
{
    GridDev g;
    if (int rc = grid_checked(grid, g, "dg_slab_ranges")) return rc;
    if (!ranges || n_parts == 0 || part >= n_parts) return fail(DG_ERR_INVALID, "dg_slab_ranges: bad part / n_parts");
    unsigned pb[4], pe[4];
    slab_planes(g, part, n_parts, pb, pe);
    const uint64_t base[4] = {0, g.nv, (uint64_t)g.nv + 2ull * g.ne_x, (uint64_t)g.nv + 2ull * (g.ne_x + (uint64_t)g.ne_y)};
    const uint64_t plane[4] = {(uint64_t)(g.n[1] + 1) * (g.n[0] + 1), (uint64_t)(g.n[1] + 1) * 2 * g.n[0], (uint64_t)(g.n[2] + 1) * 2 * g.n[1],
                               (uint64_t)(g.n[0] + 1) * 2 * g.n[2]};
    for (int a = 0; a < 4; a++) { ranges[2 * a] = base[a] + plane[a] * pb[a]; ranges[2 * a + 1] = base[a] + plane[a] * pe[a]; }
    return DG_OK;
}

int dg_sample_sdf_slab_device(const dg_mesh* m, const dg_grid_desc* grid, double sign, uint32_t part, uint32_t n_parts, double* d_full, void* stream)
{
    static const char* who = "dg_sample_sdf_slab_device";
    if (int rc = mesh_usable(m, who)) return rc;
    if (int rc = refuse_winding(m, who)) return rc;
    GridDev g;
    if (int rc = grid_checked(grid, g, who)) return rc;
    if (n_parts == 0 || part >= n_parts || !d_full) return fail(DG_ERR_INVALID, "%s: bad part / n_parts / output", who);
    if (int rc = check_handle_device(m->device, who)) return rc;
    unsigned pb[4], pe[4];
    slab_planes(g, part, n_parts, pb, pe);
    DG_LAUNCH(k1_launch_sample_slab(m->dev, g, sign, pb, pe, d_full, (cudaStream_t)stream));
    return DG_OK;
}

int dg_interleaved_slot_elems(const dg_grid_desc* grid, uint32_t n_parts, uint64_t* slot_elems)
{
    GridDev g;
    if (int rc = grid_checked(grid, g, "dg_interleaved_slot_elems")) return rc;
    InterleavedLayout L;
    if (!slot_elems || !k1_interleaved_layout(g, n_parts, L)) return fail(DG_ERR_INVALID, "dg_interleaved_slot_elems: n_parts must be 1..16");
    *slot_elems = L.slot_elems;
    return DG_OK;
}

int dg_interleaved_node_slots(const dg_grid_desc* grid, uint32_t n_parts, uint64_t l_begin, uint64_t l_end, uint32_t* part_out, uint64_t* pos_out)
{
    GridDev g;
    if (int rc = grid_checked(grid, g, "dg_interleaved_node_slots")) return rc;
    InterleavedLayout L;
    if (!k1_interleaved_layout(g, n_parts, L)) return fail(DG_ERR_INVALID, "dg_interleaved_node_slots: n_parts must be 1..16");
    const uint64_t n = grid_nodes(g);
    if (l_begin > l_end || l_end > n) return fail(DG_ERR_INVALID, "dg_interleaved_node_slots: node range outside [0, %llu]", (unsigned long long)n);
    k1_interleaved_node_slots(g, L, l_begin, l_end - l_begin, part_out, pos_out);
    return DG_OK;
}

int dg_sample_sdf_interleaved_device(const dg_mesh* m, const dg_grid_desc* grid, double sign, uint32_t part, uint32_t n_parts, double* d_slot, void* stream)
{
    static const char* who = "dg_sample_sdf_interleaved_device";
    if (int rc = mesh_usable(m, who)) return rc;
    if (int rc = refuse_winding(m, who)) return rc;
    GridDev g;
    if (int rc = grid_checked(grid, g, who)) return rc;
    InterleavedLayout L;
    if (!k1_interleaved_layout(g, n_parts, L) || part >= n_parts || !d_slot) return fail(DG_ERR_INVALID, "%s: bad part / n_parts (1..16) / output", who);
    if (int rc = check_handle_device(m->device, who)) return rc;
    DG_LAUNCH(k1_launch_sample_interleaved(m->dev, g, sign, L, part, d_slot, (cudaStream_t)stream));
    return DG_OK;
}

int dg_interleaved_unpack_device(const dg_grid_desc* grid, uint32_t n_parts, const double* d_slots, double* d_nodes, void* stream)
{
    if (int rc = require_device()) return rc;
    GridDev g;
    if (int rc = grid_checked(grid, g, "dg_interleaved_unpack_device")) return rc;
    InterleavedLayout L;
    if (!k1_interleaved_layout(g, n_parts, L) || !d_slots || !d_nodes) return fail(DG_ERR_INVALID, "dg_interleaved_unpack_device: bad n_parts (1..16) / NULL buffer");
    DG_LAUNCH(k1_launch_unpack_interleaved(g, L, d_slots, d_nodes, (cudaStream_t)stream));
    return DG_OK;
}

int dg_node_positions(const dg_grid_desc* grid, uint64_t l_begin, uint64_t l_end, double* x_host)
{
    if (int rc = require_device()) return rc;
    if (int rc = ensure_selftest()) return rc;
    GridDev g;
    if (int rc = check_range(grid, l_begin, l_end, g, "dg_node_positions")) return rc;
    const uint64_t n = l_end - l_begin;
    if (n == 0) return DG_OK;
    if (!x_host) return fail(DG_ERR_INVALID, "dg_node_positions: output is NULL");
    DevBuf<double> d_x;
    DG_CUDA(d_x.alloc(3 * n));
    DG_LAUNCH(k1_launch_node_positions(g, l_begin, n, d_x.p, nullptr));
    DG_CUDA(cudaMemcpy(x_host, d_x.p, 3 * n * sizeof(double), cudaMemcpyDeviceToHost));
    return DG_OK;
}

int dg_build_cells(const uint32_t res[3], uint64_t c_begin, uint64_t c_end, uint32_t* cells_host)
{
    if (int rc = require_device()) return rc;
    if (!res) return fail(DG_ERR_INVALID, "dg_build_cells: NULL argument");
    dg_grid_desc d;
    const double mn[3] = {0, 0, 0}, mx[3] = {1, 1, 1};
    if (int rc = dg_grid_init(mn, mx, res, &d)) return rc;
    GridDev g;
    if (int rc = grid_checked(&d, g, "dg_build_cells")) return rc;
    const uint64_t nc = grid_cells(g);
    if (c_begin > c_end || c_end > nc) return fail(DG_ERR_INVALID, "dg_build_cells: cell range out of bounds");
    const uint64_t n = c_end - c_begin;
    if (n == 0) return DG_OK;
    if (!cells_host) return fail(DG_ERR_INVALID, "dg_build_cells: output is NULL");
    // same pooled double-buffer pipeline as dg_sample_sdf: the kernel fills one 32 MiB piece (256 Ki cells) of device scratch,
    // the copy stream DMAs it into pinned memory while the CPU moves the previous piece into the caller's array
    std::lock_guard<std::mutex> lock(g_pool.mu);
    const uint64_t piece_cells = HostPathPool::kPiece * sizeof(double) / (32 * sizeof(uint32_t));    // cells per staging buffer
    const uint64_t n_pieces = (n + piece_cells - 1) / piece_cells;
    const uint64_t piece_doubles = std::min<uint64_t>(HostPathPool::kPiece, n * 16);      // 32 uint32 = 16 doubles per cell
    DG_CUDA(g_pool.prepare(2 * piece_doubles, 2));                        // device scratch: two pieces, no larger than the request
    uint32_t* d_piece[2] = {reinterpret_cast<uint32_t*>(g_pool.d_out), reinterpret_cast<uint32_t*>(g_pool.d_out + piece_doubles)};
    for (uint64_t i = 0; i <= n_pieces; i++) {
        if (i < n_pieces) {
            const uint64_t off = i * piece_cells, cnt = (off + piece_cells <= n) ? piece_cells : n - off;
            // piece i reuses device/pinned buffer i&1: its previous user (piece i-2) was fully consumed in iteration i-1
            DG_LAUNCH(k1_launch_build_cells(g, c_begin + off, cnt, d_piece[i & 1], g_pool.s_c));
            DG_CUDA(cudaMemcpyAsync(g_pool.stage[i & 1], d_piece[i & 1], cnt * 32 * sizeof(uint32_t), cudaMemcpyDeviceToHost, g_pool.s_c));
            DG_CUDA(cudaEventRecord(g_pool.dma_ev[i & 1], g_pool.s_c));
        }
        if (i >= 1) {
            const uint64_t off = (i - 1) * piece_cells, cnt = (off + piece_cells <= n) ? piece_cells : n - off;
            DG_CUDA(cudaEventSynchronize(g_pool.dma_ev[(i - 1) & 1]));
            std::memcpy(cells_host + 32 * off, g_pool.stage[(i - 1) & 1], cnt * 32 * sizeof(uint32_t));
        }
    }
    return DG_OK;
}

// ------------------------------------------------------------------------------------------------ fields / K2
static int field_common(const dg_grid_desc* grid, dg_field** out, dg_field*& f)
{
    if (!out) return fail(DG_ERR_INVALID, "dg_field_create: out is NULL");
    *out = nullptr;
    if (int rc = require_device()) return rc;
    if (int rc = ensure_selftest()) return rc;
    GridDev g;
    if (int rc = grid_checked(grid, g, "dg_field_create")) return rc;
    f = new (std::nothrow) dg_field();
    if (!f) return fail(DG_ERR_NOMEM, "dg_field_create: out of host memory");
    f->desc = *grid; f->dev.g = g;
    return DG_OK;
}

static int field_finish(dg_field* f, const double* d_nodes, const unsigned* d_cells, cudaStream_t stream)
{
    cudaError_t e = cudaGetDevice(&f->device);
    if (e == cudaSuccess) e = f->d_packed.alloc(32 * (f->n_cells_kept ? f->n_cells_kept : 1));
    if (e == cudaSuccess && f->n_cells_kept == 0) e = cudaMemsetAsync(f->d_packed.p, 0, 32 * sizeof(double), stream);
    if (e == cudaSuccess) e = f->d_tab.alloc(f->dev.g.n[0] + f->dev.g.n[1] + f->dev.g.n[2]);
    if (e == cudaSuccess) { e = k2_launch_pack(f->dev.g, d_nodes, d_cells, f->n_cells_kept, f->d_packed.p, stream); g_launches.fetch_add(1); }
    if (e == cudaSuccess) { e = k2_launch_axis_tables(f->dev.g, f->d_tab.p, stream); g_launches.fetch_add(1); }
    if (e == cudaSuccess) { e = k3_coeff_max(f->d_packed.p, 32 * f->n_cells_kept, &f->coeff_max, stream); g_launches.fetch_add(1); }
    if (e != cudaSuccess) return fail(cuda_code(e), "dg_field_create: %s", cudaGetErrorString(e));
    f->dev.packed = f->d_packed.p;
    f->dev.cell_map = f->d_cell_map.p;
    f->dev.tab = f->d_tab.p;
    return DG_OK;
}

int dg_field_create(const dg_grid_desc* grid, const double* nodes, uint64_t n_nodes, const uint32_t* cells, uint64_t n_cells_kept,
                    const uint32_t* cell_map, dg_field** out)
{
    dg_field* f = nullptr;
    if (int rc = field_common(grid, out, f)) return rc;
    auto bail = [&](int rc) { delete f; return rc; };
    const uint64_t n_cells = grid_cells(f->dev.g);
    if (!nodes && n_nodes) return bail(fail(DG_ERR_INVALID, "dg_field_create: nodes is NULL"));
    if (!cells && n_cells_kept != n_cells) return bail(fail(DG_ERR_INVALID, "dg_field_create: cells == NULL requires n_cells_kept == nx*ny*nz"));
    if (!cell_map && n_cells_kept != n_cells)      // K2/K3 read a NULL cell map as the identity: it must then cover every grid cell
        return bail(fail(DG_ERR_INVALID, "dg_field_create: cell_map == NULL requires n_cells_kept == nx*ny*nz (pass the reduced field's cell map)"));
    if (!cells) {
        const uint64_t nn = grid_nodes(f->dev.g);
        if (n_nodes != nn) return bail(fail(DG_ERR_INVALID, "dg_field_create: closed-form cells need all %llu nodes (got %llu)",
                                            (unsigned long long)nn, (unsigned long long)n_nodes));
    } else {
        for (uint64_t i = 0; i < 32 * n_cells_kept; i++)
            if (cells[i] >= n_nodes) return bail(fail(DG_ERR_INVALID, "dg_field_create: cell table references node %u >= n_nodes", cells[i]));
    }
    if (cell_map)
        for (uint64_t i = 0; i < n_cells; i++)
            if (cell_map[i] != UINT32_MAX && cell_map[i] >= n_cells_kept)
                return bail(fail(DG_ERR_INVALID, "dg_field_create: cell_map entry %u >= n_cells_kept", cell_map[i]));
    f->n_nodes = n_nodes; f->n_cells_kept = n_cells_kept;
    DevBuf<double> d_nodes;
    DevBuf<unsigned> d_cells;
    cudaError_t e = d_nodes.alloc(n_nodes);
    if (e == cudaSuccess) e = cudaMemcpy(d_nodes.p, nodes, n_nodes * sizeof(double), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && cells) {
        e = d_cells.alloc(32 * n_cells_kept);
        if (e == cudaSuccess) e = cudaMemcpy(d_cells.p, cells, 32 * n_cells_kept * sizeof(unsigned), cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess && cell_map) {
        e = f->d_cell_map.alloc(n_cells);
        if (e == cudaSuccess) e = cudaMemcpy(f->d_cell_map.p, cell_map, n_cells * sizeof(unsigned), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) return bail(fail(cuda_code(e), "dg_field_create: %s", cudaGetErrorString(e)));
    if (int rc = field_finish(f, d_nodes.p, cells ? d_cells.p : nullptr, nullptr)) return bail(rc);
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return bail(fail(DG_ERR_CUDA, "dg_field_create: %s", cudaGetErrorString(e)));
    *out = f;
    return DG_OK;
}

int dg_field_create_device(const dg_grid_desc* grid, const double* d_nodes, uint64_t n_nodes, void* stream, dg_field** out)
{
    dg_field* f = nullptr;
    if (int rc = field_common(grid, out, f)) return rc;
    const uint64_t nn = grid_nodes(f->dev.g);
    if (!d_nodes || n_nodes != nn) { delete f; return fail(DG_ERR_INVALID, "dg_field_create_device: need all %llu node coefficients", (unsigned long long)nn); }
    f->n_nodes = n_nodes;
    f->n_cells_kept = grid_cells(f->dev.g);
    if (int rc = field_finish(f, d_nodes, nullptr, (cudaStream_t)stream)) { delete f; return rc; }
    *out = f;
    return DG_OK;
}

int dg_field_destroy(dg_field* f)
{
    delete f;
    return DG_OK;
}

int dg_field_info(const dg_field* f, uint64_t info[4])
{
    if (!f || !info) return fail(DG_ERR_INVALID, "dg_field_info: NULL argument");
    info[0] = f->n_nodes; info[1] = f->n_cells_kept;
    info[2] = f->d_packed.bytes() + f->d_cell_map.bytes() + f->d_tab.bytes(); info[3] = (uint64_t)f->device;
    return DG_OK;
}

int dg_interpolate_batch_device(const dg_field* f, const double* d_x, uint64_t n, double* d_phi, double* d_grad, void* stream)
{
    if (!f) return fail(DG_ERR_INVALID, "dg_interpolate_batch_device: field is NULL");
    if (n && (!d_x || !d_phi)) return fail(DG_ERR_INVALID, "dg_interpolate_batch_device: x / phi is NULL");
    if (int rc = check_handle_device(f->device, "dg_interpolate_batch_device")) return rc;
    DG_LAUNCH(k2_launch_interpolate(f->dev, d_x, n, d_phi, d_grad, (cudaStream_t)stream));
    return DG_OK;
}

int dg_interpolate_hessian_batch_device(const dg_field* f, const double* d_x, uint64_t n, double* d_phi, double* d_grad, double* d_hess, void* stream)
{
    if (!f) return fail(DG_ERR_INVALID, "dg_interpolate_hessian_batch_device: field is NULL");
    if (n && (!d_x || !d_phi || !d_grad || !d_hess)) return fail(DG_ERR_INVALID, "dg_interpolate_hessian_batch_device: x / phi / grad / hess is NULL");
    if (int rc = check_handle_device(f->device, "dg_interpolate_hessian_batch_device")) return rc;
    DG_LAUNCH(k2_launch_interpolate(f->dev, d_x, n, d_phi, d_grad, (cudaStream_t)stream, d_hess));
    return DG_OK;
}

// Host-buffer path of K2: a three-slot pipeline.  Each slot owns device buffers for one chunk of queries, a stream and an event;
// chunk c runs H2D -> kernel -> D2H on slot c % 3, so the uploads, kernels and downloads of neighbouring chunks overlap on the two
// DMA directions of the link.  Caller memory that is already page-locked (cudaMallocHost / cudaHostRegister / torch pin_memory) is
// DMA'd directly; pageable memory goes through pooled pinned staging buffers, copied in and out by a few host threads while the
// other slots are in flight.  Calls are serialised per process (pool mutex).
namespace {
struct InterpPool {
    static constexpr int kSlots = 3;
    static constexpr uint64_t kChunk = 1u << 19;                 // queries per chunk: 12 MiB up, 16 MiB down
    std::mutex mu;
    int device = -1;
    uint64_t cap = 0;                                            // queries per slot currently allocated
    double* d_x[kSlots] = {}; double* d_phi[kSlots] = {}; double* d_grad[kSlots] = {};
    double* h_in[kSlots] = {}; double* h_out[kSlots] = {};       // pinned staging (allocated on first pageable call)
    double* d_hess[kSlots] = {}; double* h_hess[kSlots] = {};    // Hessian outputs and their pinned staging (first Hessian call only)
    cudaStream_t st[kSlots] = {}; cudaEvent_t done[kSlots] = {};
    void release()
    {
        for (int i = 0; i < kSlots; i++) {
            if (d_x[i]) cudaFree(d_x[i]); if (d_phi[i]) cudaFree(d_phi[i]); if (d_grad[i]) cudaFree(d_grad[i]);
            if (h_in[i]) cudaFreeHost(h_in[i]); if (h_out[i]) cudaFreeHost(h_out[i]);
            if (d_hess[i]) cudaFree(d_hess[i]); if (h_hess[i]) cudaFreeHost(h_hess[i]);
            if (st[i]) cudaStreamDestroy(st[i]); if (done[i]) cudaEventDestroy(done[i]);
            d_x[i] = d_phi[i] = d_grad[i] = h_in[i] = h_out[i] = d_hess[i] = h_hess[i] = nullptr; st[i] = nullptr; done[i] = nullptr;
        }
        cap = 0;
    }
    cudaError_t prepare(uint64_t chunk, bool need_stage_in, bool need_stage_out, bool need_hess)
    {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev != device) { release(); device = dev; }
        if (chunk > cap) { release(); device = dev; }
        if (cap == 0) {
            for (int i = 0; i < kSlots && e == cudaSuccess; i++) {
                e = cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking);
                if (e == cudaSuccess) e = cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming);
                if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&d_x[i]), chunk * 3 * sizeof(double));
                if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&d_phi[i]), chunk * sizeof(double));
                if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&d_grad[i]), chunk * 3 * sizeof(double));
            }
            if (e != cudaSuccess) { release(); return e; }
            cap = chunk;
        }
        for (int i = 0; i < kSlots && e == cudaSuccess; i++) {
            if (need_stage_in && !h_in[i]) e = cudaMallocHost(reinterpret_cast<void**>(&h_in[i]), cap * 3 * sizeof(double));
            if (e == cudaSuccess && need_stage_out && !h_out[i]) e = cudaMallocHost(reinterpret_cast<void**>(&h_out[i]), cap * 4 * sizeof(double));
            if (e == cudaSuccess && need_hess && !d_hess[i]) e = cudaMalloc(reinterpret_cast<void**>(&d_hess[i]), cap * 9 * sizeof(double));
            if (e == cudaSuccess && need_hess && need_stage_out && !h_hess[i]) e = cudaMallocHost(reinterpret_cast<void**>(&h_hess[i]), cap * 9 * sizeof(double));
        }
        if (e != cudaSuccess) release();
        return e;
    }
};
InterpPool g_ipool;

void threaded_copy(void* dst, const void* src, size_t bytes, unsigned nt)
{
    if (nt <= 1 || bytes < (1u << 20)) { std::memcpy(dst, src, bytes); return; }
    std::vector<std::thread> th;
    const size_t per = ((bytes + nt - 1) / nt + 63) & ~size_t(63);
    for (unsigned k = 1; k < nt; k++) {
        const size_t b = k * per, e = std::min(bytes, b + per);
        if (b < e) th.emplace_back([=]() { std::memcpy(static_cast<char*>(dst) + b, static_cast<const char*>(src) + b, e - b); });
    }
    std::memcpy(dst, src, std::min(bytes, per));
    for (auto& t : th) t.join();
}
}  // namespace

// hess (nullable; grad must then be given too) selects K2's Hessian mode; its buffers join the pool at the first call that passes it
static int dg_interpolate_batch_impl(const dg_field* f, const double* x, uint64_t n, double* phi, double* grad, double* hess, const char* who)
{
    if (!f) return fail(DG_ERR_INVALID, "%s: field is NULL", who);
    if (n == 0) return DG_OK;
    if (!x || !phi) return fail(DG_ERR_INVALID, "%s: x / phi is NULL", who);
    if (int rc = check_handle_device(f->device, who)) return rc;
    std::lock_guard<std::mutex> lock(g_ipool.mu);
    constexpr int S = InterpPool::kSlots;
    const uint64_t chunk = std::min<uint64_t>(InterpPool::kChunk, n);
    const bool x_direct = is_pinned_host(x), out_direct = is_pinned_host(phi) && is_pinned_host(grad) && is_pinned_host(hess);
    DG_CUDA(g_ipool.prepare(std::max<uint64_t>(chunk, g_ipool.cap), !x_direct, !out_direct, hess != nullptr));
    const unsigned nt = std::max(1u, std::min(4u, host_threads() / 4));      // copy threads of the staged (pageable) path, started per chunk
    const uint64_t n_chunks = (n + chunk - 1) / chunk;
    auto unstage = [&](uint64_t c) {                      // results of chunk c: pinned staging -> caller memory
        const uint64_t off = c * chunk, cnt = std::min(chunk, n - off);
        const double* src = g_ipool.h_out[c % S];
        threaded_copy(phi + off, src, cnt * sizeof(double), nt);
        if (grad) threaded_copy(grad + 3 * off, src + g_ipool.cap, 3 * cnt * sizeof(double), nt);
        if (hess) threaded_copy(hess + 9 * off, g_ipool.h_hess[c % S], 9 * cnt * sizeof(double), nt);
    };
    for (uint64_t c = 0; c < n_chunks; c++) {
        const int s = (int)(c % S);
        const uint64_t off = c * chunk, cnt = std::min(chunk, n - off);
        if (c >= (uint64_t)S) {                           // the slot's previous chunk must have left the device buffers (and staging)
            DG_CUDA(cudaEventSynchronize(g_ipool.done[s]));
            if (!out_direct) unstage(c - S);
        }
        const double* src = x + 3 * off;
        if (!x_direct) { threaded_copy(g_ipool.h_in[s], src, 3 * cnt * sizeof(double), nt); src = g_ipool.h_in[s]; }
        DG_CUDA(cudaMemcpyAsync(g_ipool.d_x[s], src, 3 * cnt * sizeof(double), cudaMemcpyHostToDevice, g_ipool.st[s]));
        DG_LAUNCH(k2_launch_interpolate(f->dev, g_ipool.d_x[s], cnt, g_ipool.d_phi[s], grad ? g_ipool.d_grad[s] : nullptr, g_ipool.st[s],
                                        hess ? g_ipool.d_hess[s] : nullptr));
        double* dst_phi = out_direct ? phi + off : g_ipool.h_out[s];
        double* dst_grad = out_direct ? grad + 3 * off : g_ipool.h_out[s] + g_ipool.cap;
        DG_CUDA(cudaMemcpyAsync(dst_phi, g_ipool.d_phi[s], cnt * sizeof(double), cudaMemcpyDeviceToHost, g_ipool.st[s]));
        if (grad) DG_CUDA(cudaMemcpyAsync(dst_grad, g_ipool.d_grad[s], 3 * cnt * sizeof(double), cudaMemcpyDeviceToHost, g_ipool.st[s]));
        if (hess) DG_CUDA(cudaMemcpyAsync(out_direct ? hess + 9 * off : g_ipool.h_hess[s], g_ipool.d_hess[s], 9 * cnt * sizeof(double),
                                          cudaMemcpyDeviceToHost, g_ipool.st[s]));
        DG_CUDA(cudaEventRecord(g_ipool.done[s], g_ipool.st[s]));
    }
    for (uint64_t c = (n_chunks > (uint64_t)S ? n_chunks - S : 0); c < n_chunks; c++) {
        DG_CUDA(cudaEventSynchronize(g_ipool.done[c % S]));
        if (!out_direct) unstage(c);
    }
    return DG_OK;
}

int dg_interpolate_batch(const dg_field* f, const double* x, uint64_t n, double* phi, double* grad)
{
    static const char* who = "dg_interpolate_batch";
    return guarded(who, [&]() { return dg_interpolate_batch_impl(f, x, n, phi, grad, nullptr, who); });
}

int dg_interpolate_hessian_batch(const dg_field* f, const double* x, uint64_t n, double* phi, double* grad, double* hess)
{
    static const char* who = "dg_interpolate_hessian_batch";
    if (n && (!phi || !grad || !hess)) return fail(DG_ERR_INVALID, "%s: phi / grad / hess is NULL", who);
    return guarded(who, [&]() { return dg_interpolate_batch_impl(f, x, n, phi, grad, hess, who); });
}

int dg_shape_functions(const double* xi, uint64_t n, double* N, double* dN)
{
    if (int rc = require_device()) return rc;
    if (int rc = ensure_selftest()) return rc;
    if (n == 0) return DG_OK;
    if (!xi || !N) return fail(DG_ERR_INVALID, "dg_shape_functions: NULL argument");
    return stage_on_device(n, n, {{xi, 3 * sizeof(double)}}, {{N, 32 * sizeof(double)}, {dN, 96 * sizeof(double)}},
                           [](void* const* in, void* const* out, uint64_t, uint64_t c) -> int {
                               DG_LAUNCH(k2_launch_shape_functions((const double*)in[0], c, (double*)out[0], (double*)out[1], nullptr));
                               return DG_OK;
                           });
}

// ------------------------------------------------------------------------------------------------ K3
// the argument checks of the density and the volume map over nodes [b, e) of f; why: the map's own check of its scalars (nullptr: valid)
static int node_map_check(const dg_field* f, uint64_t b, uint64_t e, const char* why, const void* out, const char* who)
{
    if (!f) return fail(DG_ERR_INVALID, "%s: field is NULL", who);
    GridDev g;
    if (int rc = check_range(&f->desc, b, e, g, who)) return rc;
    if (why) return fail(DG_ERR_INVALID, "%s: %s", who, why);
    if (e > b && !out) return fail(DG_ERR_INVALID, "%s: output is NULL", who);
    return check_handle_device(f->device, who);
}

static const char* density_args_invalid(double h, double) { return (h > 0.0) ? nullptr : "smoothing length must be > 0"; }

// the volume map's arguments: h finite and > 0 (c1 = 0.5 * (-inf + inf) would make every offset NaN), scale finite
static const char* volume_args_invalid(double h, double scale)
{
    if (!(h > 0.0) || !std::isfinite(h)) return "smoothing length must be finite and > 0";
    if (!std::isfinite(scale)) return "scale must be finite";
    return nullptr;
}

static int density_launch(const dg_field* f, double h, double rho0, int no_reduction, uint64_t l_begin, uint64_t n, double* d_out, cudaStream_t st)
{
    DG_LAUNCH(k3_launch_density(f->dev, f->coeff_max, h, rho0, no_reduction, l_begin, n, d_out, st));
    return DG_OK;
}

static int volume_launch(const dg_field* f, double h, double scale, int no_reduction, uint64_t l_begin, uint64_t n, double* d_out, cudaStream_t st)
{
    DG_LAUNCH(k3_launch_volume(f->dev, h, scale, no_reduction, l_begin, n, d_out, st));
    return DG_OK;
}

int dg_density_map_device(const dg_field* f, double h, double rho0, int no_reduction, uint64_t l_begin, uint64_t l_end, double* d_out,
                          void* stream)
{
    if (int rc = node_map_check(f, l_begin, l_end, density_args_invalid(h, rho0), d_out, "dg_density_map_device")) return rc;
    return density_launch(f, h, rho0, no_reduction, l_begin, l_end - l_begin, d_out, (cudaStream_t)stream);
}

int dg_density_map(const dg_field* f, double h, double rho0, int no_reduction, uint64_t l_begin, uint64_t l_end, double* out_host)
{
    if (int rc = node_map_check(f, l_begin, l_end, density_args_invalid(h, rho0), out_host, "dg_density_map")) return rc;
    const uint64_t n = l_end - l_begin;
    return stage_on_device(n, n, {}, {{out_host, sizeof(double)}}, [&](void* const*, void* const* out, uint64_t b, uint64_t c) {
        return density_launch(f, h, rho0, no_reduction, l_begin + b, c, (double*)out[0], nullptr);
    });
}

int dg_volume_map_device(const dg_field* f, double h, double scale, int no_reduction, uint64_t l_begin, uint64_t l_end, double* d_out,
                         void* stream)
{
    if (int rc = node_map_check(f, l_begin, l_end, volume_args_invalid(h, scale), d_out, "dg_volume_map_device")) return rc;
    return volume_launch(f, h, scale, no_reduction, l_begin, l_end - l_begin, d_out, (cudaStream_t)stream);
}

int dg_volume_map(const dg_field* f, double h, double scale, int no_reduction, uint64_t l_begin, uint64_t l_end, double* out_host)
{
    if (int rc = node_map_check(f, l_begin, l_end, volume_args_invalid(h, scale), out_host, "dg_volume_map")) return rc;
    const uint64_t n = l_end - l_begin;
    return stage_on_device(n, n, {}, {{out_host, sizeof(double)}}, [&](void* const*, void* const* out, uint64_t b, uint64_t c) {
        return volume_launch(f, h, scale, no_reduction, l_begin + b, c, (double*)out[0], nullptr);
    });
}

// reduceField with its index passes on the GPU (k4_reduce.cu); the swap-walk compaction and the tie-order-preserving sort stay on the host
static int reduce_field_gpu(const GridDev& g, double* nodes, uint64_t n_nodes, const uint8_t* keep_node, uint32_t* cells, uint64_t n_cells_in,
                            uint32_t* cell_map, uint64_t n_cells_grid, bool force_std_sort, ReduceStats& st)
{
    auto t0 = std::chrono::steady_clock::now();
    auto lap = [&]() { const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); t0 = std::chrono::steady_clock::now(); return ms; };
    const uint64_t tile = k4_tile(), n_tiles = (n_cells_in + tile - 1) / tile;
    DevBuf<double> d_nodes, d_nodes_out;
    DevBuf<unsigned char> d_keep, d_cell_keep, d_used;
    DevBuf<unsigned> d_cells, d_cells_out, d_cell_map, d_tile, d_bad, d_perm, d_order, d_new_id;
    DevBuf<unsigned long long> d_key;
    // ---- 1. surviving cells, cell map, compacted rows (:1076-1098)
    DG_CUDA(d_nodes.alloc(n_nodes)); DG_CUDA(d_keep.alloc(n_nodes)); DG_CUDA(d_cells.alloc(32 * n_cells_in)); DG_CUDA(d_cells_out.alloc(32 * n_cells_in));
    DG_CUDA(d_cell_keep.alloc(n_cells_in)); DG_CUDA(d_cell_map.alloc(n_cells_in)); DG_CUDA(d_tile.alloc(n_tiles)); DG_CUDA(d_bad.alloc(1)); DG_CUDA(d_used.alloc(n_nodes));
    DG_CUDA(cudaMemcpyAsync(d_keep.p, keep_node, n_nodes, cudaMemcpyHostToDevice, nullptr));
    DG_CUDA(cudaMemcpyAsync(d_cells.p, cells, 32 * n_cells_in * sizeof(unsigned), cudaMemcpyHostToDevice, nullptr));
    DG_CUDA(cudaMemcpyAsync(d_nodes.p, nodes, n_nodes * sizeof(double), cudaMemcpyHostToDevice, nullptr));
    DG_CUDA(cudaMemsetAsync(d_bad.p, 0, sizeof(unsigned), nullptr));
    DG_CUDA(cudaMemsetAsync(d_used.p, 0, n_nodes, nullptr));
    DG_LAUNCH(k4_launch_cell_keep(d_cells.p, n_cells_in, d_keep.p, (unsigned)n_nodes, d_cell_keep.p, d_bad.p, nullptr));
    DG_LAUNCH(k4_launch_tile_count(d_cell_keep.p, n_cells_in, d_tile.p, nullptr));
    std::vector<unsigned> tile_cnt(n_tiles);
    unsigned bad = 0;
    if (n_tiles) DG_CUDA(cudaMemcpy(tile_cnt.data(), d_tile.p, n_tiles * sizeof(unsigned), cudaMemcpyDeviceToHost));
    DG_CUDA(cudaMemcpy(&bad, d_bad.p, sizeof bad, cudaMemcpyDeviceToHost));
    if (bad) return fail(DG_ERR_INVALID, "dg_reduce_field: a cell refers to a node id >= n_nodes");
    uint64_t kept_cells = 0;
    for (uint64_t t = 0; t < n_tiles; t++) { const unsigned c = tile_cnt[t]; tile_cnt[t] = (unsigned)kept_cells; kept_cells += c; }     // exclusive scan of ~n/1024 counts
    if (n_tiles) DG_CUDA(cudaMemcpyAsync(d_tile.p, tile_cnt.data(), n_tiles * sizeof(unsigned), cudaMemcpyHostToDevice, nullptr));
    DG_LAUNCH(k4_launch_cell_compact(d_cells.p, n_cells_in, d_cell_keep.p, d_tile.p, d_cells_out.p, d_cell_map.p, nullptr));
    DG_LAUNCH(k4_launch_mark_used(d_cells_out.p, 32 * kept_cells, d_used.p, nullptr));
    if (n_cells_in) DG_CUDA(cudaMemcpyAsync(cell_map, d_cell_map.p, n_cells_in * sizeof(unsigned), cudaMemcpyDeviceToHost, nullptr));
    std::vector<uint8_t> used(n_nodes);
    DG_CUDA(cudaMemcpy(used.data(), d_used.p, n_nodes, cudaMemcpyDeviceToHost));
    for (uint64_t i = n_cells_in; i < n_cells_grid; i++) cell_map[i] = (uint32_t)i;                     // resize + iota (:1076-1078) for cells the field never had
    st.cells_out = kept_cells;
    st.ms_cells = lap();
    // ---- 2. surviving nodes: the reference's swap walk on a permutation (host, serial by nature)
    std::vector<uint32_t> perm;
    const uint64_t m = reduce_swap_walk(used.data(), n_nodes, perm);
    st.nodes_out = m;
    st.ms_nodes = lap();
    // ---- 3. Z-curve keys on the GPU, the order among them on the host (std::sort's tie order)
    DG_CUDA(d_perm.alloc(m)); DG_CUDA(d_key.alloc(m)); DG_CUDA(d_order.alloc(m)); DG_CUDA(d_new_id.alloc(n_nodes)); DG_CUDA(d_nodes_out.alloc(m));
    if (m) DG_CUDA(cudaMemcpyAsync(d_perm.p, perm.data(), m * sizeof(unsigned), cudaMemcpyHostToDevice, nullptr));
    DG_LAUNCH(k4_launch_morton_keys(g, d_perm.p, m, d_key.p, nullptr));
    std::vector<unsigned long long> key(m);
    if (m) DG_CUDA(cudaMemcpy(key.data(), d_key.p, m * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    std::vector<KeyPos> kp(m);
    parallel_for(m, [&](uint64_t b0, uint64_t e0) { for (uint64_t i = b0; i < e0; i++) { kp[i].key = key[i]; kp[i].pos = (uint32_t)i; } });
    std::vector<uint32_t> order;
    reduce_order_survivors(kp, force_std_sort, order, st.tie_path);
    st.ms_sort = lap();
    // ---- 4. new ids, renumbered rows, gathered coefficients (:1158-1173)
    if (m) DG_CUDA(cudaMemcpyAsync(d_order.p, order.data(), m * sizeof(unsigned), cudaMemcpyHostToDevice, nullptr));
    DG_LAUNCH(k4_launch_renumber(d_perm.p, d_order.p, m, d_nodes.p, d_new_id.p, d_nodes_out.p, d_cells_out.p, 32 * kept_cells, nullptr));
    if (kept_cells) DG_CUDA(cudaMemcpyAsync(cells, d_cells_out.p, 32 * kept_cells * sizeof(unsigned), cudaMemcpyDeviceToHost, nullptr));
    if (m) DG_CUDA(cudaMemcpyAsync(nodes, d_nodes_out.p, m * sizeof(double), cudaMemcpyDeviceToHost, nullptr));
    DG_CUDA(cudaDeviceSynchronize());
    st.ms_write = lap();
    return DG_OK;
}

int dg_reduce_field(const dg_grid_desc* grid, double* nodes, uint64_t n_nodes, const uint8_t* keep_node, uint32_t* cells, uint64_t n_cells_in,
                    uint32_t* cell_map, uint32_t flags, uint64_t* n_nodes_out, uint64_t* n_cells_out, double* timings_ms)
{
    return guarded("dg_reduce_field", [&]() -> int {
        GridDev g;
        if (int rc = grid_checked(grid, g, "dg_reduce_field")) return rc;
        const uint64_t n_grid_nodes = grid_nodes(g), n_grid_cells = grid_cells(g);
        if (!nodes || !keep_node || !cell_map || (n_cells_in && !cells) || !n_nodes_out || !n_cells_out)
            return fail(DG_ERR_INVALID, "dg_reduce_field: NULL argument");
        if (n_nodes != n_grid_nodes)          // node ids must be the grid's own numbering: their positions feed the Z-curve key (:1113)
            return fail(DG_ERR_INVALID, "dg_reduce_field: the field has %llu nodes, the grid %llu (already reduced?)", (unsigned long long)n_nodes,
                        (unsigned long long)n_grid_nodes);
        if (n_cells_in > n_grid_cells) return fail(DG_ERR_INVALID, "dg_reduce_field: more cells than the grid has");
        ReduceStats st; const char* err = "";
        const char* env = std::getenv("DG_REDUCE_FIELD_HOST");
        const bool host_passes = (flags & DG_REDUCE_HOST_PASSES) != 0 || (env && env[0] == '1');
        if (host_passes) {
            if (!reduce_field_host(g, nodes, n_nodes, keep_node, cells, n_cells_in, cell_map, n_grid_cells, (flags & DG_REDUCE_REFERENCE_SORT) != 0, st, &err))
                return fail(DG_ERR_INVALID, "dg_reduce_field: %s", err);
        } else {
            if (int rc = require_device()) return rc;
            if (int rc = reduce_field_gpu(g, nodes, n_nodes, keep_node, cells, n_cells_in, cell_map, n_grid_cells, (flags & DG_REDUCE_REFERENCE_SORT) != 0, st)) return rc;
        }
        *n_nodes_out = st.nodes_out; *n_cells_out = st.cells_out;
        if (timings_ms) { timings_ms[0] = st.ms_cells; timings_ms[1] = st.ms_nodes; timings_ms[2] = st.ms_sort; timings_ms[3] = st.ms_write; timings_ms[4] = (double)st.tie_path; }
        return DG_OK;
    });
}

// ------------------------------------------------------------------------------------------------ reduced fields on the device
// reduceField(id, pred) for a dense field that is already on the device and a predicate of the node value alone (K4ValuePred): every array
// the size of the grid (coefficients, cell flags, node marks, the swap-walk positions, new ids) lives on the device only.  The host holds one
// count per 1024 flags for the scans and the survivors' Z-curve keys for the tie-order-preserving sort; the results stay on the device in a
// dg_reduced_band (a reduced field kept on its device) until dg_reduced_band_copy.
struct dg_reduced_band {
    dg_grid_desc desc;                   // the grid it was made for: dg_field_create_reduced builds its field on it
    DevBuf<double> d_nodes;
    DevBuf<unsigned> d_cells, d_cell_map;
    uint64_t n_nodes = 0, n_cells = 0, n_grid_cells = 0;
    int device = 0;
};

namespace {
// ms since the last lap
struct StageClock {
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    double lap()
    {
        const auto t = std::chrono::steady_clock::now();
        const double ms = std::chrono::duration<double, std::milli>(t - t0).count();
        t0 = t;
        return ms;
    }
};

// the rows of the field being reduced: an uploaded table of n_cells rows, or (d_cells == nullptr) the closed form of every grid cell
struct DenseRows {
    const unsigned* d_cells;
    uint64_t n_cells;
};
}  // namespace

// kept cells (:1081-1098), first half: d_cell_keep[c] = some node of row c is kept by pred, or -- d_mask != nullptr -- has a nonzero byte in
// d_mask (a node predicate already combined with v != DBL_MAX).  Uploaded rows are checked on the way: a row that names a node >= n is
// refused, as dg_reduce_field refuses it.  Synchronises `st`.
static int device_cell_flags(const GridDev& g, const double* d_dense, uint64_t n, const DenseRows& rows, const K4ValuePred& pred,
                             DevBuf<unsigned char>& d_cell_keep, const char* who, cudaStream_t st, const unsigned char* d_mask = nullptr)
{
    DG_CUDA(d_cell_keep.alloc(rows.n_cells));
    if (!rows.d_cells) {
        if (d_mask) DG_LAUNCH(k4_launch_closed_cell_keep_mask(g, d_mask, rows.n_cells, d_cell_keep.p, st));
        else DG_LAUNCH(k4_launch_closed_cell_keep(g, d_dense, rows.n_cells, pred, d_cell_keep.p, st));
        DG_CUDA(cudaStreamSynchronize(st));
        return DG_OK;
    }
    DevBuf<unsigned char> d_keep;
    DevBuf<unsigned> d_bad;
    DG_CUDA(d_bad.alloc(1));
    DG_CUDA(cudaMemsetAsync(d_bad.p, 0, sizeof(unsigned), st));
    if (!d_mask) {
        DG_CUDA(d_keep.alloc(n));
        DG_LAUNCH(k4_launch_node_keep(d_dense, n, pred, d_keep.p, st));
        d_mask = d_keep.p;
    }
    DG_LAUNCH(k4_launch_cell_keep(rows.d_cells, rows.n_cells, d_mask, (unsigned)n, d_cell_keep.p, d_bad.p, st));
    unsigned bad = 0;
    DG_CUDA(cudaMemcpyAsync(&bad, d_bad.p, sizeof bad, cudaMemcpyDeviceToHost, st));
    DG_CUDA(cudaStreamSynchronize(st));
    if (bad) return fail(DG_ERR_INVALID, "%s: a cell refers to a node id >= n_nodes", who);
    return DG_OK;
}

// the rest of reduceField (:1076-1173) into `out`: cell map + kept rows, surviving nodes by the swap walk, their Z-curve order, renumbered
// rows and gathered coefficients.  ms[0..4) += kept cells, node compaction, sort, write-back; each stage ends with a synchronise.
static int device_reduce(const GridDev& g, const double* d_dense, uint64_t n, const DenseRows& rows, const unsigned char* d_cell_keep,
                         uint64_t n_grid_cells, bool reference_sort, dg_reduced_band& out, double ms[4], int& tie_path, StageClock& clock,
                         cudaStream_t st)
{
    const uint64_t tile = k4_tile();
    // ---- kept cells, second half: cell map + the kept rows, order kept; cells the field has no row for map to themselves (:1076-1078)
    uint64_t kept_cells = 0;
    {
        DevBuf<unsigned> d_tile;
        DG_CUDA(d_tile.alloc((rows.n_cells + tile - 1) / tile)); DG_CUDA(out.d_cell_map.alloc(n_grid_cells));
        DG_LAUNCH(k4_scan_flags(d_cell_keep, rows.n_cells, d_tile.p, kept_cells, st));
        DG_CUDA(out.d_cells.alloc(32 * kept_cells));
        if (rows.d_cells)
            DG_LAUNCH(k4_launch_cell_compact(rows.d_cells, rows.n_cells, d_cell_keep, d_tile.p, out.d_cells.p, out.d_cell_map.p, st));
        else
            DG_LAUNCH(k4_launch_closed_cell_compact(g, rows.n_cells, d_cell_keep, d_tile.p, out.d_cells.p, out.d_cell_map.p, st));
        DG_LAUNCH(k4_launch_iota(out.d_cell_map.p, rows.n_cells, n_grid_cells, st));
        DG_CUDA(cudaStreamSynchronize(st));
    }
    out.n_cells = kept_cells;
    out.n_grid_cells = n_grid_cells;
    ms[0] += clock.lap();
    // ---- surviving nodes = nodes of kept cells (:1117-1134), compacted by the reference's swap walk (:1135-1156) on the device
    DevBuf<unsigned> d_walk;
    uint64_t m_nodes = 0;
    {
        DevBuf<unsigned char> d_used;
        DevBuf<unsigned> d_tile, d_flag;
        DG_CUDA(d_used.alloc(n)); DG_CUDA(d_tile.alloc((n + tile - 1) / tile)); DG_CUDA(d_flag.alloc(1)); DG_CUDA(d_walk.alloc(n));
        DG_CUDA(cudaMemsetAsync(d_used.p, 0, n, st));
        DG_LAUNCH(k4_launch_mark_used(out.d_cells.p, 32 * kept_cells, d_used.p, st));
        unsigned rounds = 0;
        DG_LAUNCH(k4_swap_walk(d_used.p, n, d_tile.p, d_flag.p, d_walk.p, m_nodes, rounds, st));
        DG_CUDA(cudaStreamSynchronize(st));
    }
    out.n_nodes = m_nodes;
    ms[1] += clock.lap();
    // ---- Z-curve keys in swap-walk position order on the device; their order on the host (std::sort's order among equal keys)
    std::vector<uint32_t> order;
    {
        DevBuf<unsigned long long> d_key;
        DG_CUDA(d_key.alloc(m_nodes));
        DG_LAUNCH(k4_launch_morton_keys(g, d_walk.p, m_nodes, d_key.p, st));
        std::vector<KeyPos> kp(m_nodes);
        {
            std::vector<unsigned long long> key(m_nodes);
            if (m_nodes) DG_CUDA(cudaMemcpyAsync(key.data(), d_key.p, m_nodes * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
            DG_CUDA(cudaStreamSynchronize(st));
            parallel_for(m_nodes, [&](uint64_t b0, uint64_t e0) { for (uint64_t i = b0; i < e0; i++) { kp[i].key = key[i]; kp[i].pos = (uint32_t)i; } });
        }
        reduce_order_survivors(kp, reference_sort, order, tie_path);
    }
    ms[2] += clock.lap();
    // ---- new ids, renumbered rows, gathered coefficients (:1158-1173) into the handle's buffers
    {
        DevBuf<unsigned> d_order, d_new_id;
        DG_CUDA(d_order.alloc(m_nodes)); DG_CUDA(d_new_id.alloc(n)); DG_CUDA(out.d_nodes.alloc(m_nodes));
        if (m_nodes) DG_CUDA(cudaMemcpyAsync(d_order.p, order.data(), m_nodes * sizeof(unsigned), cudaMemcpyHostToDevice, st));
        DG_LAUNCH(k4_launch_renumber(d_walk.p, d_order.p, m_nodes, d_dense, d_new_id.p, out.d_nodes.p, out.d_cells.p, 32 * kept_cells, st));
        DG_CUDA(cudaStreamSynchronize(st));
    }
    ms[3] += clock.lap();
    return DG_OK;
}

// the reduction of a field made on the device (band, function, uploaded field): rows from `rows`, keep flags from d_mask (NULL: v != DBL_MAX
// alone), the device_reduce stages
static int reduce_device_field(const GridDev& g, const double* d_values, uint64_t n, const DenseRows& rows, const unsigned char* d_mask,
                               uint32_t flags, dg_reduced_band& out, double ms[5], int& tie_path, StageClock& clock, const char* who, cudaStream_t st)
{
    DevBuf<unsigned char> d_cell_keep;
    if (int rc = device_cell_flags(g, d_values, n, rows, K4ValuePred{K4_KEEP_ANY, 0.0, 0.0, 0.0}, d_cell_keep, who, st, d_mask)) return rc;
    return device_reduce(g, d_values, n, rows, d_cell_keep.p, grid_cells(g), (flags & DG_REDUCE_REFERENCE_SORT) != 0, out, ms + 1, tie_path, clock, st);
}

// timings_ms[0..7) of the reduced forms made by reduce_device_field: ms[0..5), the tie path, the total ms
static void reduced_timings(double* timings_ms, const double ms[5], int tie_path, std::chrono::steady_clock::time_point t_start)
{
    if (!timings_ms) return;
    for (int k = 0; k < 5; k++) timings_ms[k] = ms[k];
    timings_ms[5] = (double)tie_path;
    timings_ms[6] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count();
}


// addFunction(func, verbose, band predicate) + reduceField(id, always true) on one GPU
int dg_reduced_band_create(const dg_mesh* m, const dg_grid_desc* grid, double sign, double band, uint32_t flags, dg_reduced_band** out,
                           double* timings_ms)
{
    static const char* who = "dg_reduced_band_create";
    return guarded(who, [&]() -> int {
        if (!out) return fail(DG_ERR_INVALID, "%s: out is NULL", who);
        *out = nullptr;
        if (int rc = mesh_usable(m, who)) return rc;
        GridDev g;
        if (int rc = grid_checked(grid, g, who)) return rc;
        if (int rc = check_band(band, who)) return rc;
        if (int rc = check_reduce_flags(flags, who)) return rc;
        const uint64_t n = grid_nodes(g);
        if (int rc = require_device()) return rc;
        if (int rc = check_handle_device(m->device, who)) return rc;
        StageClock clock;
        const auto t_start = clock.t0;
        const cudaStream_t st = nullptr;
        double ms[5] = {0, 0, 0, 0, 0};
        std::unique_ptr<dg_reduced_band> h(new dg_reduced_band());
        h->desc = *grid;
        DG_CUDA(cudaGetDevice(&h->device));
        // ---- 1. the dense band coefficients (addFunction(func, pred), :806-817), on the device only
        DevBuf<double> d_dense;
        DG_CUDA(d_dense.alloc(n));
        if (int rc = dg_sample_sdf_band_device(m, grid, sign, band, 0, n, d_dense.p, st)) return rc;
        DG_CUDA(cudaStreamSynchronize(st));
        ms[0] = clock.lap();
        // ---- 2.-5. reduceField(id, always true): a node is kept iff its coefficient is not DBL_MAX; rows from the closed form
        int tie_path = 0;
        if (int rc = reduce_device_field(g, d_dense.p, n, DenseRows{nullptr, grid_cells(g)}, nullptr, flags, *h, ms, tie_path, clock, who, st)) return rc;
        reduced_timings(timings_ms, ms, tie_path, t_start);
        *out = h.release();
        return DG_OK;
    });
}

// What a reduced node map (GenerateDensityMap's pattern) takes from its node function: the entry point's name, the check of its
// arguments (nullptr when they are valid), the K3 kernel that samples every node with the sample predicate on, and field 1's predicate.
struct ReducedNodeMap {
    const char* who;
    const char* (*args_invalid)(double h, double param);
    cudaError_t (*launch)(const dg_field& f, double h, double param, uint64_t n, double* d_out, cudaStream_t st);
    K4ValuePred keep1;
};

// GenerateDensityMap with reduction (cmd/generate_density_map/main.cpp:117-147) on one GPU, for the density map and the volume map: the node
// function (K3) on the uploaded SDF field, then reduceField of the SDF field over its own rows with the tool's predicate, and of the new
// field over the closed-form rows with m.keep1.
static int reduced_node_map_create_impl(const ReducedNodeMap& m, const dg_grid_desc* grid, const double* sdf_nodes, uint64_t n_nodes,
                                        const uint32_t* sdf_cells, uint64_t n_cells, const uint32_t* sdf_cell_map, double h, double param,
                                        uint32_t flags, dg_reduced_band** sdf_out, dg_reduced_band** density_out, double* timings_ms)
{
    const char* who = m.who;
    if (!sdf_out || !density_out) return fail(DG_ERR_INVALID, "%s: out is NULL", who);
    *sdf_out = nullptr; *density_out = nullptr;
    GridDev g;
    if (int rc = grid_checked(grid, g, who)) return rc;
    const uint64_t n = grid_nodes(g), n_grid_cells = grid_cells(g);
    if (!sdf_nodes || !sdf_cell_map || (n_cells && !sdf_cells)) return fail(DG_ERR_INVALID, "%s: NULL argument", who);
    if (n_nodes != n)                     // node ids must be the grid's own numbering: their positions feed the Z-curve key (:1113)
        return fail(DG_ERR_INVALID, "%s: the SDF field has %llu nodes, the grid %llu (already reduced?)", who, (unsigned long long)n_nodes,
                    (unsigned long long)n);
    if (n_cells > n_grid_cells) return fail(DG_ERR_INVALID, "%s: more cells than the grid has", who);
    if (const char* why = m.args_invalid(h, param)) return fail(DG_ERR_INVALID, "%s: %s", who, why);
    if (int rc = check_reduce_flags(flags, who)) return rc;
    if (int rc = require_device()) return rc;
    if (int rc = ensure_selftest()) return rc;
    // the tool's SDF predicate (main.cpp:139) with its bounds computed as its lambda computes them
    const double cell_diag = k3_cell_diag(g);
    const K4ValuePred sdf_pred{K4_KEEP_SDF, -6.0 * h, 2.0 * h, cell_diag};
    const K4ValuePred density_pred = m.keep1;
    const bool reference_sort = (flags & DG_REDUCE_REFERENCE_SORT) != 0;
    StageClock clock;
    const auto t_start = clock.t0;
    const cudaStream_t st = nullptr;
    double ms[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};       // upload + pack, density, field 0: 4 stages, field 1: 4 stages
    int tie[2] = {0, 0};
    std::unique_ptr<dg_reduced_band> r0(new dg_reduced_band()), r1(new dg_reduced_band());
    DG_CUDA(cudaGetDevice(&r0->device));
    r1->device = r0->device;
    r0->desc = r1->desc = *grid;
    // ---- 1. upload the SDF field; flag the kept cells of its reduction (this checks the rows) and check the cell map before K2 packs
    //         through them (dg_field_create's checks); pack the SDF field for K3
    DevBuf<double> d_sdf, d_density;
    DevBuf<unsigned> d_cells;
    DevBuf<unsigned char> d_cell_keep0;
    std::unique_ptr<dg_field> f(new dg_field());
    f->desc = *grid; f->dev.g = g; f->n_nodes = n; f->n_cells_kept = n_cells;
    DG_CUDA(d_sdf.alloc(n)); DG_CUDA(d_cells.alloc(32 * n_cells)); DG_CUDA(f->d_cell_map.alloc(n_grid_cells));
    DG_CUDA(cudaMemcpyAsync(d_sdf.p, sdf_nodes, n * sizeof(double), cudaMemcpyHostToDevice, st));
    if (n_cells) DG_CUDA(cudaMemcpyAsync(d_cells.p, sdf_cells, 32 * n_cells * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    DG_CUDA(cudaMemcpyAsync(f->d_cell_map.p, sdf_cell_map, n_grid_cells * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    DG_CUDA(cudaStreamSynchronize(st));
    ms[0] = clock.lap();
    if (int rc = device_cell_flags(g, d_sdf.p, n, DenseRows{d_cells.p, n_cells}, sdf_pred, d_cell_keep0, who, st)) return rc;
    ms[2] = clock.lap();                                   // counted as field 0's kept cells
    {
        DevBuf<unsigned> d_bad;
        unsigned bad = 0;
        DG_CUDA(d_bad.alloc(1));
        DG_CUDA(cudaMemsetAsync(d_bad.p, 0, sizeof(unsigned), st));
        DG_LAUNCH(k4_launch_cell_map_check(f->d_cell_map.p, n_grid_cells, n_cells, d_bad.p, st));
        DG_CUDA(cudaMemcpyAsync(&bad, d_bad.p, sizeof bad, cudaMemcpyDeviceToHost, st));
        DG_CUDA(cudaStreamSynchronize(st));
        if (bad) return fail(DG_ERR_INVALID, "%s: a cell_map entry is >= n_cells", who);
    }
    if (int rc = field_finish(f.get(), d_sdf.p, d_cells.p, st)) return rc;
    DG_CUDA(cudaStreamSynchronize(st));
    ms[0] += clock.lap();
    // ---- 2. addFunction(node_func, verbose, pred) (main.cpp:96-133): K3 over every node, predicate on
    DG_CUDA(d_density.alloc(n));
    DG_LAUNCH(m.launch(*f, h, param, n, d_density.p, st));
    DG_CUDA(cudaStreamSynchronize(st));
    ms[1] = clock.lap();
    // ---- 3. the packed SDF field is not needed any more: free it before reducing anything
    f.reset();
    // ---- 4. reduceField(0, -6h < v + cell_diag && v - cell_diag < 2h) over the SDF field's own rows
    if (int rc = device_reduce(g, d_sdf.p, n, DenseRows{d_cells.p, n_cells}, d_cell_keep0.p, n_grid_cells, reference_sort, *r0, ms + 2, tie[0], clock, st))
        return rc;
    d_cell_keep0.release(); d_cells.release(); d_sdf.release();
    // ---- 5. reduceField(1, keep1) over the closed-form rows of the new field (addSampledFunction's cells, identity map)
    {
        const DenseRows rows1{nullptr, n_grid_cells};
        DevBuf<unsigned char> d_cell_keep1;
        if (int rc = device_cell_flags(g, d_density.p, n, rows1, density_pred, d_cell_keep1, who, st)) return rc;
        if (int rc = device_reduce(g, d_density.p, n, rows1, d_cell_keep1.p, n_grid_cells, reference_sort, *r1, ms + 6, tie[1], clock, st)) return rc;
    }
    if (timings_ms) {
        for (int k = 0; k < 10; k++) timings_ms[k] = ms[k];
        timings_ms[10] = (double)tie[0]; timings_ms[11] = (double)tie[1];
        timings_ms[12] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count();
    }
    *sdf_out = r0.release(); *density_out = r1.release();
    return DG_OK;
}

int dg_reduced_density_map_create(const dg_grid_desc* grid, const double* sdf_nodes, uint64_t n_nodes, const uint32_t* sdf_cells, uint64_t n_cells,
                                  const uint32_t* sdf_cell_map, double h, double rho0, uint32_t flags, dg_reduced_band** sdf_out,
                                  dg_reduced_band** density_out, double* timings_ms)
{
    // GenerateDensityMap's second predicate, 0 <= v && v <= 3 rho0 (main.cpp:140)
    const ReducedNodeMap m{"dg_reduced_density_map_create",
                           density_args_invalid,
                           [](const dg_field& f, double h_, double rho0_, uint64_t n, double* d_out, cudaStream_t st) {
                               return k3_launch_density(f.dev, f.coeff_max, h_, rho0_, 0, 0, n, d_out, st);
                           },
                           K4ValuePred{K4_KEEP_RANGE, 0.0, 3.0 * rho0, 0.0}};
    return guarded("dg_reduced_density_map_create", [&]() {
        return reduced_node_map_create_impl(m, grid, sdf_nodes, n_nodes, sdf_cells, n_cells, sdf_cell_map, h, rho0, flags, sdf_out, density_out, timings_ms);
    });
}

int dg_reduced_volume_map_create(const dg_grid_desc* grid, const double* sdf_nodes, uint64_t n_nodes, const uint32_t* sdf_cells, uint64_t n_cells,
                                 const uint32_t* sdf_cell_map, double h, double scale, uint32_t flags, dg_reduced_band** sdf_out,
                                 dg_reduced_band** volume_out, double* timings_ms)
{
    // the volume field keeps 0 <= v (and != DBL_MAX, as every reduceField): K4_KEEP_RANGE with b = +inf
    const ReducedNodeMap m{"dg_reduced_volume_map_create", volume_args_invalid,
                           [](const dg_field& f, double h_, double scale_, uint64_t n, double* d_out, cudaStream_t st) {
                               return k3_launch_volume(f.dev, h_, scale_, 0, 0, n, d_out, st);
                           },
                           K4ValuePred{K4_KEEP_RANGE, 0.0, INFINITY, 0.0}};
    return guarded("dg_reduced_volume_map_create", [&]() {
        return reduced_node_map_create_impl(m, grid, sdf_nodes, n_nodes, sdf_cells, n_cells, sdf_cell_map, h, scale, flags, sdf_out, volume_out, timings_ms);
    });
}

// ------------------------------------------------------------------------------------------------ user functions on the GPU (device callbacks)
// addFunction(func, verbose, pred) and reduceField(id, pred) for the caller's own GPU code: the library produces the node positions of each
// chunk of ids on the device and calls the callbacks for it on the calling thread (ctypes callbacks need that), on the library's call stream.
namespace {
struct DeviceCallbacks {
    dg_device_function func = nullptr; void* fu = nullptr;
    dg_device_sample_predicate sample = nullptr; void* su = nullptr;
    dg_device_node_predicate node = nullptr; void* nu = nullptr;
};

// The stream the device-callback calls work on: one per device, created at first use and kept.  It is a BLOCKING stream, so its work starts
// after the work the caller queued before the call on the legacy default stream (torch's default stream, and CUDA code that names no
// stream): a callback that reads data produced just before the call sees it.  Kept rather than created per call, so that what the caller's
// allocator caches for the callbacks' temporaries (torch tags freed blocks with the stream they were used on) serves every later call.
std::mutex g_call_stream_mu;
std::vector<cudaStream_t> g_call_streams;

int call_stream(cudaStream_t& s)
{
    int dev = 0, n_dev = 0;
    DG_CUDA(cudaGetDevice(&dev));
    DG_CUDA(cudaGetDeviceCount(&n_dev));
    std::lock_guard<std::mutex> lock(g_call_stream_mu);
    if (g_call_streams.size() < (size_t)n_dev) g_call_streams.resize((size_t)n_dev, nullptr);
    if (!g_call_streams[dev]) DG_CUDA(cudaStreamCreateWithFlags(&g_call_streams[dev], cudaStreamDefault));
    s = g_call_streams[dev];
    return DG_OK;
}

// the call's work on the call stream has finished when the call returns, on every path (its buffers are freed after it)
struct CallStreamSync {
    cudaStream_t s = nullptr;
    ~CallStreamSync() { if (s) cudaStreamSynchronize(s); }
};
}  // namespace

static uint64_t callback_chunk(uint64_t chunk_nodes, uint64_t n) { return std::max<uint64_t>(1, std::min<uint64_t>(chunk_nodes ? chunk_nodes : (1ull << 24), n)); }

// Runs the callbacks over nodes [0, n) chunk by chunk, in ascending order: positions (k1_launch_node_positions: the bits of dg_node_positions),
// then cb.sample -> a chunk mask, cb.func -> d_values + b and DBL_MAX where the mask is 0 (:806-817), then cb.node -> d_keep + b, ANDed with
// v != DBL_MAX (:1073).  cb.func == NULL: d_values already holds the field.  ms_callbacks += host time inside the callbacks.  Synchronises `st`.
static int run_device_callbacks(const GridDev& g, uint64_t n, uint64_t chunk_nodes, const DeviceCallbacks& cb, double* d_values, unsigned char* d_keep,
                                double& ms_callbacks, const char* who, cudaStream_t st)
{
    const uint64_t chunk = callback_chunk(chunk_nodes, n);
    DevBuf<double> d_x;
    DevBuf<unsigned char> d_smask;
    DG_CUDA(d_x.alloc(3 * chunk));
    if (cb.sample) DG_CUDA(d_smask.alloc(chunk));
    auto call = [&](const char* name, uint64_t b, uint64_t e, auto&& f) -> int {
        const auto t0 = std::chrono::steady_clock::now();
        const int rc = f();
        ms_callbacks += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (rc == 0) return DG_OK;
        cudaStreamSynchronize(st);                  // whatever the callbacks enqueued has finished before the buffers are freed
        cudaGetLastError();
        return fail(DG_ERR_CALLBACK, "%s: the %s callback returned %d for the chunk of nodes [%llu, %llu)", who, name, rc, (unsigned long long)b,
                    (unsigned long long)e);
    };
    for (uint64_t b = 0; b < n; b += chunk) {
        const uint64_t cnt = std::min(chunk, n - b), e = b + cnt;
        DG_LAUNCH(k1_launch_node_positions(g, b, cnt, d_x.p, st));
        if (cb.sample) {
            if (int rc = call("sample predicate", b, e, [&] { return cb.sample(cb.su, d_x.p, cnt, d_smask.p, st); })) return rc;
        }
        if (cb.func) {
            if (int rc = call("function", b, e, [&] { return cb.func(cb.fu, d_x.p, cb.sample ? d_smask.p : nullptr, cnt, d_values + b, st); })) return rc;
            if (cb.sample) DG_LAUNCH(k4_launch_sample_mask_apply(d_values + b, d_smask.p, cnt, st));
        }
        if (cb.node) {
            if (int rc = call("node predicate", b, e, [&] { return cb.node(cb.nu, d_x.p, d_values + b, cnt, d_keep + b, st); })) return rc;
            DG_LAUNCH(k4_launch_node_mask_combine(d_keep + b, d_values + b, cnt, st));
        }
    }
    DG_CUDA(cudaStreamSynchronize(st));
    return DG_OK;
}

// checks shared by the three entry points: the grid (grids of 2^31 nodes or more are refused), then a device
static int device_callback_setup(const dg_grid_desc* grid, GridDev& g, uint64_t& n, const char* who)
{
    if (int rc = grid_checked(grid, g, who)) return rc;
    n = grid_nodes(g);
    if (int rc = require_device()) return rc;
    return ensure_selftest();
}

int dg_add_function_device(const dg_grid_desc* grid, dg_device_function func, void* fu, dg_device_sample_predicate pred, void* pu,
                           uint64_t chunk_nodes, double* nodes_host, uint32_t* cells_host, uint32_t* cell_map_host, double* timings_ms)
{
    static const char* who = "dg_add_function_device";
    return guarded(who, [&]() -> int {
        if (!func) return fail(DG_ERR_INVALID, "%s: the function callback is NULL", who);
        if (!nodes_host) return fail(DG_ERR_INVALID, "%s: nodes output is NULL", who);
        GridDev g; uint64_t n = 0;
        if (int rc = device_callback_setup(grid, g, n, who)) return rc;
        const auto t0 = std::chrono::steady_clock::now();
        auto ms_since = [&](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count(); };
        // host threads pre-fault nodes_host and write the connectivity + cell map (dg_add_function_sdf's HostTablesJob) while the callbacks run
        HostTablesJob job;
        job.start(g, n, nodes_host, cells_host, cell_map_host);
        double ms_callbacks = 0.0;
        int rc = DG_OK;
        {
            CallStreamSync st;
            DevBuf<double> d_values;
            if (int e = call_stream(st.s)) return e;
            DG_CUDA(d_values.alloc(n));
            DeviceCallbacks cb;
            cb.func = func; cb.fu = fu; cb.sample = pred; cb.su = pu;
            rc = run_device_callbacks(g, n, chunk_nodes, cb, d_values.p, nullptr, ms_callbacks, who, st.s);
            if (rc == DG_OK) {
                // the values -> nodes_host through dg_add_function_sdf's pinned double buffer, the table workers sharing the copies
                std::lock_guard<std::mutex> lock(g_pool.mu);
                DG_CUDA(g_pool.prepare(0, 1));
                DG_CUDA(cudaEventRecord(g_pool.chunk_ev[0], st.s));
                rc = drain_to_host_locked(d_values.p, n, n, nodes_host, &job);
            }
        }
        const double ms_nodes = ms_since(t0);
        job.finish();
        if (rc == DG_OK && timings_ms) {
            timings_ms[0] = ms_since(t0); timings_ms[1] = ms_nodes; timings_ms[2] = timings_ms[0]; timings_ms[3] = job.ms_prefault;
            timings_ms[4] = (double)job.n_workers; timings_ms[5] = ms_callbacks;
        }
        return rc;
    });
}

int dg_reduced_function_create(const dg_grid_desc* grid, dg_device_function func, void* fu, dg_device_sample_predicate sample_pred, void* su,
                               dg_device_node_predicate reduce_pred, void* ru, uint64_t chunk_nodes, uint32_t flags, dg_reduced_band** out,
                               double* timings_ms)
{
    static const char* who = "dg_reduced_function_create";
    return guarded(who, [&]() -> int {
        if (!out) return fail(DG_ERR_INVALID, "%s: out is NULL", who);
        *out = nullptr;
        if (!func) return fail(DG_ERR_INVALID, "%s: the function callback is NULL", who);
        if (int rc = check_reduce_flags(flags, who)) return rc;
        GridDev g; uint64_t n = 0;
        if (int rc = device_callback_setup(grid, g, n, who)) return rc;
        StageClock clock;
        const auto t_start = clock.t0;
        double ms[5] = {0, 0, 0, 0, 0}, ms_callbacks = 0.0;
        int tie_path = 0;
        std::unique_ptr<dg_reduced_band> h(new dg_reduced_band());
        h->desc = *grid;
        DG_CUDA(cudaGetDevice(&h->device));
        CallStreamSync st;
        if (int rc = call_stream(st.s)) return rc;
        // ---- 1. addFunction(func, verbose, sample_pred) into a dense array on the device; the reduce predicate's mask per chunk meanwhile
        DevBuf<double> d_values;
        DevBuf<unsigned char> d_keep;
        DG_CUDA(d_values.alloc(n));
        if (reduce_pred) DG_CUDA(d_keep.alloc(n));
        DeviceCallbacks cb;
        cb.func = func; cb.fu = fu; cb.sample = sample_pred; cb.su = su; cb.node = reduce_pred; cb.nu = ru;
        if (int rc = run_device_callbacks(g, n, chunk_nodes, cb, d_values.p, d_keep.p, ms_callbacks, who, st.s)) return rc;
        ms[0] = clock.lap();
        // ---- 2.-5. reduceField(id, reduce_pred) over the closed-form rows of the new field (addFunction's cells, identity map)
        if (int rc = reduce_device_field(g, d_values.p, n, DenseRows{nullptr, grid_cells(g)}, d_keep.p, flags, *h, ms, tie_path, clock, who, st.s)) return rc;
        reduced_timings(timings_ms, ms, tie_path, t_start);
        if (timings_ms) timings_ms[7] = ms_callbacks;
        *out = h.release();
        return DG_OK;
    });
}

int dg_reduce_field_device(const dg_grid_desc* grid, const double* nodes, uint64_t n_nodes, const uint32_t* cells, uint64_t n_cells,
                           dg_device_node_predicate pred, void* pu, uint64_t chunk_nodes, uint32_t flags, dg_reduced_band** out,
                           double* timings_ms)
{
    static const char* who = "dg_reduce_field_device";
    return guarded(who, [&]() -> int {
        if (!out) return fail(DG_ERR_INVALID, "%s: out is NULL", who);
        *out = nullptr;
        if (!pred) return fail(DG_ERR_INVALID, "%s: the node predicate callback is NULL", who);
        if (!nodes || (n_cells && !cells)) return fail(DG_ERR_INVALID, "%s: NULL argument", who);
        if (int rc = check_reduce_flags(flags, who)) return rc;
        GridDev g; uint64_t n = 0;
        if (int rc = device_callback_setup(grid, g, n, who)) return rc;
        if (n_nodes != n)                     // node ids must be the grid's own numbering: their positions feed the Z-curve key (:1113)
            return fail(DG_ERR_INVALID, "%s: the field has %llu nodes, the grid %llu (already reduced?)", who, (unsigned long long)n_nodes, (unsigned long long)n);
        if (n_cells > grid_cells(g)) return fail(DG_ERR_INVALID, "%s: more cells than the grid has", who);
        StageClock clock;
        const auto t_start = clock.t0;
        double ms[5] = {0, 0, 0, 0, 0}, ms_callbacks = 0.0;
        int tie_path = 0;
        std::unique_ptr<dg_reduced_band> h(new dg_reduced_band());
        h->desc = *grid;
        DG_CUDA(cudaGetDevice(&h->device));
        CallStreamSync st;
        if (int rc = call_stream(st.s)) return rc;
        // ---- 1. upload the field and its rows; the predicate's mask per chunk, ANDed with v != DBL_MAX (the rows are checked by the cell flags)
        DevBuf<double> d_values;
        DevBuf<unsigned> d_cells;
        DevBuf<unsigned char> d_keep;
        DG_CUDA(d_values.alloc(n)); DG_CUDA(d_cells.alloc(32 * n_cells)); DG_CUDA(d_keep.alloc(n));
        DG_CUDA(cudaMemcpyAsync(d_values.p, nodes, n * sizeof(double), cudaMemcpyHostToDevice, st.s));
        if (n_cells) DG_CUDA(cudaMemcpyAsync(d_cells.p, cells, 32 * n_cells * sizeof(unsigned), cudaMemcpyHostToDevice, st.s));
        DeviceCallbacks cb;
        cb.node = pred; cb.nu = pu;
        if (int rc = run_device_callbacks(g, n, chunk_nodes, cb, d_values.p, d_keep.p, ms_callbacks, who, st.s)) return rc;
        ms[0] = clock.lap();
        // ---- 2.-5. reduceField over the uploaded rows
        if (int rc = reduce_device_field(g, d_values.p, n, DenseRows{d_cells.p, n_cells}, d_keep.p, flags, *h, ms, tie_path, clock, who, st.s)) return rc;
        reduced_timings(timings_ms, ms, tie_path, t_start);
        if (timings_ms) timings_ms[7] = ms_callbacks;
        *out = h.release();
        return DG_OK;
    });
}

int dg_reduced_band_sizes(const dg_reduced_band* h, uint64_t* n_nodes, uint64_t* n_cells)
{
    if (!h || !n_nodes || !n_cells) return fail(DG_ERR_INVALID, "dg_reduced_band_sizes: NULL argument");
    *n_nodes = h->n_nodes; *n_cells = h->n_cells;
    return DG_OK;
}

int dg_reduced_band_copy(const dg_reduced_band* h, double* nodes, uint32_t* cells, uint32_t* cell_map)
{
    if (!h) return fail(DG_ERR_INVALID, "dg_reduced_band_copy: handle is NULL");
    if ((!nodes && h->n_nodes) || (!cells && h->n_cells) || !cell_map) return fail(DG_ERR_INVALID, "dg_reduced_band_copy: NULL output");
    if (int rc = check_handle_device(h->device, "dg_reduced_band_copy")) return rc;
    if (h->n_nodes) DG_CUDA(cudaMemcpy(nodes, h->d_nodes.p, h->n_nodes * sizeof(double), cudaMemcpyDeviceToHost));
    if (h->n_cells) DG_CUDA(cudaMemcpy(cells, h->d_cells.p, 32 * h->n_cells * sizeof(unsigned), cudaMemcpyDeviceToHost));
    if (h->n_grid_cells) DG_CUDA(cudaMemcpy(cell_map, h->d_cell_map.p, h->n_grid_cells * sizeof(unsigned), cudaMemcpyDeviceToHost));
    return DG_OK;
}

int dg_reduced_band_destroy(dg_reduced_band* h)
{
    delete h;
    return DG_OK;
}

// dg_field_create of the handle's own arrays, device to device: K2's pack reads the handle's rows and nodes, the cell map is copied.  The
// library made the rows and the cell map, so dg_field_create's host checks have nothing to find.
int dg_field_create_reduced(const dg_reduced_band* h, dg_field** out)
{
    static const char* who = "dg_field_create_reduced";
    if (!out) return fail(DG_ERR_INVALID, "%s: out is NULL", who);
    *out = nullptr;
    if (!h) return fail(DG_ERR_INVALID, "%s: handle is NULL", who);
    dg_field* f = nullptr;
    if (int rc = field_common(&h->desc, out, f)) return rc;
    std::unique_ptr<dg_field> own(f);
    if (int rc = check_handle_device(h->device, who)) return rc;
    f->n_nodes = h->n_nodes; f->n_cells_kept = h->n_cells;
    DG_CUDA(f->d_cell_map.alloc(h->n_grid_cells));
    if (h->n_grid_cells) DG_CUDA(cudaMemcpyAsync(f->d_cell_map.p, h->d_cell_map.p, h->n_grid_cells * sizeof(unsigned), cudaMemcpyDeviceToDevice, nullptr));
    if (int rc = field_finish(f, h->d_nodes.p, h->d_cells.p, nullptr)) return rc;
    DG_CUDA(cudaDeviceSynchronize());
    *out = own.release();
    return DG_OK;
}

// ------------------------------------------------------------------------------------------------ K6: level sets (marching tetrahedra)
// The mesh stays on the field's device in the handle until dg_isosurface_copy[_device].
struct dg_isosurface {
    DevBuf<double> d_vertices;
    DevBuf<unsigned> d_triangles;
    uint64_t n_vertices = 0, n_triangles = 0;
    int device = 0;
};

// values, classify, scans, emit (k6_isosurface.cu); each stage ends with a synchronise.  Device memory: 8 B per lattice point of values,
// 7 B per point of edge flags, 1 B per lattice cell of counts, 1/8 B per point of chunk ranks, the tile arrays, one chunk of positions
// (24 B x min(Np, 2^24)), then 24 B per vertex and 12 B per triangle of output.
int dg_isosurface_create(const dg_field* f, double iso, uint32_t s, dg_isosurface** out, double* timings_ms)
{
    static const char* who = "dg_isosurface_create";
    return guarded(who, [&]() -> int {
        if (!out) return fail(DG_ERR_INVALID, "%s: out is NULL", who);
        *out = nullptr;
        if (!f) return fail(DG_ERR_INVALID, "%s: field is NULL", who);
        if (!std::isfinite(iso)) return fail(DG_ERR_INVALID, "%s: iso must be finite (got %g)", who, iso);
        if (s == 0 || s > K6_MAX_SUBDIVISIONS) return fail(DG_ERR_INVALID, "%s: subdivisions must be 1..%u (got %u)", who, K6_MAX_SUBDIVISIONS, s);
        uint64_t np = 0;
        const K6Lattice L = k6_lattice(f->dev.g, s, np);
        if (np >= (1ull << 31))
            return fail(DG_ERR_INVALID, "%s: the lattice of %llu points (%u x %u x %u) has 2^31 points or more; use fewer subdivisions", who,
                        (unsigned long long)np, L.np[0], L.np[1], L.np[2]);
        if (int rc = check_handle_device(f->device, who)) return rc;
        const uint64_t n_cells = (uint64_t)(L.np[0] - 1) * (L.np[1] - 1) * (L.np[2] - 1);
        const uint64_t n_edges = 7 * np, tile = k6_tile();
        StageClock clock;
        const auto t_start = clock.t0;
        const cudaStream_t st = nullptr;
        double ms[4] = {0, 0, 0, 0};
        std::unique_ptr<dg_isosurface> h(new dg_isosurface());
        h->device = f->device;
        // ---- values: lattice positions per chunk, K2 value-only
        DevBuf<double> d_values;
        DG_CUDA(d_values.alloc(np));
        {
            DevBuf<double> d_x;
            const uint64_t chunk = std::min<uint64_t>(np, K6_CHUNK);
            DG_CUDA(d_x.alloc(3 * chunk));
            for (uint64_t b = 0; b < np; b += chunk) {
                const uint64_t n = std::min(chunk, np - b);
                DG_LAUNCH(k6_launch_positions(L, b, n, d_x.p, st));
                DG_LAUNCH(k2_launch_interpolate(f->dev, d_x.p, n, d_values.p + b, nullptr, st));
            }
            DG_CUDA(cudaStreamSynchronize(st));
        }
        ms[0] = clock.lap();
        // ---- classify: triangle count per lattice cell, flags of the crossing edges (rounded up to whole 32-edge chunks, which emit reads)
        DevBuf<unsigned char> d_count, d_flags;
        DG_CUDA(d_count.alloc(n_cells));
        DG_CUDA(d_flags.alloc((n_edges + 31) / 32 * 32));
        DG_CUDA(cudaMemsetAsync(d_flags.p, 0, d_flags.bytes(), st));
        DG_LAUNCH(k6_launch_classify(L, d_values.p, iso, d_count.p, d_flags.p, st));
        DG_CUDA(cudaStreamSynchronize(st));
        ms[1] = clock.lap();
        // ---- scans: triangles per tile of cells, vertices per tile of edges; both totals must fit the uint32 indices of the output
        DevBuf<unsigned> d_tri_tile, d_edge_tile;
        DG_CUDA(d_tri_tile.alloc((n_cells + tile - 1) / tile));
        DG_CUDA(d_edge_tile.alloc((n_edges + tile - 1) / tile));
        uint64_t n_tri = 0, n_vert = 0;
        DG_LAUNCH(k6_scan_counts(d_count.p, n_cells, d_tri_tile.p, n_tri, st));
        DG_LAUNCH(k4_scan_flags(d_flags.p, n_edges, d_edge_tile.p, n_vert, st));
        if (n_vert >= (1ull << 32)) return fail(DG_ERR_INVALID, "%s: %llu vertices do not fit uint32 indices; use fewer subdivisions", who, (unsigned long long)n_vert);
        if (n_tri >= (1ull << 32)) return fail(DG_ERR_INVALID, "%s: %llu triangles do not fit uint32 counts; use fewer subdivisions", who, (unsigned long long)n_tri);
        ms[2] = clock.lap();
        // ---- emit: vertices at their ranks (and the rank of every 32-edge chunk), then the triangles
        if (n_vert) {
            DevBuf<unsigned> d_chunk;
            DG_CUDA(d_chunk.alloc((n_edges + 31) / 32));
            DG_CUDA(h->d_vertices.alloc(3 * n_vert));
            DG_CUDA(h->d_triangles.alloc(3 * n_tri));
            DG_LAUNCH(k6_launch_vertices(L, d_values.p, iso, d_flags.p, n_edges, d_edge_tile.p, d_chunk.p, h->d_vertices.p, st));
            DG_LAUNCH(k6_launch_triangles(L, d_values.p, iso, d_count.p, d_tri_tile.p, d_flags.p, d_chunk.p, h->d_triangles.p, st));
            DG_CUDA(cudaStreamSynchronize(st));
        }
        h->n_vertices = n_vert; h->n_triangles = n_tri;
        ms[3] = clock.lap();
        if (timings_ms) {
            for (int k = 0; k < 4; k++) timings_ms[k] = ms[k];
            timings_ms[4] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count();
        }
        *out = h.release();
        return DG_OK;
    });
}

int dg_isosurface_sizes(const dg_isosurface* s, uint64_t* n_vertices, uint64_t* n_triangles)
{
    if (!s || !n_vertices || !n_triangles) return fail(DG_ERR_INVALID, "dg_isosurface_sizes: NULL argument");
    *n_vertices = s->n_vertices; *n_triangles = s->n_triangles;
    return DG_OK;
}

int dg_isosurface_copy(const dg_isosurface* s, double* vertices, uint32_t* triangles)
{
    if (!s) return fail(DG_ERR_INVALID, "dg_isosurface_copy: handle is NULL");
    if ((!vertices && s->n_vertices) || (!triangles && s->n_triangles)) return fail(DG_ERR_INVALID, "dg_isosurface_copy: NULL output");
    if (int rc = check_handle_device(s->device, "dg_isosurface_copy")) return rc;
    if (s->n_vertices) DG_CUDA(cudaMemcpy(vertices, s->d_vertices.p, 3 * s->n_vertices * sizeof(double), cudaMemcpyDeviceToHost));
    if (s->n_triangles) DG_CUDA(cudaMemcpy(triangles, s->d_triangles.p, 3 * s->n_triangles * sizeof(unsigned), cudaMemcpyDeviceToHost));
    return DG_OK;
}

int dg_isosurface_copy_device(const dg_isosurface* s, double* d_vertices, uint32_t* d_triangles, void* stream)
{
    if (!s) return fail(DG_ERR_INVALID, "dg_isosurface_copy_device: handle is NULL");
    if ((!d_vertices && s->n_vertices) || (!d_triangles && s->n_triangles)) return fail(DG_ERR_INVALID, "dg_isosurface_copy_device: NULL output");
    if (int rc = check_handle_device(s->device, "dg_isosurface_copy_device")) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    if (s->n_vertices) DG_CUDA(cudaMemcpyAsync(d_vertices, s->d_vertices.p, 3 * s->n_vertices * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (s->n_triangles) DG_CUDA(cudaMemcpyAsync(d_triangles, s->d_triangles.p, 3 * s->n_triangles * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
    return DG_OK;
}

int dg_isosurface_destroy(dg_isosurface* s)
{
    delete s;
    return DG_OK;
}

// ------------------------------------------------------------------------------------------------ K7: ray casts
static int raycast_check(const dg_field* f, const void* o, const void* d, uint64_t n, double iso, double t_min, double t_max, const void* t_lo,
                         const void* t_hi, const void* status, const char* who)
{
    if (!f) return fail(DG_ERR_INVALID, "%s: field is NULL", who);
    if (n && (!o || !d || !t_lo || !t_hi || !status)) return fail(DG_ERR_INVALID, "%s: origins / directions / t_lo / t_hi / status is NULL", who);
    if (!std::isfinite(iso)) return fail(DG_ERR_INVALID, "%s: iso must be finite (got %g)", who, iso);
    if (std::isnan(t_min) || std::isnan(t_max)) return fail(DG_ERR_INVALID, "%s: t_min and t_max must not be NaN", who);
    if (t_min > t_max) return fail(DG_ERR_INVALID, "%s: t_min > t_max (%g > %g)", who, t_min, t_max);
    return check_handle_device(f->device, who);
}

int dg_field_raycast_device(const dg_field* f, const double* d_o, const double* d_d, uint64_t n, double iso, double t_min, double t_max,
                            double* d_t_lo, double* d_t_hi, int32_t* d_status, void* stream)
{
    if (int rc = raycast_check(f, d_o, d_d, n, iso, t_min, t_max, d_t_lo, d_t_hi, d_status, "dg_field_raycast_device")) return rc;
    if (n) DG_LAUNCH(k7_launch_raycast(f->dev, d_o, d_d, n, iso, t_min, t_max, d_t_lo, d_t_hi, d_status, (cudaStream_t)stream));
    return DG_OK;
}

// host arrays: chunks of 2^20 rays (64 MiB of device buffers)
int dg_field_raycast(const dg_field* f, const double* o, const double* d, uint64_t n, double iso, double t_min, double t_max, double* t_lo,
                     double* t_hi, int32_t* status)
{
    static const char* who = "dg_field_raycast";
    return guarded(who, [&]() -> int {
        if (int rc = raycast_check(f, o, d, n, iso, t_min, t_max, t_lo, t_hi, status, who)) return rc;
        if (n == 0) return DG_OK;
        return stage_on_device(n, std::min<uint64_t>(n, 1ull << 20), {{o, 3 * sizeof(double)}, {d, 3 * sizeof(double)}},
                               {{t_lo, sizeof(double)}, {t_hi, sizeof(double)}, {status, sizeof(int32_t)}},
                               [&](void* const* in, void* const* out, uint64_t, uint64_t c) -> int {
                                   DG_LAUNCH(k7_launch_raycast(f->dev, (const double*)in[0], (const double*)in[1], c, iso, t_min, t_max, (double*)out[0],
                                                               (double*)out[1], (int32_t*)out[2], nullptr));
                                   return DG_OK;
                               });
    });
}

// ------------------------------------------------------------------------------------------------ K9: ray casts on a mesh
static int mesh_raycast_check(const dg_mesh* m, const void* o, const void* d, uint64_t n, double t_min, double t_max, const void* t,
                              const void* id, const void* status, const char* who)
{
    if (int rc = mesh_usable(m, who)) return rc;
    if (n && (!o || !d || !t || !id || !status)) return fail(DG_ERR_INVALID, "%s: origins / directions / t / triangle_id / status is NULL", who);
    if (std::isnan(t_min) || std::isnan(t_max)) return fail(DG_ERR_INVALID, "%s: t_min and t_max must not be NaN", who);
    if (t_min > t_max) return fail(DG_ERR_INVALID, "%s: t_min > t_max (%g > %g)", who, t_min, t_max);
    if (m->dev.stack_depth > K9_MAX_STACK) return fail(DG_ERR_INVALID, "%s: tree too deep for the ray walk", who);
    return check_handle_device(m->device, who);
}

static int mesh_raycast_launch(const dg_mesh* m, const double* d_o, const double* d_d, uint64_t n, double t_min, double t_max, double* d_t,
                               int32_t* d_id, double* d_bary, int32_t* d_status, cudaStream_t st, const char* who)
{
    const WindDev* wd = nullptr;
    if (int rc = winding_dev(m, wd, who)) return rc;
    DG_LAUNCH(k9_launch_mesh_raycast(m->dev, *wd, d_o, d_d, n, t_min, t_max, d_t, d_id, d_bary, d_status, st));
    return DG_OK;
}

int dg_mesh_raycast_device(const dg_mesh* m, const double* d_o, const double* d_d, uint64_t n, double t_min, double t_max, double* d_t,
                           int32_t* d_id, double* d_bary, int32_t* d_status, void* stream)
{
    static const char* who = "dg_mesh_raycast_device";
    if (int rc = mesh_raycast_check(m, d_o, d_d, n, t_min, t_max, d_t, d_id, d_status, who)) return rc;
    if (n == 0) return DG_OK;
    return mesh_raycast_launch(m, d_o, d_d, n, t_min, t_max, d_t, d_id, d_bary, d_status, (cudaStream_t)stream, who);
}

// host arrays: chunks of 2^20 rays
int dg_mesh_raycast(const dg_mesh* m, const double* o, const double* d, uint64_t n, double t_min, double t_max, double* t, int32_t* id,
                    double* bary, int32_t* status)
{
    static const char* who = "dg_mesh_raycast";
    return guarded(who, [&]() -> int {
        if (int rc = mesh_raycast_check(m, o, d, n, t_min, t_max, t, id, status, who)) return rc;
        if (n == 0) return DG_OK;
        return stage_on_device(n, std::min<uint64_t>(n, 1ull << 20), {{o, 3 * sizeof(double)}, {d, 3 * sizeof(double)}},
                               {{t, sizeof(double)}, {id, sizeof(int32_t)}, {status, sizeof(int32_t)}, {bary, 3 * sizeof(double)}},
                               [&](void* const* in, void* const* out, uint64_t, uint64_t c) {
                                   return mesh_raycast_launch(m, (const double*)in[0], (const double*)in[1], c, t_min, t_max, (double*)out[0],
                                                              (int32_t*)out[1], (double*)out[3], (int32_t*)out[2], nullptr, who);
                               });
    });
}

int dg_obj_read(const char* path, double** vertices, uint64_t* n_vertices, uint32_t** triangles, uint64_t* n_triangles)
{
    if (!path || !vertices || !n_vertices || !triangles || !n_triangles) return fail(DG_ERR_INVALID, "dg_obj_read: NULL argument");
    *vertices = nullptr; *triangles = nullptr; *n_vertices = 0; *n_triangles = 0;
    ObjData d; std::string err;
    if (!read_obj(path, d, err)) return fail(err.rfind("Cannot open", 0) == 0 || err.rfind("short read", 0) == 0 ? DG_ERR_IO : DG_ERR_INVALID, "dg_obj_read: %s", err.c_str());
    double* v = static_cast<double*>(std::malloc(std::max<size_t>(1, d.vertices.size() * sizeof(double))));
    uint32_t* f = static_cast<uint32_t*>(std::malloc(std::max<size_t>(1, d.faces.size() * sizeof(uint32_t))));
    if (!v || !f) { std::free(v); std::free(f); return fail(DG_ERR_NOMEM, "dg_obj_read: out of host memory"); }
    if (!d.vertices.empty()) std::memcpy(v, d.vertices.data(), d.vertices.size() * sizeof(double));
    if (!d.faces.empty()) std::memcpy(f, d.faces.data(), d.faces.size() * sizeof(uint32_t));
    *vertices = v; *triangles = f; *n_vertices = d.vertices.size() / 3; *n_triangles = d.faces.size() / 3;
    return DG_OK;
}

void dg_obj_free(double* vertices, uint32_t* triangles)
{
    std::free(vertices); std::free(triangles);
}

}  // extern "C"
