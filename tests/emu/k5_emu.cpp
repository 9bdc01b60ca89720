// tests/emu/k5_emu.cpp -- TEST INFRASTRUCTURE: the product's K5 translation unit (discregrid_b200/csrc/k5_winding.cu: k5_atan2, the records,
// the walk and the launchers) compiled for the CPU through tests/emu/cuda_emu.h, plus a small extern "C" surface for
// tests/test_winding_emulated.py.  Linked alone into build/bin/libk5emu.so and, with the other emulated TUs, into build/bin/libdgemu.so.
//
// The walk's stack here is a static array of K5_MAX_STACK entries per lane, while the device gets exactly the dynamic shared memory the
// launcher asks for (stack_depth x K5_THREADS x 8 B).  So that a stack_depth too small for some tree cannot pass here unnoticed, every
// launch of this TU fills the entries past the launcher's shared-memory size with a canary first and checks them afterwards; a changed
// canary fails the launch (cudaErrorLaunchFailure, as the device's out-of-bounds shared-memory write would).
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/dg_launch.h"
#include "../../discregrid_b200/csrc/k5_winding.h"

namespace dgb {
uint2 k5_stack[K5_MAX_STACK * K5_THREADS];          // the one block that runs at a time

namespace k5_emu_guard {
constexpr size_t CAPACITY = sizeof(k5_stack) / sizeof(uint2);
constexpr unsigned CANARY_X = 0xC0DEC0DEu, CANARY_Y = 0xFEEDFACEu;   // no walk entry: both halves of one are < 2^25
inline cudaError_t g_status = cudaSuccess;

// the launch's first stack entry the device would not have
inline size_t first_guarded(size_t smem) { return smem / sizeof(uint2); }

inline bool fill(size_t smem)
{
    if (first_guarded(smem) > CAPACITY) {
        std::fprintf(stderr, "k5_emu: the launch asks for %zu B of shared memory, more than the emulated stack holds\n", smem);
        return false;
    }
    for (size_t i = first_guarded(smem); i < CAPACITY; i++) k5_stack[i] = make_uint2(CANARY_X, CANARY_Y);
    return true;
}

inline bool intact(size_t smem)
{
    for (size_t i = first_guarded(smem); i < CAPACITY; i++)
        if (k5_stack[i].x != CANARY_X || k5_stack[i].y != CANARY_Y) {
            std::fprintf(stderr, "k5_emu: stack overrun: entry %zu (depth %zu of lane %zu) written past the %zu B of shared memory of the launch\n",
                         i, i / K5_THREADS, i % K5_THREADS, smem);
            return false;
        }
    return true;
}

template <class F> inline void launch(unsigned grid, unsigned block, size_t smem, const F& body)
{
    if (!fill(smem)) { g_status = cudaErrorInvalidValue; return; }
    dg_emu::launch(grid, block, smem, body);
    if (!intact(smem)) g_status = cudaErrorLaunchFailure;
}

inline cudaError_t after_launch() { const cudaError_t e = g_status; g_status = cudaSuccess; return e; }
}  // namespace k5_emu_guard
}  // namespace dgb

#undef DG_KERNEL_LAUNCH
#undef DG_AFTER_LAUNCH
#define DG_KERNEL_LAUNCH(kernel, grid, block, smem, stream, ...) \
    dgb::k5_emu_guard::launch((unsigned)(grid), (unsigned)(block), (size_t)(smem), [&]() { kernel(__VA_ARGS__); })
#define DG_AFTER_LAUNCH() dgb::k5_emu_guard::after_launch()
#include "../../discregrid_b200/csrc/k5_winding.cu"

using namespace dgb;

namespace {
struct EmuWinding {
    HostBvh host;
    RawVec<WindLeaf> leaves;
    RawVec<WindClusterPair> clusters;
    WindDev dev;
};
}  // namespace

extern "C" {

void emu_k5_atan2(const double* y, const double* x, uint64_t n, double* out)
{
    for (uint64_t i = 0; i < n; i++) out[i] = k5_atan2_host(y[i], x[i]);
}

void* emu_winding_create(const double* V, uint64_t nV, const uint32_t* F, uint64_t nT)
{
    auto* m = new EmuWinding();
    const char* err = "";
    if (!build_host_bvh(V, nV, F, nT, m->host, &err, false)) { std::fprintf(stderr, "emu_winding_create: %s\n", err); delete m; return nullptr; }
    build_winding_records(m->host, m->leaves, m->clusters);
    m->dev.leaves = m->leaves.data(); m->dev.clusters = m->clusters.data();
    m->dev.n_tri = (int)nT;
    m->dev.stack_depth = m->host.max_depth > 1 ? m->host.max_depth - 1 : 1;
    return m;
}
void emu_winding_destroy(void* h) { delete (EmuWinding*)h; }
int emu_winding_stack_depth(void* h) { return ((EmuWinding*)h)->dev.stack_depth; }
// leaf position -> triangle id; leaves[T][9]; clusters[T][2][16] (p, n, M, r of the left then the right child)
void emu_winding_records(void* h, int32_t* order, double* leaves, double* clusters)
{
    auto* m = (EmuWinding*)h;
    const uint64_t T = m->host.n_triangles;
    if (order) std::memcpy(order, m->host.order.data(), T * sizeof(int32_t));
    if (leaves) std::memcpy(leaves, m->leaves.data(), T * sizeof(WindLeaf));
    if (clusters) std::memcpy(clusters, m->clusters.data(), T * sizeof(WindClusterPair));
}
int emu_winding_number(void* h, const double* pts, uint64_t n, double beta, double* w)
{
    return (int)k5_launch_winding(((EmuWinding*)h)->dev, pts, n, beta, w, nullptr);
}
// the same launch with a stack of `stack_depth` entries per lane instead of the tree's own: a depth that is too small must fail the launch
int emu_winding_number_with_depth(void* h, const double* pts, uint64_t n, double beta, int stack_depth, double* w)
{
    WindDev d = ((EmuWinding*)h)->dev;
    d.stack_depth = stack_depth;
    return (int)k5_launch_winding(d, pts, n, beta, w, nullptr);
}

}  // extern "C"
