// tests/emu/k5_emu.cpp -- TEST INFRASTRUCTURE: the product's K5 translation unit (discregrid_b200/csrc/k5_winding.cu: k5_atan2, the records,
// the walk and the launchers) compiled for the CPU through tests/emu/cuda_emu.h, plus a small extern "C" surface for
// tests/test_winding_emulated.py.  Linked alone into build/bin/libk5emu.so and, with the other emulated TUs, into build/bin/libdgemu.so.
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/k5_winding.cu"

namespace dgb {
uint2 k5_stack[K5_MAX_STACK * K5_THREADS];          // the one block that runs at a time
}  // namespace dgb

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

}  // extern "C"
