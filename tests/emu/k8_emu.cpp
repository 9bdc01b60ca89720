// tests/emu/k8_emu.cpp -- TEST INFRASTRUCTURE: the product's K8 translation unit (discregrid_b200/csrc/k8_refit.cu: the refit passes and their
// launcher) compiled for the CPU through tests/emu/cuda_emu.h, plus a small extern "C" surface for tests/test_refit_emulated.py.  Linked with
// k5_emu.cpp into build/bin/libk8emu.so and, with the other emulated TUs, into build/bin/libdgemu.so.
#define DG_EMU 1
#include "cuda_emu.h"

// __reduce_max_sync (sm_80+ redux.sync.max.u32) from the emulation's ballot: the maximum's bits from the top, one ballot per bit
inline unsigned __reduce_max_sync(unsigned mask, unsigned v)
{
    unsigned r = 0;
    for (int bit = 31; bit >= 0; bit--) {
        const unsigned cand = r | (1u << bit);
        if (__ballot_sync(mask, v >= cand) != 0u) r = cand;
    }
    return r;
}

#include "../../discregrid_b200/csrc/k8_refit.cu"
#include "../../discregrid_b200/csrc/k1_sdf.h"

using namespace dgb;

namespace {
// a mesh's records as dg_mesh holds them on the device (here: host memory), with the refit's tables and scratch
struct EmuRefit {
    HostBvh host;
    RefitTopoHost topo;
    RawVec<SpherePair> spheres;
    RawVec<LeafRecord> leaves;
    RawVec<LeafF> leaves_f;
    RawVec<PseudoNormals> normals;
    RawVec<float4> nodes_f;
    RawVec<WindLeaf> wind_leaves;
    RawVec<WindClusterPair> wind_clusters;
    double bounds[5] = {0, 0, 0, 0, 0};
    std::vector<uint32_t> F;
    std::vector<double> V;
    std::vector<RefitSums> sums;
    std::vector<RefitBounds> part;
    std::vector<double> d_bounds, pn_tri, angle, pn_vert, pn_edge;
};
}  // namespace

extern "C" {

void emu_k8_acos(const double* x, uint64_t n, double* out)
{
    for (uint64_t i = 0; i < n; i++) out[i] = k8_acos_host(x[i]);
}

int emu_refit_nodef_stride(void) { return K1_NODEF_STRIDE; }

// dg_mesh_create's records (host build, with the fp32 leaf shadows and the winding records)
void* emu_refit_create(const double* V, uint64_t nV, const uint32_t* F, uint64_t nT)
{
    auto* m = new EmuRefit();
    const char* err = "";
    if (!build_host_bvh(V, nV, F, nT, m->host, &err, true)) { std::fprintf(stderr, "emu_refit_create: %s\n", err); delete m; return nullptr; }
    m->spheres = m->host.spheres; m->leaves = m->host.leaves; m->leaves_f = m->host.leaves_f; m->normals = m->host.normals;
    m->nodes_f.resize(nT * K1_NODEF_STRIDE);
    pack_node_records(m->host, K1_NODEF_STRIDE, reinterpret_cast<float*>(m->nodes_f.data()));
    build_winding_records(m->host, m->wind_leaves, m->wind_clusters);
    for (int d = 0; d < 3; d++) m->bounds[d] = m->host.center[d];
    m->bounds[3] = m->host.half_extent; m->bounds[4] = 1.0;
    m->F.assign(F, F + 3 * nT);
    k8_build_topology(m->host, m->topo);
    m->V.resize(3 * nV); m->sums.resize(nT); m->part.resize(k8_bounds_entries(nV)); m->d_bounds.resize(5);
    m->pn_tri.resize(3 * nT); m->angle.resize(3 * nT); m->pn_vert.resize(3 * nV); m->pn_edge.resize(9 * nT);
    return m;
}
void emu_refit_destroy(void* h) { delete (EmuRefit*)h; }

// every record recomputed from V (the count of the build); with_k5 = 0 leaves the winding records as they are
int emu_refit(void* h, const double* V, int with_k5)
{
    auto* m = (EmuRefit*)h;
    std::memcpy(m->V.data(), V, m->V.size() * sizeof(double));
    RefitDev r;
    r.V = m->V.data(); r.n_vertices = m->host.n_vertices; r.n_tri = (int)m->host.n_triangles; r.levels = m->host.max_depth;
    r.F = m->F.data(); r.f_leaf = m->topo.f_leaf.data(); r.order = m->host.order.data(); r.inc_begin = m->topo.inc_begin.data();
    r.inc = m->topo.inc.data(); r.nodes = m->topo.nodes.data();
    r.sums = m->sums.data(); r.part = m->part.data(); r.bounds = m->d_bounds.data();
    r.pn_tri = m->pn_tri.data(); r.angle = m->angle.data(); r.pn_vert = m->pn_vert.data(); r.pn_edge = m->pn_edge.data();
    r.spheres = m->spheres.data(); r.leaves = m->leaves.data(); r.leaves_f = m->leaves_f.data(); r.normals = m->normals.data();
    r.nodes_f = m->nodes_f.data(); r.nodef_stride = K1_NODEF_STRIDE;
    if (with_k5) { r.wind_leaves = m->wind_leaves.data(); r.wind_clusters = m->wind_clusters.data(); }
    const cudaError_t e = k8_launch_refit(r, m->topo.level_begin, true, nullptr);
    if (e != cudaSuccess) return (int)e;
    std::memcpy(m->bounds, m->d_bounds.data(), sizeof m->bounds);
    return 0;
}

// only the winding records, as the library builds them at their first use after a refit
int emu_refit_winding_only(void* h)
{
    auto* m = (EmuRefit*)h;
    RefitDev r;
    r.V = m->V.data(); r.n_vertices = m->host.n_vertices; r.n_tri = (int)m->host.n_triangles; r.levels = m->host.max_depth;
    r.F = m->F.data(); r.f_leaf = m->topo.f_leaf.data(); r.order = m->host.order.data(); r.inc_begin = m->topo.inc_begin.data();
    r.inc = m->topo.inc.data(); r.nodes = m->topo.nodes.data(); r.sums = m->sums.data();
    r.wind_leaves = m->wind_leaves.data(); r.wind_clusters = m->wind_clusters.data();
    return (int)k8_launch_refit(r, m->topo.level_begin, false, nullptr);
}

// order[T]; leaves[T][16] (LeafRecord bytes); leaves_f[T][16] floats; spheres[T][8]; nodes_f[T][4 * stride] floats; normals[T][21];
// bounds[5] (centre, half extent, finite); wind_leaves[T][9]; wind_clusters[T][2][16].  Any pointer may be NULL.
void emu_refit_records(void* h, int32_t* order, void* leaves, float* leaves_f, double* spheres, float* nodes_f, double* normals, double* bounds,
                       double* wind_leaves, double* wind_clusters)
{
    auto* m = (EmuRefit*)h;
    const uint64_t T = m->host.n_triangles;
    if (order) std::memcpy(order, m->host.order.data(), T * sizeof(int32_t));
    if (leaves) std::memcpy(leaves, m->leaves.data(), T * sizeof(LeafRecord));
    if (leaves_f) std::memcpy(leaves_f, m->leaves_f.data(), T * sizeof(LeafF));
    if (spheres) std::memcpy(spheres, m->spheres.data(), T * sizeof(SpherePair));
    if (nodes_f) std::memcpy(nodes_f, m->nodes_f.data(), m->nodes_f.size() * sizeof(float4));
    if (normals) std::memcpy(normals, m->normals.data(), T * sizeof(PseudoNormals));
    if (bounds) std::memcpy(bounds, m->bounds, sizeof m->bounds);
    if (wind_leaves) std::memcpy(wind_leaves, m->wind_leaves.data(), T * sizeof(WindLeaf));
    if (wind_clusters) std::memcpy(wind_clusters, m->wind_clusters.data(), T * sizeof(WindClusterPair));
}

}  // extern "C"
