// tests/emu/k9_emu.cpp -- TEST INFRASTRUCTURE: the product's mesh ray-cast kernel (discregrid_b200/csrc/k9_mesh_raycast.cu) compiled for the
// CPU through tests/emu/cuda_emu.h.  Part of build/bin/libdgemu.so as it is; with K9_EMU_SURFACE it also exports a small extern "C" surface
// for tests/test_mesh_raycast_emulated.py and tools/mesh_raycast_bench.py (build/bin/libk9emu.so, and libk9emu_nocull.so with K9_CULL=0).
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/k9_mesh_raycast.cu"

#if K9_EMU_SURFACE
using namespace dgb;

namespace {
// a mesh's records as dg_mesh_create and the first winding-number call leave them on the device (here: host memory)
struct EmuMeshRay {
    HostBvh host;
    RawVec<float4> nodes_f;
    RawVec<WindLeaf> wind_leaves;
    RawVec<WindClusterPair> wind_clusters;
    DeviceBvh dev;
    WindDev wind;
};
}  // namespace

extern "C" {

void* emu_k9_create(const double* V, uint64_t nV, const uint32_t* F, uint64_t nT)
{
    auto* m = new EmuMeshRay();
    const char* err = "";
    if (!build_host_bvh(V, nV, F, nT, m->host, &err, true)) { std::fprintf(stderr, "emu_k9_create: %s\n", err); delete m; return nullptr; }
    m->nodes_f.resize(nT * K1_NODEF_STRIDE);
    pack_node_records(m->host, K1_NODEF_STRIDE, reinterpret_cast<float*>(m->nodes_f.data()));
    build_winding_records(m->host, m->wind_leaves, m->wind_clusters);
    m->dev.leaves = m->host.leaves.data();
    m->dev.nodes_f = m->nodes_f.data();
    for (int d = 0; d < 3; d++) m->dev.ctr[d] = m->host.center[d];
    m->dev.half_extent = (float)m->host.half_extent * 1.0000002f;       // rounded up, as dg_mesh_create
    m->dev.n_tri = (int)nT;
    m->dev.stack_depth = m->host.max_depth > 1 ? m->host.max_depth - 1 : 1;
    m->wind.leaves = m->wind_leaves.data(); m->wind.clusters = m->wind_clusters.data();
    m->wind.n_tri = (int)nT; m->wind.stack_depth = m->dev.stack_depth;
    return m;
}
void emu_k9_destroy(void* h) { delete (EmuMeshRay*)h; }
int emu_k9_cull(void) { return K9_CULL; }
int emu_k9_raycast(void* h, const double* o, const double* d, uint64_t n, double t_min, double t_max, double* t, int32_t* id, double* bary,
                   int32_t* status)
{
    auto* m = (EmuMeshRay*)h;
    return (int)k9_launch_mesh_raycast(m->dev, m->wind, o, d, n, t_min, t_max, t, id, bary, status, nullptr);
}
// counters since the last reset: boxes tested, triangles tested, rays
void emu_k9_counters(unsigned long long* out)
{
    out[0] = dg_emu::g_counters[8]; out[1] = dg_emu::g_counters[9]; out[2] = dg_emu::g_counters[10];
}
void emu_k9_counters_reset(void) { dg_emu::g_counters[8] = dg_emu::g_counters[9] = dg_emu::g_counters[10] = 0; }

}  // extern "C"
#endif
