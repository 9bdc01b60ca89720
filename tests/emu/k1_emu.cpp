// tests/emu/k1_emu.cpp -- TEST INFRASTRUCTURE: the product's K1 translation unit (discregrid_b200/csrc/k1_sdf.cu: traversal kernels AND
// their launchers) compiled for the CPU through tests/emu/cuda_emu.h, plus a small extern "C" surface for tests/test_k1_emulated.py.
// "Device" pointers are host pointers; the mesh is built by the product's host builder exactly as dg_mesh_create does.
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/k1_sdf.cu"

namespace dgb {
namespace {
alignas(16) unsigned char k1_smem[1 << 18];          // the one block that runs at a time
}
}  // namespace dgb

using namespace dgb;

namespace {
struct EmuMesh {
    HostBvh host;
    std::vector<float4> nodes_f;
    DeviceBvh dev;
};

bool to_grid(const double* gd /*mn3 mx3 cell3 inv3*/, const uint32_t* res, GridDev& g)
{
    for (int k = 0; k < 3; k++) { g.mn[k] = gd[k]; g.mx[k] = gd[3 + k]; g.cell[k] = gd[6 + k]; g.inv[k] = gd[9 + k]; g.n[k] = res[k]; if (!res[k]) return false; }
    const unsigned nx = g.n[0], ny = g.n[1], nz = g.n[2];
    g.nv = (nx + 1) * (ny + 1) * (nz + 1);
    g.ne_x = nx * (ny + 1) * (nz + 1); g.ne_y = (nx + 1) * ny * (nz + 1); g.ne_z = (nx + 1) * (ny + 1) * nz;
    return true;
}
}  // namespace

extern "C" {

void* emu_mesh_create(const double* V, uint64_t nV, const uint32_t* F, uint64_t nT)
{
    auto* m = new EmuMesh();
    const char* err = "";
    if (!build_host_bvh(V, nV, F, nT, m->host, &err, true)) { std::fprintf(stderr, "emu_mesh_create: %s\n", err); delete m; return nullptr; }
    // the interleaved fp32 node record, as dg_mesh_create lays it out
    m->nodes_f.assign((size_t)nT * K1_NODEF_STRIDE, make_float4(0.f, 0.f, 0.f, 0.f));
    pack_node_records(m->host, K1_NODEF_STRIDE, reinterpret_cast<float*>(m->nodes_f.data()));
    DeviceBvh& d = m->dev;
    d.spheres = m->host.spheres.data(); d.leaves = m->host.leaves.data(); d.normals = m->host.normals.data();
    d.leaves_f = m->host.leaves_f.data();
    d.nodes_f = m->nodes_f.data();
    for (int k = 0; k < 3; k++) d.ctr[k] = m->host.center[k];
    d.half_extent = (float)m->host.half_extent * 1.0000002f;
    d.n_tri = (int)nT;
    d.stack_depth = m->host.max_depth > 1 ? m->host.max_depth - 1 : 1;
    return m;
}
void emu_mesh_destroy(void* h) { delete (EmuMesh*)h; }

int emu_sample_sdf(void* h, const double* gd, const uint32_t* res, double sign, uint64_t l_begin, uint64_t l_end, double* out)
{
    GridDev g; if (!to_grid(gd, res, g)) return -1;
    return (int)k1_launch_sample_nodes(((EmuMesh*)h)->dev, g, sign, l_begin, l_end - l_begin, out, nullptr);
}
int emu_sample_interleaved(void* h, const double* gd, const uint32_t* res, double sign, uint32_t part, uint32_t n_parts, double* slots, uint64_t* slot_elems)
{
    GridDev g; if (!to_grid(gd, res, g)) return -1;
    InterleavedLayout L; if (!k1_interleaved_layout(g, n_parts, L)) return -2;
    *slot_elems = L.slot_elems;
    if (!slots) return 0;
    return (int)k1_launch_sample_interleaved(((EmuMesh*)h)->dev, g, sign, L, part, slots + (size_t)part * L.slot_elems, nullptr);
}
int emu_unpack_interleaved(const double* gd, const uint32_t* res, uint32_t n_parts, const double* slots, double* nodes)
{
    GridDev g; if (!to_grid(gd, res, g)) return -1;
    InterleavedLayout L; if (!k1_interleaved_layout(g, n_parts, L)) return -2;
    return (int)k1_launch_unpack_interleaved(g, L, slots, nodes, nullptr);
}
int emu_sample_slab(void* h, const double* gd, const uint32_t* res, double sign, const uint32_t* plane_begin, const uint32_t* plane_end, double* full)
{
    GridDev g; if (!to_grid(gd, res, g)) return -1;
    return (int)k1_launch_sample_slab(((EmuMesh*)h)->dev, g, sign, plane_begin, plane_end, full, nullptr);
}
int emu_mesh_distance(void* h, const double* pts, uint64_t n, int is_signed, double* dist, double* nearp, int32_t* ent, int32_t* tri)
{
    return (int)k1_launch_distance(((EmuMesh*)h)->dev, pts, n, is_signed, dist, nearp, ent, tri, nullptr);
}
int emu_node_positions(const double* gd, const uint32_t* res, uint64_t l_begin, uint64_t l_end, double* x)
{
    GridDev g; if (!to_grid(gd, res, g)) return -1;
    return (int)k1_launch_node_positions(g, l_begin, l_end - l_begin, x, nullptr);
}
int emu_build_cells(const double* gd, const uint32_t* res, uint64_t c_begin, uint64_t c_end, uint32_t* cells)
{
    GridDev g; if (!to_grid(gd, res, g)) return -1;
    return (int)k1_launch_build_cells(g, c_begin, c_end - c_begin, cells, nullptr);
}
void emu_counters(unsigned long long* out /*32*/, int reset) { for (int i = 0; i < 32; i++) { out[i] = dg_emu::g_counters[i]; if (reset) dg_emu::g_counters[i] = 0; } }
// block ids in the order the last sampling launches ran them (cleared by reading)
uint64_t emu_block_trace(uint32_t* out, uint64_t cap) { const uint64_t n = dg_emu::g_block_trace.size(); for (uint64_t i = 0; i < n && i < cap; i++) out[i] = dg_emu::g_block_trace[i]; dg_emu::g_block_trace.clear(); return n; }

}  // extern "C"
