// tests/emu/k3_emu.cpp -- TEST INFRASTRUCTURE: the product's K3 translation unit (k3_density.cu) compiled for the CPU, and the
// extern "C" surface of the emulated field / interpolate / density-map path for tests/test_k23_emulated.py.
#define DG_EMU 1
#include "cuda_emu.h"
#include "../../discregrid_b200/csrc/k3_density.cu"
#include "../../discregrid_b200/csrc/k2_interp.h"

using namespace dgb;

namespace {
struct EmuField {
    FieldDev dev;
    double* packed = nullptr;
    std::vector<double2> tab;
    std::vector<unsigned> cell_map;
    double coeff_max = 0.0;
    ~EmuField() { std::free(packed); }
};
bool to_grid(const double* gd, const uint32_t* res, GridDev& g)
{
    for (int k = 0; k < 3; k++) { g.mn[k] = gd[k]; g.mx[k] = gd[3 + k]; g.cell[k] = gd[6 + k]; g.inv[k] = gd[9 + k]; g.n[k] = res[k]; if (!res[k]) return false; }
    const unsigned nx = g.n[0], ny = g.n[1], nz = g.n[2];
    g.nv = (nx + 1) * (ny + 1) * (nz + 1);
    g.ne_x = nx * (ny + 1) * (nz + 1); g.ne_y = (nx + 1) * ny * (nz + 1); g.ne_z = (nx + 1) * (ny + 1) * nz;
    return true;
}
}  // namespace

extern "C" {

// what dg_field_create does: packed 256-byte cell blocks (pack_cells_kernel), per-axis tables (axis_tables_kernel), cell map
void* emu_field_create(const double* gd, const uint32_t* res, const double* nodes, const uint32_t* cells /*nullable*/, uint64_t n_cells_kept,
                       const uint32_t* cell_map /*nullable*/)
{
    auto* f = new EmuField();
    if (!to_grid(gd, res, f->dev.g)) { delete f; return nullptr; }
    const uint64_t n_cells = (uint64_t)res[0] * res[1] * res[2];
    const size_t blocks = n_cells_kept ? n_cells_kept : 1;
    f->packed = static_cast<double*>(std::aligned_alloc(256, blocks * 256));
    std::memset(f->packed, 0, blocks * 256);
    f->tab.resize(res[0] + res[1] + res[2]);
    if (cell_map) f->cell_map.assign(cell_map, cell_map + n_cells);
    if (k2_launch_pack(f->dev.g, nodes, cells, n_cells_kept, f->packed, nullptr) != cudaSuccess) { delete f; return nullptr; }
    if (k2_launch_axis_tables(f->dev.g, f->tab.data(), nullptr) != cudaSuccess) { delete f; return nullptr; }
    if (k3_coeff_max(f->packed, 32 * n_cells_kept, &f->coeff_max, nullptr) != cudaSuccess) { delete f; return nullptr; }
    f->dev.packed = f->packed; f->dev.tab = f->tab.data(); f->dev.cell_map = cell_map ? f->cell_map.data() : nullptr;
    return f;
}
void emu_field_destroy(void* h) { delete (EmuField*)h; }
int emu_interpolate(void* h, const double* x, uint64_t n, double* phi, double* grad)
{
    return (int)k2_launch_interpolate(((EmuField*)h)->dev, x, n, phi, grad, nullptr);
}
int emu_shape_functions(const double* xi, uint64_t n, double* N, double* dN) { return (int)k2_launch_shape_functions(xi, n, N, dN, nullptr); }
int emu_density_map(void* h, double hh, double rho0, int no_reduction, uint64_t l_begin, uint64_t l_end, double* out)
{
    const EmuField* f = (EmuField*)h;
    return (int)k3_launch_density(f->dev, f->coeff_max, hh, rho0, no_reduction, l_begin, l_end - l_begin, out, nullptr);
}

}  // extern "C"
