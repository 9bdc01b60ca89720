// Launch interface of the K2 kernels (k2_interp.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "dg_device.cuh"

namespace dgb {

constexpr int K2_THREADS = 128;

struct FieldDev {                   // device-resident field (see k2_interp.cu for the layout rationale)
    GridDev g;
    const double* packed = nullptr;     // [max(1, n_cells_kept)][32], 256-byte aligned blocks
    const unsigned* cell_map = nullptr; // [nx*ny*nz] or nullptr (identity)
    const double2* tab = nullptr;       // [nx + ny + nz] per-axis (c0, c1)
};

cudaError_t k2_launch_pack(const GridDev& g, const double* d_nodes, const unsigned* d_cells, uint64_t n_cells_kept,
                           double* d_packed, cudaStream_t stream);
cudaError_t k2_launch_axis_tables(const GridDev& g, double2* d_tab, cudaStream_t stream);
// d_grad nullable (value only); d_hess nullable, and when given d_grad must be too: the Hessian mode, hess[n][3][3] row-major
cudaError_t k2_launch_interpolate(const FieldDev& f, const double* d_x, uint64_t n, double* d_phi, double* d_grad,
                                  cudaStream_t stream, double* d_hess = nullptr);
cudaError_t k2_launch_shape_functions(const double* d_xi, uint64_t n, double* d_N, double* d_dN, cudaStream_t stream);

}  // namespace dgb
