// Launch interface of the K3 kernel (k3_density.cu): GenerateDensityMap's per-node function.
#pragma once
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>
#include "k2_interp.h"

namespace dgb {
// GenerateDensityMap's cell_diag = cellSize().norm() (main.cpp:117): the value K3's predicate uses, and the SDF field's reduceField with it
double k3_cell_diag(const GridDev& g);
// max |c| over the n packed coefficients c != DBL_MAX, +inf if one of them is NaN or +-inf; synchronises `stream`
cudaError_t k3_coeff_max(const double* d_packed, uint64_t n, double* out, cudaStream_t stream);
// coeff_max: k3_coeff_max of f's packed coefficients (it decides whether points outside the kernel support may be skipped)
cudaError_t k3_launch_density(const FieldDev& f, double coeff_max, double h, double rho0, int no_reduction, uint64_t l_begin,
                              uint64_t count, double* d_out, cudaStream_t stream);
// the volume map (contract in k3_density.cu): scale * the quadrature of the inside indicator over the ball of radius h, per node.
// h finite and > 0, scale finite: the caller's to check
cudaError_t k3_launch_volume(const FieldDev& f, double h, double scale, int no_reduction, uint64_t l_begin, uint64_t count, double* d_out,
                             cudaStream_t stream);
// the volume map's quadrature points inside the ball of radius h, in quadrature order: (xi.x, xi.y, xi.z, wijk) per point
std::vector<double> k3_volume_points(double h);
}
