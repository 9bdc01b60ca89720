// Launch interface of K7 (k7_raycast.cu): first crossings of a level set along rays.  Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "k2_interp.h"

namespace dgb {

constexpr int K7_THREADS = 128;
constexpr int K7_DEPTH = 5;                  // D of the contract: depth of the Bernstein descent below a segment

// per ray i: origin o[3 i..], direction d[3 i..]; t_lo[i], t_hi[i], status[i] as in the contract of k7_raycast.cu.  iso finite, t_min <= t_max,
// neither NaN (the caller checks)
cudaError_t k7_launch_raycast(const FieldDev& f, const double* d_o, const double* d_d, uint64_t n, double iso, double t_min, double t_max,
                              double* d_t_lo, double* d_t_hi, int32_t* d_status, cudaStream_t stream);

}  // namespace dgb
