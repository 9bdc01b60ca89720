// Launch interface of K9 (k9_mesh_raycast.cu): first hits of rays and segments on a triangle mesh.  Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "k1_sdf.h"
#include "k5_winding.h"

namespace dgb {

constexpr int K9_THREADS = 128;
constexpr int K9_MAX_STACK = 32;   // deferred siblings per lane; as K5_MAX_STACK, a tree of < 2^25 triangles has at most 26 levels

// per ray i: origin o[3 i..], direction d[3 i..]; t[i], triangle_id[i], barycentric[3 i..] (may be NULL) and status[i] as in the contract
// of k9_mesh_raycast.cu.  t_min <= t_max, neither NaN; m.stack_depth <= K9_MAX_STACK (the caller checks).  `w` holds the vertices in leaf
// order (K5's WindLeaf records), `m` the tree (fp32 child boxes, leaf records for the ids).
cudaError_t k9_launch_mesh_raycast(const DeviceBvh& m, const WindDev& w, const double* d_o, const double* d_d, uint64_t n, double t_min,
                                   double t_max, double* d_t, int32_t* d_id, double* d_bary, int32_t* d_status, cudaStream_t stream);

}  // namespace dgb
