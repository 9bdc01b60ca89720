// Launch interface of K12 (k12_raycast_grad.cu): the vector-Jacobian products of the two ray casts, K9's on a mesh and K7's on a field.
// Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "k10_distance_grad.h"
#include "k11_field_grad.h"

namespace dgb {

constexpr int K12_THREADS = 128;

// what K9 returned for n rays, the positions the backward differentiates at and the upstream gradients
struct K12MeshRays {
    const double* d = nullptr;                          // [n][3] directions
    const double* t = nullptr;                          // [n] hit parameter
    const int32_t* id = nullptr;                        // [n] triangle id, -1: miss
    const double* bary = nullptr;                       // [n][3] weights of F[id][0..2] (read by the vertex sums only)
    const double* V = nullptr;                          // [nV][3] vertex positions
    const double* grad_t = nullptr;                     // [n] nullable: zeros
    const double* grad_bary = nullptr;                  // [n][3] nullable: zeros
    uint64_t n = 0;
};

// bytes of device scratch k12_launch_mesh_vjp needs (0 unless grad_vertices is wanted)
uint64_t k12_mesh_scratch_bytes(uint64_t n, int n_tri, bool grad_origins, bool grad_vertices);
// grad_origins, grad_directions [n][3] and grad_vertices [nV][3], each nullable (grad_vertices is overwritten, 0 where nothing arrives).
// topo.F is read for every ray; the incidences only for grad_vertices.  The triangle ids must have passed k10_launch_check; n < 2^32 - 1.
// Queued on `stream`, no host synchronisation.
cudaError_t k12_launch_mesh_vjp(const K10Topo& topo, const K12MeshRays& r, double* d_grad_origins, double* d_grad_directions,
                                double* d_grad_vertices, void* scratch, cudaStream_t stream);

// what K7 returned for n rays and the upstream gradients of its bracket
struct K12FieldRays {
    const double* o = nullptr;                          // [n][3] origins
    const double* d = nullptr;                          // [n][3] directions
    const double* t_lo = nullptr;                       // [n]
    const int32_t* status = nullptr;                    // [n] DG_RAY_MISS (0) or a crossing
    const double* grad_t_lo = nullptr;                  // [n] nullable: zeros
    const double* grad_t_hi = nullptr;                  // [n] nullable: zeros
    uint64_t n = 0;
};

// bytes of device scratch k12_launch_field_vjp needs; n_cells_kept is the trainable field's when grad_nodes is wanted
uint64_t k12_field_scratch_bytes(uint64_t n, uint64_t n_cells_kept, bool grad_nodes);
// grad_origins, grad_directions [n][3] and grad_nodes [n_nodes] (each nullable; grad_nodes needs tf, a trainable field whose tf->f is f,
// and is overwritten).  K2's gradient mode evaluates the field at the rays' crossings; K11 sums the node gradient.  n < 2^32 - 1.  Queued
// on `stream`, no host synchronisation.
cudaError_t k12_launch_field_vjp(const FieldDev& f, const K11Field* tf, const K12FieldRays& r, double* d_grad_origins, double* d_grad_directions,
                                 double* d_grad_nodes, void* scratch, cudaStream_t stream);

}  // namespace dgb
