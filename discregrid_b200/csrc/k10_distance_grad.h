// Launch interface of K10 (k10_distance_grad.cu): the vector-Jacobian product of the mesh distance with respect to the query points and
// the mesh's vertices.  Host-callable, no kernel code here.  The forward with the barycentric weights is K1's (k1_launch_distance_bary).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace dgb {

constexpr int K10_THREADS = 128;
constexpr unsigned K10_FAN = 32;                       // the fixed tree of the segment sums reduces groups of 32

// the mesh's topology: F [T][3] by triangle id, and K8's vertex -> (triangle, slot) incidences (RefitTopoHost::inc_begin / inc)
struct K10Topo {
    const uint32_t* F = nullptr;
    const uint32_t* inc_begin = nullptr;                // [nV + 1]
    const uint32_t* inc = nullptr;                      // [3T]: 3 * triangle + slot
    uint64_t n_vertices = 0;
    int n_tri = 0;
};

// the saved forward outputs and the upstream gradient of n queries
struct K10Query {
    const double* x = nullptr;                          // [n][3] points
    const double* dist = nullptr;                       // [n] signed or unsigned distance
    const double* near = nullptr;                       // [n][3] nearest point
    const int32_t* tri = nullptr;                       // [n] triangle id, -1: none
    const double* bary = nullptr;                       // [n][3] weights of F[tri][0..2]
    const double* g = nullptr;                          // [n] upstream gradient of the distance
    uint64_t n = 0;
};

// counts the triangle ids outside [-1, n_tri) into *d_bad (zeroed first)
cudaError_t k10_launch_check(const int32_t* d_tri, uint64_t n, int n_tri, unsigned* d_bad, cudaStream_t stream);
// bytes of device scratch k10_launch_vjp needs (0 when grad_vertices is not wanted)
uint64_t k10_scratch_bytes(uint64_t n, int n_tri, bool grad_points, bool grad_vertices);
// grad_points [n][3] and grad_vertices [nV][3] (each nullable; grad_vertices is overwritten, 0 where nothing arrives).  Queued on `stream`,
// no host synchronisation.  The triangle ids must have passed k10_launch_check.
cudaError_t k10_launch_vjp(const K10Topo& topo, const K10Query& q, double* d_grad_points, double* d_grad_vertices, void* scratch,
                           cudaStream_t stream);

// The vertex passes of k10_launch_vjp on their own (sort, contributions, segments, levels, vertices), for a caller that computed the
// per-query gradient itself (K12's ray casts): query q with key[q] = t + 1 (0: takes no part) gives -(bary[q][i] * g[q][k]) to slot i of
// triangle t, summed as K10's contract states.  grad_vertices [nV][3] is overwritten; n < 2^32 - 1.  Queued on `stream`.
uint64_t k10_scatter_scratch_bytes(uint64_t n, int n_tri);
cudaError_t k10_launch_scatter(const K10Topo& topo, uint64_t n, const double* d_g, const uint32_t* d_key, const double* d_bary,
                               double* d_grad_vertices, void* scratch, cudaStream_t stream);

}  // namespace dgb
