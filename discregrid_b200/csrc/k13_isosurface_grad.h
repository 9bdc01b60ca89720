// Launch interface of K13 (k13_isosurface_grad.cu): the vector-Jacobian product of K6's level-set vertices in a trainable field's node
// values.  Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "k6_isosurface.h"
#include "k11_field_grad.h"

namespace dgb {

constexpr int K13_THREADS = 128;

// *d_bad <- how many of the n edge ids are not edges of L (lin(p) >= Np, or q = p + delta_d leaves the lattice).  Queued on `stream`.
cudaError_t k13_launch_check(const K6Lattice& L, const uint64_t* d_edge_ids, uint64_t n, unsigned* d_bad, cudaStream_t stream);
// bytes of device scratch k13_launch_vjp needs for n vertices on a trainable field of n_cells_kept cells
uint64_t k13_scratch_bytes(uint64_t n, uint64_t n_cells_kept);
// grad_nodes [tf.n_nodes] (overwritten) from the upstream d_grad_vertices [n][3] of the vertices on the edges d_edge_ids [n], extracted from
// tf at iso on the lattice L.  The edge ids must have passed k13_launch_check; 2n < 2^32 - 1.  Queued on `stream`, no host synchronisation.
cudaError_t k13_launch_vjp(const K11Field& tf, const K6Lattice& L, double iso, const uint64_t* d_edge_ids, uint64_t n,
                           const double* d_grad_vertices, double* d_grad_nodes, void* scratch, cudaStream_t stream);

}  // namespace dgb
