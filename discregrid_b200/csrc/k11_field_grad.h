// Launch interface of K11 (k11_field_grad.cu): the vector-Jacobian product of K2's interpolate with respect to a field's node values, and
// the tables a trainable field keeps for it.  Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "k2_interp.h"

namespace dgb {

constexpr int K11_THREADS = 128;
constexpr unsigned K11_FAN = 32;                       // the tree of the segment sums reduces groups of 32 (K10's R)

// a trainable field: K2's device field plus the tables of dg_field_create_trainable
struct K11Field {
    FieldDev f;
    const uint32_t* inc_begin = nullptr;               // [n_nodes + 1]: node v's incidences are inc[inc_begin[v] .. inc_begin[v + 1])
    const uint32_t* inc = nullptr;                     // [32 n_cells_kept]: 32 * cell + slot, ascending per node
    const unsigned char* has_max = nullptr;            // [n_cells_kept]: the cell's block holds a DBL_MAX coefficient
    uint64_t n_nodes = 0, n_cells_kept = 0;
};

// has_max[c] = (some packed[c][j] == DBL_MAX)
cudaError_t k11_launch_flags(const double* d_packed, uint64_t n_cells_kept, unsigned char* d_has_max, cudaStream_t stream);
// bytes of device scratch k11_launch_incidence needs
uint64_t k11_incidence_scratch_bytes(uint64_t n_cells_kept);
// the node -> (cell, slot) table of a field: d_cells [n_cells_kept][32] node ids, or NULL for the closed-form table of a dense grid.
// Requires 32 n_cells_kept < 2^32 and every node id below n_nodes.  Queued on `stream`.
cudaError_t k11_launch_incidence(const GridDev& g, const unsigned* d_cells, uint64_t n_cells_kept, uint64_t n_nodes, uint32_t* d_inc_begin,
                                 uint32_t* d_inc, void* scratch, cudaStream_t stream);
// bytes of device scratch k11_launch_vjp needs for n queries
uint64_t k11_scratch_bytes(uint64_t n, uint64_t n_cells_kept);
// grad_nodes [n_nodes] (overwritten) from gphi [n] and ggrad [n][3] (either nullable, not both); n < 2^32 - 1.  Queued on `stream`, no host
// synchronisation.
cudaError_t k11_launch_vjp(const K11Field& f, const double* d_x, uint64_t n, const double* d_gphi, const double* d_ggrad, double* d_grad_nodes,
                           void* scratch, cudaStream_t stream);

}  // namespace dgb
