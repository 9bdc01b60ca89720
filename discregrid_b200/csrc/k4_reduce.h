// Launch interface of the reduceField index kernels (k4_reduce.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "dg_device.cuh"

namespace dgb {

unsigned k4_tile();          // entries per tile of the counting / compaction passes
cudaError_t k4_launch_cell_keep(const unsigned* d_cells, uint64_t n_cells, const unsigned char* d_keep_node, unsigned n_nodes, unsigned char* d_cell_keep,
                                unsigned* d_bad, cudaStream_t stream);
cudaError_t k4_launch_tile_count(const unsigned char* d_flag, uint64_t n, unsigned* d_tile_count, cudaStream_t stream);
cudaError_t k4_launch_cell_compact(const unsigned* d_cells, uint64_t n_cells, const unsigned char* d_cell_keep, const unsigned* d_tile_offset,
                                   unsigned* d_cells_out, unsigned* d_cell_map, cudaStream_t stream);
cudaError_t k4_launch_mark_used(const unsigned* d_cells_out, uint64_t n_entries, unsigned char* d_used, cudaStream_t stream);
cudaError_t k4_launch_morton_keys(const GridDev& g, const unsigned* d_perm, uint64_t m, unsigned long long* d_key, cudaStream_t stream);
cudaError_t k4_launch_renumber(const unsigned* d_perm, const unsigned* d_order, uint64_t m, const double* d_nodes, unsigned* d_new_id, double* d_nodes_out,
                               unsigned* d_cells_out, uint64_t n_entries, cudaStream_t stream);

// reduceField predicates that depend on the node value v alone.  A node is kept iff v != DBL_MAX (:1073) and
//   K4_KEEP_ANY   : always (the reduced narrow band)
//   K4_KEEP_SDF   : a < v + c && v - c < b   (GenerateDensityMap's SDF field: a = -6h, b = 2h, c = cell diagonal; main.cpp:139)
//   K4_KEEP_RANGE : a <= v && v <= b          (its density field: a = 0, b = 3 rho0; main.cpp:140)
enum K4KeepKind { K4_KEEP_ANY = 0, K4_KEEP_SDF = 1, K4_KEEP_RANGE = 2 };
struct K4ValuePred {
    K4KeepKind kind;
    double a, b, c;
};
// d_keep[i] = predicate of d_nodes[i], for rows read through k4_launch_cell_keep
cudaError_t k4_launch_node_keep(const double* d_nodes, uint64_t n, const K4ValuePred& p, unsigned char* d_keep, cudaStream_t stream);
// cell flags and compaction with the closed-form rows (cell_node_id) of the dense coefficients d_nodes
cudaError_t k4_launch_closed_cell_keep(const GridDev& g, const double* d_nodes, uint64_t n_cells, const K4ValuePred& p, unsigned char* d_cell_keep,
                                       cudaStream_t stream);
// the same cell flags from a node mask (0 = not kept) instead of a value predicate
cudaError_t k4_launch_closed_cell_keep_mask(const GridDev& g, const unsigned char* d_keep_node, uint64_t n_cells, unsigned char* d_cell_keep, cudaStream_t stream);
// node masks of device callbacks: d_values[i] = DBL_MAX where d_keep[i] == 0 (a sample predicate, :817); d_keep[i] = d_keep[i] != 0 &&
// d_values[i] != DBL_MAX, as 0 / 1 (a reduce predicate, :1073)
cudaError_t k4_launch_sample_mask_apply(double* d_values, const unsigned char* d_keep, uint64_t n, cudaStream_t stream);
cudaError_t k4_launch_node_mask_combine(unsigned char* d_keep, const double* d_values, uint64_t n, cudaStream_t stream);
cudaError_t k4_launch_closed_cell_compact(const GridDev& g, uint64_t n_cells, const unsigned char* d_cell_keep, const unsigned* d_tile_offset,
                                          unsigned* d_cells_out, unsigned* d_cell_map, cudaStream_t stream);
// d_bad[0] becomes non-zero when an entry of d_cell_map[0..n) is neither 0xffffffff nor < n_rows
cudaError_t k4_launch_cell_map_check(const unsigned* d_cell_map, uint64_t n, uint64_t n_rows, unsigned* d_bad, cudaStream_t stream);
// d_out[i] = i for i in [begin, end)
cudaError_t k4_launch_iota(unsigned* d_out, uint64_t begin, uint64_t end, cudaStream_t stream);
// d_tile (ceil(n / k4_tile()) entries) <- exclusive scan of the set flags per tile; total = number of set flags.  Synchronises `stream`.
cudaError_t k4_scan_flags(const unsigned char* d_flag, uint64_t n, unsigned* d_tile, uint64_t& total, cudaStream_t stream);
// The reference's swap-walk compaction (:1135-1156, reduce_swap_walk) on the device: m = number of used positions, d_walk[0..m) = the
// node at each position afterwards.  d_walk: n entries, d_tile: ceil(n / k4_tile()), d_flag: 1.  rounds = pointer-jumping rounds run.
cudaError_t k4_swap_walk(const unsigned char* d_used, uint64_t n, unsigned* d_tile, unsigned* d_flag, unsigned* d_walk, uint64_t& m, unsigned& rounds,
                         cudaStream_t stream);

}  // namespace dgb
