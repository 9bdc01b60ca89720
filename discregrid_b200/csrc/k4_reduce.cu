// K4: the index passes of CubicLagrangeDiscreteGrid::reduceField (cubic_lagrange_discrete_grid.cpp:1065-1174) on the GPU -- SURVEY 8(f) N3.
//
// reduceField keeps the cells that own at least one node the predicate accepted, keeps the nodes those cells refer to, renumbers the
// nodes in Z-curve order and rewrites the connectivity.  The reference does it with one std::set of back-references per node; what it
// computes is a renumbering, and everything except two steps is data-parallel:
//   kernels here : keep flag per cell (:1081-1098) . cell map + compaction of the surviving rows . marks of the surviving nodes (:1117-1134)
//                  . Morton key of every survivor (zValue, :583-601 / z_sort_table.hpp:119-134) . new node ids, renumbered rows, gathered
//                  coefficients (:1158-1173)
//   host (reduce_field.cpp): the reference's back-to-front swap compaction replayed on a permutation array (:1135-1156, O(n), inherently
//                  serial) and the sort of the survivors by key, whose order among EQUAL keys is libstdc++'s introsort's (reduce_field.h).
// The reduced narrow band (dg_reduced_band_create), the reduced density map (dg_reduced_density_map_create) and the reductions of fields
// sampled by device callbacks (dg_reduced_function_create, dg_reduce_field_device) run the same passes on the device only: keep flags from
// a value predicate or a node mask, cell flags and rows from an uploaded table or from the closed form instead of a cell table, and the swap
// walk itself as pointer jumping (swap_walk_*); the sort of the survivors stays on the host.
// All kernels are warp-synchronous (ballot / popc), so tests/emu runs them unchanged.  Integer work, bit-exact by construction; the one
// floating-point step (the key's cast of inv * x) uses the reference's operations in the reference's order (no FMA: -fmad=false).
#include "k4_reduce.h"
#include "dg_launch.h"

#include <cfloat>
#include <climits>
#include <vector>

namespace dgb {
namespace {

constexpr unsigned TILE = 1024;                       // cells per warp in the counting / compaction passes

// keep flag per cell: any of its 32 nodes kept?  One warp per cell, lane j reads entry j.  bad[0] is set when an entry is not a node id.
__global__ void cell_keep_kernel(const unsigned* __restrict__ cells, unsigned long long n_cells, const unsigned char* __restrict__ keep_node,
                                 unsigned n_nodes, unsigned char* __restrict__ cell_keep, unsigned* __restrict__ bad)
{
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const bool live = warp < n_cells;                 // whole warps: uniform
    unsigned v = 0;
    if (live) v = __ldg(cells + warp * 32ull + lane);
    const bool oob = live && v >= n_nodes;
    const unsigned any_bad = __ballot_sync(0xffffffffu, oob);
    const unsigned any_keep = __ballot_sync(0xffffffffu, live && !oob && keep_node[v] != 0);
    if (live && lane == 0) {
        if (any_bad) atomicAdd(bad, 1u);
        cell_keep[warp] = (any_keep && !any_bad) ? 1 : 0;
    }
}

// number of set flags per tile of TILE entries (one warp per tile)
__global__ void tile_count_kernel(const unsigned char* __restrict__ flag, unsigned long long n, unsigned* __restrict__ tile_count)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long base = tile * TILE;
    if (base >= n) return;                            // whole warps
    unsigned cnt = 0;
    for (unsigned k = 0; k < TILE; k += 32) {
        const unsigned long long i = base + k + lane;
        cnt += (unsigned)__popc(__ballot_sync(0xffffffffu, i < n && flag[i] != 0));
    }
    if (lane == 0) tile_count[tile] = cnt;
}

// cell_map (:1076-1097) and the surviving rows moved to the front, order kept: one warp per tile, tile_offset = exclusive scan of the counts
__global__ void cell_compact_kernel(const unsigned* __restrict__ cells, unsigned long long n_cells, const unsigned char* __restrict__ cell_keep,
                                    const unsigned* __restrict__ tile_offset, unsigned* __restrict__ cells_out, unsigned* __restrict__ cell_map)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long base = tile * TILE;
    if (base >= n_cells) return;
    unsigned run = tile_offset[tile];
    const unsigned lt = (1u << lane) - 1u;
    for (unsigned k = 0; k < TILE; k += 32) {
        const unsigned long long c = base + k + lane;
        const bool kept = c < n_cells && cell_keep[c] != 0;
        const unsigned m = __ballot_sync(0xffffffffu, kept);
        if (c < n_cells) cell_map[c] = kept ? run + (unsigned)__popc(m & lt) : 0xffffffffu;
        // the warp copies the kept rows of this chunk, 128 bytes at a time
        unsigned rest = m, r = run;
        while (rest) {
            const unsigned src_lane = (unsigned)__ffs((int)rest) - 1u;
            rest &= rest - 1u;
            const unsigned long long src = base + k + src_lane;
            cells_out[(unsigned long long)r * 32ull + lane] = __ldg(cells + src * 32ull + lane);
            r++;
        }
        run += (unsigned)__popc(m);
    }
}

__global__ void mark_used_kernel(const unsigned* __restrict__ cells_out, unsigned long long n_entries, unsigned char* __restrict__ used)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_entries) used[cells_out[i]] = 1;
}

// morton_lut (z_sort_table.hpp:119-134): only the LOW 16 bits of each coordinate reach the key (x at bit 0, y at bit 1, z at bit 2)
__device__ __forceinline__ unsigned long long spread16(unsigned long long v)
{
    v &= 0xffffull;
    v = (v | v << 16) & 0x0000ff0000ffull;
    v = (v | v << 8) & 0x00f00f00f00full;
    v = (v | v << 4) & 0x0c30c30c30c3ull;
    v = (v | v << 2) & 0x249249249249ull;
    return v;
}

// key[i] = zValue(indexToNodePosition(perm[i]), 4 * min(inv_cell_size))   (:1113-1114, :583-601)
__global__ void morton_key_kernel(GridDev g, const unsigned* __restrict__ perm, unsigned long long m, double inv, unsigned long long* __restrict__ key)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    double x[3];
    node_position(g, perm[i], x[0], x[1], x[2]);
    unsigned p[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int c = (x[k] >= 0.0) ? static_cast<int>(inv * x[k]) : static_cast<int>(inv * x[k]) - 1;             // :589-592
        p[k] = static_cast<unsigned>(static_cast<long long>(c) - (static_cast<long long>(INT_MIN) + 1));          // :595-598
    }
    key[i] = spread16(p[0]) | (spread16(p[1]) << 1) | (spread16(p[2]) << 2);
}

// rank r holds the node that sat at position order[r]: new id of that node = r; its coefficient moves to r (:1158-1173)
__global__ void renumber_nodes_kernel(const unsigned* __restrict__ perm, const unsigned* __restrict__ order, unsigned long long m,
                                      const double* __restrict__ nodes, unsigned* __restrict__ new_id, double* __restrict__ nodes_out)
{
    const unsigned long long r = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= m) return;
    const unsigned v = perm[order[r]];
    new_id[v] = (unsigned)r;
    nodes_out[r] = nodes[v];
}

__global__ void renumber_cells_kernel(unsigned* __restrict__ cells_out, unsigned long long n_entries, const unsigned* __restrict__ new_id)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_entries) cells_out[i] = new_id[cells_out[i]];
}

// ---- reduction on the device only (dg_reduced_band_create, dg_reduced_density_map_create): the same passes on a dense field whose keep
// flags come from a value predicate (K4ValuePred), with the rows of the cells either uploaded or taken from the closed form (cell_node_id)
// instead of a 32-index table of the whole grid.

// pred(x, v) && v != DBL_MAX (:1069-1074) for the predicates that depend on v alone, in the expression order of the reference's tool:
// v + c and v - c are rounded first, then compared with the bounds as given (no rearranged bounds)
template <int KIND>
__device__ __forceinline__ bool value_kept(const K4ValuePred& p, double v)
{
    if (KIND == K4_KEEP_SDF) return (p.a < v + p.c && v - p.c < p.b) && v != DBL_MAX;
    if (KIND == K4_KEEP_RANGE) return (p.a <= v && v <= p.b) && v != DBL_MAX;
    return v != DBL_MAX;
}

// keep flag per node of a dense field (for rows read through cell_keep_kernel)
template <int KIND>
__global__ void node_keep_kernel(const double* __restrict__ nodes, unsigned long long n, K4ValuePred p, unsigned char* __restrict__ keep)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keep[i] = value_kept<KIND>(p, __ldg(nodes + i)) ? 1 : 0;
}

// addFunction(func, verbose, pred) stores DBL_MAX where the sample predicate rejects (:817): v = keep ? v : DBL_MAX
__global__ void sample_mask_apply_kernel(double* __restrict__ values, const unsigned char* __restrict__ keep, unsigned long long n)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && keep[i] == 0) values[i] = DBL_MAX;
}

// reduceField keeps node l iff pred(x_l, c_l) && c_l != DBL_MAX (:1069-1074): keep = keep && v != DBL_MAX, as 0 / 1
__global__ void node_mask_combine_kernel(unsigned char* __restrict__ keep, const double* __restrict__ values, unsigned long long n)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keep[i] = (keep[i] != 0 && __ldg(values + i) != DBL_MAX) ? 1 : 0;
}

__device__ __forceinline__ void cell_ijk(const GridDev& g, unsigned long long c, unsigned& i, unsigned& j, unsigned& k)
{
    const unsigned long long s = (unsigned long long)g.n[0] * g.n[1];
    k = (unsigned)(c / s);
    const unsigned t = (unsigned)(c - (unsigned long long)k * s);
    j = t / g.n[0]; i = t - j * g.n[0];
}

// where a node's keep decision comes from: a value predicate of its coefficient, or a node mask computed beforehand (a device predicate
// combined with v != DBL_MAX by node_mask_combine_kernel)
template <int KIND>
struct ValueKeep {
    const double* __restrict__ nodes;
    K4ValuePred p;
    __device__ __forceinline__ bool operator()(unsigned l) const { return value_kept<KIND>(p, __ldg(nodes + l)); }
};
struct MaskKeep {
    const unsigned char* __restrict__ keep;
    __device__ __forceinline__ bool operator()(unsigned l) const { return __ldg(keep + l) != 0; }
};

// keep flag per cell: one warp per cell, lane j asks `keep` about the cell's closed-form node j
template <class Keep>
__global__ void closed_cell_keep_kernel(GridDev g, Keep keep, unsigned long long n_cells, unsigned char* __restrict__ cell_keep)
{
    const unsigned long long c = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const bool live = c < n_cells;                    // whole warps: uniform
    bool kept = false;
    if (live) {
        unsigned i, j, k;
        cell_ijk(g, c, i, j, k);
        kept = keep(cell_node_id(g, i, j, k, lane));
    }
    const unsigned any = __ballot_sync(0xffffffffu, kept);
    if (live && lane == 0) cell_keep[c] = any ? 1 : 0;
}

// bad[0] += 1 per warp that sees a cell map entry that is neither 0xffffffff nor a row id < n_rows
__global__ void cell_map_check_kernel(const unsigned* __restrict__ cell_map, unsigned long long n, unsigned long long n_rows, unsigned* __restrict__ bad)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool b = false;
    if (i < n) { const unsigned v = cell_map[i]; b = v != 0xffffffffu && v >= n_rows; }
    if (__ballot_sync(0xffffffffu, b) && (threadIdx.x & 31u) == 0) atomicAdd(bad, 1u);
}

// cell_map[i] = i on [begin, end): the reference's resize + iota (:1076-1078) for cells a field never had rows for
__global__ void iota_kernel(unsigned* __restrict__ out, unsigned long long begin, unsigned long long end)
{
    const unsigned long long i = begin + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < end) out[i] = (unsigned)i;
}

// cell_map and the closed-form rows of the kept cells, order kept: cell_compact_kernel with the rows computed instead of copied
__global__ void closed_cell_compact_kernel(GridDev g, unsigned long long n_cells, const unsigned char* __restrict__ cell_keep,
                                           const unsigned* __restrict__ tile_offset, unsigned* __restrict__ cells_out, unsigned* __restrict__ cell_map)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long base = tile * TILE;
    if (base >= n_cells) return;
    unsigned run = tile_offset[tile];
    const unsigned lt = (1u << lane) - 1u;
    for (unsigned k = 0; k < TILE; k += 32) {
        const unsigned long long c = base + k + lane;
        const bool kept = c < n_cells && cell_keep[c] != 0;
        const unsigned m = __ballot_sync(0xffffffffu, kept);
        if (c < n_cells) cell_map[c] = kept ? run + (unsigned)__popc(m & lt) : 0xffffffffu;
        unsigned rest = m, r = run;
        while (rest) {
            const unsigned src_lane = (unsigned)__ffs((int)rest) - 1u;
            rest &= rest - 1u;
            unsigned ci, cj, ck;
            cell_ijk(g, base + k + src_lane, ci, cj, ck);
            cells_out[(unsigned long long)r * 32ull + lane] = cell_node_id(g, ci, cj, ck, lane);
            r++;
        }
        run += (unsigned)__popc(m);
    }
}

// The reference's back-to-front swap walk (:1135-1156) in parallel.  With m used positions, a used position p < m keeps its node; a dead
// position p < m ends up holding the first USED position of q0 = m + dead(p), q_{i+1} = m + dead(q_i), where dead(q) = number of dead
// positions before q (the k-th dead position from the front is swapped with position m + k).  walk[q] = q for a used q, m + dead(q) for a
// dead one; tile_offset = exclusive scan of the used counts per tile, so dead(q) = q - used positions before q.
__global__ void swap_walk_start_kernel(const unsigned char* __restrict__ used, unsigned long long n, unsigned long long m,
                                       const unsigned* __restrict__ tile_offset, unsigned* __restrict__ walk)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long base = tile * TILE;
    if (base >= n) return;
    unsigned long long run = tile_offset[tile];
    const unsigned lt = (1u << lane) - 1u;
    for (unsigned k = 0; k < TILE; k += 32) {
        const unsigned long long q = base + k + lane;
        const bool u = q < n && used[q] != 0;
        const unsigned mask = __ballot_sync(0xffffffffu, u);
        if (q < n) walk[q] = u ? (unsigned)q : (unsigned)(m + (q - (run + (unsigned)__popc(mask & lt))));
        run += (unsigned)__popc(mask);
    }
}

// one round of pointer jumping over [m, n): walk[q] <- walk[walk[q]].  In place: a value read while another thread rewrites it is either
// the old or the new pointer, both further along the same chain, so a round advances every pointer at least as far as a double-buffered one.
__global__ void swap_walk_jump_kernel(unsigned* walk, unsigned long long m, unsigned long long n, unsigned* __restrict__ changed)
{
    const unsigned long long q = m + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool moved = false;
    if (q < n) {
        const unsigned a = walk[q], b = walk[a];
        if (b != a) { walk[q] = b; moved = true; }
    }
    if (__ballot_sync(0xffffffffu, moved) && (threadIdx.x & 31u) == 0) atomicAdd(changed, 1u);
}

// positions [0, m): walk[p] = p (used) or a position >= m whose pointer now names the used position at the end of its chain
__global__ void swap_walk_finish_kernel(unsigned* walk, unsigned long long m)
{
    const unsigned long long p = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < m) walk[p] = walk[walk[p]];
}

inline unsigned blocks_for(unsigned long long threads, unsigned block) { return (unsigned)((threads + block - 1) / block); }

}  // namespace

unsigned k4_tile() { return TILE; }

cudaError_t k4_launch_cell_keep(const unsigned* d_cells, uint64_t n_cells, const unsigned char* d_keep_node, unsigned n_nodes, unsigned char* d_cell_keep,
                                unsigned* d_bad, cudaStream_t stream)
{
    if (n_cells == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(cell_keep_kernel, blocks_for(n_cells * 32ull, 128), 128, 0, stream, d_cells, (unsigned long long)n_cells, d_keep_node, n_nodes, d_cell_keep, d_bad);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_tile_count(const unsigned char* d_flag, uint64_t n, unsigned* d_tile_count, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    const uint64_t tiles = (n + TILE - 1) / TILE;
    DG_KERNEL_LAUNCH(tile_count_kernel, blocks_for(tiles * 32ull, 128), 128, 0, stream, d_flag, (unsigned long long)n, d_tile_count);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_cell_compact(const unsigned* d_cells, uint64_t n_cells, const unsigned char* d_cell_keep, const unsigned* d_tile_offset,
                                   unsigned* d_cells_out, unsigned* d_cell_map, cudaStream_t stream)
{
    if (n_cells == 0) return cudaSuccess;
    const uint64_t tiles = (n_cells + TILE - 1) / TILE;
    DG_KERNEL_LAUNCH(cell_compact_kernel, blocks_for(tiles * 32ull, 128), 128, 0, stream, d_cells, (unsigned long long)n_cells, d_cell_keep, d_tile_offset, d_cells_out, d_cell_map);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_mark_used(const unsigned* d_cells_out, uint64_t n_entries, unsigned char* d_used, cudaStream_t stream)
{
    if (n_entries == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(mark_used_kernel, blocks_for(n_entries, 256), 256, 0, stream, d_cells_out, (unsigned long long)n_entries, d_used);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_morton_keys(const GridDev& g, const unsigned* d_perm, uint64_t m, unsigned long long* d_key, cudaStream_t stream)
{
    if (m == 0) return cudaSuccess;
    double inv = g.inv[0]; if (g.inv[1] < inv) inv = g.inv[1]; if (g.inv[2] < inv) inv = g.inv[2];
    inv = 4.0 * inv;                                                                                    // 4.0 * m_inv_cell_size.minCoeff(), :1114
    DG_KERNEL_LAUNCH(morton_key_kernel, blocks_for(m, 256), 256, 0, stream, g, d_perm, (unsigned long long)m, inv, d_key);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_renumber(const unsigned* d_perm, const unsigned* d_order, uint64_t m, const double* d_nodes, unsigned* d_new_id, double* d_nodes_out,
                               unsigned* d_cells_out, uint64_t n_entries, cudaStream_t stream)
{
    if (m) { DG_KERNEL_LAUNCH(renumber_nodes_kernel, blocks_for(m, 256), 256, 0, stream, d_perm, d_order, (unsigned long long)m, d_nodes, d_new_id, d_nodes_out); }
    if (n_entries) { DG_KERNEL_LAUNCH(renumber_cells_kernel, blocks_for(n_entries, 256), 256, 0, stream, d_cells_out, (unsigned long long)n_entries, d_new_id); }
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_node_keep(const double* d_nodes, uint64_t n, const K4ValuePred& p, unsigned char* d_keep, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    const unsigned blocks = blocks_for(n, 256);
    switch (p.kind) {
    case K4_KEEP_ANY: DG_KERNEL_LAUNCH(node_keep_kernel<K4_KEEP_ANY>, blocks, 256, 0, stream, d_nodes, (unsigned long long)n, p, d_keep); break;
    case K4_KEEP_SDF: DG_KERNEL_LAUNCH(node_keep_kernel<K4_KEEP_SDF>, blocks, 256, 0, stream, d_nodes, (unsigned long long)n, p, d_keep); break;
    case K4_KEEP_RANGE: DG_KERNEL_LAUNCH(node_keep_kernel<K4_KEEP_RANGE>, blocks, 256, 0, stream, d_nodes, (unsigned long long)n, p, d_keep); break;
    default: return cudaErrorInvalidValue;
    }
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_closed_cell_keep(const GridDev& g, const double* d_nodes, uint64_t n_cells, const K4ValuePred& p, unsigned char* d_cell_keep,
                                       cudaStream_t stream)
{
    if (n_cells == 0) return cudaSuccess;
    const unsigned blocks = blocks_for(n_cells * 32ull, 128);
    const unsigned long long nc = n_cells;
    switch (p.kind) {
    case K4_KEEP_ANY: DG_KERNEL_LAUNCH(closed_cell_keep_kernel<ValueKeep<K4_KEEP_ANY>>, blocks, 128, 0, stream, g, ValueKeep<K4_KEEP_ANY>{d_nodes, p}, nc, d_cell_keep); break;
    case K4_KEEP_SDF: DG_KERNEL_LAUNCH(closed_cell_keep_kernel<ValueKeep<K4_KEEP_SDF>>, blocks, 128, 0, stream, g, ValueKeep<K4_KEEP_SDF>{d_nodes, p}, nc, d_cell_keep); break;
    case K4_KEEP_RANGE: DG_KERNEL_LAUNCH(closed_cell_keep_kernel<ValueKeep<K4_KEEP_RANGE>>, blocks, 128, 0, stream, g, ValueKeep<K4_KEEP_RANGE>{d_nodes, p}, nc, d_cell_keep); break;
    default: return cudaErrorInvalidValue;
    }
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_closed_cell_keep_mask(const GridDev& g, const unsigned char* d_keep_node, uint64_t n_cells, unsigned char* d_cell_keep, cudaStream_t stream)
{
    if (n_cells == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(closed_cell_keep_kernel<MaskKeep>, blocks_for(n_cells * 32ull, 128), 128, 0, stream, g, MaskKeep{d_keep_node}, (unsigned long long)n_cells,
                     d_cell_keep);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_sample_mask_apply(double* d_values, const unsigned char* d_keep, uint64_t n, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(sample_mask_apply_kernel, blocks_for(n, 256), 256, 0, stream, d_values, d_keep, (unsigned long long)n);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_node_mask_combine(unsigned char* d_keep, const double* d_values, uint64_t n, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(node_mask_combine_kernel, blocks_for(n, 256), 256, 0, stream, d_keep, d_values, (unsigned long long)n);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_closed_cell_compact(const GridDev& g, uint64_t n_cells, const unsigned char* d_cell_keep, const unsigned* d_tile_offset,
                                          unsigned* d_cells_out, unsigned* d_cell_map, cudaStream_t stream)
{
    if (n_cells == 0) return cudaSuccess;
    const uint64_t tiles = (n_cells + TILE - 1) / TILE;
    DG_KERNEL_LAUNCH(closed_cell_compact_kernel, blocks_for(tiles * 32ull, 128), 128, 0, stream, g, (unsigned long long)n_cells, d_cell_keep, d_tile_offset,
                     d_cells_out, d_cell_map);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_cell_map_check(const unsigned* d_cell_map, uint64_t n, uint64_t n_rows, unsigned* d_bad, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(cell_map_check_kernel, blocks_for(n, 256), 256, 0, stream, d_cell_map, (unsigned long long)n, (unsigned long long)n_rows, d_bad);
    return DG_AFTER_LAUNCH();
}

cudaError_t k4_launch_iota(unsigned* d_out, uint64_t begin, uint64_t end, cudaStream_t stream)
{
    if (end <= begin) return cudaSuccess;
    DG_KERNEL_LAUNCH(iota_kernel, blocks_for(end - begin, 256), 256, 0, stream, d_out, (unsigned long long)begin, (unsigned long long)end);
    return DG_AFTER_LAUNCH();
}

// exclusive scan of per-tile counts on the host (one entry per TILE flags) through d_tile, in place; returns the total
static cudaError_t scan_tile_counts(unsigned* d_tile, uint64_t n_tiles, uint64_t& total, cudaStream_t stream)
{
    std::vector<unsigned> cnt(n_tiles);
    total = 0;
    if (n_tiles == 0) return cudaSuccess;
    cudaError_t e = cudaMemcpyAsync(cnt.data(), d_tile, n_tiles * sizeof(unsigned), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return e;
    for (uint64_t t = 0; t < n_tiles; t++) { const unsigned c = cnt[t]; cnt[t] = (unsigned)total; total += c; }
    e = cudaMemcpyAsync(d_tile, cnt.data(), n_tiles * sizeof(unsigned), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);         // cnt goes out of scope
    return e;
}

cudaError_t k4_scan_flags(const unsigned char* d_flag, uint64_t n, unsigned* d_tile, uint64_t& total, cudaStream_t stream)
{
    cudaError_t e = k4_launch_tile_count(d_flag, n, d_tile, stream);
    if (e != cudaSuccess) return e;
    return scan_tile_counts(d_tile, (n + TILE - 1) / TILE, total, stream);
}

cudaError_t k4_swap_walk(const unsigned char* d_used, uint64_t n, unsigned* d_tile, unsigned* d_flag, unsigned* d_walk, uint64_t& m, unsigned& rounds,
                         cudaStream_t stream)
{
    rounds = 0;
    cudaError_t e = k4_scan_flags(d_used, n, d_tile, m, stream);
    if (e != cudaSuccess || m == 0) return e;
    const uint64_t tiles = (n + TILE - 1) / TILE;
    DG_KERNEL_LAUNCH(swap_walk_start_kernel, blocks_for(tiles * 32ull, 128), 128, 0, stream, d_used, (unsigned long long)n, (unsigned long long)m, d_tile, d_walk);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    // a chain visits distinct positions of [m, n), so ceil(log2(n - m)) rounds reach its end; stop as soon as a round moves nothing
    unsigned max_rounds = 0;
    while ((1ull << max_rounds) < n - m) max_rounds++;
    for (unsigned r = 0; r < max_rounds; r++) {
        unsigned changed = 0;
        if ((e = cudaMemsetAsync(d_flag, 0, sizeof(unsigned), stream)) != cudaSuccess) return e;
        DG_KERNEL_LAUNCH(swap_walk_jump_kernel, blocks_for(n - m, 256), 256, 0, stream, d_walk, (unsigned long long)m, (unsigned long long)n, d_flag);
        if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
        if ((e = cudaMemcpyAsync(&changed, d_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
        rounds++;
        if (!changed) break;
    }
    if (m) { DG_KERNEL_LAUNCH(swap_walk_finish_kernel, blocks_for(m, 256), 256, 0, stream, d_walk, (unsigned long long)m); }
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
