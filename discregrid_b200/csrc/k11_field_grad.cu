// K11: the vector-Jacobian product of K2's interpolate with respect to a field's node values (dg_interpolate_vjp): for upstream gradients of
// phi and of grad at n query points, the gradient of the loss with respect to every node value, summed in a fixed order.
//
// NUMERICAL CONTRACT (fp64, no FMA: the TU is compiled with -fmad=false; the library's own, the reference has no such derivative).  A field
// has packed blocks c[cell][0..31]; query q has point x_q, upstream gradient of phi gphi[q] (nullable) and of grad ggrad[q][3] (nullable),
// at least one of the two given.
//   Validity: q contributes iff K2 would not return its sentinel for x_q on the field's current coefficients: x_q inside the domain (NaN
//       fails), the cell located exactly as in interpolate_kernel (including the clamp of each index to n - 1) not removed by the cell map,
//       and no DBL_MAX among the cell's 32 coefficients.
//   Factors: N_j and D_jk are the expressions K2 multiplies c_j by in the value and in the gradient sum, in the same operation order
//       (shape_rows.cuh, shared with shape_functions_kernel: what dg_shape_functions returns as N and dN), at xi = c0 * x - c1 from K2's
//       per-axis table.  The VJP is therefore the transpose of K2's linear map in the coefficients, up to the rounding of the products.
//   Contribution of q to slot j: start from the first present term and add the others left to right:
//       gphi * N_j,   (ggrad_0 * c0_x) * D_j0,   (ggrad_1 * c0_y) * D_j1,   (ggrad_2 * c0_z) * D_j2.
//       An absent upstream adds nothing (it is not added as +0.0).
//   Segments: key = kept cell index + 1, 0 for a sentinel query; the queries stably sorted by key, so in ascending q within a cell.  The
//       segment of (cell, j) is the list of the contributions to j of that cell's queries, in that order.
//   Segment sum R (K10's, word for word): while the list has more than one entry, replace each aligned group of 32 consecutive entries (the
//       last may be shorter) by its tree sum; the one entry left is R.  Tree sum of y_0 .. y_{m-1}: for s = 1, 2, 4, 8, 16, y_i = y_i + y_{i+s}
//       for every i that is a multiple of 2s with i + s < m; the result is y_0.
//   Nodes: grad_nodes[v] = ((+0.0 + R_1) + R_2) + ..., over v's incidences (cell, j) in ascending 32 * cell + j whose segment is not empty.
//       A node that receives nothing gets +0.0.  Skipping an empty segment and adding +0.0 for it give the same bits: the fold starts at
//       +0.0, and a sum of which one operand is +0.0 is never -0.0 in round-to-nearest (x + (+0.0) is x for x != -0.0 and +0.0 for
//       x = -0.0), so the fold never holds -0.0 and adding +0.0 to it changes nothing.  An implementation may zero-fill instead of flagging.
//   The bits depend only on the field's topology, the points and the upstream gradients: not on the coefficient values (except through the
//   DBL_MAX test), the launch geometry, the stream or the run.  No gradient in x comes from this pass (K2's gradient and Hessian modes give it).
//
// Passes (all warp-synchronous, no double atomics, so that tests/emu runs every one):
//   keys     : one thread per query: the key above.
//   sort     : radix_sort_pairs of the keys with the query indices, bit_width(n_cells_kept) key bits.
//   segments : the first and last sorted position of each cell; then per cell the number of its aligned groups of 32 queries, scanned into
//              group offsets (the sort's scan), and the first sorted position of every group.
//   level 1  : one warp per group: each lane evaluates its query's 32 rows and, slot by slot, the warp's shuffle tree sums the group's
//              contributions in the contract's order.  Lane j stores slot j, so a group leaves one 256-byte block: about 8 B per query
//              above 256 B per touched cell, not a block per query.  The group count is known only on the device, so the scratch is sized
//              for the most groups n queries can make, min(n, ceil(n / 32) + min(n, n_cells_kept)).
//   levels   : for cells with more than 32 queries, S = 1, 32, 1024, ...: one thread per group whose offset in its cell is a multiple of
//              32 S sums, slot by slot, the <= 32 blocks S apart in place with the tree; a level no cell needs returns at once (a flag
//              the count pass sets).  After the last level the first block of a cell holds its 32 segment sums R.
//   nodes    : one thread per node over its incidences (the trainable field's table: radix_sort_pairs of (node id, 32 * cell + j)).
#include "k11_field_grad.h"
#include "radix_sort.h"
#include "dg_launch.h"
#include "shape_rows.cuh"

#include <cfloat>
#include <climits>

namespace dgb {
namespace {

constexpr unsigned K11_FULL = 0xffffffffu;
constexpr unsigned K11_EMPTY = 0xffffffffu;                        // seg_begin of a cell no query reaches
constexpr unsigned K11_MAX_BLOCKS = 4096;                          // grid-stride launches over a count known only on the device
constexpr int K11_MAX_LEVELS = 8;                                  // levels above the first: 32^7 > 2^32 groups of one cell

// K2's cell location (interpolate_kernel): false for the sentinel cases other than DBL_MAX
__device__ __forceinline__ bool k11_locate(const GridDev& g, const unsigned* __restrict__ cell_map, double x, double y, double z, unsigned& mi0,
                                           unsigned& mi1, unsigned& mi2, unsigned& cell)
{
    if (!((g.mn[0] <= x) && (x <= g.mx[0]) && (g.mn[1] <= y) && (y <= g.mx[1]) && (g.mn[2] <= z) && (z <= g.mx[2]))) return false;
    mi0 = (unsigned)((x - g.mn[0]) * g.inv[0]);
    mi1 = (unsigned)((y - g.mn[1]) * g.inv[1]);
    mi2 = (unsigned)((z - g.mn[2]) * g.inv[2]);
    if (mi0 >= g.n[0]) mi0 = g.n[0] - 1;
    if (mi1 >= g.n[1]) mi1 = g.n[1] - 1;
    if (mi2 >= g.n[2]) mi2 = g.n[2] - 1;
    const unsigned i = g.n[1] * g.n[0] * mi2 + g.n[0] * mi1 + mi0;
    cell = cell_map ? __ldg(cell_map + i) : i;
    return cell != UINT_MAX;
}

__global__ void __launch_bounds__(K11_THREADS)
k11_flags_kernel(const double* __restrict__ packed, unsigned long long n_cells, unsigned char* __restrict__ has_max)
{
    const unsigned long long c = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (c >= n_cells) return;
    bool m = false;
    for (int j = 0; j < 32; j++) m |= (packed[32 * c + j] == DBL_MAX);
    has_max[c] = m ? 1 : 0;
}

// node id of incidence idx = 32 * cell + slot
__global__ void __launch_bounds__(K11_THREADS)
k11_inc_key_kernel(GridDev g, const unsigned* __restrict__ cells, unsigned long long n32, uint32_t* __restrict__ key)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (idx >= n32) return;
    if (cells) { key[idx] = cells[idx]; return; }
    const unsigned c = (unsigned)(idx >> 5), jn = (unsigned)(idx & 31u);
    const unsigned nxy = g.n[0] * g.n[1];
    const unsigned k = c / nxy, t = c - k * nxy, j = t / g.n[0], i = t - j * g.n[0];
    key[idx] = cell_node_id(g, i, j, k, jn);
}

// inc_begin from the node ids sorted: every node id in (previous id, this id] starts here; the last position also ends the nodes above it
__global__ void __launch_bounds__(K11_THREADS)
k11_inc_begin_kernel(const uint32_t* __restrict__ skey, unsigned long long n32, unsigned long long n_nodes, uint32_t* __restrict__ inc_begin)
{
    const unsigned long long p = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (p >= n32) return;
    const unsigned long long k = skey[p];
    const unsigned long long first = p == 0 ? 0 : (unsigned long long)skey[p - 1] + 1;
    for (unsigned long long v = first; v <= k; v++) inc_begin[v] = (uint32_t)p;
    if (p + 1 == n32)
        for (unsigned long long v = k + 1; v <= n_nodes; v++) inc_begin[v] = (uint32_t)n32;
}

__global__ void __launch_bounds__(K11_THREADS)
k11_key_kernel(K11Field f, const double* __restrict__ xq, unsigned long long n, uint32_t* __restrict__ key)
{
    const unsigned long long q = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (q >= n) return;
    unsigned mi0, mi1, mi2, cell;
    const bool valid = k11_locate(f.f.g, f.f.cell_map, xq[3 * q], xq[3 * q + 1], xq[3 * q + 2], mi0, mi1, mi2, cell) && !f.has_max[cell];
    key[q] = valid ? cell + 1u : 0u;
}

__global__ void __launch_bounds__(K11_THREADS)
k11_segment_kernel(unsigned long long n, const uint32_t* __restrict__ skey, uint32_t* __restrict__ seg_begin, uint32_t* __restrict__ seg_end)
{
    const unsigned long long p = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (p >= n) return;
    const uint32_t k = skey[p];
    if (k == 0u) return;
    if (p == 0 || skey[p - 1] != k) seg_begin[k] = (uint32_t)p;
    if (p + 1 == n || skey[p + 1] != k) seg_end[k] = (uint32_t)(p + 1);
}

// the number of aligned groups of 32 queries of each key (0 for key 0, the sentinels, and for the entry past the last key); deep[L] = 1 when
// some cell has more than 32^L groups, i.e. needs the level with S = 32^L (every writer stores the same 1)
__global__ void __launch_bounds__(K11_THREADS)
k11_count_kernel(unsigned long long n_keys, const uint32_t* __restrict__ seg_begin, const uint32_t* __restrict__ seg_end, uint32_t* __restrict__ goff,
                 uint32_t* __restrict__ deep)
{
    const unsigned long long k = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (k > n_keys) return;
    const bool touched = k >= 1 && k < n_keys && seg_begin[k] != K11_EMPTY;
    const uint32_t ng = touched ? (seg_end[k] - seg_begin[k] + K11_FAN - 1) / K11_FAN : 0u;
    goff[k] = ng;
    unsigned long long S = 1;
    for (int L = 0; L < K11_MAX_LEVELS && ng > S; L++, S *= K11_FAN) deep[L] = 1u;
}

__global__ void __launch_bounds__(K11_THREADS)
k11_group_kernel(unsigned long long n, const uint32_t* __restrict__ skey, const uint32_t* __restrict__ seg_begin, const uint32_t* __restrict__ goff,
                 uint32_t* __restrict__ gstart)
{
    const unsigned long long p = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (p >= n) return;
    const uint32_t k = skey[p];
    if (k == 0u) return;
    const uint32_t off = (uint32_t)p - seg_begin[k];
    if (off % K11_FAN == 0) gstart[goff[k] + off / K11_FAN] = (uint32_t)p;
}

// level 1: one warp per group (grid-stride over the groups; *total is the group count)
__global__ void __launch_bounds__(K11_THREADS)
k11_first_level_kernel(K11Field f, const double* __restrict__ xq, const double* __restrict__ gphi, const double* __restrict__ ggrad,
                       const uint32_t* __restrict__ skey, const uint32_t* __restrict__ sval, const uint32_t* __restrict__ seg_end,
                       const uint32_t* __restrict__ gstart, const uint32_t* __restrict__ total, double* __restrict__ part)
{
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long warp0 = ((unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x) >> 5;
    const unsigned long long n_warps = ((unsigned long long)gridDim.x * K11_THREADS) >> 5;
    const unsigned long long n_groups = *total;
    const GridDev& g = f.f.g;
    for (unsigned long long grp = warp0; grp < n_groups; grp += n_warps) {            // warp-uniform
        const uint32_t p = gstart[grp];
        const uint32_t left = seg_end[skey[p]] - p;
        const unsigned m = left < K11_FAN ? left : K11_FAN;
        const unsigned long long q = sval[p + (lane < m ? lane : m - 1)];               // lanes past the group shadow its last query
        const double x = xq[3 * q], y = xq[3 * q + 1], z = xq[3 * q + 2];
        unsigned mi0 = 0, mi1 = 0, mi2 = 0, cell = 0;
        k11_locate(g, f.f.cell_map, x, y, z, mi0, mi1, mi2, cell);                       // valid: the key was not 0
        const double2 tx = __ldg(f.f.tab + mi0), ty = __ldg(f.f.tab + g.n[0] + mi1), tz = __ldg(f.f.tab + g.n[0] + g.n[1] + mi2);
        const double gp = gphi ? gphi[q] : 0.0;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        if (ggrad) { a0 = ggrad[3 * q] * tx.x; a1 = ggrad[3 * q + 1] * ty.x; a2 = ggrad[3 * q + 2] * tz.x; }
        double mine = 0.0;
        shape_rows(tx.x * x - tx.y, ty.x * y - ty.y, tz.x * z - tz.y, [&](int j, double nj, double d0, double d1, double d2) {
            double t;
            if (gphi) {
                t = gp * nj;
                if (ggrad) { t = t + a0 * d0; t = t + a1 * d1; t = t + a2 * d2; }
            } else {
                t = a0 * d0; t = t + a1 * d1; t = t + a2 * d2;
            }
#pragma unroll
            for (unsigned s = 1; s < K11_FAN; s <<= 1) {
                const double o = __shfl_down_sync(K11_FULL, t, s);
                if ((lane & (2 * s - 1)) == 0 && lane + s < m) t = t + o;
            }
            const double r = __shfl_sync(K11_FULL, t, 0);
            if (lane == (unsigned)j) mine = r;
        });
        part[grp * K11_FAN + lane] = mine;
    }
}

// one level above the first: the blocks S apart of the group that starts at grp, in place, slot by slot (grid-stride over the groups);
// returns at once when no cell needs the level (*deep == 0)
__global__ void __launch_bounds__(K11_THREADS)
k11_level_kernel(const uint32_t* __restrict__ skey, const uint32_t* __restrict__ gstart, const uint32_t* __restrict__ goff,
                 const uint32_t* __restrict__ total, const uint32_t* __restrict__ deep, unsigned long long S, double* __restrict__ part)
{
    if (*deep == 0u) return;
    const unsigned long long n_groups = *total;
    const unsigned long long stride = (unsigned long long)gridDim.x * K11_THREADS;
    for (unsigned long long grp = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x; grp < n_groups; grp += stride) {
        const uint32_t key = skey[gstart[grp]];
        const unsigned long long g0 = goff[key], ng = goff[key + 1] - g0, local = grp - g0;
        if (local % (K11_FAN * S) != 0) continue;
        const unsigned long long left = (ng - local + S - 1) / S;
        const int m = left < K11_FAN ? (int)left : (int)K11_FAN;
        if (m < 2) continue;
        for (unsigned j = 0; j < K11_FAN; j++) {
            double y[K11_FAN];
#pragma unroll
            for (int i = 0; i < (int)K11_FAN; i++) y[i] = (i < m) ? part[(grp + i * S) * K11_FAN + j] : 0.0;
#pragma unroll
            for (int s = 1; s < (int)K11_FAN; s <<= 1)
#pragma unroll
                for (int i = 0; i < (int)K11_FAN; i += 2 * s)
                    if (i + s < m) y[i] = y[i] + y[i + s];
            part[grp * K11_FAN + j] = y[0];
        }
    }
}

__global__ void __launch_bounds__(K11_THREADS)
k11_node_kernel(K11Field f, const uint32_t* __restrict__ seg_begin, const uint32_t* __restrict__ goff, const double* __restrict__ part,
                double* __restrict__ grad_nodes)
{
    const unsigned long long v = (unsigned long long)blockIdx.x * K11_THREADS + threadIdx.x;
    if (v >= f.n_nodes) return;
    double acc = 0.0;
    for (uint32_t k = f.inc_begin[v]; k < f.inc_begin[v + 1]; k++) {
        const uint32_t e = f.inc[k];
        const uint32_t key = e / K11_FAN + 1u;
        if (seg_begin[key] == K11_EMPTY) continue;                   // no query in this cell
        acc = acc + part[(unsigned long long)goff[key] * K11_FAN + e % K11_FAN];
    }
    grad_nodes[v] = acc;
}

unsigned k11_blocks(uint64_t n) { return (unsigned)((n + K11_THREADS - 1) / K11_THREADS); }
unsigned k11_stride_blocks(uint64_t threads) { const uint64_t b = (threads + K11_THREADS - 1) / K11_THREADS; return (unsigned)(b < K11_MAX_BLOCKS ? (b ? b : 1) : K11_MAX_BLOCKS); }
uint64_t k11_align(uint64_t b) { return (b + 255) & ~(uint64_t)255; }
int k11_bit_width(uint64_t v) { int b = 0; while (b < 64 && (v >> b) != 0) b++; return b > 0 ? b : 1; }
// an upper bound on the groups of n queries: each holds at least one query, and all but one per touched cell hold 32
uint64_t k11_group_bound(uint64_t n, uint64_t n_cells) { const uint64_t b = (n + K11_FAN - 1) / K11_FAN + (n < n_cells ? n : n_cells); return b < n ? b : n; }

}  // namespace

cudaError_t k11_launch_flags(const double* d_packed, uint64_t n_cells_kept, unsigned char* d_has_max, cudaStream_t stream)
{
    if (n_cells_kept == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(k11_flags_kernel, k11_blocks(n_cells_kept), K11_THREADS, 0, stream, d_packed, (unsigned long long)n_cells_kept, d_has_max);
    return DG_AFTER_LAUNCH();
}

uint64_t k11_incidence_scratch_bytes(uint64_t n_cells_kept)
{
    const uint64_t n32 = 32 * n_cells_kept;
    return 2 * k11_align(4 * n32) + radix_sort_scratch_bytes(n32);
}

cudaError_t k11_launch_incidence(const GridDev& g, const unsigned* d_cells, uint64_t n_cells_kept, uint64_t n_nodes, uint32_t* d_inc_begin,
                                 uint32_t* d_inc, void* scratch, cudaStream_t stream)
{
    const unsigned long long n32 = 32ull * n_cells_kept;
    if (n32 >= (1ull << 32)) return cudaErrorInvalidValue;
    if (n32 == 0) return cudaMemsetAsync(d_inc_begin, 0, 4 * (n_nodes + 1), stream);
    char* s = static_cast<char*>(scratch);
    uint32_t* key = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * n32);
    uint32_t* skey = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * n32);
    cudaError_t e;
    DG_KERNEL_LAUNCH(k11_inc_key_kernel, k11_blocks(n32), K11_THREADS, 0, stream, g, d_cells, n32, key);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if ((e = radix_sort_pairs(key, nullptr, n32, k11_bit_width(n_nodes ? n_nodes - 1 : 0), skey, d_inc, s, stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k11_inc_begin_kernel, k11_blocks(n32), K11_THREADS, 0, stream, skey, n32, (unsigned long long)n_nodes, d_inc_begin);
    return DG_AFTER_LAUNCH();
}

uint64_t k11_scratch_bytes(uint64_t n, uint64_t n_cells_kept)
{
    if (n == 0) return 0;
    const uint64_t keys = n_cells_kept + 1, groups = k11_group_bound(n, n_cells_kept);
    return 3 * k11_align(4 * n) + radix_sort_scratch_bytes(n) + 2 * k11_align(4 * keys) + k11_align(4 * (keys + 1)) + k11_align(4 * K11_MAX_LEVELS) +
           exclusive_scan_scratch_bytes(keys + 1) + k11_align(4 * groups) + k11_align(8 * K11_FAN * groups);
}

cudaError_t k11_launch_vjp(const K11Field& f, const double* d_x, uint64_t n, const double* d_gphi, const double* d_ggrad, double* d_grad_nodes,
                           void* scratch, cudaStream_t stream)
{
    if (!d_gphi && !d_ggrad) return cudaErrorInvalidValue;
    if (n == 0) return f.n_nodes ? cudaMemsetAsync(d_grad_nodes, 0, f.n_nodes * sizeof(double), stream) : cudaSuccess;
    if (n >= (1ull << 32) - 1) return cudaErrorInvalidValue;           // sorted positions are uint32, 0xffffffff marks an empty segment
    const uint64_t keys = f.n_cells_kept + 1, groups = k11_group_bound(n, f.n_cells_kept);
    char* s = static_cast<char*>(scratch);
    uint32_t* key = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * n);
    uint32_t* skey = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * n);
    uint32_t* sval = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * n);
    void* sort_scratch = s; s += radix_sort_scratch_bytes(n);
    uint32_t* seg_begin = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * keys);
    uint32_t* seg_end = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * keys);
    uint32_t* goff = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * (keys + 1));    // goff[keys]: the group count
    uint32_t* deep = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * K11_MAX_LEVELS);
    void* scan_scratch = s; s += exclusive_scan_scratch_bytes(keys + 1);
    uint32_t* gstart = reinterpret_cast<uint32_t*>(s); s += k11_align(4 * groups);
    double* part = reinterpret_cast<double*>(s);
    const unsigned long long nn = n;
    cudaError_t e;
    DG_KERNEL_LAUNCH(k11_key_kernel, k11_blocks(n), K11_THREADS, 0, stream, f, d_x, nn, key);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if ((e = radix_sort_pairs(key, nullptr, n, k11_bit_width(f.n_cells_kept), skey, sval, sort_scratch, stream)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(seg_begin, 0xff, 4 * keys, stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k11_segment_kernel, k11_blocks(n), K11_THREADS, 0, stream, nn, skey, seg_begin, seg_end);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(deep, 0, 4 * K11_MAX_LEVELS, stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k11_count_kernel, k11_blocks(keys + 1), K11_THREADS, 0, stream, (unsigned long long)keys, seg_begin, seg_end, goff, deep);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if ((e = exclusive_scan_u32(goff, keys + 1, scan_scratch, stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k11_group_kernel, k11_blocks(n), K11_THREADS, 0, stream, nn, skey, seg_begin, goff, gstart);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    const uint32_t* total = goff + keys;
    DG_KERNEL_LAUNCH(k11_first_level_kernel, k11_stride_blocks(32 * groups), K11_THREADS, 0, stream, f, d_x, d_gphi, d_ggrad, skey, sval, seg_end,
                     gstart, total, part);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    const unsigned long long max_groups = (nn + K11_FAN - 1) / K11_FAN;     // of one cell: the levels a call may need; deep[L] says which it does
    int L = 0;
    for (unsigned long long S = 1; S < max_groups; S *= K11_FAN, L++) {
        DG_KERNEL_LAUNCH(k11_level_kernel, k11_stride_blocks(groups), K11_THREADS, 0, stream, skey, gstart, goff, total, deep + L, S, part);
        if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    }
    if (f.n_nodes == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(k11_node_kernel, k11_blocks(f.n_nodes), K11_THREADS, 0, stream, f, seg_begin, goff, part, d_grad_nodes);
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
