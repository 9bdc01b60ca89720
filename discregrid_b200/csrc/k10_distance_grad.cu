// K10: the vector-Jacobian product of the mesh distance (dg_mesh_distance_vjp): for an upstream gradient g of the distances of n queries,
// the gradient with respect to the query points and the deterministic gradient with respect to the mesh's vertices.  The forward that
// feeds it is K1's: mesh_distance_bary_kernel (k1_sdf.cu), a separate __global__ next to mesh_distance_kernel with the same inlined walk
// and finish_query, which also writes the weights; mesh_distance_kernel itself is unchanged.
//
// NUMERICAL CONTRACT (fp64, no FMA: the TU is compiled with -fmad=false).  Per query q: point x, and as dg_mesh_distance[_bary] returned
// them (either sign mode) the distance d, nearest point p, triangle id t (-1: none) and weights w; upstream gradient g.
//   Weights (K1): w = (fl(fl(1 - s) - t), s, t) on the vertex slots F[t][0], F[t][1], F[t][2], with (s, t) exactly the values tri_dist2
//       produced for the winning leaf, so that p = v0 + s e0 + t e1 as finish_query computes it (leaf records: v0 = V[F[t][0]],
//       e0 = V[F[t][1]] - v0, e1 = V[F[t][2]] - v0).  NaN when t = -1.
//   d(d)/dx = (x - p) / d (the sign of d is the sign; in the winding mode the sign is piecewise constant):
//       gx[q][k] = fl(fl(g / d) * fl(x_k - p_k)), k = 0, 1, 2;  +0.0 when t == -1 or d == 0.
//   d(d)/dV[F[t][i]] = -w_i d(d)/dx (envelope theorem): the contribution of q to slot i of its triangle is c[q][i][k] = -fl(w_i * gx[q][k]).
//   Segments: the queries with t >= 0, stably sorted by t (so in ascending q within a triangle); the segment of (t, i) is the list of
//       c[q][i] over those queries, in that order.
//   Segment sum R: while the list has more than one entry, replace each aligned group of 32 consecutive entries (the last may be shorter)
//       by its tree sum; the one entry left is R.  Tree sum of y_0 .. y_{m-1}: for s = 1, 2, 4, 8, 16, y_j = y_j + y_{j+s} for every j
//       that is a multiple of 2s with j + s < m; the result is y_0.  (The groups above the first level are summed by the same tree rather
//       than left to right, so that a segment of n queries -- every query on one triangle -- takes log_32 n dependent steps, not n / 32.)
//   grad_vertices[v][k] = ((+0.0 + R_1) + R_2) + ..., R_j the segment sum of the j-th non-empty (t, i) among v's incidences in K8's order
//       (inc_begin[v] .. inc_begin[v + 1], ascending 3t + i); 0 for a vertex that receives nothing.
// The bits therefore depend on nothing but the inputs: not on the launch geometry, the stream or the run.  The backward reads no vertex
// position, so a gradient is right even when the mesh was refit again after the forward.
//
// Passes (all data-parallel; the sort is radix_sort.cu, warp-synchronous like K4, so tests/emu runs every pass):
//   point    : one thread per query: gx (into grad_points or scratch) and the sort key t + 1 (0 for t = -1, which the sort puts first).
//   sort     : radix_sort_pairs of the keys with the query indices, ceil(bit_width(T) / 8) passes.
//   contrib  : one thread per sorted position: the 9 values c[q][i][k], stored [3i + k][position] (coalesced).
//   segments : the first and last sorted position of each triangle.
//   levels   : for S = 1, 32, 1024, ... < n, one thread per sorted position whose offset in its segment is a multiple of 32 S sums the
//              <= 32 entries S apart in place with the tree.  After the last level a segment's sum sits at its first position.
//   vertices : one thread per vertex over its incidences.
// The passes after the point pass are k10_launch_scatter, which K12 (k12_raycast_grad.cu) calls with its own per-ray gradients and keys.
#include "k10_distance_grad.h"
#include "radix_sort.h"
#include "dg_launch.h"

namespace dgb {
namespace {

__global__ void __launch_bounds__(K10_THREADS)
k10_check_kernel(const int32_t* __restrict__ tri, unsigned long long n, int n_tri, unsigned* __restrict__ bad)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * K10_THREADS + threadIdx.x;
    const int t = idx < n ? tri[idx] : -1;
    const unsigned b = __ballot_sync(0xffffffffu, t < -1 || t >= n_tri);
    if (b && (threadIdx.x & 31u) == 0u) atomicAdd(bad, (unsigned)__popc(b));
}

__global__ void __launch_bounds__(K10_THREADS)
k10_point_kernel(K10Query q, double* __restrict__ gx, uint32_t* __restrict__ key)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * K10_THREADS + threadIdx.x;
    if (i >= q.n) return;
    const int t = q.tri[i];
    const double d = q.dist[i];
    double o[3] = {0.0, 0.0, 0.0};
    if (t >= 0 && d != 0.0) {
        const double s = q.g[i] / d;
        for (int k = 0; k < 3; k++) o[k] = s * (q.x[3 * i + k] - q.near[3 * i + k]);
    }
    if (gx) for (int k = 0; k < 3; k++) gx[3 * i + k] = o[k];
    if (key) key[i] = t >= 0 ? (uint32_t)t + 1u : 0u;
}

__global__ void __launch_bounds__(K10_THREADS)
k10_contrib_kernel(unsigned long long n, const uint32_t* __restrict__ skey, const uint32_t* __restrict__ sval, const double* __restrict__ gx,
                   const double* __restrict__ bary, double* __restrict__ c)
{
    const unsigned long long p = (unsigned long long)blockIdx.x * K10_THREADS + threadIdx.x;
    if (p >= n || skey[p] == 0u) return;
    const unsigned long long q = sval[p];
    const double g[3] = {gx[3 * q], gx[3 * q + 1], gx[3 * q + 2]};
    for (int i = 0; i < 3; i++) {
        const double w = bary[3 * q + i];
        for (int k = 0; k < 3; k++) c[(unsigned long long)(3 * i + k) * n + p] = -(w * g[k]);
    }
}

__global__ void __launch_bounds__(K10_THREADS)
k10_segment_kernel(unsigned long long n, const uint32_t* __restrict__ skey, uint32_t* __restrict__ seg_begin, uint32_t* __restrict__ seg_end)
{
    const unsigned long long p = (unsigned long long)blockIdx.x * K10_THREADS + threadIdx.x;
    if (p >= n) return;
    const uint32_t k = skey[p];
    if (k == 0u) return;
    if (p == 0 || skey[p - 1] != k) seg_begin[k] = (uint32_t)p;
    if (p + 1 == n || skey[p + 1] != k) seg_end[k] = (uint32_t)(p + 1);
}

// one level of the segment sums: the group of 32 entries S apart that starts at p, in place
__global__ void __launch_bounds__(K10_THREADS)
k10_level_kernel(unsigned long long n, const uint32_t* __restrict__ skey, const uint32_t* __restrict__ seg_begin,
                 const uint32_t* __restrict__ seg_end, unsigned long long S, double* __restrict__ c)
{
    const unsigned long long p = (unsigned long long)blockIdx.x * K10_THREADS + threadIdx.x;
    if (p >= n) return;
    const uint32_t key = skey[p];
    if (key == 0u) return;
    const unsigned long long b = seg_begin[key], e = seg_end[key];
    if ((p - b) % (K10_FAN * S) != 0) return;
    const unsigned long long left = (e - p + S - 1) / S;              // entries of the group
    const int m = left < K10_FAN ? (int)left : (int)K10_FAN;
    if (m < 2) return;
    for (int r = 0; r < 9; r++) {
        double* row = c + (unsigned long long)r * n + p;
        double y[K10_FAN];
#pragma unroll
        for (int j = 0; j < (int)K10_FAN; j++) y[j] = (j < m) ? row[j * S] : 0.0;
#pragma unroll
        for (int s = 1; s < (int)K10_FAN; s <<= 1)
#pragma unroll
            for (int j = 0; j < (int)K10_FAN; j += 2 * s)
                if (j + s < m) y[j] = y[j] + y[j + s];
        row[0] = y[0];
    }
}

__global__ void __launch_bounds__(K10_THREADS)
k10_vertex_kernel(K10Topo topo, unsigned long long n, const uint32_t* __restrict__ seg_begin, const double* __restrict__ c,
                  double* __restrict__ gv)
{
    const unsigned long long v = (unsigned long long)blockIdx.x * K10_THREADS + threadIdx.x;
    if (v >= topo.n_vertices) return;
    double acc[3] = {0.0, 0.0, 0.0};
    for (uint32_t k = topo.inc_begin[v]; k < topo.inc_begin[v + 1]; k++) {
        const uint32_t qi = topo.inc[k];
        const uint32_t b = seg_begin[qi / 3 + 1];
        if (b == 0xffffffffu) continue;                                // no query on this triangle
        const unsigned slot = qi % 3;
        for (int d = 0; d < 3; d++) acc[d] = acc[d] + c[(unsigned long long)(3 * slot + d) * n + b];
    }
    for (int d = 0; d < 3; d++) gv[3 * v + d] = acc[d];
}

unsigned k10_blocks(uint64_t n) { return (unsigned)((n + K10_THREADS - 1) / K10_THREADS); }
uint64_t k10_align(uint64_t b) { return (b + 255) & ~(uint64_t)255; }
int k10_key_bits(int n_tri) { int b = 0; while (b < 32 && ((uint64_t)n_tri >> b) != 0) b++; return b > 0 ? b : 1; }     // keys 0 .. T

}  // namespace

cudaError_t k10_launch_check(const int32_t* d_tri, uint64_t n, int n_tri, unsigned* d_bad, cudaStream_t stream)
{
    cudaError_t e = cudaMemsetAsync(d_bad, 0, sizeof(unsigned), stream);
    if (e != cudaSuccess || n == 0) return e;
    DG_KERNEL_LAUNCH(k10_check_kernel, k10_blocks(n), K10_THREADS, 0, stream, d_tri, (unsigned long long)n, n_tri, d_bad);
    return DG_AFTER_LAUNCH();
}

uint64_t k10_scatter_scratch_bytes(uint64_t n, int n_tri)
{
    if (n == 0) return 0;
    uint64_t b = 2 * k10_align(4 * n) + radix_sort_scratch_bytes(n);  // sorted keys, sorted query ids, the sort's own
    b += k10_align(72 * n) + 2 * k10_align(4 * ((uint64_t)n_tri + 1));
    return b;
}

uint64_t k10_scratch_bytes(uint64_t n, int n_tri, bool grad_points, bool grad_vertices)
{
    if (!grad_vertices || n == 0) return 0;
    uint64_t b = grad_points ? 0 : k10_align(24 * n);                 // gx when grad_points is not wanted
    return b + k10_align(4 * n) + k10_scatter_scratch_bytes(n, n_tri); // keys, then the scatter's
}

cudaError_t k10_launch_vjp(const K10Topo& topo, const K10Query& q, double* d_grad_points, double* d_grad_vertices, void* scratch,
                           cudaStream_t stream)
{
    const uint64_t n = q.n;
    cudaError_t e;
    if (!d_grad_vertices) {
        if (n == 0 || !d_grad_points) return cudaSuccess;
        DG_KERNEL_LAUNCH(k10_point_kernel, k10_blocks(n), K10_THREADS, 0, stream, q, d_grad_points, (uint32_t*)nullptr);
        return DG_AFTER_LAUNCH();
    }
    if (n == 0) return cudaMemsetAsync(d_grad_vertices, 0, 3 * topo.n_vertices * sizeof(double), stream);
    if (n >= (1ull << 32) - 1) return cudaErrorInvalidValue;           // sorted positions are uint32, 0xffffffff marks an empty segment
    char* s = static_cast<char*>(scratch);
    double* gx = d_grad_points;
    if (!gx) { gx = reinterpret_cast<double*>(s); s += k10_align(24 * n); }
    uint32_t* key = reinterpret_cast<uint32_t*>(s); s += k10_align(4 * n);
    DG_KERNEL_LAUNCH(k10_point_kernel, k10_blocks(n), K10_THREADS, 0, stream, q, gx, key);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    return k10_launch_scatter(topo, n, gx, key, q.bary, d_grad_vertices, s, stream);
}

cudaError_t k10_launch_scatter(const K10Topo& topo, uint64_t n, const double* gx, const uint32_t* key, const double* bary,
                               double* d_grad_vertices, void* scratch, cudaStream_t stream)
{
    cudaError_t e;
    if (n == 0) return cudaMemsetAsync(d_grad_vertices, 0, 3 * topo.n_vertices * sizeof(double), stream);
    if (n >= (1ull << 32) - 1) return cudaErrorInvalidValue;           // sorted positions are uint32, 0xffffffff marks an empty segment
    char* s = static_cast<char*>(scratch);
    uint32_t* skey = reinterpret_cast<uint32_t*>(s); s += k10_align(4 * n);
    uint32_t* sval = reinterpret_cast<uint32_t*>(s); s += k10_align(4 * n);
    void* sort_scratch = s; s += radix_sort_scratch_bytes(n);
    double* c = reinterpret_cast<double*>(s); s += k10_align(72 * n);
    uint32_t* seg_begin = reinterpret_cast<uint32_t*>(s); s += k10_align(4 * ((uint64_t)topo.n_tri + 1));
    uint32_t* seg_end = reinterpret_cast<uint32_t*>(s);
    const unsigned long long nn = n;
    if ((e = radix_sort_pairs(key, nullptr, n, k10_key_bits(topo.n_tri), skey, sval, sort_scratch, stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k10_contrib_kernel, k10_blocks(n), K10_THREADS, 0, stream, nn, skey, sval, gx, bary, c);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(seg_begin, 0xff, 4 * ((size_t)topo.n_tri + 1), stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k10_segment_kernel, k10_blocks(n), K10_THREADS, 0, stream, nn, skey, seg_begin, seg_end);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    for (unsigned long long S = 1; S < nn; S *= K10_FAN) {
        DG_KERNEL_LAUNCH(k10_level_kernel, k10_blocks(n), K10_THREADS, 0, stream, nn, skey, seg_begin, seg_end, S, c);
        if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    }
    if (topo.n_vertices == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(k10_vertex_kernel, k10_blocks(topo.n_vertices), K10_THREADS, 0, stream, topo, nn, seg_begin, c, d_grad_vertices);
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
