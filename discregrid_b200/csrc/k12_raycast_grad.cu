// K12: the vector-Jacobian products of the two ray casts (dg_mesh_raycast_vjp, dg_field_raycast_vjp): for upstream gradients of the first
// hits of n rays, the gradients with respect to the origins, the directions and the mesh's vertices or the field's node values.  The
// forwards are K9 (k9_mesh_raycast.cu) and K7 (k7_raycast.cu), unchanged; the sums reuse K10's and K11's passes, unchanged.
//
// NUMERICAL CONTRACT (IEEE fp64, no FMA: the TU is compiled with -fmad=false; the library's own, the reference has no ray casts).  Every
// dot product is ((a0 * b0 + a1 * b1) + a2 * b2) and every cross product (a x b)_k = a_{k+1} * b_{k+2} - a_{k+2} * b_{k+1} (indices mod 3),
// each product rounded on its own.  A NULL upstream gradient is read as +0.0 in the same expressions, so it gives the bits of zeros.
//
// Mesh (K9 hit).  Per ray: direction d, t, triangle id and weights b = (b0, b1, b2) as K9 returned them; v0, v1, v2 = V[F[id][0..2]] from
// the positions V the caller passes (not the mesh's records: the mesh may have been refit since the forward); upstream g_t and g_b.
//   n   = (v1 - v0) x (v2 - v0)                    (the differences per component)
//   den = n . d,   nn = n . n
//   w_k = (g_b0 * (v2_k - v1_k) + g_b1 * (v0_k - v2_k)) + g_b2 * (v1_k - v0_k)
//   a_k = (n x w)_k / nn
//   s   = (g_t + d . a) / den
//   g_o_k = a_k - s * n_k,   g_d_k = t * g_o_k
//   A ray is valid iff id >= 0, den is finite and != 0, and nn is finite and != 0; an invalid ray gets +0.0 in g_o and g_d and takes no part
//   in the vertex sums.  A grazing ray (den small against |n| |d|) gives large but finite gradients: that is the derivative, not clamped.
//   Vertex v_i of the hit triangle receives -(b_i * g_o_k) from the ray: exactly K10's contribution with gx := g_o, so grad_vertices is K10's
//   sum (sort key id + 1, segment sums R, per-vertex fold over ascending 3t + i), see k10_distance_grad.cu.  By construction the ray's
//   contributions and g_o sum to zero up to rounding (translation invariance), and g_d = t g_o because moving d by e at fixed t moves the
//   point o + t d by t e.
//
// Field (K7 hit).  Per ray: origin o, direction d, t_lo and status as K7 returned them; upstream g_lo and g_hi of t_lo and t_hi.  Both ends
//   of the bracket follow the crossing t*, so their upstreams are added.
//   x_c_k = o_k + t_lo * d_k, clamped to [mn_k, mx_k] as K7 clamps its samples (x < mn ? mn : (x > mx ? mx : x)), so that phi(x_c) has the
//           bits K7 evaluated at t_lo; +inf in every component for a ray with status DG_RAY_MISS.
//   (phi_c, grad_c) = K2's gradient mode at x_c (k2_launch_interpolate, the kernel itself: no copy of its arithmetic)
//   den  = grad_c . d
//   gphi = -(g_lo + g_hi) / den                   (the sum negated, then divided)
//   g_o_k = gphi * grad_c_k,   g_d_k = t_lo * g_o_k
//   A ray is valid iff status != DG_RAY_MISS, phi_c is finite and != DBL_MAX, and den is finite and != 0; an invalid ray gets +0.0 in g_o,
//   g_d and gphi, and its x_c is set to +inf so that it takes no part in the node sum.
//   grad_nodes = K11's VJP (k11_launch_vjp) over the points x_c with the upstream gphi alone, on a trainable field: its contract (keys,
//   segment sums, node fold) in k11_field_grad.cu.
// The bits depend on nothing but the inputs: not on the launch geometry, the stream or the run.
//
// Passes (one thread per ray, no collectives, so tests/emu runs them as they are):
//   mesh  : k12_mesh_ray_kernel writes g_o (into grad_origins or scratch), g_d and K10's sort key; then k10_launch_scatter.
//   field : k12_field_point_kernel writes x_c; K2's gradient mode; k12_field_ray_kernel writes g_o, g_d, gphi and clears x_c of invalid
//           rays; then k11_launch_vjp.
#include "k12_raycast_grad.h"
#include "k2_interp.h"
#include "dg_launch.h"

#include <cfloat>
#include <cmath>

namespace dgb {
namespace {

constexpr int K12_MISS = 0;                                           // DG_RAY_MISS of the C-ABI

__device__ __forceinline__ double k12_dot(const double a[3], const double b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
__device__ __forceinline__ void k12_cross(const double a[3], const double b[3], double c[3])
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ bool k12_finite_nonzero(double v) { return fabs(v) <= DBL_MAX && v != 0.0; }

__global__ void __launch_bounds__(K12_THREADS)
k12_mesh_ray_kernel(K12MeshRays r, const uint32_t* __restrict__ F, double* __restrict__ go, double* __restrict__ gd, uint32_t* __restrict__ key)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * K12_THREADS + threadIdx.x;
    if (i >= r.n) return;
    const int id = r.id[i];
    double g[3] = {0.0, 0.0, 0.0};
    bool valid = id >= 0;
    if (valid) {
        const uint32_t* f = F + 3ull * (unsigned)id;
        double v0[3], v1[3], v2[3], d[3], e1[3], e2[3], n[3];
        for (int k = 0; k < 3; k++) {
            v0[k] = r.V[3ull * f[0] + k]; v1[k] = r.V[3ull * f[1] + k]; v2[k] = r.V[3ull * f[2] + k];
            d[k] = r.d[3 * i + k];
            e1[k] = v1[k] - v0[k]; e2[k] = v2[k] - v0[k];
        }
        k12_cross(e1, e2, n);
        const double den = k12_dot(n, d), nn = k12_dot(n, n);
        valid = k12_finite_nonzero(den) && k12_finite_nonzero(nn);
        if (valid) {
            const double gt = r.grad_t ? r.grad_t[i] : 0.0;
            double gb[3] = {0.0, 0.0, 0.0};
            if (r.grad_bary) for (int k = 0; k < 3; k++) gb[k] = r.grad_bary[3 * i + k];
            double w[3], c[3], a[3];
            for (int k = 0; k < 3; k++) w[k] = (gb[0] * (v2[k] - v1[k]) + gb[1] * (v0[k] - v2[k])) + gb[2] * (v1[k] - v0[k]);
            k12_cross(n, w, c);
            for (int k = 0; k < 3; k++) a[k] = c[k] / nn;
            const double s = (gt + k12_dot(d, a)) / den;
            for (int k = 0; k < 3; k++) g[k] = a[k] - s * n[k];
        }
    }
    if (go) for (int k = 0; k < 3; k++) go[3 * i + k] = g[k];
    if (gd) {
        const double t = r.t[i];
        for (int k = 0; k < 3; k++) gd[3 * i + k] = valid ? t * g[k] : 0.0;
    }
    if (key) key[i] = valid ? (uint32_t)id + 1u : 0u;
}

__global__ void __launch_bounds__(K12_THREADS)
k12_field_point_kernel(GridDev g, K12FieldRays r, double* __restrict__ xc)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * K12_THREADS + threadIdx.x;
    if (i >= r.n) return;
    const bool hit = r.status[i] != K12_MISS;
    const double t = r.t_lo[i];
    for (int a = 0; a < 3; a++) {
        const double x = r.o[3 * i + a] + t * r.d[3 * i + a];
        xc[3 * i + a] = hit ? (x < g.mn[a] ? g.mn[a] : (x > g.mx[a] ? g.mx[a] : x)) : INFINITY;
    }
}

__global__ void __launch_bounds__(K12_THREADS)
k12_field_ray_kernel(K12FieldRays r, const double* __restrict__ phi, const double* __restrict__ grad, double* __restrict__ go,
                     double* __restrict__ gd, double* __restrict__ gphi, double* __restrict__ xc)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * K12_THREADS + threadIdx.x;
    if (i >= r.n) return;
    const double p = phi[i];
    double gr[3], d[3];
    for (int k = 0; k < 3; k++) { gr[k] = grad[3 * i + k]; d[k] = r.d[3 * i + k]; }
    const double den = k12_dot(gr, d);
    const bool valid = r.status[i] != K12_MISS && fabs(p) <= DBL_MAX && p != DBL_MAX && k12_finite_nonzero(den);
    double gp = 0.0, g[3] = {0.0, 0.0, 0.0};
    if (valid) {
        const double sum = (r.grad_t_lo ? r.grad_t_lo[i] : 0.0) + (r.grad_t_hi ? r.grad_t_hi[i] : 0.0);
        gp = -sum / den;
        for (int k = 0; k < 3; k++) g[k] = gp * gr[k];
    }
    if (go) for (int k = 0; k < 3; k++) go[3 * i + k] = g[k];
    if (gd) {
        const double t = r.t_lo[i];
        for (int k = 0; k < 3; k++) gd[3 * i + k] = valid ? t * g[k] : 0.0;
    }
    if (gphi) {
        gphi[i] = gp;
        if (!valid) for (int k = 0; k < 3; k++) xc[3 * i + k] = INFINITY;
    }
}

unsigned k12_blocks(uint64_t n) { return (unsigned)((n + K12_THREADS - 1) / K12_THREADS); }
uint64_t k12_align(uint64_t b) { return (b + 255) & ~(uint64_t)255; }

}  // namespace

uint64_t k12_mesh_scratch_bytes(uint64_t n, int n_tri, bool grad_origins, bool grad_vertices)
{
    if (!grad_vertices || n == 0) return 0;
    return (grad_origins ? 0 : k12_align(24 * n)) + k12_align(4 * n) + k10_scatter_scratch_bytes(n, n_tri);   // g_o, keys, K10's
}

cudaError_t k12_launch_mesh_vjp(const K10Topo& topo, const K12MeshRays& r, double* d_grad_origins, double* d_grad_directions,
                                double* d_grad_vertices, void* scratch, cudaStream_t stream)
{
    const uint64_t n = r.n;
    if (n >= (1ull << 32) - 1) return cudaErrorInvalidValue;            // K10's sorted positions are uint32
    if (!d_grad_vertices) {
        if (n == 0 || (!d_grad_origins && !d_grad_directions)) return cudaSuccess;
        DG_KERNEL_LAUNCH(k12_mesh_ray_kernel, k12_blocks(n), K12_THREADS, 0, stream, r, topo.F, d_grad_origins, d_grad_directions,
                         (uint32_t*)nullptr);
        return DG_AFTER_LAUNCH();
    }
    if (n == 0) return cudaMemsetAsync(d_grad_vertices, 0, 3 * topo.n_vertices * sizeof(double), stream);
    char* s = static_cast<char*>(scratch);
    double* go = d_grad_origins;
    if (!go) { go = reinterpret_cast<double*>(s); s += k12_align(24 * n); }
    uint32_t* key = reinterpret_cast<uint32_t*>(s); s += k12_align(4 * n);
    DG_KERNEL_LAUNCH(k12_mesh_ray_kernel, k12_blocks(n), K12_THREADS, 0, stream, r, topo.F, go, d_grad_directions, key);
    const cudaError_t e = DG_AFTER_LAUNCH();
    if (e != cudaSuccess) return e;
    return k10_launch_scatter(topo, n, go, key, r.bary, d_grad_vertices, s, stream);
}

uint64_t k12_field_scratch_bytes(uint64_t n, uint64_t n_cells_kept, bool grad_nodes)
{
    if (n == 0) return 0;
    uint64_t b = k12_align(24 * n) + k12_align(8 * n) + k12_align(24 * n);                   // x_c, phi_c, grad_c
    if (grad_nodes) b += k12_align(8 * n) + k11_scratch_bytes(n, n_cells_kept);            // gphi, K11's
    return b;
}

cudaError_t k12_launch_field_vjp(const FieldDev& f, const K11Field* tf, const K12FieldRays& r, double* d_grad_origins, double* d_grad_directions,
                                 double* d_grad_nodes, void* scratch, cudaStream_t stream)
{
    const uint64_t n = r.n;
    if (d_grad_nodes && !tf) return cudaErrorInvalidValue;
    if (n >= (1ull << 32) - 1) return cudaErrorInvalidValue;            // K11's sorted positions are uint32
    if (n == 0) return d_grad_nodes && tf->n_nodes ? cudaMemsetAsync(d_grad_nodes, 0, tf->n_nodes * sizeof(double), stream) : cudaSuccess;
    if (!d_grad_origins && !d_grad_directions && !d_grad_nodes) return cudaSuccess;
    char* s = static_cast<char*>(scratch);
    double* xc = reinterpret_cast<double*>(s); s += k12_align(24 * n);
    double* phi = reinterpret_cast<double*>(s); s += k12_align(8 * n);
    double* grad = reinterpret_cast<double*>(s); s += k12_align(24 * n);
    double* gphi = nullptr;
    if (d_grad_nodes) { gphi = reinterpret_cast<double*>(s); s += k12_align(8 * n); }
    cudaError_t e;
    DG_KERNEL_LAUNCH(k12_field_point_kernel, k12_blocks(n), K12_THREADS, 0, stream, f.g, r, xc);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if ((e = k2_launch_interpolate(f, xc, n, phi, grad, stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k12_field_ray_kernel, k12_blocks(n), K12_THREADS, 0, stream, r, phi, grad, d_grad_origins, d_grad_directions, gphi, xc);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if (!d_grad_nodes) return cudaSuccess;
    return k11_launch_vjp(*tf, xc, n, gphi, nullptr, d_grad_nodes, s, stream);
}

}  // namespace dgb
