// K13: the vector-Jacobian product of K6's level-set extraction (dg_isosurface_vjp): for the upstream gradient of the extracted vertex
// positions, the gradient with respect to the node values of a trainable field.  The forward is K6 (k6_isosurface.cu), unchanged apart from
// the edge id it keeps beside every vertex; the lattice values are K2's value-only kernel and the node sums K11's, both called as they are.
//
// NUMERICAL CONTRACT (IEEE fp64, no FMA: the TU is compiled with -fmad=false; the library's own, the reference has no level sets).
// Inputs: a trainable field holding the forward's node values, iso and s as given to the forward, n edge ids and the upstream gV[n][3].
// Lattice.  K6's, k6_lattice(field grid, s).  Refused before anything is written: iso not finite, s outside 1..16, a lattice of 2^31 points
//   or more, and any edge id that is not an edge of the lattice: lin(p) >= Np, or q = p + delta_d leaves the lattice on some axis (checked
//   on the device by k13_launch_check, one synchronise in the caller).
// Endpoints of vertex v.  p = e / 7, d = e % 7, q = p + delta_d.  x_p,a = lat_coord(a, I_a) and x_q,a = lat_coord(a, I_a + delta_d,a): K6's
//   own function (k6_isosurface.h), so K6's bits.  f_p and f_q are K2's value-only interpolate at x_p and x_q on the field's current values
//   (k2_launch_interpolate, the kernel itself), the bits of the forward's lattice values.
// Per vertex, each product and difference rounded on its own:
//   delta  = f_q - f_p
//   t      = (iso - f_p) / delta                                          (K6's bits of t)
//   g_t    = (gV0 * (x_q,0 - x_p,0) + gV1 * (x_q,1 - x_p,1)) + gV2 * (x_q,2 - x_p,2)
//   r      = g_t / delta
//   gphi_p = (t - 1.0) * r,   gphi_q = -(t * r)
//   from dt/df_p = (t - 1) / delta and dt/df_q = -t / delta.  A vertex is valid iff f_p and f_q are finite and != DBL_MAX, delta is finite and
//   != 0, and t is finite; an invalid vertex gets +0.0 at both endpoints and its two points are set to +inf, so that K11 skips them.  An
//   upstream that is not finite is not clamped: the arithmetic gives what it gives.
// Node sums.  grad_nodes is K11's VJP (k11_launch_vjp) over 2n queries: query 2v is x_p with upstream gphi_p, query 2v + 1 is x_q with
//   upstream gphi_q, the upstream is gphi alone.  K11's stable sort by cell, its tree R and its node fold fix the order (k11_field_grad.cu);
//   K11's sorted positions are uint32, so 2n < 2^32 - 1.
// The bits depend on nothing but the inputs (the field's topology and values, iso, s, the edge ids and gV): not on the launch geometry, the
// stream or the run.  First order only; not differentiable in iso; the triangle connectivity is piecewise constant and carries no gradient.
//
// Passes (one thread per edge id or vertex, no collectives apart from the check's ballot, so tests/emu runs them as they are): the edge-id
// check; k13_points_kernel writes the 2n endpoints; K2's value-only launch; k13_vertex_kernel writes gphi and sets the points of invalid
// vertices to +inf; k11_launch_vjp.
#include "k13_isosurface_grad.h"
#include "k2_interp.h"
#include "dg_launch.h"

#include <cfloat>
#include <cmath>

namespace dgb {
namespace {

__device__ __forceinline__ bool k13_finite(double v) { return fabs(v) <= DBL_MAX; }

__global__ void __launch_bounds__(K13_THREADS)
k13_check_kernel(K6Lattice L, const unsigned long long* __restrict__ edges, unsigned long long n, unsigned* __restrict__ bad)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * K13_THREADS + threadIdx.x;
    bool b = false;
    if (i < n) {
        const unsigned long long e = edges[i], lp = e / 7ull;
        const unsigned long long np = (unsigned long long)L.np[0] * L.np[1] * L.np[2];
        if (lp >= np) {
            b = true;
        } else {
            const unsigned l = (unsigned)lp, m = mask_of_dir((unsigned)(e % 7ull));
            const unsigned I = l % L.np[0], r = l / L.np[0], J = r % L.np[1], K = r / L.np[1];
            b = I + (m & 1u) >= L.np[0] || J + ((m >> 1) & 1u) >= L.np[1] || K + (m >> 2) >= L.np[2];
        }
    }
    const unsigned w = __ballot_sync(0xffffffffu, b);
    if (w && (threadIdx.x & 31u) == 0u) atomicAdd(bad, (unsigned)__popc(w));
}

// x[6 v .. 6 v + 2] = x_p, x[6 v + 3 .. 6 v + 5] = x_q
__global__ void __launch_bounds__(K13_THREADS)
k13_points_kernel(K6Lattice L, const unsigned long long* __restrict__ edges, unsigned long long n, double* __restrict__ x)
{
    const unsigned long long v = (unsigned long long)blockIdx.x * K13_THREADS + threadIdx.x;
    if (v >= n) return;
    const unsigned long long e = edges[v];
    const unsigned lp = (unsigned)(e / 7ull), dm = mask_of_dir((unsigned)(e % 7ull));
    const unsigned I = lp % L.np[0], r = lp / L.np[0], J = r % L.np[1], K = r / L.np[1];
    const unsigned ip[3] = {I, J, K};
    for (int a = 0; a < 3; a++) {
        x[6 * v + a] = lat_coord(L, a, ip[a]);
        x[6 * v + 3 + a] = lat_coord(L, a, ip[a] + ((dm >> a) & 1u));
    }
}

__global__ void __launch_bounds__(K13_THREADS)
k13_vertex_kernel(double iso, const double* __restrict__ f, const double* __restrict__ gV, unsigned long long n, double* __restrict__ x,
                  double* __restrict__ gphi)
{
    const unsigned long long v = (unsigned long long)blockIdx.x * K13_THREADS + threadIdx.x;
    if (v >= n) return;
    const double fp = f[2 * v], fq = f[2 * v + 1];
    const double delta = fq - fp;
    const double t = (iso - fp) / delta;
    const bool valid = k13_finite(fp) && fp != DBL_MAX && k13_finite(fq) && fq != DBL_MAX && k13_finite(delta) && delta != 0.0 && k13_finite(t);
    double gp = 0.0, gq = 0.0;
    if (valid) {
        double dx[3];
        for (int a = 0; a < 3; a++) dx[a] = x[6 * v + 3 + a] - x[6 * v + a];
        const double gt = (gV[3 * v] * dx[0] + gV[3 * v + 1] * dx[1]) + gV[3 * v + 2] * dx[2];
        const double r = gt / delta;
        gp = (t - 1.0) * r;
        gq = -(t * r);
    } else {
        for (int k = 0; k < 6; k++) x[6 * v + k] = INFINITY;
    }
    gphi[2 * v] = gp;
    gphi[2 * v + 1] = gq;
}

unsigned k13_blocks(uint64_t n) { return (unsigned)((n + K13_THREADS - 1) / K13_THREADS); }
uint64_t k13_align(uint64_t b) { return (b + 255) & ~(uint64_t)255; }

}  // namespace

cudaError_t k13_launch_check(const K6Lattice& L, const uint64_t* d_edge_ids, uint64_t n, unsigned* d_bad, cudaStream_t stream)
{
    cudaError_t e = cudaMemsetAsync(d_bad, 0, sizeof(unsigned), stream);
    if (e != cudaSuccess || n == 0) return e;
    DG_KERNEL_LAUNCH(k13_check_kernel, k13_blocks(n), K13_THREADS, 0, stream, L, reinterpret_cast<const unsigned long long*>(d_edge_ids),
                     (unsigned long long)n, d_bad);
    return DG_AFTER_LAUNCH();
}

uint64_t k13_scratch_bytes(uint64_t n, uint64_t n_cells_kept)
{
    if (n == 0) return 0;
    return k13_align(48 * n) + 2 * k13_align(16 * n) + k11_scratch_bytes(2 * n, n_cells_kept);   // points, values, gphi, K11's
}

cudaError_t k13_launch_vjp(const K11Field& tf, const K6Lattice& L, double iso, const uint64_t* d_edge_ids, uint64_t n,
                           const double* d_grad_vertices, double* d_grad_nodes, void* scratch, cudaStream_t stream)
{
    if (2 * n >= (1ull << 32) - 1) return cudaErrorInvalidValue;       // K11's sorted positions are uint32
    if (n == 0) return tf.n_nodes ? cudaMemsetAsync(d_grad_nodes, 0, tf.n_nodes * sizeof(double), stream) : cudaSuccess;
    const unsigned long long* edges = reinterpret_cast<const unsigned long long*>(d_edge_ids);
    char* s = static_cast<char*>(scratch);
    double* x = reinterpret_cast<double*>(s); s += k13_align(48 * n);
    double* f = reinterpret_cast<double*>(s); s += k13_align(16 * n);
    double* gphi = reinterpret_cast<double*>(s); s += k13_align(16 * n);
    cudaError_t e;
    DG_KERNEL_LAUNCH(k13_points_kernel, k13_blocks(n), K13_THREADS, 0, stream, L, edges, (unsigned long long)n, x);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    if ((e = k2_launch_interpolate(tf.f, x, 2 * n, f, nullptr, stream)) != cudaSuccess) return e;
    DG_KERNEL_LAUNCH(k13_vertex_kernel, k13_blocks(n), K13_THREADS, 0, stream, iso, f, d_grad_vertices, (unsigned long long)n, x, gphi);
    if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;
    return k11_launch_vjp(tf, x, 2 * n, gphi, nullptr, d_grad_nodes, s, stream);
}

}  // namespace dgb
