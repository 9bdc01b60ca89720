// K3: the per-node function of GenerateDensityMap, one grid node per lane.
//
// Replaces addFunction(density_func, verbose, pred) of cmd/generate_density_map/main.cpp:96-133:
//   pred(x)        : clamp x into the domain, d = interpolate(0, x); reject if d == DBL_MAX, else keep iff
//                    -6h < d + cell_diag && d - cell_diag < 2h                                  (:119-133)
//   density_func(x): d = interpolate(0, x); 0 if d > 2h, else rho0 * GaussQuadrature::integrate(
//                    xi -> gamma(x + xi) * W(xi), [-h,h]^3, p = 30)                               (:96-112)
//   gamma(y)       : d = interpolate(0, y); (d > h) ? 0 : 1 - d/h                                (:86-93)
//   integrate      : 16 x 16 x 16 Gauss points, i (x) outermost, k (z) innermost, ONE sequential accumulator
//                    res += (wi*wj*wk) * f(c0*xi + c1); res *= c0.prod()     (gauss_quadrature.cpp:5927-5960)
//   W              : cubic spline, sph_kernel.hpp:22-42
//
// The 4096-term sum is sequential in the reference, so for bit-exact parity one lane owns one node and walks
// the 4096 points in order; parallelism comes from the 10^8 nodes.  Everything that does not depend on the
// node is tabulated on the host with the reference's operation order: the 16 offsets c0*xi+c1 per axis, the
// 16 weights, and W at the 4096 points (constant / global memory).  The 32 adjacent nodes of a warp sample 32
// adjacent points at every step, i.e. one to three cells, so the 256-byte coefficient blocks are L1 hits.
//
// Points with W == 0 (outside the kernel support, ~48 % of the cube) add wijk * (gamma * 0).  That is +-0, which
// leaves the accumulator unchanged (it starts at +0 and every term is >= 0), only while gamma is finite; the
// reference adds NaN where gamma = 1 - d/h is +inf (d/h overflowed to -inf) or NaN (d is NaN), and a field may
// hold anything (dg_field_create does not look at values, a .cdf may hold NaN, inf or -DBL_MAX).  So the
// skipping kernel (SKIP_ZERO_W) runs only when gamma is finite at every point by construction:
//   * M = max |c| over the field's packed coefficients c != DBL_MAX, with M = +inf if one of them is NaN or
//     +-inf (k3_coeff_max, once per field).  A cell holding a DBL_MAX coefficient interpolates to DBL_MAX
//     whatever its other terms are, and d = DBL_MAX > h gives gamma = 0, or 1 - DBL_MAX/inf = 1 for h = inf.
//   * Otherwise d = sum_j c_j N_j(X) over a cell's 32 coefficients with X in [-1, 1]^3 up to rounding, and
//     sum_j |N_j| <= 8 there: the 8 corner functions facc (1+-x)(1+-y)(1+-z) with |facc| <= 19/64 sum to at
//     most 8 * 19/64 < 2.4 (the products sum to 8); the 8 edge functions along x, 9/64 (1-x^2)(1+-3x)(1+-y)(1+-z),
//     to 9/64 * 4 * (1-x^2) * 2 max(1, 3|x|) <= 9/64 * 4 * 4/sqrt(3) < 1.3, likewise along y and z.  Total < 6.3.
//     Each product and partial sum is then below 8 M (1 + 1e-14), so with 64 M < DBL_MAX every partial sum
//     and d are finite, and |d / h| <= 8 M / h < DBL_MAX when 64 M / h < DBL_MAX: gamma is finite.
// k3_launch_density takes M and picks the instantiation; a field that fails the bound (or h too small for
// it) samples all 4096 points as the reference does.
#include "dg_device.cuh"
#include "k3_density.h"
#include "fast_div.h"
#include "dg_launch.h"

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

namespace dgb {

namespace {

// cmd/generate_density_map/gauss_quadrature.cpp:616-632 (abscissae, p = 30) and :3422-3438 (weights); n = 16 (:100-101)
const double GA16[16] = {
    -0.989400934991649938510249739920, -0.944575023073232600268056557979, -0.865631202387831755196145877562,
    -0.755404408355002998654015300417, -0.617876244402643770570193737512, -0.458016777657227369680015272024,
    -0.281603550779258915426339626720, -0.095012509837637426635126303154, 0.095012509837637426635126303154,
    0.281603550779258915426339626720, 0.458016777657227369680015272024, 0.617876244402643770570193737512,
    0.755404408355002998654015300417, 0.865631202387831755196145877562, 0.944575023073232600268056557979,
    0.989400934991649938510249739920};
const double GW16[16] = {
    0.027152459411758110563450685504, 0.062253523938649010793788818319, 0.095158511682492036287683845330,
    0.124628971255533488315947465708, 0.149595988816575764523975067277, 0.169156519395001675443168664970,
    0.182603415044922529064663763165, 0.189450610455067447457366824892, 0.189450610455067447457366824892,
    0.182603415044922529064663763165, 0.169156519395001675443168664970, 0.149595988816575764523975067277,
    0.124628971255533488315947465708, 0.095158511682492036287683845330, 0.062253523938649010793788818319,
    0.027152459411758110563450685504};

struct QuadParams {
    double off[16];      // c0*xi + c1 per axis point (identical on the three axes: the domain is a cube)
    double w[16];
    double h, two_h, six_h_neg, rho0, c0prod, cell_diag;
    double inv_h;        // RN(1/h)
};

// value-only interpolate (cubic_lagrange_discrete_grid.cpp:977-1023) reading the packed block through L1
__device__ __forceinline__ double interp_value(const FieldDev& f, double x, double y, double z)
{
    const GridDev& g = f.g;
    if (!((g.mn[0] <= x) && (x <= g.mx[0]) && (g.mn[1] <= y) && (y <= g.mx[1]) && (g.mn[2] <= z) && (z <= g.mx[2]))) return DBL_MAX;
    unsigned mi0 = (unsigned)((x - g.mn[0]) * g.inv[0]);
    unsigned mi1 = (unsigned)((y - g.mn[1]) * g.inv[1]);
    unsigned mi2 = (unsigned)((z - g.mn[2]) * g.inv[2]);
    if (mi0 >= g.n[0]) mi0 = g.n[0] - 1;
    if (mi1 >= g.n[1]) mi1 = g.n[1] - 1;
    if (mi2 >= g.n[2]) mi2 = g.n[2] - 1;
    const unsigned i = g.n[1] * g.n[0] * mi2 + g.n[0] * mi1 + mi0;
    const unsigned cell = f.cell_map ? __ldg(f.cell_map + i) : i;
    if (cell == UINT_MAX) return DBL_MAX;
    const double2 tx = __ldg(f.tab + mi0), ty = __ldg(f.tab + g.n[0] + mi1), tz = __ldg(f.tab + g.n[0] + g.n[1] + mi2);
    const double X = tx.x * x - tx.y, Y = ty.x * y - ty.y, Z = tz.x * z - tz.y;
    const double x2 = X * X, y2 = Y * Y, z2 = Z * Z;
    const double _1mx = 1.0 - X, _1my = 1.0 - Y, _1mz = 1.0 - Z;
    const double _1px = 1.0 + X, _1py = 1.0 + Y, _1pz = 1.0 + Z;
    const double _1m3x = 1.0 - 3.0 * X, _1m3y = 1.0 - 3.0 * Y, _1m3z = 1.0 - 3.0 * Z;
    const double _1p3x = 1.0 + 3.0 * X, _1p3y = 1.0 + 3.0 * Y, _1p3z = 1.0 + 3.0 * Z;
    const double mxmy = _1mx * _1my, mxpy = _1mx * _1py, pxmy = _1px * _1my, pxpy = _1px * _1py;
    const double mxmz = _1mx * _1mz, mxpz = _1mx * _1pz, pxmz = _1px * _1mz, pxpz = _1px * _1pz;
    const double mymz = _1my * _1mz, mypz = _1my * _1pz, pymz = _1py * _1mz, pypz = _1py * _1pz;
    const double facc = 1.0 / 64.0 * (9.0 * (x2 + y2 + z2) - 19.0);
    const double fx = 9.0 / 64.0 * (1.0 - x2), fy = 9.0 / 64.0 * (1.0 - y2), fz = 9.0 / 64.0 * (1.0 - z2);
    const double fxm = fx * _1m3x, fxp = fx * _1p3x, fym = fy * _1m3y, fyp = fy * _1p3y, fzm = fz * _1m3z, fzp = fz * _1p3z;
    const double2* cb = reinterpret_cast<const double2*>(f.packed + (size_t)cell * 32);
    double phi = 0.0;
    bool missing = false;
    double2 c;
#define DG_T(cj, n) { const double c_ = (cj); missing |= (c_ == DBL_MAX); phi = phi + c_ * (n); }
    c = __ldg(cb + 0);  DG_T(c.x, facc * mxmy * _1mz) DG_T(c.y, facc * pxmy * _1mz)
    c = __ldg(cb + 1);  DG_T(c.x, facc * mxpy * _1mz) DG_T(c.y, facc * pxpy * _1mz)
    c = __ldg(cb + 2);  DG_T(c.x, facc * mxmy * _1pz) DG_T(c.y, facc * pxmy * _1pz)
    c = __ldg(cb + 3);  DG_T(c.x, facc * mxpy * _1pz) DG_T(c.y, facc * pxpy * _1pz)
    c = __ldg(cb + 4);  DG_T(c.x, fxm * mymz) DG_T(c.y, fxp * mymz)
    c = __ldg(cb + 5);  DG_T(c.x, fxm * mypz) DG_T(c.y, fxp * mypz)
    c = __ldg(cb + 6);  DG_T(c.x, fxm * pymz) DG_T(c.y, fxp * pymz)
    c = __ldg(cb + 7);  DG_T(c.x, fxm * pypz) DG_T(c.y, fxp * pypz)
    c = __ldg(cb + 8);  DG_T(c.x, fym * mxmz) DG_T(c.y, fyp * mxmz)
    c = __ldg(cb + 9);  DG_T(c.x, fym * pxmz) DG_T(c.y, fyp * pxmz)
    c = __ldg(cb + 10); DG_T(c.x, fym * mxpz) DG_T(c.y, fyp * mxpz)
    c = __ldg(cb + 11); DG_T(c.x, fym * pxpz) DG_T(c.y, fyp * pxpz)
    c = __ldg(cb + 12); DG_T(c.x, fzm * mxmy) DG_T(c.y, fzp * mxmy)
    c = __ldg(cb + 13); DG_T(c.x, fzm * mxpy) DG_T(c.y, fzp * mxpy)
    c = __ldg(cb + 14); DG_T(c.x, fzm * pxmy) DG_T(c.y, fzp * pxmy)
    c = __ldg(cb + 15); DG_T(c.x, fzm * pxpy) DG_T(c.y, fzp * pxpy)
#undef DG_T
    return missing ? DBL_MAX : phi;
}

#ifndef K3_MIN_BLOCKS
#define K3_MIN_BLOCKS 5            // blocks of 128 threads per SM the register allocation must allow; ptxas for sm_90a: 96 registers,
                                   // no spills (6 -> 80 registers and 8 B of spill stores, 8 -> 64 registers and 144 B).  H100 80GB HBM3
                                   // capped at 400 W, 128^3 bunny field: 4 / 5 / 6 / 8 -> 380 / 372-380 / 381-383 / 500 ms
#endif
template <bool SKIP_ZERO_W>
__global__ void __launch_bounds__(128, K3_MIN_BLOCKS)
density_map_kernel(FieldDev f, QuadParams qp, const double* __restrict__ Wtab, int no_reduction, unsigned l_begin,
                   unsigned long long count, double* __restrict__ out)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    double x, y, z;
    node_position(f.g, l_begin + (unsigned)idx, x, y, z);
    if (!no_reduction) {                                            // predicate, main.cpp:119-133
        const double cx = fmin(fmax(x, f.g.mn[0]), f.g.mx[0]);      // cwiseMax(min).cwiseMin(max)
        const double cy = fmin(fmax(y, f.g.mn[1]), f.g.mx[1]);
        const double cz = fmin(fmax(z, f.g.mn[2]), f.g.mx[2]);
        const double d = interp_value(f, cx, cy, cz);
        const bool keep = (d != DBL_MAX) && (qp.six_h_neg < d + qp.cell_diag) && (d - qp.cell_diag < qp.two_h);
        if (!keep) { out[idx] = DBL_MAX; return; }                  // cubic_lagrange_discrete_grid.cpp:817
    }
    const double dist = interp_value(f, x, y, z);                   // main.cpp:98
    if (dist > qp.two_h) { out[idx] = 0.0; return; }
    double res = 0.0;
    const bool fast_h = in_fast_div_range(qp.h);
    for (int i = 0; i < 16; i++) {
        const double wi = qp.w[i], sx = x + qp.off[i];
        for (int j = 0; j < 16; j++) {
            const double wij = wi * qp.w[j], sy = y + qp.off[j];
            const double* wrow = Wtab + ((i * 16 + j) * 16);
#pragma unroll 1
            for (int k = 0; k < 16; k++) {
                const double W = __ldg(wrow + k);
                if (SKIP_ZERO_W && W == 0.0) continue;               // contributes exactly +0 (see header)
                const double wijk = wij * qp.w[k];
                const double d = interp_value(f, sx, sy, z + qp.off[k]);
                // d / h with h a launch constant: the same IEEE quotient from RN(1/h) and four FMAs (fast_div.h); plain division
                // when d is zero or outside the range where nothing can over- or underflow.  The division is ~33 of the ~400
                // instructions per quadrature point, and this form was measured faster than it.
                double dq = div_by_known_reciprocal(d, qp.h, qp.inv_h);
                if (!(fast_h && in_fast_div_range(d))) dq = d / qp.h;
                const double gam = (d > qp.h) ? 0.0 : 1.0 - dq;         // main.cpp:86-93
                res = res + wijk * (gam * W);                        // gauss_quadrature.cpp:5954
            }
        }
    }
    res = res * qp.c0prod;                                           // :5958
    out[idx] = qp.rho0 * res;                                        // main.cpp:111
}

// M of the header: the bit patterns of |c| for c != DBL_MAX, maximised with atomicMax.  Non-negative doubles order like their bits, and
// |NaN| (exponent all ones, mantissa != 0) and +inf come out above every finite value.
__global__ void __launch_bounds__(256)
coeff_max_kernel(const double* __restrict__ packed, unsigned long long n, unsigned long long* __restrict__ out)
{
    unsigned long long m = 0;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
#pragma unroll 4
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const double c = __ldg(packed + i);
        const unsigned long long b = (unsigned long long)__double_as_longlong(fabs(c));
        if (c != DBL_MAX && b > m) m = b;
    }
    if (m) atomicMax(out, m);
}

}  // namespace

cudaError_t k3_coeff_max(const double* d_packed, uint64_t n, double* out, cudaStream_t stream)
{
    const unsigned blocks = (unsigned)std::min<uint64_t>((n + 255) / 256, 1024), nb = blocks ? blocks : 1;
    unsigned long long bits = 0;
#ifdef DG_EMU
    DG_KERNEL_LAUNCH(coeff_max_kernel, nb, 256, 0, stream, d_packed, (unsigned long long)n, &bits);
#else
    unsigned long long* d_bits = nullptr;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&d_bits), sizeof bits, stream);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(d_bits, 0, sizeof bits, stream);
    if (e == cudaSuccess) {
        DG_KERNEL_LAUNCH(coeff_max_kernel, nb, 256, 0, stream, d_packed, (unsigned long long)n, d_bits);
        e = DG_AFTER_LAUNCH();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&bits, d_bits, sizeof bits, cudaMemcpyDeviceToHost, stream);
    cudaFreeAsync(d_bits, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return e;
#endif
    if (bits > 0x7ff0000000000000ull) bits = 0x7ff0000000000000ull;    // NaN -> +inf
    std::memcpy(out, &bits, sizeof bits);
    return cudaSuccess;
}

// Host tables.  This TU is compiled without FP contraction on the host side as well (x86-64 baseline has no FMA;
// -ffp-contract=off is passed explicitly), so these match the reference's CPU arithmetic bit for bit.

// cell_diag = cellSize().norm(); Eigen >= 3.3 reduces a Vector3d as (a0 + a1) + a2 (main.cpp:117)
double k3_cell_diag(const GridDev& g)
{
    return std::sqrt((g.cell[0] * g.cell[0] + g.cell[1] * g.cell[1]) + g.cell[2] * g.cell[2]);
}

cudaError_t k3_launch_density(const FieldDev& f, double coeff_max, double h, double rho0, int no_reduction, uint64_t l_begin,
                              uint64_t count, double* d_out, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    // the bound of the header: W == 0 points may be skipped when 64 M and 64 M / h are finite (h > 0 is the caller's to check; h = +inf
    // passes: every point then lies outside the domain, see the header)
    const double m64 = 64.0 * coeff_max;
    const bool skip_zero_w = (m64 < DBL_MAX) && (m64 / h < DBL_MAX);
    const auto kernel = skip_zero_w ? density_map_kernel<true> : density_map_kernel<false>;
    QuadParams qp;
    // integrate(): c0 = 0.5 * diagonal, c1 = 0.5 * (min + max) of [-h, h]^3 (gauss_quadrature.cpp:5937-5938)
    const double lo = -h, hi = h;
    const double c0 = 0.5 * (hi - lo), c1 = 0.5 * (lo + hi);
    for (int i = 0; i < 16; i++) { qp.off[i] = c0 * GA16[i] + c1; qp.w[i] = GW16[i]; }
    qp.h = h; qp.two_h = 2.0 * h; qp.six_h_neg = -6.0 * h; qp.rho0 = rho0;
    qp.inv_h = 1.0 / h;
    qp.c0prod = c0 * c0 * c0;                                        // Eigen prod(): (c0*c0)*c0
    qp.cell_diag = k3_cell_diag(f.g);
    // W at the 4096 points (sph_kernel.hpp:10-42): k = 8/(pi h^3)
    const double pi = static_cast<double>(M_PI);
    const double h3 = h * h * h;
    const double kk = 8.0 / (pi * h3);
    std::vector<double> W(4096);
    for (int i = 0; i < 16; i++)
        for (int j = 0; j < 16; j++)
            for (int k = 0; k < 16; k++) {
                const double rx = qp.off[i], ry = qp.off[j], rz = qp.off[k];
                const double rl = std::sqrt((rx * rx + ry * ry) + rz * rz);
                const double q = rl / h;
                double res = 0.0;
                if (q <= 1.0) {
                    if (q <= 0.5) { const double q2 = q * q, q3 = q2 * q; res = kk * (6.0 * q3 - 6.0 * q2 + 1.0); }
                    else { const double m = 1.0 - q; res = kk * (2.0 * m * m * m); }
                }
                W[(i * 16 + j) * 16 + k] = res;
            }
    const unsigned blocks = (unsigned)((count + 127) / 128);
#ifdef DG_EMU
    DG_KERNEL_LAUNCH(kernel, blocks, 128, 0, stream, f, qp, W.data(), no_reduction, (unsigned)l_begin, (unsigned long long)count, d_out);
    return cudaSuccess;
#else
    double* d_W = nullptr;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&d_W), 4096 * sizeof(double), stream);
    if (e != cudaSuccess) return e;
    e = cudaMemcpyAsync(d_W, W.data(), 4096 * sizeof(double), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) {
        // the pageable source is staged synchronously by the runtime, so W may go out of scope afterwards
        DG_KERNEL_LAUNCH(kernel, blocks, 128, 0, stream, f, qp, d_W, no_reduction, (unsigned)l_begin, (unsigned long long)count, d_out);
        e = DG_AFTER_LAUNCH();
    }
    cudaFreeAsync(d_W, stream);
    return e;
#endif
}

// ================================================================================================ volume map
// The volume map of Bender et al. 2019 ("Volume Maps: An Implicit Boundary Representation for SPH", MIG 2019), in 3D and in fp64, as
// SPlisHSPlasH generates it with Discregrid's addFunction over an SDF grid.  The reference has no volume map; this is the library's contract,
// written in the reference's own building blocks (DESIGN section 3, "Volume map"):
//   d(y)           : interpolate(sdf, y), the bits of interp_value above (DBL_MAX outside the domain, in a removed cell, or where a
//                    coefficient is missing)
//   pred(x)        : GenerateDensityMap's sample predicate (main.cpp:119-133), unless no_reduction: clamp x into the domain,
//                    dd = d(clamp(x)); reject (DBL_MAX, :817) if dd == DBL_MAX, else keep iff -6h < dd + cell_diag && dd - cell_diag < 2h
//   volume(x)      : 0.0 if d(x) > (1.0 + 1.0) * h, else s * GaussQuadrature::integrate(g, [-h, h]^3, p = 30) with the order of
//                    gauss_quadrature.cpp:5927-5960: 16^3 points, i outermost, res += wijk * g(c0 * xi + c1), res *= c0.prod()
//   g(xi)          : 0.0 if (xi.x^2 + xi.y^2) + xi.z^2 > h * h (Eigen's squaredNorm; d is not evaluated), else gamma(d(x + xi)) with
//                    x + xi formed per component, as K3's x + off[i]
//   gamma(delta)   : 1.0 if delta <= 0; W((delta, 0, 0)) / W_zero if delta < h; 0.0 otherwise (DBL_MAX and NaN included).  W is
//                    sph_kernel.hpp:22-42's CubicKernel with radius h, W_zero = W(0) = k.
// Two consequences the kernel uses:
//   * The skip is exact.  The reference returns 0.0 for an offset outside the ball without interpolating, and wijk * 0.0 = +0 leaves
//     the accumulator (which starts at +0) unchanged whatever it holds.  So the points outside the ball are simply not visited; no
//     bound on the coefficients like K3's SKIP_ZERO_W is needed.
//   * The ball test, the offsets and wijk = (wi * wj) * wk depend on h alone.  The host tabulates the points inside the ball once per
//     call, in quadrature order (1008 of 4096 at h = 1; rounding at the sphere can change the count with h, so it is not a constant),
//     and the kernel walks that flat list with no branch on the ball.  All 32 lanes of a warp read the same entry at each step.
// rl = sqrt((delta * delta + 0 * 0) + 0 * 0) is sqrt(delta * delta): delta * delta >= +0, and adding +0 to it changes no bit.

namespace {

struct VolumeParams {
    double h, two_h, six_h_neg, scale, c0prod, cell_diag, k, w_zero;
};

#ifndef K3V_MIN_BLOCKS
#define K3V_MIN_BLOCKS 5           // blocks of 128 threads per SM the register allocation must allow; ptxas for sm_90a: see DESIGN section 4
#endif
__global__ void __launch_bounds__(128, K3V_MIN_BLOCKS)
volume_map_kernel(FieldDev f, VolumeParams vp, const double2* __restrict__ pts, unsigned n_pts, int no_reduction, unsigned l_begin,
                  unsigned long long count, double* __restrict__ out)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    double x, y, z;
    node_position(f.g, l_begin + (unsigned)idx, x, y, z);
    if (!no_reduction) {                                            // GenerateDensityMap's predicate, main.cpp:119-133
        const double cx = fmin(fmax(x, f.g.mn[0]), f.g.mx[0]);
        const double cy = fmin(fmax(y, f.g.mn[1]), f.g.mx[1]);
        const double cz = fmin(fmax(z, f.g.mn[2]), f.g.mx[2]);
        const double d = interp_value(f, cx, cy, cz);
        const bool keep = (d != DBL_MAX) && (vp.six_h_neg < d + vp.cell_diag) && (d - vp.cell_diag < vp.two_h);
        if (!keep) { out[idx] = DBL_MAX; return; }
    }
    const double dist = interp_value(f, x, y, z);
    if (dist > vp.two_h) { out[idx] = 0.0; return; }
    double res = 0.0;
#pragma unroll 1
    for (unsigned p = 0; p < n_pts; p++) {
        const double2 a = __ldg(pts + 2 * p), b = __ldg(pts + 2 * p + 1);    // (xi.x, xi.y), (xi.z, wijk)
        const double d = interp_value(f, x + a.x, y + a.y, z + b.x);
        double gam = 0.0;
        if (d <= 0.0) gam = 1.0;
        else if (d < vp.h) {                                        // W((d, 0, 0)) / W_zero, sph_kernel.hpp:22-42
            const double rl = sqrt(d * d);
            const double q = rl / vp.h;
            double W = 0.0;
            if (q <= 1.0) {
                if (q <= 0.5) { const double q2 = q * q, q3 = q2 * q; W = vp.k * (6.0 * q3 - 6.0 * q2 + 1.0); }
                else { const double m = 1.0 - q; W = vp.k * (2.0 * m * m * m); }
            }
            gam = W / vp.w_zero;
        }
        res = res + b.y * gam;                                      // gauss_quadrature.cpp:5954
    }
    res = res * vp.c0prod;                                          // :5958
    out[idx] = vp.scale * res;
}

}  // namespace

// The points of the 16^3 rule inside the ball of radius h, in quadrature order: (xi.x, xi.y, xi.z, wijk) each.  Host arithmetic without
// contraction, with the reference's expressions (gauss_quadrature.cpp:5937-5954, Eigen's squaredNorm (a0 + a1) + a2).
std::vector<double> k3_volume_points(double h)
{
    const double lo = -h, hi = h;
    const double c0 = 0.5 * (hi - lo), c1 = 0.5 * (lo + hi);
    double off[16];
    for (int i = 0; i < 16; i++) off[i] = c0 * GA16[i] + c1;
    const double hh = h * h;
    std::vector<double> pts;
    pts.reserve(4 * 1100);
    for (int i = 0; i < 16; i++) {
        const double wi = GW16[i];
        for (int j = 0; j < 16; j++) {
            const double wij = wi * GW16[j];
            for (int k = 0; k < 16; k++) {
                const double wijk = wij * GW16[k];
                if ((off[i] * off[i] + off[j] * off[j]) + off[k] * off[k] > hh) continue;
                pts.push_back(off[i]); pts.push_back(off[j]); pts.push_back(off[k]); pts.push_back(wijk);
            }
        }
    }
    return pts;
}

cudaError_t k3_launch_volume(const FieldDev& f, double h, double scale, int no_reduction, uint64_t l_begin, uint64_t count, double* d_out,
                             cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    const std::vector<double> pts = k3_volume_points(h);
    const unsigned n_pts = (unsigned)(pts.size() / 4);
    VolumeParams vp;
    const double c0 = 0.5 * (h - (-h));
    vp.h = h; vp.two_h = (1.0 + 1.0) * h; vp.six_h_neg = -6.0 * h; vp.scale = scale;
    vp.c0prod = c0 * c0 * c0;                                       // Eigen prod(): (c0*c0)*c0
    vp.cell_diag = k3_cell_diag(f.g);
    // CubicKernel::setRadius (sph_kernel.hpp:10-20): k = 8/(pi h^3), W_zero = W(0) = k * (6*0 - 6*0 + 1)
    const double pi = static_cast<double>(M_PI);
    const double h3 = h * h * h;
    vp.k = 8.0 / (pi * h3);
    vp.w_zero = vp.k * (6.0 * 0.0 - 6.0 * 0.0 + 1.0);
    const unsigned blocks = (unsigned)((count + 127) / 128);
    const double2* h_pts = reinterpret_cast<const double2*>(pts.data());
#ifdef DG_EMU
    DG_KERNEL_LAUNCH(volume_map_kernel, blocks, 128, 0, stream, f, vp, h_pts, n_pts, no_reduction, (unsigned)l_begin, (unsigned long long)count, d_out);
    return cudaSuccess;
#else
    const size_t bytes = pts.size() * sizeof(double);
    double2* d_pts = nullptr;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&d_pts), bytes ? bytes : sizeof(double2), stream);
    if (e != cudaSuccess) return e;
    if (bytes) e = cudaMemcpyAsync(d_pts, h_pts, bytes, cudaMemcpyHostToDevice, stream);   // pageable: staged before the call returns
    if (e == cudaSuccess) {
        DG_KERNEL_LAUNCH(volume_map_kernel, blocks, 128, 0, stream, f, vp, d_pts, n_pts, no_reduction, (unsigned)l_begin, (unsigned long long)count, d_out);
        e = DG_AFTER_LAUNCH();
    }
    cudaFreeAsync(d_pts, stream);
    return e;
#endif
}

}  // namespace dgb
