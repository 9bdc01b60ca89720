// K2: batched CubicLagrangeDiscreteGrid::interpolate (+ gradient), one query per lane.
//
// Replaces interpolate (cubic_lagrange_discrete_grid.cpp:977-1063), determineShapeFunctions + split interpolate
// (:901-975), shape_function_ (:339-580) and the index helpers discrete_grid.cpp:8-38.
//
// Device layout (built once by dg_field_create): the 32 coefficients of every kept cell are gathered into one
// contiguous, 256-byte-aligned block packed[cell][32] (the reference keeps a shared node array + a 32-index
// table per cell: 16 scattered 16-byte pairs per query, i.e. >= 2x the algorithmic DRAM traffic).  A query's
// compulsory traffic is then exactly 24 B (x) + 256 B (block) + 8 B (phi) [+ 24 B (grad)].
//
// Kernel: each lane locates its cell, then issues ONE bulk async copy (cp.async.bulk, the TMA engine's 1-D
// path) of its 256-byte block into the warp's shared-memory staging area and signals the warp's mbarrier.
// While the copies are in flight the lane evaluates everything that does not need coefficients (xi and all
// shape-function temporaries).  After the mbarrier flips, the 32 terms are accumulated in the reference's
// order j = 0..31, each shape function / Jacobian row evaluated on the fly (no N[32]/dN[32][3] arrays in
// registers).  Staging slots are 272 bytes apart so that the 16-byte shared loads of a quarter-warp hit
// distinct banks.  No registers are held by in-flight data, so memory-level parallelism is bounded only by
// shared memory (8.5 KB per warp).
//
// The per-axis reference-cell maps c0 = 2/denom, c1 = (hi+lo)/denom (:1000-1002) depend only on the cell
// index along that axis; they are tabulated once per field with the reference's exact operation order, which
// removes six fp64 divisions per query without changing a bit.
//
// Hessian mode (interpolate_kernel<true, true>; the reference has no Hessian, so this contract is the library's own).  phi and grad
// are computed by the same expressions in the same order as the gradient mode and have its bits.  Notation as in the code: X, Y, Z = xi,
// Lx = 1 + sx*X (_1mx / _1px), and so on.  The second derivatives of the 32 shape functions, in xi:
//   corner (sx, sy, sz), N = F*Lx*Ly*Lz/64 with F = 9(X^2+Y^2+Z^2) - 19, scale 1/64:
//     d2/dX2  = (18*(1 + 3*sx*X)) * (Ly*Lz)                       (18 * _1m3x / _1p3x, times mymz ...)
//     d2/dXdY = (sy*xsA + sx*(18Y*Ly)) * Lz                        (xsA = 18X + sx*A, the gradient's xmA / xpA)
//     d2/dXdZ = (sz*xsA + sx*(18Z*Lz)) * Ly,   d2/dYdZ = (sz*ysB + sy*(18Z*Lz)) * Lx,   d2/dY2, d2/dZ2 by permutation
//   x-edge (s, sy, sz), N = (9/64)*P*Ly*Lz with P = (1-X^2)(1+3sX) (Xm / Xp), P' = mX / pX, P'' = -2 - 18sX, scale 9/64:
//     d2/dX2 = P''*(Ly*Lz),  d2/dXdY = (sy*P')*Lz,  d2/dXdZ = (sz*P')*Ly,  d2/dYdZ = (sy*sz)*P,  d2/dY2 = d2/dZ2 = 0
//   y- and z-edges by permutation.  A sign s* is applied as an exact negation, never as a product.
// Each entry h_ab accumulates h = h + c_j * (d2 * scale) over j = 0..31 in the order of the value sum, skipping the structural zeros
// (a diagonal entry sums the 8 corners and the 8 edges along its axis, a mixed entry all 32): adding c_j * 0 would turn an infinite
// coefficient into NaN and could flip the sign of a zero.  Then H_ab = (h_ab * c0_a) * c0_b, computed once for a < b and stored at
// [a][b] and [b][a] of the row-major hess[n][3][3].  Sentinels as in the gradient mode, with all nine entries +0.0.
#include "dg_device.cuh"
#include "k2_interp.h"
#include "dg_launch.h"
#include "shape_rows.cuh"

#include <cfloat>
#include <climits>
#include <cstdint>
#include <cstring>

namespace dgb {

namespace {

constexpr int K2_SLOT_BYTES = 272;          // 256-byte block + 16 bytes of padding (bank spreading)
constexpr int K2_WARPS = K2_THREADS / 32;

#ifdef DG_EMU
// CPU emulation: "shared" addresses are plain pointers, the bulk copy is a memcpy that has completed when it returns, the mbarrier
// has nothing left to wait for (each lane only reads the slot it copied itself)
typedef uintptr_t smem_addr_t;
inline smem_addr_t smem_u32(const void* p) { return (smem_addr_t)p; }
inline void mbar_init(smem_addr_t, unsigned) {}
inline void mbar_expect_tx(smem_addr_t, unsigned) {}
inline void bulk_g2s(smem_addr_t dst, const void* src, unsigned bytes, smem_addr_t) { std::memcpy((void*)dst, src, bytes); }
inline void mbar_wait(smem_addr_t, unsigned) {}
inline void __syncwarp() {}
#else
typedef unsigned smem_addr_t;
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
#endif

// Gathers the packed per-cell blocks.  One thread per (kept cell, local node).
__global__ void pack_cells_kernel(GridDev g, const double* __restrict__ nodes, const unsigned* __restrict__ cells /*nullable*/,
                                  unsigned long long n32, double* __restrict__ packed)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n32) return;
    unsigned v;
    if (cells) v = cells[idx];
    else {
        const unsigned c = (unsigned)(idx >> 5), jn = (unsigned)(idx & 31u);
        const unsigned nxy = g.n[0] * g.n[1];
        const unsigned k = c / nxy, t = c - k * nxy, j = t / g.n[0], i = t - j * g.n[0];
        v = cell_node_id(g, i, j, k, jn);
    }
    packed[idx] = nodes[v];
}

// Per-axis reference-cell maps: tab[off_d + m] = (c0, c1) for cell index m along axis d.
// subdomain(): origin = min + double(m)*cell, max = origin + cell (discrete_grid.cpp:26-32);
// denom = max - min, c0 = 2/denom, c1 = (max+min)/denom (cubic_lagrange_discrete_grid.cpp:1000-1002).
__global__ void axis_tables_kernel(GridDev g, double2* __restrict__ tab)
{
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned n0 = g.n[0], n1 = g.n[1], n2 = g.n[2];
    if (idx >= n0 + n1 + n2) return;
    int d; unsigned m;
    if (idx < n0) { d = 0; m = idx; } else if (idx < n0 + n1) { d = 1; m = idx - n0; } else { d = 2; m = idx - n0 - n1; }
    const double lo = g.mn[d] + (double)m * g.cell[d];
    const double hi = lo + g.cell[d];
    const double denom = hi - lo;
    tab[idx] = make_double2(2.0 / denom, (hi + lo) / denom);
}

// <false, false>: value; <true, false>: value + gradient; <true, true>: value + gradient + Hessian (see the header comment)
template <bool GRAD, bool HESS>
__global__ void __launch_bounds__(K2_THREADS)
interpolate_kernel(GridDev g, const double* __restrict__ packed, const unsigned* __restrict__ cell_map /*nullable*/,
                   const double2* __restrict__ tab, const double* __restrict__ xq, unsigned long long n,
                   double* __restrict__ phi_out, double* __restrict__ grad_out, double* __restrict__ hess_out)
{
    static_assert(GRAD || !HESS, "the Hessian mode also computes the gradient");
    __shared__ __align__(16) unsigned char stage[K2_WARPS][32 * K2_SLOT_BYTES];
    __shared__ __align__(8) unsigned long long bars[K2_WARPS];

    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const unsigned long long q0 = (unsigned long long)blockIdx.x * K2_THREADS + threadIdx.x;
    if (q0 - lane >= n) return;                             // whole warp past the end
    const bool live = q0 < n;
    const unsigned long long q = live ? q0 : n - 1;         // tail lanes shadow the last query (no store)

    const smem_addr_t bar = smem_u32(&bars[warp]);
    if (lane == 0) { mbar_init(bar, 1); mbar_expect_tx(bar, 32u * 256u); }
    __syncwarp();

    const double x = xq[3 * q], y = xq[3 * q + 1], z = xq[3 * q + 2];

    // ---- cell location (:981-994).  NaN fails `contains` like Eigen's AlignedBox.
    bool valid = (g.mn[0] <= x) && (x <= g.mx[0]) && (g.mn[1] <= y) && (y <= g.mx[1]) && (g.mn[2] <= z) && (z <= g.mx[2]);
    unsigned mi0 = 0, mi1 = 0, mi2 = 0, cell = 0;
    if (valid) {
        mi0 = (unsigned)((x - g.mn[0]) * g.inv[0]);
        mi1 = (unsigned)((y - g.mn[1]) * g.inv[1]);
        mi2 = (unsigned)((z - g.mn[2]) * g.inv[2]);
        if (mi0 >= g.n[0]) mi0 = g.n[0] - 1;
        if (mi1 >= g.n[1]) mi1 = g.n[1] - 1;
        if (mi2 >= g.n[2]) mi2 = g.n[2] - 1;
        const unsigned i = g.n[1] * g.n[0] * mi2 + g.n[0] * mi1 + mi0;     // multiToSingleIndex
        cell = cell_map ? __ldg(cell_map + i) : i;
        if (cell == UINT_MAX) { valid = false; cell = 0; }                  // removed by reduceField (:993)
    }

    // ---- one bulk copy per lane: packed[cell][0..31] -> stage[warp][lane]
    const smem_addr_t slot = smem_u32(&stage[warp][lane * K2_SLOT_BYTES]);
    bulk_g2s(slot, packed + (size_t)cell * 32, 256u, bar);

    // ---- reference-cell coordinates (:996-1003) and every coefficient-independent temporary (:344-385, :440-460)
    const double2 tx = __ldg(tab + mi0), ty = __ldg(tab + g.n[0] + mi1), tz = __ldg(tab + g.n[0] + g.n[1] + mi2);
    const double X = tx.x * x - tx.y, Y = ty.x * y - ty.y, Z = tz.x * z - tz.y;     // xi = c0*x - c1
    const double x2 = X * X, y2 = Y * Y, z2 = Z * Z;
    const double _1mx = 1.0 - X, _1my = 1.0 - Y, _1mz = 1.0 - Z;
    const double _1px = 1.0 + X, _1py = 1.0 + Y, _1pz = 1.0 + Z;
    const double _1m3x = 1.0 - 3.0 * X, _1m3y = 1.0 - 3.0 * Y, _1m3z = 1.0 - 3.0 * Z;
    const double _1p3x = 1.0 + 3.0 * X, _1p3y = 1.0 + 3.0 * Y, _1p3z = 1.0 + 3.0 * Z;
    const double mxmy = _1mx * _1my, mxpy = _1mx * _1py, pxmy = _1px * _1my, pxpy = _1px * _1py;
    const double mxmz = _1mx * _1mz, mxpz = _1mx * _1pz, pxmz = _1px * _1mz, pxpz = _1px * _1pz;
    const double mymz = _1my * _1mz, mypz = _1my * _1pz, pymz = _1py * _1mz, pypz = _1py * _1pz;
    const double _1mx2 = 1.0 - x2, _1my2 = 1.0 - y2, _1mz2 = 1.0 - z2;
    const double facc = 1.0 / 64.0 * (9.0 * (x2 + y2 + z2) - 19.0);                   // :388
    const double fx = 9.0 / 64.0 * _1mx2, fy = 9.0 / 64.0 * _1my2, fz = 9.0 / 64.0 * _1mz2;   // :400,412,424
    const double fxm = fx * _1m3x, fxp = fx * _1p3x, fym = fy * _1m3y, fyp = fy * _1p3y, fzm = fz * _1m3z, fzp = fz * _1p3z;

    double xmA = 0, xpA = 0, ymB = 0, ypB = 0, zmC = 0, zpC = 0, mX = 0, pX = 0, Xm = 0, Xp = 0, mY = 0, pY = 0, Ym = 0, Yp = 0,
           mZ = 0, pZ = 0, Zm = 0, Zp = 0;
    if (GRAD) {
        const double A = 9.0 * (3.0 * x2 + y2 + z2) - 19.0;                           // :440-442
        const double B = 9.0 * (x2 + 3.0 * y2 + z2) - 19.0;
        const double C = 9.0 * (x2 + y2 + 3.0 * z2) - 19.0;
        const double _18x = 18.0 * X, _18y = 18.0 * Y, _18z = 18.0 * Z;
        xmA = _18x - A; xpA = _18x + A; ymB = _18y - B; ypB = _18y + B; zmC = _18z - C; zpC = _18z + C;   // :455-460
        const double _3m9x2 = 3.0 - 9.0 * x2, _3m9y2 = 3.0 - 9.0 * y2, _3m9z2 = 3.0 - 9.0 * z2;
        const double _2x = 2.0 * X, _2y = 2.0 * Y, _2z = 2.0 * Z;
        mX = -_3m9x2 - _2x; pX = _3m9x2 - _2x; Xm = _1mx2 * _1m3x; Xp = _1mx2 * _1p3x;                    // :489-492
        mY = -_3m9y2 - _2y; pY = _3m9y2 - _2y; Ym = _1my2 * _1m3y; Yp = _1my2 * _1p3y;                    // :518-521
        mZ = -_3m9z2 - _2z; pZ = _3m9z2 - _2z; Zm = _1mz2 * _1m3z; Zp = _1mz2 * _1p3z;                    // :547-550
    }
    // Hessian-mode temporaries: 18(1 -+ 3X) of the corners' d2/dX2, 18X*(1 -+ X) of their mixed terms, P'' = -2 -+ 18X of the x-edges
    double d2xm = 0, d2xp = 0, d2ym = 0, d2yp = 0, d2zm = 0, d2zp = 0, x18m = 0, x18p = 0, y18m = 0, y18p = 0, z18m = 0, z18p = 0,
           ddXm = 0, ddXp = 0, ddYm = 0, ddYp = 0, ddZm = 0, ddZp = 0;
    if (HESS) {
        const double _18x = 18.0 * X, _18y = 18.0 * Y, _18z = 18.0 * Z;
        d2xm = 18.0 * _1m3x; d2xp = 18.0 * _1p3x; d2ym = 18.0 * _1m3y; d2yp = 18.0 * _1p3y; d2zm = 18.0 * _1m3z; d2zp = 18.0 * _1p3z;
        x18m = _18x * _1mx; x18p = _18x * _1px; y18m = _18y * _1my; y18p = _18y * _1py; z18m = _18z * _1mz; z18p = _18z * _1pz;
        ddXm = -2.0 + _18x; ddXp = -2.0 - _18x; ddYm = -2.0 + _18y; ddYp = -2.0 - _18y; ddZm = -2.0 + _18z; ddZp = -2.0 - _18z;
    }

    // ---- wait for the warp's 32 blocks
    mbar_wait(bar, 0);
    const double2* cb = reinterpret_cast<const double2*>(&stage[warp][lane * K2_SLOT_BYTES]);

    double phi = 0.0, g0 = 0.0, g1 = 0.0, g2 = 0.0;
    bool missing = false;
    // one term of the sequential sums (:1044-1060); corner rows are scaled by /64, edge rows by *(9/64) (:487, :576)
#define DG_CORNER(cj, n, dx, dy, dz)                                         \
    {                                                                        \
        const double c_ = (cj);                                              \
        missing |= (c_ == DBL_MAX);                                          \
        phi = phi + c_ * (n);                                                \
        if (GRAD) { g0 = g0 + c_ * ((dx) * 0.015625); g1 = g1 + c_ * ((dy) * 0.015625); g2 = g2 + c_ * ((dz) * 0.015625); } \
    }
#define DG_EDGE(cj, n, dx, dy, dz)                                           \
    {                                                                        \
        const double c_ = (cj);                                              \
        missing |= (c_ == DBL_MAX);                                          \
        phi = phi + c_ * (n);                                                \
        if (GRAD) { g0 = g0 + c_ * ((dx) * (9.0 / 64.0)); g1 = g1 + c_ * ((dy) * (9.0 / 64.0)); g2 = g2 + c_ * ((dz) * (9.0 / 64.0)); } \
    }
    // Hessian terms of one node, given by its signs (m = -1, p = +1); an edge's own axis sign is S.  Structural zeros are not added.
    double hxx = 0.0, hxy = 0.0, hxz = 0.0, hyy = 0.0, hyz = 0.0, hzz = 0.0;
#define DG_SG_m(v) (-(v))
#define DG_SG_p(v) (v)
#define DG_SG2_mm(v) (v)
#define DG_SG2_mp(v) (-(v))
#define DG_SG2_pm(v) (-(v))
#define DG_SG2_pp(v) (v)
#define DG_CORNER_H(cj, SX, SY, SZ)                                                                                   \
    if (HESS) {                                                                                                       \
        const double c_ = (cj);                                                                                       \
        hxx = hxx + c_ * ((d2x##SX * SY##y##SZ##z) * 0.015625);                                                       \
        hyy = hyy + c_ * ((d2y##SY * SX##x##SZ##z) * 0.015625);                                                       \
        hzz = hzz + c_ * ((d2z##SZ * SX##x##SY##y) * 0.015625);                                                       \
        hxy = hxy + c_ * (((DG_SG_##SY(x##SX##A) + DG_SG_##SX(y18##SY)) * _1##SZ##z) * 0.015625);                    \
        hxz = hxz + c_ * (((DG_SG_##SZ(x##SX##A) + DG_SG_##SX(z18##SZ)) * _1##SY##y) * 0.015625);                    \
        hyz = hyz + c_ * (((DG_SG_##SZ(y##SY##B) + DG_SG_##SY(z18##SZ)) * _1##SX##x) * 0.015625);                    \
    }
#define DG_XEDGE_H(cj, S, SY, SZ)                                                                                     \
    if (HESS) {                                                                                                       \
        const double c_ = (cj);                                                                                       \
        hxx = hxx + c_ * ((ddX##S * SY##y##SZ##z) * (9.0 / 64.0));                                                    \
        hxy = hxy + c_ * ((DG_SG_##SY(S##X) * _1##SZ##z) * (9.0 / 64.0));                                             \
        hxz = hxz + c_ * ((DG_SG_##SZ(S##X) * _1##SY##y) * (9.0 / 64.0));                                             \
        hyz = hyz + c_ * (DG_SG2_##SY##SZ(X##S) * (9.0 / 64.0));                                                      \
    }
#define DG_YEDGE_H(cj, SX, S, SZ)                                                                                     \
    if (HESS) {                                                                                                       \
        const double c_ = (cj);                                                                                       \
        hyy = hyy + c_ * ((ddY##S * SX##x##SZ##z) * (9.0 / 64.0));                                                    \
        hxy = hxy + c_ * ((DG_SG_##SX(S##Y) * _1##SZ##z) * (9.0 / 64.0));                                             \
        hxz = hxz + c_ * (DG_SG2_##SX##SZ(Y##S) * (9.0 / 64.0));                                                      \
        hyz = hyz + c_ * ((DG_SG_##SZ(S##Y) * _1##SX##x) * (9.0 / 64.0));                                             \
    }
#define DG_ZEDGE_H(cj, SX, SY, S)                                                                                     \
    if (HESS) {                                                                                                       \
        const double c_ = (cj);                                                                                       \
        hzz = hzz + c_ * ((ddZ##S * SX##x##SY##y) * (9.0 / 64.0));                                                    \
        hxy = hxy + c_ * (DG_SG2_##SX##SY(Z##S) * (9.0 / 64.0));                                                      \
        hxz = hxz + c_ * ((DG_SG_##SX(S##Z) * _1##SY##y) * (9.0 / 64.0));                                             \
        hyz = hyz + c_ * ((DG_SG_##SY(S##Z) * _1##SX##x) * (9.0 / 64.0));                                             \
    }
    double2 c;
    // corners (:389-396, :462-485)
    c = cb[0];
    DG_CORNER(c.x, facc * mxmy * _1mz, xmA * mymz, mxmz * ymB, mxmy * zmC) DG_CORNER_H(c.x, m, m, m)
    DG_CORNER(c.y, facc * pxmy * _1mz, xpA * mymz, pxmz * ymB, pxmy * zmC) DG_CORNER_H(c.y, p, m, m)
    c = cb[1];
    DG_CORNER(c.x, facc * mxpy * _1mz, xmA * pymz, mxmz * ypB, mxpy * zmC) DG_CORNER_H(c.x, m, p, m)
    DG_CORNER(c.y, facc * pxpy * _1mz, xpA * pymz, pxmz * ypB, pxpy * zmC) DG_CORNER_H(c.y, p, p, m)
    c = cb[2];
    DG_CORNER(c.x, facc * mxmy * _1pz, xmA * mypz, mxpz * ymB, mxmy * zpC) DG_CORNER_H(c.x, m, m, p)
    DG_CORNER(c.y, facc * pxmy * _1pz, xpA * mypz, pxpz * ymB, pxmy * zpC) DG_CORNER_H(c.y, p, m, p)
    c = cb[3];
    DG_CORNER(c.x, facc * mxpy * _1pz, xmA * pypz, mxpz * ypB, mxpy * zpC) DG_CORNER_H(c.x, m, p, p)
    DG_CORNER(c.y, facc * pxpy * _1pz, xpA * pypz, pxpz * ypB, pxpy * zpC) DG_CORNER_H(c.y, p, p, p)
    // x edges (:403-410, :493-516)
    c = cb[4];
    DG_EDGE(c.x, fxm * mymz, mX * mymz, -Xm * _1mz, -Xm * _1my) DG_XEDGE_H(c.x, m, m, m)
    DG_EDGE(c.y, fxp * mymz, pX * mymz, -Xp * _1mz, -Xp * _1my) DG_XEDGE_H(c.y, p, m, m)
    c = cb[5];
    DG_EDGE(c.x, fxm * mypz, mX * mypz, -Xm * _1pz, Xm * _1my) DG_XEDGE_H(c.x, m, m, p)
    DG_EDGE(c.y, fxp * mypz, pX * mypz, -Xp * _1pz, Xp * _1my) DG_XEDGE_H(c.y, p, m, p)
    c = cb[6];
    DG_EDGE(c.x, fxm * pymz, mX * pymz, Xm * _1mz, -Xm * _1py) DG_XEDGE_H(c.x, m, p, m)
    DG_EDGE(c.y, fxp * pymz, pX * pymz, Xp * _1mz, -Xp * _1py) DG_XEDGE_H(c.y, p, p, m)
    c = cb[7];
    DG_EDGE(c.x, fxm * pypz, mX * pypz, Xm * _1pz, Xm * _1py) DG_XEDGE_H(c.x, m, p, p)
    DG_EDGE(c.y, fxp * pypz, pX * pypz, Xp * _1pz, Xp * _1py) DG_XEDGE_H(c.y, p, p, p)
    // y edges (:415-422, :522-545)
    c = cb[8];
    DG_EDGE(c.x, fym * mxmz, -Ym * _1mz, mY * mxmz, -Ym * _1mx) DG_YEDGE_H(c.x, m, m, m)
    DG_EDGE(c.y, fyp * mxmz, -Yp * _1mz, pY * mxmz, -Yp * _1mx) DG_YEDGE_H(c.y, m, p, m)
    c = cb[9];
    DG_EDGE(c.x, fym * pxmz, Ym * _1mz, mY * pxmz, -Ym * _1px) DG_YEDGE_H(c.x, p, m, m)
    DG_EDGE(c.y, fyp * pxmz, Yp * _1mz, pY * pxmz, -Yp * _1px) DG_YEDGE_H(c.y, p, p, m)
    c = cb[10];
    DG_EDGE(c.x, fym * mxpz, -Ym * _1pz, mY * mxpz, Ym * _1mx) DG_YEDGE_H(c.x, m, m, p)
    DG_EDGE(c.y, fyp * mxpz, -Yp * _1pz, pY * mxpz, Yp * _1mx) DG_YEDGE_H(c.y, m, p, p)
    c = cb[11];
    DG_EDGE(c.x, fym * pxpz, Ym * _1pz, mY * pxpz, Ym * _1px) DG_YEDGE_H(c.x, p, m, p)
    DG_EDGE(c.y, fyp * pxpz, Yp * _1pz, pY * pxpz, Yp * _1px) DG_YEDGE_H(c.y, p, p, p)
    // z edges (:427-434, :551-574)
    c = cb[12];
    DG_EDGE(c.x, fzm * mxmy, -Zm * _1my, -Zm * _1mx, mZ * mxmy) DG_ZEDGE_H(c.x, m, m, m)
    DG_EDGE(c.y, fzp * mxmy, -Zp * _1my, -Zp * _1mx, pZ * mxmy) DG_ZEDGE_H(c.y, m, m, p)
    c = cb[13];
    DG_EDGE(c.x, fzm * mxpy, -Zm * _1py, Zm * _1mx, mZ * mxpy) DG_ZEDGE_H(c.x, m, p, m)
    DG_EDGE(c.y, fzp * mxpy, -Zp * _1py, Zp * _1mx, pZ * mxpy) DG_ZEDGE_H(c.y, m, p, p)
    c = cb[14];
    DG_EDGE(c.x, fzm * pxmy, Zm * _1my, -Zm * _1px, mZ * pxmy) DG_ZEDGE_H(c.x, p, m, m)
    DG_EDGE(c.y, fzp * pxmy, Zp * _1my, -Zp * _1px, pZ * pxmy) DG_ZEDGE_H(c.y, p, m, p)
    c = cb[15];
    DG_EDGE(c.x, fzm * pxpy, Zm * _1py, Zm * _1px, mZ * pxpy) DG_ZEDGE_H(c.x, p, p, m)
    DG_EDGE(c.y, fzp * pxpy, Zp * _1py, Zp * _1px, pZ * pxpy) DG_ZEDGE_H(c.y, p, p, p)
#undef DG_CORNER
#undef DG_EDGE
#undef DG_CORNER_H
#undef DG_XEDGE_H
#undef DG_YEDGE_H
#undef DG_ZEDGE_H
#undef DG_SG_m
#undef DG_SG_p
#undef DG_SG2_mm
#undef DG_SG2_mp
#undef DG_SG2_pm
#undef DG_SG2_pp

    if (!live) return;
    if (!valid || missing) {                        // sentinel paths (:981-982, :993-994, :1015-1018, :1050-1054)
        phi_out[q] = DBL_MAX;
        if (GRAD) { grad_out[3 * q] = 0.0; grad_out[3 * q + 1] = 0.0; grad_out[3 * q + 2] = 0.0; }
        if (HESS) { for (int k = 0; k < 9; k++) hess_out[9 * q + k] = 0.0; }
        return;
    }
    phi_out[q] = phi;
    if (GRAD) {                                     // gradient->array() *= c0.array()  (:1060)
        grad_out[3 * q] = g0 * tx.x;
        grad_out[3 * q + 1] = g1 * ty.x;
        grad_out[3 * q + 2] = g2 * tz.x;
    }
    if (HESS) {                                     // d2/dx_a dx_b = (h_ab * c0_a) * c0_b, one value for [a][b] and [b][a]
        const double Hxx = (hxx * tx.x) * tx.x, Hxy = (hxy * tx.x) * ty.x, Hxz = (hxz * tx.x) * tz.x;
        const double Hyy = (hyy * ty.x) * ty.x, Hyz = (hyz * ty.x) * tz.x, Hzz = (hzz * tz.x) * tz.x;
        double* h = hess_out + 9 * q;
        h[0] = Hxx; h[1] = Hxy; h[2] = Hxz;
        h[3] = Hxy; h[4] = Hyy; h[5] = Hyz;
        h[6] = Hxz; h[7] = Hyz; h[8] = Hzz;
    }
}

// shape_function_ alone (diagnostics / dg_shape_functions): the rows of shape_rows.cuh, one thread per point.
__global__ void shape_functions_kernel(const double* __restrict__ xi, unsigned long long n, double* __restrict__ N, double* __restrict__ dN)
{
    const unsigned long long q = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    double* Nq = N + 32 * q;
    double* Dq = dN ? dN + 96 * q : nullptr;
    shape_rows(xi[3 * q], xi[3 * q + 1], xi[3 * q + 2], [&](int j, double nj, double d0, double d1, double d2) {
        Nq[j] = nj;
        if (Dq) { Dq[3 * j] = d0; Dq[3 * j + 1] = d1; Dq[3 * j + 2] = d2; }
    });
}

}  // namespace

cudaError_t k2_launch_pack(const GridDev& g, const double* d_nodes, const unsigned* d_cells, uint64_t n_cells_kept,
                           double* d_packed, cudaStream_t stream)
{
    if (n_cells_kept == 0) return cudaSuccess;
    const unsigned long long n32 = (unsigned long long)n_cells_kept * 32ull;
    DG_KERNEL_LAUNCH(pack_cells_kernel, (unsigned)((n32 + 255) / 256), 256, 0, stream, g, d_nodes, d_cells, n32, d_packed);
    return DG_AFTER_LAUNCH();
}

cudaError_t k2_launch_axis_tables(const GridDev& g, double2* d_tab, cudaStream_t stream)
{
    const unsigned n = g.n[0] + g.n[1] + g.n[2];
    DG_KERNEL_LAUNCH(axis_tables_kernel, (n + 127) / 128, 128, 0, stream, g, d_tab);
    return DG_AFTER_LAUNCH();
}

cudaError_t k2_launch_interpolate(const FieldDev& f, const double* d_x, uint64_t n, double* d_phi, double* d_grad,
                                  cudaStream_t stream, double* d_hess)
{
    if (n == 0) return cudaSuccess;
    if (d_hess && !d_grad) return cudaErrorInvalidValue;
    const unsigned blocks = (unsigned)((n + K2_THREADS - 1) / K2_THREADS);
    if (d_hess)
        DG_KERNEL_LAUNCH((interpolate_kernel<true, true>), blocks, K2_THREADS, 0, stream, f.g, f.packed, f.cell_map, f.tab, d_x, (unsigned long long)n, d_phi, d_grad, d_hess);
    else if (d_grad)
        DG_KERNEL_LAUNCH((interpolate_kernel<true, false>), blocks, K2_THREADS, 0, stream, f.g, f.packed, f.cell_map, f.tab, d_x, (unsigned long long)n, d_phi, d_grad, nullptr);
    else
        DG_KERNEL_LAUNCH((interpolate_kernel<false, false>), blocks, K2_THREADS, 0, stream, f.g, f.packed, f.cell_map, f.tab, d_x, (unsigned long long)n, d_phi, nullptr, nullptr);
    return DG_AFTER_LAUNCH();
}

cudaError_t k2_launch_shape_functions(const double* d_xi, uint64_t n, double* d_N, double* d_dN, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(shape_functions_kernel, (unsigned)((n + 127) / 128), 128, 0, stream, d_xi, (unsigned long long)n, d_N, d_dN);
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
