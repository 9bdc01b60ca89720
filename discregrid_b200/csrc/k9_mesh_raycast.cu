// K9: the first hit of each of n rays (or segments) on a triangle mesh, through the sphere tree's fp32 child boxes.  One thread per ray.
//
// The reference has no such function, so this contract is the library's own.  tests/mesh_raycast_ref.py restates it in numpy as a brute-force
// loop over every triangle, and the tests compare t, triangle_id, barycentric and status bit for bit.
//
// Inputs.  Rays i = 0..n-1 with origin o[3] and direction d[3]; one interval [t_min, t_max] for all rays, neither bound NaN, t_min <= t_max,
//   either bound may be infinite.  A segment x0 -> x1 is the ray (x0, x1 - x0) on [0, 1].  The ray misses if o or d is not finite, or d = 0.
// Triangle test (Woop, Benthin and Wald, "Watertight ray/triangle intersection", JCGT 2013), IEEE fp64 without contraction.  The vertices
//   are V[F[id]] exactly, as K5's WindLeaf records hold them (never v0 + e0 of the LeafRecord, which is rounded per triangle).
//   - kz = the axis of largest |d_a| (the first on ties), kx = (kz + 1) % 3, ky = (kx + 1) % 3; kx and ky swap when d[kz] < 0.
//   - Sx = d[kx] / d[kz], Sy = d[ky] / d[kz], Sz = 1.0 / d[kz].
//   - For each vertex P of (v0, v1, v2) -> (A, B, C): p = P - o (three subtractions), Px = p[kx] - Sx * p[kz], Py = p[ky] - Sy * p[kz],
//     Pz = Sz * p[kz].
//   - U = Cx * By - Cy * Bx, V = Ax * Cy - Ay * Cx, W = Bx * Ay - By * Ax.
//   - det = (U + V) + W, T = (U * Az + V * Bz) + W * Cz, t = T / det.
//   - zl = min(Az, Bz, Cz) and zh = max(Az, Bz, Cz) as (a < b ? a : b) folded left to right (and (a < b ? b : a)); tol = max(|zl|, |zh|) *
//     2^-49 (the same fold).
//   Accept iff all of:
//     (U >= 0 && V >= 0 && W >= 0) || (U <= 0 && V <= 0 && W <= 0)        (the positive form, so that NaN rejects)
//     det != 0
//     !(Ax > 0 && Bx > 0 && Cx > 0) && !(Ax < 0 && Bx < 0 && Cx < 0), and the same for y   (the origin lies in the sheared bounding box)
//     zl - tol <= t && t <= zh + tol                                       (t lies in the hull of Az, Bz, Cz, widened by tol)
//     t_min <= t && t <= t_max                                             (inclusive; NaN rejects)
// Why it is watertight.  A vertex's sheared coordinates depend only on the vertex and the ray, so a shared edge gives the same sheared
//   vertices in both of its triangles, and IEEE fl(a*b) - fl(c*d) is exactly antisymmetric: the two triangles' edge functions for that edge
//   are exact negatives.  A ray through the edge is therefore accepted by at least one of them.  More generally the sheared vertices of a
//   closed mesh form a closed piecewise-linear surface around the origin of the sheared frame, so the line x = y = 0 meets the exact hull of
//   some triangle's sheared vertices; the computed signs of that triangle's edge functions are then the exact ones or zero (rounding is
//   monotone), so it passes the sign test, and its origin lies in its bounding box.  The two conditions beyond the paper never reject such a
//   triangle: its t is a convex combination of Az, Bz, Cz up to about 6 ulp of max |Z| (U, V, W share a sign), well inside tol, unless every
//   product U * Az ... is subnormal.
// Why the two extra conditions.  For a ray that lies in a triangle's plane (to rounding), the paper's test alone accepts triangles far from
//   the ray: the sheared vertices then lie on a line through the origin, U, V and W are rounding noise and share a sign about one time in ten,
//   and T / det is noise too when det is subnormal.  No bound on a box could then say which boxes hold no acceptable triangle.  With the
//   bounding-box and hull conditions an accepted triangle has its origin inside its sheared bounding box and its t inside its widened z range,
//   and both are bounded by the box of any subtree that holds it (below).
// Result per ray.  Among the accepted triangles, the lexicographic minimum of (t, id), id the original triangle index; t values compare as
//   numbers (-0.0 == +0.0, the lower id wins) and the reported t has the winner's bits.  This does not depend on the traversal order, so a
//   brute-force loop over all triangles is an exact oracle.  Outputs: t[i], triangle_id[i], barycentric[3 i..] = (U / det, V / det, W / det)
//   (the weights of v0, v1, v2 of F[id]; may be NULL), status[i] = DG_RAY_ENTER (1) when det > 0, DG_RAY_LEAVE (2) when det < 0.  det > 0 is
//   the side from which a ray enters a closed, outward-oriented mesh (det = -(n . d) up to the positive scale of the shear, n = the
//   triangle's (v1 - v0) x (v2 - v0); tests/test_mesh_raycast_emulated.py pins it with box.obj).  A miss gives DG_RAY_MISS (0), t = +inf,
//   id = -1 and barycentric = NaN (0x7ff8000000000000).
//
// Culling (changes no result).  A subtree is skipped only when no triangle under it can be accepted with a t that could still win:
//   1. Box in doubles.  The fp32 child boxes are lo_f = round_down(fl(b_lo - ctr)), hi_f = round_up(fl(b_hi - ctr)) (make_box_shadow), with
//      |b - ctr| <= half_extent.  With He = 2 * half_extent and s_a = (|ctr_a| + He) * 2^-50, L_a = fl(fl(ctr_a + lo_f) - s_a) and
//      H_a = fl(fl(ctr_a + hi_f) + s_a) bound every vertex coordinate of the subtree: the three roundings (b - ctr; ctr + lo_f; +- s_a) add
//      at most 2^-53 (2 |ctr_a| + 3 He) < s_a.
//   2. Monotone bounds of the computed test.  IEEE rounding is monotone, so the computed Pz = fl(Sz * fl(P[kz] - o[kz])) is monotone in
//      P[kz] (increasing iff Sz > 0), and the computed Px = fl(fl(P[kx] - o[kx]) - fl(Sx * fl(P[kz] - o[kz]))) is increasing in P[kx] and
//      monotone in P[kz] (decreasing iff Sx >= 0).  Evaluating the same expressions at the box corners therefore bounds the computed
//      sheared coordinates of every vertex under the subtree: Xlo <= Px <= Xhi, Ylo <= Py <= Yhi, Zlo <= Pz <= Zhi, with no error term.
//   3. Cull iff Xlo > 0 || Xhi < 0 || Ylo > 0 || Yhi < 0 (the bounding-box condition then fails for every triangle under it), or
//      t_enter > best || t_exit < t_min, where tolb = max(|Zlo|, |Zhi|) * 2^-49, t_enter = Zlo - tolb, t_exit = Zhi + tolb and best is the t
//      of the current best hit (t_max before the first).  An accepted triangle has zl >= Zlo and tol <= tolb, so t >= fl(zl - tol) >= t_enter
//      (monotone again); likewise t <= t_exit.  The comparison with best is strict: a tie at equal t can still be won by a lower id.
//   A NaN bound compares false and culls nothing.  Culling is off for the whole ray (every subtree is visited) when half_extent is not finite
//   (a non-finite vertex, as K1 switches its filters off), when Sz is not finite, or when some |o_a| or |ctr_a| + 2 He exceeds 2^1020 (so
//   that no box coordinate minus the origin overflows).  K9_CULL=0 compiles culling out (tests/emu builds both and compares them).
//
// Traversal (a choice that changes no result).  The implicit tree of K1: a node is the leaf range [b, e), its children split at
// m = (b + e) >> 1 and their boxes are float4s 2..4 of the K1_NODEF_STRIDE record at nodes_f[m].  A child of one triangle is tested at once;
// of two internal children that pass the nearer (smaller t_enter) is visited first and the other is pushed with its t_enter, which is checked
// against best again when it is popped (at most stack_depth entries).  LeafRecord::tri_id is read only where an id is needed: at a tie and
// for a new best.  No warp collectives, so tests/emu runs the kernel as it is.  A one-triangle mesh has no internal node: its triangle is
// tested directly.
#include "k9_mesh_raycast.h"
#include "dg_launch.h"

#include <cfloat>
#include <cmath>

#ifndef K9_CULL
#define K9_CULL 1
#endif
#ifdef DG_EMU
#define K9_COUNT(i) (dg_emu::g_counters[(i)]++)            // tests/emu counters: 8 boxes tested, 9 triangles tested, 10 rays
#else
#define K9_COUNT(i)
#endif

namespace dgb {
namespace {

constexpr int K9_MISS = 0, K9_ENTER = 1, K9_LEAVE = 2;       // DG_RAY_MISS, DG_RAY_ENTER, DG_RAY_LEAVE of the C-ABI

struct K9Ray {
    double ox, oy, oz;                                // o[kx], o[ky], o[kz]
    int kx, ky, kz;
    double Sx, Sy, Sz;
};

// p[k] by selects, so that arrays indexed by the ray's axes stay in registers
__device__ __forceinline__ double k9_sel(const double* p, int k) { return k == 0 ? p[0] : (k == 1 ? p[1] : p[2]); }

struct K9Hit {
    double t, U, V, W, det;
};

// the contract's triangle test on the vertices v[9]; true with the hit's t, U, V, W and det when accepted
__device__ __forceinline__ bool k9_triangle(const K9Ray& r, const double* v, double t_min, double t_max, K9Hit& h)
{
    double X[3], Y[3], Z[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const double px = k9_sel(v + 3 * k, r.kx) - r.ox, py = k9_sel(v + 3 * k, r.ky) - r.oy, pz = k9_sel(v + 3 * k, r.kz) - r.oz;
        X[k] = px - r.Sx * pz;
        Y[k] = py - r.Sy * pz;
        Z[k] = r.Sz * pz;
    }
    const double U = X[2] * Y[1] - Y[2] * X[1];
    const double V = X[0] * Y[2] - Y[0] * X[2];
    const double W = X[1] * Y[0] - Y[1] * X[0];
    if (!((U >= 0.0 && V >= 0.0 && W >= 0.0) || (U <= 0.0 && V <= 0.0 && W <= 0.0))) return false;
    const double det = (U + V) + W;
    if (det == 0.0) return false;
    if ((X[0] > 0.0 && X[1] > 0.0 && X[2] > 0.0) || (X[0] < 0.0 && X[1] < 0.0 && X[2] < 0.0)) return false;
    if ((Y[0] > 0.0 && Y[1] > 0.0 && Y[2] > 0.0) || (Y[0] < 0.0 && Y[1] < 0.0 && Y[2] < 0.0)) return false;
    const double T = (U * Z[0] + V * Z[1]) + W * Z[2];
    const double t = T / det;
    double zl = Z[0] < Z[1] ? Z[0] : Z[1];
    zl = zl < Z[2] ? zl : Z[2];
    double zh = Z[0] < Z[1] ? Z[1] : Z[0];
    zh = zh < Z[2] ? Z[2] : zh;
    const double tol = (fabs(zl) < fabs(zh) ? fabs(zh) : fabs(zl)) * 0x1p-49;
    if (!(zl - tol <= t && t <= zh + tol)) return false;
    if (!(t_min <= t && t <= t_max)) return false;
    h.t = t; h.U = U; h.V = V; h.W = W; h.det = det;
    return true;
}

// per-ray constants of the box test: the origin, and the slack that turns an fp32 box into doubles bounding its vertices
struct K9Cull {
    double ctr[3], s[3];
};

// the contract's bounds of one child box (lo, hi: fp32, relative to ctr): false when culled, else its t_enter
__device__ __forceinline__ bool k9_box(const K9Ray& r, const K9Cull& c, const float* lo, const float* hi, double t_min, double best,
                                       double& t_enter)
{
    double L[3], H[3];
#pragma unroll
    for (int a = 0; a < 3; a++) {
        L[a] = (c.ctr[a] + (double)lo[a]) - c.s[a];
        H[a] = (c.ctr[a] + (double)hi[a]) + c.s[a];
    }
    const double Lx = k9_sel(L, r.kx), Ly = k9_sel(L, r.ky), Lz = k9_sel(L, r.kz);
    const double Hx = k9_sel(H, r.kx), Hy = k9_sel(H, r.ky), Hz = k9_sel(H, r.kz);
    const double zlo = r.Sz * ((r.Sz > 0.0 ? Lz : Hz) - r.oz);
    const double zhi = r.Sz * ((r.Sz > 0.0 ? Hz : Lz) - r.oz);
    const double tolb = (fabs(zlo) < fabs(zhi) ? fabs(zhi) : fabs(zlo)) * 0x1p-49;
    t_enter = zlo - tolb;
    const double t_exit = zhi + tolb;
    if (t_enter > best || t_exit < t_min) return false;
    const double xlo = (Lx - r.ox) - r.Sx * ((r.Sx >= 0.0 ? Hz : Lz) - r.oz);
    const double xhi = (Hx - r.ox) - r.Sx * ((r.Sx >= 0.0 ? Lz : Hz) - r.oz);
    if (xlo > 0.0 || xhi < 0.0) return false;
    const double ylo = (Ly - r.oy) - r.Sy * ((r.Sy >= 0.0 ? Hz : Lz) - r.oz);
    const double yhi = (Hy - r.oy) - r.Sy * ((r.Sy >= 0.0 ? Lz : Hz) - r.oz);
    return !(ylo > 0.0 || yhi < 0.0);
}

struct K9Best {
    double t;
    int id;
    K9Hit h;
};

// tests the triangle at leaf position p and keeps it when (t, id) beats the best
__device__ __forceinline__ void k9_leaf(const K9Ray& r, const DeviceBvh& m, const WindLeaf* __restrict__ wl, int p, double t_min, double t_max,
                                        K9Best& b)
{
    K9_COUNT(9);
    double v[9];
    const double* src = wl[p].v;
#pragma unroll
    for (int k = 0; k < 9; k++) v[k] = __ldg(src + k);
    K9Hit h;
    if (!k9_triangle(r, v, t_min, t_max, h)) return;
    if (b.id >= 0 && h.t > b.t) return;
    const int id = __ldg(&m.leaves[p].tri_id);
    if (b.id >= 0 && h.t == b.t && id >= b.id) return;
    b.t = h.t; b.id = id; b.h = h;
}

__global__ void __launch_bounds__(K9_THREADS)
mesh_raycast_kernel(DeviceBvh m, const WindLeaf* __restrict__ wl, const double* __restrict__ o_in, const double* __restrict__ d_in,
                    unsigned long long n, double t_min, double t_max, double* __restrict__ t_out, int* __restrict__ id_out,
                    double* __restrict__ bary_out, int* __restrict__ status_out)
{
    const unsigned long long q = (unsigned long long)blockIdx.x * K9_THREADS + threadIdx.x;
    if (q >= n) return;
    K9_COUNT(10);
    K9Ray r;
    double o[3], d[3];
    bool finite = true, nonzero = false;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        o[a] = o_in[3 * q + a]; d[a] = d_in[3 * q + a];
        finite &= fabs(o[a]) <= DBL_MAX && fabs(d[a]) <= DBL_MAX;
        nonzero |= d[a] != 0.0;
    }
    K9Best b;
    b.t = t_max; b.id = -1;
    if (finite && nonzero) {
        int kz = 0;
        if (fabs(d[1]) > fabs(d[0])) kz = 1;
        if (fabs(d[2]) > fabs(k9_sel(d, kz))) kz = 2;
        int kx = kz + 1 == 3 ? 0 : kz + 1;
        int ky = kx + 1 == 3 ? 0 : kx + 1;
        if (k9_sel(d, kz) < 0.0) { const int s = kx; kx = ky; ky = s; }
        r.kx = kx; r.ky = ky; r.kz = kz;
        r.ox = k9_sel(o, kx); r.oy = k9_sel(o, ky); r.oz = k9_sel(o, kz);
        const double dx = k9_sel(d, kx), dy = k9_sel(d, ky), dz = k9_sel(d, kz);
        r.Sx = dx / dz; r.Sy = dy / dz; r.Sz = 1.0 / dz;

        K9Cull c;
        const double He = 2.0 * (double)m.half_extent;
        bool cull = K9_CULL && fabs(He) <= DBL_MAX && fabs(r.Sz) <= DBL_MAX;
#pragma unroll
        for (int a = 0; a < 3; a++) {
            c.ctr[a] = m.ctr[a];
            c.s[a] = (fabs(m.ctr[a]) + He) * 0x1p-50;
            cull = cull && fabs(o[a]) <= 0x1p1020 && fabs(m.ctr[a]) + He <= 0x1p1020;
        }
        if (m.n_tri == 1) {
            k9_leaf(r, m, wl, 0, t_min, t_max, b);
        } else {
            int stk_b[K9_MAX_STACK], stk_e[K9_MAX_STACK];
            double stk_t[K9_MAX_STACK];
            int sp = 0;
            int nb = 0, ne = m.n_tri;                                           // the current internal node [nb, ne)
            for (;;) {
                const int mid = (nb + ne) >> 1;
                const float4* rec = m.nodes_f + (size_t)mid * K1_NODEF_STRIDE;
                const float4 q0 = __ldg(rec + 2), q1 = __ldg(rec + 3), q2 = __ldg(rec + 4);
                const float l_lo[3] = {q0.x, q0.y, q0.z}, l_hi[3] = {q0.w, q1.x, q1.y};
                const float r_lo[3] = {q1.z, q1.w, q2.x}, r_hi[3] = {q2.y, q2.z, q2.w};
                double tl = -INFINITY, tr = -INFINITY;
                K9_COUNT(8); K9_COUNT(8);
                bool hl = !cull || k9_box(r, c, l_lo, l_hi, t_min, b.t, tl);
                bool hr = !cull || k9_box(r, c, r_lo, r_hi, t_min, b.t, tr);
                if (hl && mid - nb == 1) { k9_leaf(r, m, wl, nb, t_min, t_max, b); hl = false; }
                if (hr && ne - mid == 1) { k9_leaf(r, m, wl, mid, t_min, t_max, b); hr = false; }
                if (hl && hr) {
                    const bool left_first = !(tr < tl);
                    stk_b[sp] = left_first ? mid : nb; stk_e[sp] = left_first ? ne : mid; stk_t[sp] = left_first ? tr : tl; sp++;
                    if (left_first) ne = mid; else nb = mid;
                } else if (hl) {
                    ne = mid;
                } else if (hr) {
                    nb = mid;
                } else {
                    bool found = false;
                    while (sp > 0) {
                        sp--;
                        if (cull && stk_t[sp] > b.t) continue;                  // a better hit was found since it was pushed
                        nb = stk_b[sp]; ne = stk_e[sp]; found = true;
                        break;
                    }
                    if (!found) break;
                }
            }
        }
    }
    if (b.id >= 0) {
        t_out[q] = b.t;
        id_out[q] = b.id;
        if (bary_out) {
            bary_out[3 * q] = b.h.U / b.h.det; bary_out[3 * q + 1] = b.h.V / b.h.det; bary_out[3 * q + 2] = b.h.W / b.h.det;
        }
        status_out[q] = b.h.det > 0.0 ? K9_ENTER : K9_LEAVE;
    } else {
        t_out[q] = INFINITY;
        id_out[q] = -1;
        if (bary_out) {
            const double nan = __longlong_as_double(0x7ff8000000000000LL);
            bary_out[3 * q] = nan; bary_out[3 * q + 1] = nan; bary_out[3 * q + 2] = nan;
        }
        status_out[q] = K9_MISS;
    }
}

}  // namespace

cudaError_t k9_launch_mesh_raycast(const DeviceBvh& m, const WindDev& w, const double* d_o, const double* d_d, uint64_t n, double t_min,
                                   double t_max, double* d_t, int32_t* d_id, double* d_bary, int32_t* d_status, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((n + K9_THREADS - 1) / K9_THREADS);
    DG_KERNEL_LAUNCH(mesh_raycast_kernel, blocks, K9_THREADS, 0, stream, m, w.leaves, d_o, d_d, (unsigned long long)n, t_min, t_max, d_t,
                     (int*)d_id, d_bary, (int*)d_status);
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
