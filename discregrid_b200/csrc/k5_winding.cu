// K5: generalized winding numbers (Barill et al. 2018, "Fast Winding Numbers for Soups and Clouds") over the reference's sphere tree,
// and the winding sign mode of the signed distance built on them.  Beyond the reference, which signs with the angle-weighted
// pseudonormal (TriangleMeshDistance.h:269-308) -- a rule that is only right for closed manifold meshes.
//
// NUMERICAL CONTRACT (fp64, no FMA: the TU is compiled with -fmad=false, the host part with -ffp-contract=off)
//   Leaf records, in leaf order (HostBvh::order): the three vertices V[F[t]] as given -- not v0 + e0, which is not v1 bit for bit.
//   Exact term of a triangle at x: a = v0 - x, b = v1 - x, c = v2 - x (componentwise), |u| = sqrt((ux*ux + uy*uy) + uz*uz),
//       k = b x c = (by*cz - bz*cy, bz*cx - bx*cz, bx*cy - by*cx),  det = (ax*kx + ay*ky) + az*kz,
//       a.b = (ax*bx + ay*by) + az*bz,  b.c likewise,  c.a = (cx*ax + cy*ay) + cz*az,
//       den = (((|a|*|b|)*|c| + (a.b)*|c|) + (b.c)*|a|) + (c.a)*|b|,      Omega = 2.0 * k5_atan2(det, den)   (Van Oosterom-Strackee)
//   k5_atan2: written with IEEE + - * / sqrt and comparisons only (no libm), so the device, the CPU emulation and a numpy restatement agree
//       bit for bit; the reduction and the polynomial are fdlibm's atan (intervals 7/16, 11/16, 19/16, 39/16; atanhi/atanlo; 11 odd
//       coefficients), the quadrant logic fdlibm's atan2 with the exponent tests replaced by q = |y|/|x| > 2^60 and (x < 0 and q < 2^-60).
//       atan2(+-0, -x) = +-pi (x = -0 included), atan2(+-0, +x) = +-0, NaN in -> NaN out.  Within 2 ulp of a correctly rounded atan2.
//   Cluster records (host, build_winding_records) for every subtree of more than one triangle.  Per triangle first:
//       e0 = v1 - v0, e1 = v2 - v0, an = 0.5 * (e0 x e1) (same cross-product form), a = |an|, c = ((v0 + v1) + v2) / 3.0,
//       and the subtree sums A = a, AC = a*c, CS = c, N = an, cnt = 1, p~ = c, M = 0.
//   Then for the node with split position m: every sum is (left-subtree sum) + (right-subtree sum),
//       p~ = A > 0 ? AC / A : CS / cnt        (area-weighted centroid; the plain mean of the centroids for zero area)
//       n~ = N
//       M[j][k] = (M_L[j][k] + (p_L[j] - p~[j]) * N_L[k]) + (M_R[j][k] + (p_R[j] - p~[j]) * N_R[k])
//                 which is sum_t a_t (c_t - p~) (x) n_t regrouped, the first moment about p~
//       r_c = sqrt(max over the subtree's vertices v of |v - p~|^2)
//   stored as the spheres are: the children of the node with split position m at clusters[m].l / .r, the root at clusters[0].l.
//   Far-field term of a cluster at x: r = p~ - x, r2 = (rx*rx + ry*ry) + rz*rz; the cluster is far iff r2 > (beta*r_c) * (beta*r_c);
//       |r|^3 = r2 * sqrt(r2), |r|^5 = |r|^3 * r2, n.r = (nx*rx + ny*ry) + nz*rz, tr = (M00 + M11) + M22,
//       (Mr)_j = (Mj0*rx + Mj1*ry) + Mj2*rz, rMr = (rx*(Mr)_0 + ry*(Mr)_1) + rz*(Mr)_2,
//       term = (n.r / |r|^3 + tr / |r|^3) - (3.0 * rMr) / |r|^5      (dipole + first moment of the expansion of grad 1/(4 pi |r|))
//       A single triangle is always summed exactly.
//   The sum: the walk starts at the root and stops at far clusters and at triangles (the "cut").  S is the fp64 left fold, from 0.0, of the
//       cut's terms in increasing leaf position (left-child-first pre-order), w = S / 12.566370614359172 (the double nearest 4 pi).  Any walk
//       that adds in this order gives these bits.  beta = +inf: no cluster is far, the exact sum over all triangles.  beta >= 1 or +inf.
//   Sign rule: inside iff w > 0.5 (strict: on-surface points of flat or convex pieces, w = 1/2, 1/4, 1/8, stay +0 as with the reference's
//       >= 0); value = sign * (inside ? -d_u : d_u) with d_u the unsigned distance of K1 (same bits as the pseudonormal mode's magnitude).
//       Where the pseudonormal mode writes a sentinel (DBL_MAX outside a band; DBL_MAX for a query no triangle accepts, DESIGN §2 (v)), the
//       winding mode writes the same bits.
#include "k5_winding.h"
#include "dg_launch.h"       // DG_KERNEL_LAUNCH: <<<>>> on the device, fibers under tests/emu (DG_EMU)
#include "k5_atan2.h"

#include <cfloat>
#include <cmath>
#include <cstring>
#include <future>
#include <algorithm>

namespace dgb {

// ------------------------------------------------------------------------------------------------ arithmetic (host and device)
// k5_atan2 and its helpers: k5_atan2.h (shared with the refit, k8_refit.cu)
double k5_atan2_host(double y, double x) { return k5_atan2(y, x); }

// solid angle of the triangle v[9] seen from p (exact term)
DG_HD double k5_solid_angle(const double* __restrict__ v, double px, double py, double pz)
{
    const double ax = v[0] - px, ay = v[1] - py, az = v[2] - pz;
    const double bx = v[3] - px, by = v[4] - py, bz = v[5] - pz;
    const double cx = v[6] - px, cy = v[7] - py, cz = v[8] - pz;
    const double la = sqrt(ax * ax + ay * ay + az * az), lb = sqrt(bx * bx + by * by + bz * bz), lc = sqrt(cx * cx + cy * cy + cz * cz);
    const double kx = by * cz - bz * cy, ky = bz * cx - bx * cz, kz = bx * cy - by * cx;
    const double det = ax * kx + ay * ky + az * kz;
    const double ab = ax * bx + ay * by + az * bz, bc = bx * cx + by * cy + bz * cz, ca = cx * ax + cy * ay + cz * az;
    const double den = la * lb * lc + ab * lc + bc * la + ca * lb;
    return 2.0 * k5_atan2(det, den);
}

DG_HD double k5_far_term(const WindCluster& c, double rx, double ry, double rz, double r2)
{
    const double r3 = r2 * sqrt(r2), r5 = r3 * r2;
    const double dip = c.n[0] * rx + c.n[1] * ry + c.n[2] * rz;
    const double tr = c.M[0] + c.M[4] + c.M[8];
    const double m0 = c.M[0] * rx + c.M[1] * ry + c.M[2] * rz;
    const double m1 = c.M[3] * rx + c.M[4] * ry + c.M[5] * rz;
    const double m2 = c.M[6] * rx + c.M[7] * ry + c.M[8] * rz;
    const double rmr = rx * m0 + ry * m1 + rz * m2;
    return (dip / r3 + tr / r3) - (3.0 * rmr) / r5;
}

// ------------------------------------------------------------------------------------------------ the walk
#ifdef DG_EMU
extern uint2 k5_stack[];                           // defined by the emulation TU (one block runs at a time)
#else
extern __shared__ uint2 k5_stack[];
#endif

// S of the contract: pre-order, left child first; the deferred right children [m, e) wait on the lane's stack (k5_stack[depth][lane]), and
// their record is clusters[m].r, that of a left child [b, m) clusters[m].l
__device__ __forceinline__ double k5_winding_sum(const WindDev& m, double px, double py, double pz, double beta)
{
    uint2* stack = k5_stack + threadIdx.x;
    double S = 0.0;
    unsigned b = 0, e = (unsigned)m.n_tri, rec = 0;
    bool right = false;
    int sp = 0;
    for (;;) {
        if (e - b == 1u) {
            S = S + k5_solid_angle(m.leaves[b].v, px, py, pz);
        } else {
            const WindCluster& c = right ? m.clusters[rec].r : m.clusters[rec].l;
            const double rx = c.p[0] - px, ry = c.p[1] - py, rz = c.p[2] - pz;
            const double r2 = rx * rx + ry * ry + rz * rz;
            const double br = beta * c.r;
            if (r2 > br * br) {
                S = S + k5_far_term(c, rx, ry, rz, r2);
            } else {
                const unsigned mid = (b + e) >> 1;
                stack[(size_t)sp * K5_THREADS] = make_uint2(mid, e);
                sp++;
                e = mid; rec = mid; right = false;
                continue;
            }
        }
        if (sp == 0) break;
        sp--;
        const uint2 t = stack[(size_t)sp * K5_THREADS];
        b = t.x; e = t.y; rec = t.x; right = true;
    }
    return S;
}

__global__ void __launch_bounds__(K5_THREADS)
winding_number_kernel(WindDev m, const double* __restrict__ pts, unsigned long long n, double beta, double* __restrict__ w)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * K5_THREADS + threadIdx.x;
    if (idx >= n) return;
    w[idx] = k5_winding_sum(m, pts[3 * idx], pts[3 * idx + 1], pts[3 * idx + 2], beta) / k5::FOUR_PI;
}

// the node pass: one lane per node id, so the lanes of a warp are neighbouring nodes of one node array
__global__ void __launch_bounds__(K5_THREADS)
winding_sign_nodes_kernel(WindDev m, GridDev g, unsigned l_begin, unsigned long long count, double sign, double band, double beta,
                          double* __restrict__ vals)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * K5_THREADS + threadIdx.x;
    if (idx >= count) return;
    const double v = vals[idx];
    if (v == DBL_MAX) {            // outside the band, or no triangle accepted: K1's own epilogue with `sign`
        vals[idx] = (fabs(v) <= band) ? ((sign == 1.0) ? v : sign * v) : DBL_MAX;
        return;
    }
    double px, py, pz;
    node_position(g, l_begin + (unsigned)idx, px, py, pz);
    const double du = fabs(v);
    const double s = (k5_winding_sum(m, px, py, pz, beta) / k5::FOUR_PI > 0.5) ? -du : du;
    vals[idx] = (sign == 1.0) ? s : sign * s;
}

__global__ void __launch_bounds__(K5_THREADS)
winding_sign_points_kernel(WindDev m, const double* __restrict__ pts, unsigned long long n, double beta, double* __restrict__ dist)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * K5_THREADS + threadIdx.x;
    if (idx >= n) return;
    const double d = dist[idx];
    if (d == DBL_MAX) return;
    const double w = k5_winding_sum(m, pts[3 * idx], pts[3 * idx + 1], pts[3 * idx + 2], beta) / k5::FOUR_PI;
    dist[idx] = (w > 0.5) ? -d : d;
}

// ------------------------------------------------------------------------------------------------ launchers
static size_t k5_smem_bytes(const WindDev& m) { return (size_t)m.stack_depth * K5_THREADS * sizeof(uint2); }
static unsigned k5_blocks(uint64_t n) { return (unsigned)((n + K5_THREADS - 1) / K5_THREADS); }

cudaError_t k5_launch_winding(const WindDev& m, const double* d_pts, uint64_t n, double beta, double* d_w, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(winding_number_kernel, k5_blocks(n), K5_THREADS, k5_smem_bytes(m), stream, m, d_pts, (unsigned long long)n, beta, d_w);
    return DG_AFTER_LAUNCH();
}

cudaError_t k5_launch_sign_nodes(const WindDev& m, const GridDev& g, double sign, double band, double beta, uint64_t l_begin, uint64_t count,
                                 double* d_vals, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(winding_sign_nodes_kernel, k5_blocks(count), K5_THREADS, k5_smem_bytes(m), stream, m, g, (unsigned)l_begin,
                     (unsigned long long)count, sign, band, beta, d_vals);
    return DG_AFTER_LAUNCH();
}

cudaError_t k5_launch_sign_points(const WindDev& m, const double* d_pts, uint64_t n, double beta, double* d_dist, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(winding_sign_points_kernel, k5_blocks(n), K5_THREADS, k5_smem_bytes(m), stream, m, d_pts, (unsigned long long)n, beta, d_dist);
    return DG_AFTER_LAUNCH();
}

// ------------------------------------------------------------------------------------------------ host: the records
namespace {
struct WindSums { double A, AC[3], CS[3], N[3], p[3], M[9], cnt; };

struct WindBuilder {
    const HostBvh& h;
    RawVec<WindClusterPair>& out;
    int par_levels;

    const double* vert(int32_t tri, int k) const { return &h.V[3 * (size_t)h.F[3 * (size_t)tri + k]]; }

    WindSums leaf(int32_t tri) const
    {
        const double* v0 = vert(tri, 0); const double* v1 = vert(tri, 1); const double* v2 = vert(tri, 2);
        const double e0[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]}, e1[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
        WindSums s;
        s.N[0] = 0.5 * (e0[1] * e1[2] - e0[2] * e1[1]);
        s.N[1] = 0.5 * (e0[2] * e1[0] - e0[0] * e1[2]);
        s.N[2] = 0.5 * (e0[0] * e1[1] - e0[1] * e1[0]);
        s.A = std::sqrt(s.N[0] * s.N[0] + s.N[1] * s.N[1] + s.N[2] * s.N[2]);
        for (int d = 0; d < 3; d++) {
            const double c = (v0[d] + v1[d] + v2[d]) / 3.0;
            s.CS[d] = c; s.p[d] = c; s.AC[d] = s.A * c;
        }
        for (int k = 0; k < 9; k++) s.M[k] = 0.0;
        s.cnt = 1.0;
        return s;
    }

    WindSums build(int b, int e, WindCluster* slot, int depth)
    {
        if (e - b == 1) return leaf(h.order[b]);
        const int m = (b + e) >> 1;
        WindClusterPair& pr = out[m];
        WindSums L, R;
        if (depth <= par_levels && e - b >= 4096) {
            auto left = std::async(std::launch::async, [&, b, m, depth]() { return build(b, m, &pr.l, depth + 1); });
            R = build(m, e, &pr.r, depth + 1);
            L = left.get();
        } else {
            L = build(b, m, &pr.l, depth + 1);
            R = build(m, e, &pr.r, depth + 1);
        }
        WindSums s;
        s.A = L.A + R.A; s.cnt = L.cnt + R.cnt;
        for (int d = 0; d < 3; d++) { s.AC[d] = L.AC[d] + R.AC[d]; s.CS[d] = L.CS[d] + R.CS[d]; s.N[d] = L.N[d] + R.N[d]; }
        for (int d = 0; d < 3; d++) s.p[d] = (s.A > 0.0) ? s.AC[d] / s.A : s.CS[d] / s.cnt;
        for (int j = 0; j < 3; j++)
            for (int k = 0; k < 3; k++)
                s.M[3 * j + k] = (L.M[3 * j + k] + (L.p[j] - s.p[j]) * L.N[k]) + (R.M[3 * j + k] + (R.p[j] - s.p[j]) * R.N[k]);
        double r2 = 0.0;
        for (int i = b; i < e; i++)
            for (int k = 0; k < 3; k++) {
                const double* v = vert(h.order[i], k);
                const double dx = v[0] - s.p[0], dy = v[1] - s.p[1], dz = v[2] - s.p[2];
                r2 = std::max(r2, dx * dx + dy * dy + dz * dz);
            }
        for (int d = 0; d < 3; d++) { slot->p[d] = s.p[d]; slot->n[d] = s.N[d]; }
        for (int k = 0; k < 9; k++) slot->M[k] = s.M[k];
        slot->r = std::sqrt(r2);
        return s;
    }
};
}  // namespace

void build_winding_records(const HostBvh& h, RawVec<WindLeaf>& leaves, RawVec<WindClusterPair>& clusters)
{
    const uint64_t nT = h.n_triangles;
    leaves.resize(nT);
    clusters.resize(nT);
    parallel_for(nT, [&](uint64_t p0, uint64_t p1) {
        for (uint64_t pos = p0; pos < p1; pos++) {
            const uint32_t* t = &h.F[3 * (size_t)h.order[pos]];
            for (int k = 0; k < 3; k++)
                for (int d = 0; d < 3; d++) leaves[pos].v[3 * k + d] = h.V[3 * (size_t)t[k] + d];
            std::memset(&clusters[pos], 0, sizeof(WindClusterPair));          // leaf children and the root's right slot stay zero
        }
    });
    unsigned hw = host_threads(); if (hw == 0) hw = 1; if (hw > 64) hw = 64;
    int lv = 0; while ((1u << (lv + 1)) <= hw && lv < 6) lv++;
    WindBuilder bld{h, clusters, lv};
    bld.build(0, (int)nT, &clusters[0].l, 1);
}

}  // namespace dgb
