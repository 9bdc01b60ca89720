// Per-record expressions of the mesh's device records, written once for the host builder (bvh_build.cpp, g++ -ffp-contract=off) and for
// the device refit (k8_refit.cu, nvcc -fmad=false): a record computed from the same vertices has the same bits on both sides.
// max / min are std::max / std::max's own comparisons (first argument kept on ties and when the second is NaN); rounding to fp32 is
// IEEE round-to-nearest, and nextafterf is exact on both sides.
#pragma once
#include <cfloat>
#include <cmath>
#include "bvh_build.h"
#include "dg_device.cuh"

namespace dgb {
#if !defined(__CUDACC__)
using std::fabs; using std::isfinite; using std::nextafterf; using std::sqrt;
#endif

DG_HD double rec_max(double a, double b) { return (a < b) ? b : a; }   // std::max(a, b)
DG_HD double rec_min(double a, double b) { return (b < a) ? b : a; }   // std::min(a, b)

// fp32 bounds rounded outward: down(v) <= v <= up(v) for every finite v
DG_HD float rec_down(double v) { const float f = (float)v; return ((double)f > v) ? nextafterf(f, -INFINITY) : f; }
DG_HD float rec_up(double v) { const float f = (float)v; return ((double)f < v) ? nextafterf(f, INFINITY) : f; }

// the 128-byte leaf record of the triangle (v0, v1, v2) (TriangleMeshDistance.h:567-575, 675, 693)
DG_HD void make_leaf_record(const double* v0, const double* v1, const double* v2, int32_t id, LeafRecord& L)
{
    double e0[3], e1[3];
    for (int d = 0; d < 3; d++) { e0[d] = v1[d] - v0[d]; e1[d] = v2[d] - v0[d]; }
    for (int d = 0; d < 3; d++) { L.v0[d] = v0[d]; L.e0[d] = e0[d]; L.e1[d] = e1[d]; }
    L.a00 = e0[0] * e0[0] + e0[1] * e0[1] + e0[2] * e0[2];
    L.a01 = e0[0] * e1[0] + e0[1] * e1[1] + e0[2] * e1[2];
    L.a11 = e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2];
    L.det = fabs(L.a00 * L.a11 - L.a01 * L.a01);
    L.inv_det = 1 / L.det;
    L.denom = L.a00 - 2 * L.a01 + L.a11;
    L.tri_id = id; L._pad = 0;
}

// fp32 shadow of a leaf record relative to `center` (all products in fp64, rounded once)
DG_HD void make_leaf_shadow(const LeafRecord& L, const double* center, LeafF& f)
{
    double e2[3], n3[3];
    for (int d = 0; d < 3; d++) { f.v0[d] = (float)(L.v0[d] - center[d]); f.e0[d] = (float)L.e0[d]; f.e1[d] = (float)L.e1[d]; e2[d] = L.e1[d] - L.e0[d]; }
    n3[0] = L.e0[1] * L.e1[2] - L.e0[2] * L.e1[1]; n3[1] = L.e0[2] * L.e1[0] - L.e0[0] * L.e1[2]; n3[2] = L.e0[0] * L.e1[1] - L.e0[1] * L.e1[0];
    f.d00 = (float)L.a00; f.d01 = (float)L.a01; f.d11 = (float)L.a11; f.d22 = (float)(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
    // UNIT normal: the filter's (w.n)^2 then scales like a squared distance and stays a normal fp32 number wherever the filter runs
    // (e0 x e1 scales like length^2, so with it (w.n)^2 overflows fp32 for meshes of size ~1e6 and goes subnormal at ~1e-7).  Zero
    // area (or a non-finite mesh): n = 0, i.e. no plane bound.  The max-component scaling keeps n.n clear of fp64 under/overflow.
    const double s = rec_max(fabs(n3[0]), rec_max(fabs(n3[1]), fabs(n3[2])));
    const double len = (s > 0 && isfinite(s)) ? s * sqrt((n3[0] / s) * (n3[0] / s) + (n3[1] / s) * (n3[1] / s) + (n3[2] / s) * (n3[2] / s)) : 0.0;
    for (int d = 0; d < 3; d++) f.n[d] = (len > 0) ? (float)(n3[d] / len) : 0.f;
}

// bounding sphere of one triangle (TriangleMeshDistance.h:451-458): centre ((a + b) + c) / 3, radius the max of the three distances
DG_HD void make_leaf_sphere(const double* a, const double* b, const double* c, double* ctr, double& r)
{
    for (int d = 0; d < 3; d++) ctr[d] = ((a[d] + b[d]) + c[d]) / 3.0;
    double l[3];
    const double* v[3] = {a, b, c};
    for (int k = 0; k < 3; k++) {
        const double x = v[k][0] - ctr[0], y = v[k][1] - ctr[1], z = v[k][2] - ctr[2];
        l[k] = sqrt(x * x + y * y + z * z);
    }
    r = rec_max(rec_max(l[0], l[1]), l[2]);
}

// axis-aligned box of one triangle as its parent records it: {lo, hi} = std::min / std::max of the three vertices, nested left to right
DG_HD void make_leaf_box(const double* a, const double* b, const double* c, double* box)
{
    for (int d = 0; d < 3; d++) { box[d] = rec_min(rec_min(a[d], b[d]), c[d]); box[3 + d] = rec_max(rec_max(a[d], b[d]), c[d]); }
}

// fp32 shadow of a sphere pair relative to `center`
DG_HD void make_sphere_shadow(const SpherePair& sp, const double* center, SpherePairF& f)
{
    for (int d = 0; d < 3; d++) { f.lc[d] = (float)(sp.lc[d] - center[d]); f.rc[d] = (float)(sp.rc[d] - center[d]); }
    f.lr = (float)sp.lr; f.rr = (float)sp.rr;
}

// fp32 child boxes (bx = {left lo, left hi, right lo, right hi}) relative to `center`, rounded outward
DG_HD void make_box_shadow(const double* bx, const double* center, BoxPairF& q)
{
    for (int d = 0; d < 3; d++) {
        q.l_lo[d] = rec_down(bx[d] - center[d]); q.l_hi[d] = rec_up(bx[3 + d] - center[d]);
        q.r_lo[d] = rec_down(bx[6 + d] - center[d]); q.r_hi[d] = rec_up(bx[9 + d] - center[d]);
    }
}

}  // namespace dgb
