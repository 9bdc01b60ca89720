// K8: refit of a mesh's device records to new vertex positions V' (dg_mesh_refit).  The triangles and the leaf order of the build stay, so
// the implicit tree (node = leaf range [b, e), split m = (b + e) >> 1, bvh_build.h) keeps its topology and every record the kernels read is
// recomputed from V' alone, by data-parallel passes over the T triangles and the tree's levels.
//
// NUMERICAL CONTRACT (fp64, no FMA: the TU is compiled with -fmad=false, the host part with -ffp-contract=off).  n = triangles under a node.
//   Leaf records, fp32 leaf shadows, leaf spheres ((a + b) + c) / 3 with the max of the three norms, the fp32 sphere shadows and the
//       outward rounding of the child boxes: the expressions of bvh_records.h, which bvh_build.cpp uses too, on V'.
//   Centre and half extent: bvh_build.cpp's formula on V' (per coordinate lo = std::min, hi = std::max from +-DBL_MAX, NaN skipped, ties
//       kept by the first vertex; centre 0.5 * (lo + hi); any non-finite vertex or extent: half extent +inf, non-finite centre
//       coordinates 0).  The refit folds runs of K8_BOUNDS_GROUP vertices in order, then runs of partial bounds in order: the same result.
//   Internal sphere of node [b, e): S = S(left) + S(right) componentwise, a leaf's S = (v0 + v1) + v2; centre c = S / (double)(3n);
//       radius sqrt(max over the node's vertices v of dot(c - v, c - v)), the max skipping NaN (std::max(r2, d2) from 0.0).  The max is
//       exact and independent of order.  This is where the refit differs from the build, which sums the node's 3n vertices one after
//       the other in the arrangement the node had before its own sort: replaying that would need one stored permutation per level and a
//       chain of 3T dependent additions at the root.  A refit to the build's own vertices therefore moves internal sphere centres by a
//       few ulp and radii with them.
//   Child boxes: per coordinate the min and max of the vertices under each child; a leaf child's box is make_leaf_box, an internal
//       child's folds its children's boxes with std::min / std::max from +-DBL_MAX (NaN skipped).  For values that are not NaN and
//       not a mix of -0 and +0 this equals the build's box exactly.
//   Pseudonormals: the host builder's expressions and summation orders (vertex sums in (triangle, slot) incidence order; an edge's
//       first term assigned, later ones added, in triangle index order), except the angle acos(|u.v|), which is
//       k8_acos(x) = k5_atan2(sqrt((1.0 - x) * (1.0 + x)), x): 0 at x = 1, NaN for x > 1 or NaN, IEEE operations only, so that the device,
//       the CPU emulation and numpy agree bit for bit (CUDA's acos and glibc's do not).  dg_mesh_create keeps std::acos, so a refit to the
//       build's own vertices gives pseudonormals a few ulp away from the build's.
//   K5 records: k5_winding.cu's contract with V' as the vertices (the sums are already bottom-up there; r_c is the same exact max).
//   Unchanged: the watertight flags, the stack depth, the sign mode and beta.
#include "k8_refit.h"
#include "bvh_records.h"
#include "dg_launch.h"       // DG_KERNEL_LAUNCH: <<<>>> on the device, fibers under tests/emu (DG_EMU)
#include "k5_atan2.h"

#include <cfloat>
#include <cmath>
#include <cstring>
#include <algorithm>

namespace dgb {

DG_HD double k8_acos(double x) { return k5_atan2(sqrt((1.0 - x) * (1.0 + x)), x); }
double k8_acos_host(double x) { return k8_acos(x); }

namespace {

DG_HD double k8_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }      // Vec3r::dot, left to right
DG_HD void k8_unit(const double* a, double* out) { const double l = sqrt(k8_dot(a, a)); out[0] = a[0] / l; out[1] = a[1] / l; out[2] = a[2] / l; }
DG_HD void k8_sub(const double* a, const double* b, double* out) { out[0] = a[0] - b[0]; out[1] = a[1] - b[1]; out[2] = a[2] - b[2]; }

// the leaf-level sums of K5 (build_winding_records' leaf()) and of the sphere tree
struct LeafSums { double S[3], lo[3], hi[3], A, AC[3], CS[3], N[3], p[3], M[9], cnt; };

DG_HD void k8_leaf_sums(const double* v0, const double* v1, const double* v2, LeafSums& s)
{
    for (int d = 0; d < 3; d++) {
        s.S[d] = (v0[d] + v1[d]) + v2[d];
        s.lo[d] = rec_min(rec_min(rec_min(DBL_MAX, v0[d]), v1[d]), v2[d]);
        s.hi[d] = rec_max(rec_max(rec_max(-DBL_MAX, v0[d]), v1[d]), v2[d]);
    }
    const double e0[3] = {v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2]}, e1[3] = {v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2]};
    s.N[0] = 0.5 * (e0[1] * e1[2] - e0[2] * e1[1]);
    s.N[1] = 0.5 * (e0[2] * e1[0] - e0[0] * e1[2]);
    s.N[2] = 0.5 * (e0[0] * e1[1] - e0[1] * e1[0]);
    s.A = sqrt(s.N[0] * s.N[0] + s.N[1] * s.N[1] + s.N[2] * s.N[2]);
    for (int d = 0; d < 3; d++) {
        const double c = (v0[d] + v1[d] + v2[d]) / 3.0;
        s.CS[d] = c; s.p[d] = c; s.AC[d] = s.A * c;
    }
    for (int k = 0; k < 9; k++) s.M[k] = 0.0;
    s.cnt = 1.0;
}

DG_HD void k8_node_to_leafsums(const RefitSums& n, LeafSums& s)
{
    for (int d = 0; d < 3; d++) { s.S[d] = n.S[d]; s.lo[d] = n.lo[d]; s.hi[d] = n.hi[d]; s.AC[d] = n.AC[d]; s.CS[d] = n.CS[d]; s.N[d] = n.N[d]; s.p[d] = n.p[d]; }
    for (int k = 0; k < 9; k++) s.M[k] = n.M[k];
    s.A = n.A; s.cnt = n.cnt;
}

__device__ __forceinline__ const double* k8_vert(const RefitDev& r, uint32_t v) { return r.V + 3 * (size_t)v; }

// ------------------------------------------------------------------------------------------------ pass 1: centre and half extent
__global__ void __launch_bounds__(K8_THREADS)
k8_bounds_vertices_kernel(const double* __restrict__ V, unsigned long long nV, unsigned long long n_out, RefitBounds* __restrict__ out)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * K8_THREADS + threadIdx.x;
    if (idx >= n_out) return;
    RefitBounds b;
    for (int d = 0; d < 3; d++) { b.lo[d] = DBL_MAX; b.hi[d] = -DBL_MAX; }
    bool finite = true;
    const unsigned long long i1 = ((idx + 1) * K8_BOUNDS_GROUP < nV) ? (idx + 1) * K8_BOUNDS_GROUP : nV;
    for (unsigned long long i = idx * K8_BOUNDS_GROUP; i < i1; i++)
        for (int d = 0; d < 3; d++) {
            const double v = V[3 * i + d];
            b.lo[d] = rec_min(b.lo[d], v); b.hi[d] = rec_max(b.hi[d], v);
            finite = finite && isfinite(v);
        }
    b.finite = finite ? 1 : 0; b._pad = 0;
    out[idx] = b;
}

__global__ void __launch_bounds__(K8_THREADS)
k8_bounds_fold_kernel(const RefitBounds* __restrict__ in, unsigned long long n_in, unsigned long long n_out, RefitBounds* __restrict__ out)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * K8_THREADS + threadIdx.x;
    if (idx >= n_out) return;
    RefitBounds b;
    for (int d = 0; d < 3; d++) { b.lo[d] = DBL_MAX; b.hi[d] = -DBL_MAX; }
    int finite = 1;
    const unsigned long long j1 = ((idx + 1) * K8_BOUNDS_GROUP < n_in) ? (idx + 1) * K8_BOUNDS_GROUP : n_in;
    for (unsigned long long j = idx * K8_BOUNDS_GROUP; j < j1; j++) {
        for (int d = 0; d < 3; d++) { b.lo[d] = rec_min(b.lo[d], in[j].lo[d]); b.hi[d] = rec_max(b.hi[d], in[j].hi[d]); }
        finite &= in[j].finite;
    }
    b.finite = finite; b._pad = 0;
    out[idx] = b;
}

// bvh_build.cpp: centre, half extent and the rule for non-finite vertices
__global__ void k8_bounds_final_kernel(const RefitBounds* __restrict__ in, double* __restrict__ bounds)
{
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const RefitBounds b = in[0];
    double c[3], he = 0;
    for (int d = 0; d < 3; d++) { c[d] = 0.5 * (b.lo[d] + b.hi[d]); he = rec_max(he, rec_max(b.hi[d] - c[d], c[d] - b.lo[d])); }
    if (!b.finite || !isfinite(he)) { he = INFINITY; for (int d = 0; d < 3; d++) if (!isfinite(c[d])) c[d] = 0.0; }
    for (int d = 0; d < 3; d++) bounds[d] = c[d];
    bounds[3] = he;
    bounds[4] = b.finite ? 1.0 : 0.0;
}

// ------------------------------------------------------------------------------------------------ pass 2: one thread per leaf position
__global__ void __launch_bounds__(K8_THREADS)
k8_leaf_kernel(RefitDev r)
{
    const int pos = (int)(blockIdx.x * K8_THREADS + threadIdx.x);
    if (pos >= r.n_tri) return;
    const uint32_t* t = r.f_leaf + 3 * (size_t)pos;
    const double* a = k8_vert(r, t[0]); const double* b = k8_vert(r, t[1]); const double* c = k8_vert(r, t[2]);
    const int id = r.order[pos];
    if (r.leaves) {
        LeafRecord L;
        make_leaf_record(a, b, c, id, L);
        r.leaves[pos] = L;
        if (r.leaves_f) { LeafF f; make_leaf_shadow(L, r.bounds, f); r.leaves_f[pos] = f; }
    }
    int lb = 0, le = r.n_tri, parent = -1, side = 0;                 // the leaf's parent: halve [0, T) down to [pos, pos + 1)
    while (le - lb > 1) { const int m = (lb + le) >> 1; parent = m; if (pos < m) { le = m; side = 0; } else { lb = m; side = 1; } }
    if (r.spheres) {
        if (pos == 0) { SpherePair z; memset(&z, 0, sizeof z); r.spheres[0] = z; }       // index 0 is no node's split position
        if (parent >= 0) {
            double ctr[3], rad;
            make_leaf_sphere(a, b, c, ctr, rad);
            SpherePair& sp = r.spheres[parent];
            double* sc = side ? sp.rc : sp.lc;
            sc[0] = ctr[0]; sc[1] = ctr[1]; sc[2] = ctr[2];
            if (side) sp.rr = rad; else sp.lr = rad;
            make_leaf_box(a, b, c, &r.sums[parent].box[6 * side]);
        }
    }
    if (r.pn_tri) {                                                   // bvh_build.cpp, pseudonormals (TriangleMeshDistance.h:394-400)
        double u[3], v[3], w[3], n[3], x[3], y[3];
        k8_sub(b, a, u); k8_sub(c, a, v);
        x[0] = u[1] * v[2] - u[2] * v[1]; x[1] = -u[0] * v[2] + u[2] * v[0]; x[2] = u[0] * v[1] - u[1] * v[0];
        k8_unit(x, n);
        double* pt = r.pn_tri + 3 * (size_t)id;
        pt[0] = n[0]; pt[1] = n[1]; pt[2] = n[2];
        double* an = r.angle + 3 * (size_t)id;
        k8_unit(u, x); k8_unit(v, y); an[0] = k8_acos(fabs(k8_dot(x, y)));
        k8_sub(a, b, w); k8_unit(w, x); k8_sub(c, b, w); k8_unit(w, y); an[1] = k8_acos(fabs(k8_dot(x, y)));
        k8_sub(b, c, w); k8_unit(w, x); k8_sub(a, c, w); k8_unit(w, y); an[2] = k8_acos(fabs(k8_dot(x, y)));
    }
    if (r.wind_leaves) {
        WindLeaf wl;
        for (int d = 0; d < 3; d++) { wl.v[d] = a[d]; wl.v[3 + d] = b[d]; wl.v[6 + d] = c[d]; }
        r.wind_leaves[pos] = wl;
    }
    if (r.wind_clusters) {                                            // leaf children and the root's right slot stay zero
        WindCluster z;
        memset(&z, 0, sizeof z);
        if (parent >= 0) { if (side) r.wind_clusters[parent].r = z; else r.wind_clusters[parent].l = z; }
        if (pos == 0) { r.wind_clusters[0].r = z; if (r.n_tri == 1) r.wind_clusters[0].l = z; }
    }
}

// ------------------------------------------------------------------------------------------------ pass 3: pseudonormals
__global__ void __launch_bounds__(K8_THREADS)
k8_vertex_normal_kernel(RefitDev r)
{
    const unsigned long long v = (unsigned long long)blockIdx.x * K8_THREADS + threadIdx.x;
    if (v >= r.n_vertices) return;
    double acc[3] = {0, 0, 0};
    for (uint32_t k = r.inc_begin[v]; k < r.inc_begin[v + 1]; k++) {
        const uint32_t q = r.inc[k];
        const double al = r.angle[q];
        const double* n = r.pn_tri + 3 * (size_t)(q / 3);
        acc[0] = acc[0] + al * n[0]; acc[1] = acc[1] + al * n[1]; acc[2] = acc[2] + al * n[2];
    }
    k8_unit(acc, r.pn_vert + 3 * v);
}

// one thread per (triangle, slot): the triangles around the edge's lower vertex, in index order
__global__ void __launch_bounds__(K8_THREADS)
k8_edge_normal_kernel(RefitDev r)
{
    const unsigned long long q = (unsigned long long)blockIdx.x * K8_THREADS + threadIdx.x;
    if (q >= 3ull * (unsigned long long)r.n_tri) return;
    const uint32_t* t = r.F + 3 * (q / 3);
    const int s = (int)(q % 3);
    const uint32_t ea = (s == 1) ? t[1] : t[0], eb = (s == 0) ? t[1] : t[2];     // E01, E12, E02
    const uint32_t lo = ea < eb ? ea : eb, hi = ea < eb ? eb : ea;
    double acc[3] = {0, 0, 0};
    int count = 0;
    uint32_t prev_tri = 0xffffffffu;
    for (uint32_t k = r.inc_begin[lo]; k < r.inc_begin[lo + 1]; k++) {
        const uint32_t tri = r.inc[k] / 3;
        if (tri == prev_tri) continue;                                // vertex repeated inside one triangle
        prev_tri = tri;
        const uint32_t* u = r.F + 3 * (size_t)tri;
        const uint32_t ua[3] = {u[0], u[1], u[0]}, ub[3] = {u[1], u[2], u[2]};
        const double* pt = r.pn_tri + 3 * (size_t)tri;
        for (int j = 0; j < 3; j++) {
            const uint32_t l2 = ua[j] < ub[j] ? ua[j] : ub[j], h2 = ua[j] < ub[j] ? ub[j] : ua[j];
            if (l2 == lo && h2 == hi) {
                if (count == 0) { acc[0] = pt[0]; acc[1] = pt[1]; acc[2] = pt[2]; }
                else { acc[0] = acc[0] + pt[0]; acc[1] = acc[1] + pt[1]; acc[2] = acc[2] + pt[2]; }
                count++;
            }
        }
    }
    k8_unit(acc, r.pn_edge + 3 * q);
}

// the 7 x 3 block of each leaf position: V0 V1 V2 E01 E12 E02 F
__global__ void __launch_bounds__(K8_THREADS)
k8_scatter_normals_kernel(RefitDev r)
{
    const int pos = (int)(blockIdx.x * K8_THREADS + threadIdx.x);
    if (pos >= r.n_tri) return;
    const uint32_t* t = r.f_leaf + 3 * (size_t)pos;
    const size_t id = (size_t)r.order[pos];
    const double* src[7] = {r.pn_vert + 3 * (size_t)t[0], r.pn_vert + 3 * (size_t)t[1], r.pn_vert + 3 * (size_t)t[2],
                            r.pn_edge + 9 * id, r.pn_edge + 9 * id + 3, r.pn_edge + 9 * id + 6, r.pn_tri + 3 * id};
    PseudoNormals N;
    for (int k = 0; k < 7; k++) for (int d = 0; d < 3; d++) N.n[k][d] = src[k][d];
    r.normals[pos] = N;
}

// ------------------------------------------------------------------------------------------------ pass 4: bottom-up sums, one level
__device__ __forceinline__ void k8_child(const RefitDev& r, int b, int e, LeafSums& s)
{
    if (e - b == 1) {
        const uint32_t* t = r.f_leaf + 3 * (size_t)b;
        k8_leaf_sums(k8_vert(r, t[0]), k8_vert(r, t[1]), k8_vert(r, t[2]), s);
    } else {
        k8_node_to_leafsums(r.sums[(b + e) >> 1], s);
    }
}

__global__ void __launch_bounds__(K8_THREADS)
k8_sums_kernel(RefitDev r, unsigned first, unsigned count)
{
    const unsigned idx = blockIdx.x * K8_THREADS + threadIdx.x;
    if (idx >= count) return;
    const RefitNodeRef nd = r.nodes[first + idx];
    const int m = (nd.b + nd.e) >> 1;
    LeafSums L, R;
    k8_child(r, nd.b, m, L);
    k8_child(r, m, nd.e, R);
    RefitSums& s = r.sums[m];
    const double cnt3 = (double)(3 * (nd.e - nd.b));
    for (int d = 0; d < 3; d++) {
        s.S[d] = L.S[d] + R.S[d];
        s.c[d] = s.S[d] / cnt3;
        s.lo[d] = rec_min(L.lo[d], R.lo[d]);
        s.hi[d] = rec_max(L.hi[d], R.hi[d]);
    }
    if (m - nd.b > 1) for (int d = 0; d < 3; d++) { s.box[d] = L.lo[d]; s.box[3 + d] = L.hi[d]; }        // leaf children: k8_leaf_kernel
    if (nd.e - m > 1) for (int d = 0; d < 3; d++) { s.box[6 + d] = R.lo[d]; s.box[9 + d] = R.hi[d]; }
    // K5 (build_winding_records)
    s.A = L.A + R.A; s.cnt = L.cnt + R.cnt;
    for (int d = 0; d < 3; d++) { s.AC[d] = L.AC[d] + R.AC[d]; s.CS[d] = L.CS[d] + R.CS[d]; s.N[d] = L.N[d] + R.N[d]; }
    for (int d = 0; d < 3; d++) s.p[d] = (s.A > 0.0) ? s.AC[d] / s.A : s.CS[d] / s.cnt;
    for (int j = 0; j < 3; j++)
        for (int k = 0; k < 3; k++)
            s.M[3 * j + k] = (L.M[3 * j + k] + (L.p[j] - s.p[j]) * L.N[k]) + (R.M[3 * j + k] + (R.p[j] - s.p[j]) * R.N[k]);
    s.r2s = 0ull; s.r2k = 0ull;                                       // +0.0: the radius pass only raises them
}

// ------------------------------------------------------------------------------------------------ pass 5: radii
// max of non-negative fp64 bit patterns over the warp, as two 32-bit reductions (high word, then the low word of the lanes that hold it)
__device__ __forceinline__ unsigned long long k8_warp_max_u64(unsigned long long v)
{
    const unsigned hi = __reduce_max_sync(0xffffffffu, (unsigned)(v >> 32));
    const unsigned lo = __reduce_max_sync(0xffffffffu, ((unsigned)(v >> 32) == hi) ? (unsigned)v : 0u);
    return ((unsigned long long)hi << 32) | lo;
}

// one thread per leaf position (every lane of every warp runs the same number of steps): the leaf's three vertices raise the two r^2 maxima
// of each of its ancestors.  Where the whole warp sits under one ancestor (every level near the root) the warp reduces first, so that one
// atomic per warp and level reaches that node.
__global__ void __launch_bounds__(K8_THREADS)
k8_radius_kernel(RefitDev r)
{
    const int pos = (int)(blockIdx.x * K8_THREADS + threadIdx.x);
    const bool live = pos < r.n_tri;
    double v[3][3];
    if (live) {
        const uint32_t* t = r.f_leaf + 3 * (size_t)pos;
        for (int k = 0; k < 3; k++) { const double* p = k8_vert(r, t[k]); v[k][0] = p[0]; v[k][1] = p[1]; v[k][2] = p[2]; }
    }
    int lb = 0, le = r.n_tri;
    for (int lev = 0; lev < r.levels - 1; lev++) {
        const bool act = live && le - lb > 1;
        const int m = act ? (lb + le) >> 1 : 0;
        unsigned long long ks = 0ull, kk = 0ull;
        if (act) {
            const RefitSums& s = r.sums[m];
            double r2 = 0.0, q2 = 0.0;
            for (int k = 0; k < 3; k++) {
                const double d[3] = {s.c[0] - v[k][0], s.c[1] - v[k][1], s.c[2] - v[k][2]};
                r2 = rec_max(r2, k8_dot(d, d));                      // bvh_build.cpp: ctr - v
                const double dx = v[k][0] - s.p[0], dy = v[k][1] - s.p[1], dz = v[k][2] - s.p[2];
                q2 = rec_max(q2, dx * dx + dy * dy + dz * dz);       // k5_winding.cu: v - p~
            }
            ks = (unsigned long long)__double_as_longlong(r2);
            kk = (unsigned long long)__double_as_longlong(q2);
        }
        const unsigned key = act ? (unsigned)m : 0xffffffffu;
        const unsigned kmax = __reduce_max_sync(0xffffffffu, key);
        if (__ballot_sync(0xffffffffu, key == kmax) == 0xffffffffu) {
            if (key != 0xffffffffu) {
                ks = k8_warp_max_u64(ks);
                kk = k8_warp_max_u64(kk);
                if ((threadIdx.x & 31u) == 0u) { atomicMax(&r.sums[m].r2s, ks); atomicMax(&r.sums[m].r2k, kk); }
            }
        } else if (act) {
            atomicMax(&r.sums[m].r2s, ks); atomicMax(&r.sums[m].r2k, kk);
        }
        if (act) { if (pos < m) le = m; else lb = m; }
    }
}

// ------------------------------------------------------------------------------------------------ pass 6: internal spheres and clusters
__global__ void __launch_bounds__(K8_THREADS)
k8_finalize_kernel(RefitDev r, unsigned count)
{
    const unsigned idx = blockIdx.x * K8_THREADS + threadIdx.x;
    if (idx >= count) return;
    const RefitNodeRef nd = r.nodes[idx];
    const RefitSums& s = r.sums[(nd.b + nd.e) >> 1];
    if (r.spheres && nd.parent >= 0) {                                // the root's sphere is unused, as in the reference
        SpherePair& sp = r.spheres[nd.parent];
        double* sc = nd.side ? sp.rc : sp.lc;
        sc[0] = s.c[0]; sc[1] = s.c[1]; sc[2] = s.c[2];
        const double rad = sqrt(__longlong_as_double((long long)s.r2s));
        if (nd.side) sp.rr = rad; else sp.lr = rad;
    }
    if (r.wind_clusters) {
        WindCluster& w = nd.parent < 0 ? r.wind_clusters[0].l : (nd.side ? r.wind_clusters[nd.parent].r : r.wind_clusters[nd.parent].l);
        for (int d = 0; d < 3; d++) { w.p[d] = s.p[d]; w.n[d] = s.N[d]; }
        for (int k = 0; k < 9; k++) w.M[k] = s.M[k];
        w.r = sqrt(__longlong_as_double((long long)s.r2k));
    }
}

// ------------------------------------------------------------------------------------------------ pass 7: fp32 node records
__global__ void __launch_bounds__(K8_THREADS)
k8_pack_kernel(RefitDev r)
{
    const int m = (int)(blockIdx.x * K8_THREADS + threadIdx.x);
    if (m >= r.n_tri) return;
    float rec[4 * K8_MAX_NODEF_STRIDE];
    for (int k = 0; k < 4 * r.nodef_stride; k++) rec[k] = 0.f;
    SpherePairF f;
    make_sphere_shadow(r.spheres[m], r.bounds, f);
    memcpy(rec, &f, sizeof f);
    if (m != 0) { BoxPairF q; make_box_shadow(r.sums[m].box, r.bounds, q); memcpy(rec + 8, &q, sizeof q); }
    float4* out = r.nodes_f + (size_t)m * r.nodef_stride;
    for (int k = 0; k < r.nodef_stride; k++) out[k] = make_float4(rec[4 * k], rec[4 * k + 1], rec[4 * k + 2], rec[4 * k + 3]);
}

unsigned k8_blocks(uint64_t n) { return (unsigned)((n + K8_THREADS - 1) / K8_THREADS); }

}  // namespace

// ------------------------------------------------------------------------------------------------ host
uint64_t k8_bounds_entries(uint64_t nV)
{
    const uint64_t n1 = (nV + K8_BOUNDS_GROUP - 1) / K8_BOUNDS_GROUP, n2 = (n1 + K8_BOUNDS_GROUP - 1) / K8_BOUNDS_GROUP;
    return n1 + std::max<uint64_t>(n2, 1);
}

void k8_build_topology(const HostBvh& h, RefitTopoHost& out)
{
    const uint64_t nT = h.n_triangles, nV = h.n_vertices;
    out.f_leaf.resize(3 * nT);
    for (uint64_t p = 0; p < nT; p++)
        for (int k = 0; k < 3; k++) out.f_leaf[3 * p + k] = h.F[3 * (size_t)h.order[p] + k];
    out.inc_begin.assign(nV + 1, 0);
    out.inc.resize(3 * nT);
    for (uint64_t i = 0; i < 3 * nT; i++) out.inc_begin[h.F[i] + 1]++;
    for (uint64_t v = 0; v < nV; v++) out.inc_begin[v + 1] += out.inc_begin[v];
    std::vector<uint32_t> cursor(out.inc_begin.begin(), out.inc_begin.end() - 1);
    for (uint64_t i = 0; i < 3 * nT; i++) out.inc[cursor[h.F[i]]++] = (uint32_t)i;
    // internal nodes breadth first: the root, then depth 1, ...
    out.nodes.clear(); out.level_begin.assign(1, 0);
    if (nT > 1) out.nodes.push_back({0, (int32_t)nT, -1, 0});
    for (size_t lev0 = 0; lev0 < out.nodes.size();) {
        const size_t lev1 = out.nodes.size();
        out.level_begin.push_back((uint32_t)lev1);
        for (size_t i = lev0; i < lev1; i++) {
            const RefitNodeRef nd = out.nodes[i];
            const int m = (nd.b + nd.e) >> 1;
            if (m - nd.b > 1) out.nodes.push_back({nd.b, m, m, 0});
            if (nd.e - m > 1) out.nodes.push_back({m, nd.e, m, 1});
        }
        lev0 = lev1;
    }
    if (out.level_begin.back() != out.nodes.size()) out.level_begin.push_back((uint32_t)out.nodes.size());
}

cudaError_t k8_launch_refit(const RefitDev& r0, const std::vector<uint32_t>& level_begin, bool k1, cudaStream_t stream)
{
    RefitDev r = r0;
    if (r.nodef_stride < 5 || r.nodef_stride > K8_MAX_NODEF_STRIDE) return cudaErrorInvalidValue;     // k8_pack_kernel's staging array
    if (!k1) { r.spheres = nullptr; r.leaves = nullptr; r.leaves_f = nullptr; r.normals = nullptr; r.nodes_f = nullptr; r.pn_tri = nullptr; }
    const uint64_t T = (uint64_t)r.n_tri, nV = r.n_vertices;
    cudaError_t e;
#define K8_LAUNCH(kernel, n, ...)                                                            \
    do {                                                                                     \
        DG_KERNEL_LAUNCH(kernel, k8_blocks(n), K8_THREADS, 0, stream, __VA_ARGS__);          \
        if ((e = DG_AFTER_LAUNCH()) != cudaSuccess) return e;                                \
    } while (0)
    if (k1) {
        uint64_t n = (nV + K8_BOUNDS_GROUP - 1) / K8_BOUNDS_GROUP;
        const uint64_t n1 = n;
        RefitBounds* cur = r.part;
        K8_LAUNCH(k8_bounds_vertices_kernel, n, r.V, (unsigned long long)nV, (unsigned long long)n, cur);
        bool in_first = true;
        while (n > 1) {
            const uint64_t nn = (n + K8_BOUNDS_GROUP - 1) / K8_BOUNDS_GROUP;
            RefitBounds* nxt = in_first ? r.part + n1 : r.part;
            K8_LAUNCH(k8_bounds_fold_kernel, nn, cur, (unsigned long long)n, (unsigned long long)nn, nxt);
            cur = nxt; n = nn; in_first = !in_first;
        }
        K8_LAUNCH(k8_bounds_final_kernel, 1, cur, r.bounds);
    }
    K8_LAUNCH(k8_leaf_kernel, T, r);
    if (k1) {
        K8_LAUNCH(k8_vertex_normal_kernel, nV, r);
        K8_LAUNCH(k8_edge_normal_kernel, 3 * T, r);
        K8_LAUNCH(k8_scatter_normals_kernel, T, r);
    }
    const int n_levels = (int)level_begin.size() - 1;
    if (n_levels > 0 && level_begin.back() > 0) {
        for (int d = n_levels - 1; d >= 0; d--) {
            const unsigned first = level_begin[d], count = level_begin[d + 1] - level_begin[d];
            if (count) K8_LAUNCH(k8_sums_kernel, count, r, first, count);
        }
        K8_LAUNCH(k8_radius_kernel, T, r);
        K8_LAUNCH(k8_finalize_kernel, level_begin.back(), r, (unsigned)level_begin.back());
    }
    if (k1) K8_LAUNCH(k8_pack_kernel, T, r);
#undef K8_LAUNCH
    return cudaSuccess;
}

}  // namespace dgb
