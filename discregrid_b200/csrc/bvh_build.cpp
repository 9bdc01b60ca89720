// See bvh_build.h.  Compiled with -ffp-contract=off: every expression below must round exactly like the
// reference's x86-64 build (no FMA), because these values feed bit-exact device comparisons.
#include "bvh_build.h"
#include "bvh_records.h"
#include "sort_replay.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <atomic>
#include <future>
#include <thread>
#include <unordered_map>

namespace dgb {
namespace {

struct P3 { double x, y, z; };
inline P3 operator-(P3 a, P3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline P3 operator+(P3 a, P3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline double dot3(P3 a, P3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }          // Vec3r::dot, left to right
inline double len(P3 a) { return std::sqrt(dot3(a, a)); }
inline P3 unit(P3 a) { const double l = len(a); return {a.x / l, a.y / l, a.z / l}; }  // Vec3r::normalized
inline P3 crs(P3 a, P3 b) { return {a.y * b.z - a.z * b.y, -a.x * b.z + a.z * b.x, a.x * b.y - a.y * b.x}; }
inline double at(const P3& p, int d) { return d == 0 ? p.x : (d == 1 ? p.y : p.z); }

struct Builder {
    const P3* V;
    const uint32_t* F;
    HostBvh& out;
    std::vector<int32_t>& order;           // current arrangement of triangle ids (the reference sorts structs in place)
    struct Key { double k; int32_t id; };
    std::vector<Key> keys;                 // scratch for the sort (same comparisons => same permutation as the reference)
    std::atomic<int> max_depth{0};
    int par_levels = 0;                    // subtrees of the first `par_levels` levels are built by separate threads
    unsigned hw_threads = 1;               // host threads the whole build may use
    bool replay_ok = false;                // sort_replay_matches_std_sort()

    inline P3 vert(int32_t tri, int k) const { return V[F[3 * (size_t)tri + k]]; }

    // bounding sphere of the node covering [b, e) in the CURRENT arrangement (TriangleMeshDistance.h:451-491)
    // also returns the axis-aligned box of the node's vertices in box[6] = {lo, hi}
    void build(int b, int e, double sc[3], double& sr, double box[6], int depth)
    {
        { int cur = max_depth.load(std::memory_order_relaxed); while (depth > cur && !max_depth.compare_exchange_weak(cur, depth)) {} }
        const int n = e - b;
        if (n == 1) {                                        // bvh_records.h, shared with the device refit
            const P3 a = vert(order[b], 0), bb = vert(order[b], 1), c = vert(order[b], 2);
            make_leaf_sphere(&a.x, &bb.x, &c.x, sc, sr);
            make_leaf_box(&a.x, &bb.x, &c.x, box);
            return;
        }
        double top[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX}, bot[3] = {DBL_MAX, DBL_MAX, DBL_MAX};
        P3 ctr = {0, 0, 0};
        for (int i = b; i < e; i++)
            for (int k = 0; k < 3; k++) {
                const P3 p = vert(order[i], k);
                ctr = ctr + p;                               // sequential, arrangement order matters for rounding
                top[0] = std::max(top[0], p.x); top[1] = std::max(top[1], p.y); top[2] = std::max(top[2], p.z);
                bot[0] = std::min(bot[0], p.x); bot[1] = std::min(bot[1], p.y); bot[2] = std::min(bot[2], p.z);
            }
        const double cnt = (double)(3 * n);
        ctr = {ctr.x / cnt, ctr.y / cnt, ctr.z / cnt};
        for (int d = 0; d < 3; d++) { box[d] = bot[d]; box[3 + d] = top[d]; }
        const double diag[3] = {top[0] - bot[0], top[1] - bot[1], top[2] - bot[2]};
        int split = 0;                                       // std::max_element: first maximum
        if (diag[1] > diag[split]) split = 1;
        if (diag[2] > diag[split]) split = 2;
        double r2 = 0.0;
        for (int i = b; i < e; i++)
            for (int k = 0; k < 3; k++) { const P3 d = ctr - vert(order[i], k); r2 = std::max(r2, dot3(d, d)); }
        sc[0] = ctr.x; sc[1] = ctr.y; sc[2] = ctr.z; sr = std::sqrt(r2);

        // unstable std::sort on the first vertex's coordinate (TriangleMeshDistance.h:494-499)
        for (int i = b; i < e; i++) keys[i] = {at(vert(order[i], 0), split), order[i]};
        {
            auto by_key = [](const Key& x, const Key& y) { return x.k < y.k; };
            // near the root one sort is most of the critical path: same comparisons and swaps as std::sort, on the threads this
            // subtree may use (sort_replay.h); the arrangement -- ties included -- is the one std::sort leaves
            const unsigned share = hw_threads >> (depth - 1 < 16 ? depth - 1 : 16);
            if (n >= 32768 && share >= 2 && replay_ok) replay_sort(keys.data() + b, (uint64_t)n, by_key, share);
            else std::sort(keys.begin() + b, keys.begin() + e, by_key);
        }
        for (int i = b; i < e; i++) order[i] = keys[i].id;

        const int m = (b + e) >> 1;
        SpherePair& sp = out.spheres[m];
        double* bx = &out.boxes[12 * (size_t)m];
        // the two subtrees touch disjoint ranges of `order`/`keys` and disjoint records: build them concurrently near the root.
        // Every node is still processed by exactly the reference's sequence of operations, so the tree is unchanged.
        if (depth <= par_levels && n >= 4096) {
            auto left = std::async(std::launch::async, [&, b, m, depth, bx]() { build(b, m, sp.lc, sp.lr, bx, depth + 1); });
            build(m, e, sp.rc, sp.rr, bx + 6, depth + 1);
            left.get();
        } else {
            build(b, m, sp.lc, sp.lr, bx, depth + 1);
            build(m, e, sp.rc, sp.rr, bx + 6, depth + 1);
        }
    }
};

}  // namespace

bool build_host_bvh(const double* Vd, uint64_t nV, const uint32_t* F, uint64_t nT, HostBvh& out, const char** err, bool with_leaf_shadow)
{
    if (!Vd || !F || nT == 0 || nV == 0) { *err = "empty triangle list or vertex list"; return false; }
    if (nT >= (1ull << 25) || nV > (uint64_t)0x7fffffff) { *err = "mesh too large (< 2^25 triangles; int32 vertex indices as in the reference)"; return false; }
    for (uint64_t i = 0; i < 3 * nT; i++) if (F[i] >= nV) { *err = "triangle index out of range"; return false; }
    const P3* V = reinterpret_cast<const P3*>(Vd);
    const int T = (int)nT;
    out = HostBvh();
    out.n_vertices = nV; out.n_triangles = nT;
    out.V.assign(Vd, Vd + 3 * nV);
    out.F.assign(F, F + 3 * nT);
    out.spheres.resize(nT);
    std::memset(&out.spheres[0], 0, sizeof(SpherePair));               // index 0 is no node's split position
    out.order.resize(nT);
    for (int i = 0; i < T; i++) out.order[i] = i;

    Builder bld{V, F, out, out.order};
    bld.keys.resize(nT);
    { unsigned hw = host_threads(); if (hw == 0) hw = 1; if (hw > 64) hw = 64;
      int lv = 0; while ((1u << (lv + 1)) <= hw && lv < 6) lv++; bld.par_levels = lv; bld.hw_threads = hw;
      bld.replay_ok = nT >= 32768 && sort_replay_matches_std_sort(); }
    double root_c[3], root_r, root_box[6];
    out.boxes.resize(12 * nT);
    std::memset(out.boxes.data(), 0, 12 * sizeof(double));
    bld.build(0, T, root_c, root_r, root_box, 1);
    out.max_depth = bld.max_depth.load();      // root sphere is computed and unused, as in the reference (:125,357)

    // ---- pseudonormals (TriangleMeshDistance.h:359-420), in the reference's arrays first.
    // The reference accumulates into per-vertex / per-edge sums while looping over the triangles in index order (an
    // unordered_map keyed by the vertex pair for the edges).  The same sums, term by term in the same order, are produced
    // here from a vertex -> (triangle, slot) incidence list, which makes every stage a parallel loop.
    out.pn_tri.resize(3 * nT); out.pn_edge.resize(9 * nT); out.pn_vert.resize(3 * nV);          // every entry is written below
    P3* pt = reinterpret_cast<P3*>(out.pn_tri.data());
    P3* pe = reinterpret_cast<P3*>(out.pn_edge.data());
    P3* pv = reinterpret_cast<P3*>(out.pn_vert.data());
    std::vector<double> angle(3 * nT);
    parallel_for(nT, [&](uint64_t i0, uint64_t i1) {
        for (uint64_t i = i0; i < i1; i++) {
            const uint32_t* t = F + 3 * i;
            const P3 a = V[t[0]], b = V[t[1]], c = V[t[2]];
            pt[i] = unit(crs(b - a, c - a));                                                  // :394
            angle[3 * i + 0] = std::acos(std::abs(dot3(unit(b - a), unit(c - a))));          // :398-400
            angle[3 * i + 1] = std::acos(std::abs(dot3(unit(a - b), unit(c - b))));
            angle[3 * i + 2] = std::acos(std::abs(dot3(unit(b - c), unit(a - c))));
        }
    });
    // incidence list in (triangle, slot) order
    std::vector<uint32_t> inc_begin(nV + 1, 0), inc(3 * nT);
    for (uint64_t i = 0; i < 3 * nT; i++) inc_begin[F[i] + 1]++;
    for (uint64_t v = 0; v < nV; v++) inc_begin[v + 1] += inc_begin[v];
    {
        std::vector<uint32_t> cursor(inc_begin.begin(), inc_begin.end() - 1);
        for (uint64_t i = 0; i < 3 * nT; i++) inc[cursor[F[i]]++] = (uint32_t)i;              // entry = 3*triangle + slot
    }
    parallel_for(nV, [&](uint64_t v0, uint64_t v1) {
        for (uint64_t v = v0; v < v1; v++) {
            P3 acc = {0, 0, 0};                                                               // :385
            for (uint32_t k = inc_begin[v]; k < inc_begin[v + 1]; k++) {
                const double al = angle[inc[k]];
                const P3 n = pt[inc[k] / 3];
                acc = acc + P3{al * n.x, al * n.y, al * n.z};                                 // :401-403
            }
            pv[v] = unit(acc);                                                                // :411-413 (same divisions)
        }
    });
    std::atomic<int> flags{0};
    parallel_for(nT, [&](uint64_t i0, uint64_t i1) {
        int local = 0;
        for (uint64_t i = i0; i < i1; i++) {
            const uint32_t* t = F + 3 * i;
            const uint32_t ea[3] = {t[0], t[1], t[0]}, eb[3] = {t[1], t[2], t[2]};           // E01, E12, E02 (:406-408, :417-419)
            for (int s = 0; s < 3; s++) {
                const uint32_t lo = std::min(ea[s], eb[s]), hi = std::max(ea[s], eb[s]);
                P3 acc = {0, 0, 0};
                int count = 0;
                uint32_t prev_tri = 0xffffffffu;
                for (uint32_t k = inc_begin[lo]; k < inc_begin[lo + 1]; k++) {               // triangles touching `lo`, in index order
                    const uint32_t tri = inc[k] / 3;
                    if (tri == prev_tri) continue;                                            // vertex repeated inside one triangle
                    prev_tri = tri;
                    const uint32_t* u = F + 3 * (size_t)tri;
                    const uint32_t ua[3] = {u[0], u[1], u[0]}, ub[3] = {u[1], u[2], u[2]};
                    for (int q = 0; q < 3; q++)
                        if (std::min(ua[q], ub[q]) == lo && std::max(ua[q], ub[q]) == hi) {
                            acc = (count == 0) ? pt[tri] : acc + pt[tri];                     // first: assignment (:368), then += (:372)
                            count++;
                        }
                }
                pe[3 * i + s] = unit(acc);
                if (count == 1) local |= 1; else if (count > 2) local |= 2;                   // :422-438
            }
        }
        flags.fetch_or(local);
    });
    out.flags = flags.load();

    // ---- device records in leaf order
    out.leaves.resize(nT);
    out.normals.resize(nT);
    parallel_for(nT, [&](uint64_t p0, uint64_t p1) {
        for (uint64_t pos = p0; pos < p1; pos++) {
            const int id = out.order[pos];
            const uint32_t* t = F + 3 * (size_t)id;
            const P3 v0 = V[t[0]], v1 = V[t[1]], v2 = V[t[2]];
            make_leaf_record(&v0.x, &v1.x, &v2.x, id, out.leaves[pos]);      // TriangleMeshDistance.h:567-575 (bvh_records.h)
            PseudoNormals& N = out.normals[pos];
            const P3 src[7] = {pv[t[0]], pv[t[1]], pv[t[2]], pe[3 * id + 0], pe[3 * id + 1], pe[3 * id + 2], pt[id]};
            for (int k = 0; k < 7; k++) { N.n[k][0] = src[k].x; N.n[k][1] = src[k].y; N.n[k][2] = src[k].z; }
        }
    });

    // ---- fp32 shadow of the sphere pairs (filter only), relative to the bounding-box centre
    {
        double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
        for (uint64_t i = 0; i < nV; i++) for (int d = 0; d < 3; d++) { lo[d] = std::min(lo[d], Vd[3 * i + d]); hi[d] = std::max(hi[d], Vd[3 * i + d]); }
        out.half_extent = 0;
        for (int d = 0; d < 3; d++) { out.center[d] = 0.5 * (lo[d] + hi[d]); out.half_extent = std::max(out.half_extent, std::max(hi[d] - out.center[d], out.center[d] - lo[d])); }
        // a NaN coordinate slips through min / max: with any non-finite vertex the fp32 shadows mean nothing.  half_extent = +inf switches every
        // fp32 filter of K1 off (E = inf: all decisions in fp64, exactly the reference's, NaN comparisons included) and sends the packet walk's
        // lanes to the per-lane walk.
        bool finite = true;
        for (uint64_t i = 0; i < 3 * nV && finite; i++) finite = std::isfinite(Vd[i]);
        if (!finite || !std::isfinite(out.half_extent)) { out.half_extent = INFINITY; for (int d = 0; d < 3; d++) if (!std::isfinite(out.center[d])) out.center[d] = 0.0; }
        out.spheres_f.resize(nT);
        out.boxes_f.resize(nT);
        // child boxes are rounded outward so that the fp32 box contains the fp64 one
        parallel_for(nT, [&](uint64_t m0, uint64_t m1) {
            for (uint64_t m = m0; m < m1; m++) {
                make_sphere_shadow(out.spheres[m], out.center, out.spheres_f[m]);
                BoxPairF& q = out.boxes_f[m];
                if (m == 0) { std::memset(&q, 0, sizeof q); continue; }
                make_box_shadow(&out.boxes[12 * m], out.center, q);
            }
        });
        RawVec<double>().swap(out.boxes);
        // fp32 triangle shadows in leaf order (all products formed in fp64, then rounded once)
        if (with_leaf_shadow) out.leaves_f.resize(nT);
        if (with_leaf_shadow) parallel_for(nT, [&](uint64_t p0, uint64_t p1) {
            for (uint64_t pos = p0; pos < p1; pos++) make_leaf_shadow(out.leaves[pos], out.center, out.leaves_f[pos]);
        });
    }

    return true;
}

void pack_node_records(const HostBvh& h, int stride, float* out)
{
    const uint64_t nT = h.n_triangles;
    parallel_for(nT, [&](uint64_t m0, uint64_t m1) {
        for (uint64_t m = m0; m < m1; m++) {
            float* rec = out + m * (uint64_t)stride * 4;
            std::memset(rec, 0, (size_t)stride * 16);
            std::memcpy(rec, &h.spheres_f[m], sizeof(SpherePairF));
            std::memcpy(rec + 8, &h.boxes_f[m], sizeof(BoxPairF));
        }
    });
}

namespace {
int export_rec(const HostBvh& bvh, int b, int e, int& next, double* spheres, int32_t* kids)
{
    const int id = next++;
    if (e - b == 1) {
        if (kids) { kids[2 * id] = -1; kids[2 * id + 1] = bvh.order[b]; }
        if (spheres) std::memset(spheres + 8 * (size_t)id, 0, 8 * sizeof(double));   // reference leaves hold default spheres
        return id;
    }
    const int m = (b + e) >> 1;
    if (spheres) std::memcpy(spheres + 8 * (size_t)id, &bvh.spheres[m], 8 * sizeof(double));
    const int l = export_rec(bvh, b, m, next, spheres, kids);
    const int r = export_rec(bvh, m, e, next, spheres, kids);
    if (kids) { kids[2 * id] = l; kids[2 * id + 1] = r; }
    return id;
}
}  // namespace

void export_reference_tree(const HostBvh& bvh, double* spheres, int32_t* kids)
{
    int next = 0;
    export_rec(bvh, 0, (int)bvh.n_triangles, next, spheres, kids);
}

}  // namespace dgb
