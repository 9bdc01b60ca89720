// Host-side construction of the mesh-distance acceleration data, laid out for the sm_90a traversal kernel.
//
// What is built is *numerically* the reference's structure (TriangleMeshDistance.h:336-512: median-split
// bounding-sphere tree ordered by std::sort on the first vertex, angle-weighted pseudonormals) because the
// query result -- including which of several equidistant triangles wins and therefore the sign -- depends
// on the traversal order (TriangleMeshDistance.h:528, 542-560).  The *layout* is new:
//
//   * no node array and no child pointers.  After construction the triangles sit in "leaf order"
//     (position 0..T-1).  A tree node is the half-open range [b, e) of leaf positions it covers; its
//     children are [b, m) and [m, e) with m = (b + e) >> 1 (== (int)(0.5*(b+e)), TriangleMeshDistance.h:502).
//     Every internal node has a distinct m in [1, T-1], so the pair of child spheres is stored at
//     spheres[m] -- one 64-byte, 64-byte-aligned record = two 32-byte sectors.
//   * one 128-byte record per triangle (leaf order) with every point-independent quantity of
//     point_triangle_sq_unsigned precomputed with the reference's exact operation order:
//     v0, e0 = v1-v0, e1 = v2-v0, a00, a01, a11, det = |a00*a11 - a01*a01|, 1/det, a00 - 2*a01 + a11, id.
//   * one 7x3 block of pseudonormals per triangle (leaf order), indexed directly by NearestEntity
//     (V0,V1,V2,E01,E12,E02,F), so the sign needs a single 24-byte gather.
#pragma once
#include <cstdint>
#include <algorithm>
#include <memory>
#include <thread>
#include <type_traits>
#include <utility>
#include <vector>

namespace dgb {

// std::vector whose resize() leaves trivially-constructible elements uninitialised: the big record arrays are written exactly once,
// by parallel loops, and zero-filling them first (serially, touching every page) cost as much as filling them
template <class T>
struct DefaultInitAllocator : std::allocator<T> {
    template <class U> struct rebind { using other = DefaultInitAllocator<U>; };
    using std::allocator<T>::allocator;
    template <class U> void construct(U* p) noexcept(std::is_nothrow_default_constructible<U>::value) { ::new (static_cast<void*>(p)) U; }
    template <class U, class... A> void construct(U* p, A&&... a) { ::new (static_cast<void*>(p)) U(std::forward<A>(a)...); }
};
template <class T> using RawVec = std::vector<T, DefaultInitAllocator<T>>;

// Host threads this process can really run: the scheduler affinity mask, capped by the cgroup CPU quota (a container that sees 128
// logical CPUs but is throttled to a 16-CPU quota runs 128 busy threads SLOWER than 16).  host_threads.cpp.
unsigned host_threads();

// static partition of [0, n) over the usable host threads; fn(begin, end)
template <class Fn>
void parallel_for(uint64_t n, Fn fn)
{
    unsigned nt = host_threads();
    if (nt == 0) nt = 1;
    if (nt > 32) nt = 32;
    if (n < 4096 || nt == 1) { fn(0, n); return; }
    std::vector<std::thread> th;
    const uint64_t per = (n + nt - 1) / nt;
    for (unsigned k = 0; k < nt; k++) {
        const uint64_t b = k * per, e = std::min(n, b + per);
        if (b >= e) break;
        th.emplace_back([=, &fn]() { fn(b, e); });
    }
    for (auto& t : th) t.join();
}


struct alignas(64) SpherePair {   // children of the internal node whose split position is the array index
    double lc[3], lr;             // left child sphere  (TriangleMeshDistance.h:105)
    double rc[3], rr;             // right child sphere (TriangleMeshDistance.h:106)
};
static_assert(sizeof(SpherePair) == 64, "SpherePair must be 64 bytes");

// fp32 shadow of SpherePair, relative to HostBvh::center: used only to FILTER traversal decisions (k1_sdf.cu); every decision
// the fp32 interval cannot certify is re-taken from the fp64 record, so results do not depend on these values.
struct alignas(32) SpherePairF {
    float lc[3], lr;
    float rc[3], rr;
};
static_assert(sizeof(SpherePairF) == 32, "SpherePairF must be 32 bytes");

// fp32 axis-aligned boxes (relative to HostBvh::center, rounded OUTWARD) of the two children of an internal node: a second,
// tighter lower bound used only to SKIP subtrees that provably cannot change the result (k1_sdf.cu, "hopeless" test).
struct alignas(16) BoxPairF {
    float l_lo[3], l_hi[3];
    float r_lo[3], r_hi[3];
};
static_assert(sizeof(BoxPairF) == 48, "BoxPairF must be 48 bytes");

struct alignas(128) LeafRecord {
    double v0[3];
    double e0[3];
    double e1[3];
    double a00, a01, a11;
    double det, inv_det, denom;   // |a00*a11-a01*a01|, 1/det, (a00 - 2*a01) + a11
    int32_t tri_id;               // original triangle index (Result::triangle_id)
    int32_t _pad;
};
static_assert(sizeof(LeafRecord) == 128, "LeafRecord must be 128 bytes");

// fp32 shadow of a triangle (relative to HostBvh::center), used only to REJECT leaf tests that provably cannot be accepted
// (k1_sdf.cu, leaf_lower_bound): v0, e0, e1, |e0|^2, e0.e1, |e1|^2, |e1-e0|^2, n = unit normal (e0 x e1) / |e0 x e1| (0 for zero area).
// Never contributes a value to the result.
struct alignas(64) LeafF {
    float v0[3], e0[3], e1[3];
    float d00, d01, d11, d22;
    float n[3];
};
static_assert(sizeof(LeafF) == 64, "LeafF must be 64 bytes");

struct PseudoNormals { double n[7][3]; };   // V0 V1 V2 E01 E12 E02 F
static_assert(sizeof(PseudoNormals) == 168, "PseudoNormals must be 168 bytes");

struct HostBvh {
    uint64_t n_vertices = 0, n_triangles = 0;
    RawVec<SpherePair> spheres;             // [T]  (index 0 unused, zeroed)
    RawVec<SpherePairF> spheres_f;          // [T]  fp32 shadow, relative to `center`
    RawVec<BoxPairF> boxes_f;               // [T]  fp32 child boxes, relative to `center`, rounded outward
    RawVec<double> boxes;                   // [T][12] fp64 child boxes (build scratch)
    double center[3] = {0, 0, 0};           // bounding-box centre of the vertices
    double half_extent = 0;                 // max |v - center|_inf over the vertices
    RawVec<LeafRecord> leaves;              // [T]
    RawVec<LeafF> leaves_f;                 // [T]  fp32 shadow, relative to `center`
    RawVec<PseudoNormals> normals;          // [T]
    std::vector<int32_t> order;             // leaf position -> triangle id
    int max_depth = 0;                      // number of levels (root = 1)
    int flags = 0;                          // bit0: edge with a single triangle; bit1: edge with > 2 triangles
    // reference-numbered copies for dg_mesh_tree / dg_mesh_pseudonormals (diagnostics, built on demand)
    std::vector<double> V;                  // nV x 3
    std::vector<uint32_t> F;                // nT x 3
    RawVec<double> pn_tri, pn_edge, pn_vert;
};

// The fp32 record of every internal node as the traversal kernels read it (index = split position m, `stride` float4s each):
// [sphere pair, 32 B][box pair, 48 B] (+ padding).
void pack_node_records(const HostBvh& h, int stride, float* out /* n_triangles * stride * 4 floats */);

// Returns false (and leaves *err) on invalid input.
bool build_host_bvh(const double* V, uint64_t nV, const uint32_t* F, uint64_t nT, HostBvh& out, const char** err,
                    bool with_leaf_shadow = false);

// Re-expresses the implicit tree in the reference's explicit pre-order numbering (diagnostics only).
void export_reference_tree(const HostBvh& bvh, double* spheres /*(2T-1) x 8*/, int32_t* kids /*(2T-1) x 2*/);

}  // namespace dgb
