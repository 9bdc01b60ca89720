// Launch interface of K8 (k8_refit.cu): refits a mesh's device records to new vertex positions, topology and leaf order kept.
// Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>
#include "bvh_build.h"
#include "k5_winding.h"

namespace dgb {

constexpr int K8_THREADS = 128;
constexpr int K8_BOUNDS_GROUP = 64;     // vertices (first pass) or partial bounds (later passes) folded in order by one thread
constexpr int K8_MAX_NODEF_STRIDE = 8;  // float4s of an fp32 node record the packing pass can stage (K1_NODEF_STRIDE is 5 or 6)

// an internal node of the implicit tree: leaf positions [b, e), split m = (b + e) >> 1, parent split (-1 for the root), side in the parent
struct RefitNodeRef { int32_t b, e, parent, side; };

// per internal node (index = split position m): the bottom-up sums and the two r^2 maxima (fp64 bit patterns, atomicMax)
struct RefitSums {
    double S[3], c[3];                  // vertex sum, sphere centre S / (3n)
    double lo[3], hi[3];                // box of the node's vertices (NaN skipped), for the parent's box
    double box[12];                     // the two child boxes as the fp32 records round them: {l lo, l hi, r lo, r hi}
    double A, AC[3], CS[3], N[3], p[3], M[9], cnt;   // K5 cluster sums (k5_winding.cu)
    unsigned long long r2s, r2k;        // max |c - v|^2 and max |v - p~|^2 over the node's vertices
};
static_assert(sizeof(RefitSums) == 392, "RefitSums must be 392 bytes");

struct RefitBounds { double lo[3], hi[3]; int finite, _pad; };    // partial bounds of a contiguous run of vertices, folded in order
static_assert(sizeof(RefitBounds) == 56, "RefitBounds must be 56 bytes");

// topology tables, built once on the host from F and the leaf order
struct RefitTopoHost {
    std::vector<uint32_t> f_leaf;       // [T][3] vertex ids of the triangle at each leaf position
    std::vector<uint32_t> inc_begin;    // [nV + 1] vertex -> incidences (CSR)
    std::vector<uint32_t> inc;          // [3T] incidences in (triangle, slot) order: 3 * triangle + slot
    std::vector<RefitNodeRef> nodes;    // internal nodes, root first, grouped by depth
    std::vector<uint32_t> level_begin;  // nodes of depth d (root: 0) are nodes[level_begin[d], level_begin[d + 1])
};
void k8_build_topology(const HostBvh& h, RefitTopoHost& out);
// partial-bounds entries the bounds passes need (both ping-pong buffers together)
uint64_t k8_bounds_entries(uint64_t n_vertices);

struct RefitDev {
    // inputs
    const double* V = nullptr;          // [nV][3] the new positions
    uint64_t n_vertices = 0;
    int n_tri = 0, levels = 1;          // levels = HostBvh::max_depth
    const uint32_t* F = nullptr;        // [T][3] by triangle id
    const uint32_t* f_leaf = nullptr;   // [T][3] by leaf position
    const int32_t* order = nullptr;     // [T] leaf position -> triangle id
    const uint32_t* inc_begin = nullptr;
    const uint32_t* inc = nullptr;
    const RefitNodeRef* nodes = nullptr;
    // scratch
    RefitSums* sums = nullptr;          // [T]
    RefitBounds* part = nullptr;        // [k8_bounds_entries(nV)]
    double* bounds = nullptr;           // [5]: centre, half extent, finite (1.0 / 0.0)
    double* pn_tri = nullptr;           // [T][3]  by triangle id
    double* angle = nullptr;            // [T][3]
    double* pn_vert = nullptr;          // [nV][3]
    double* pn_edge = nullptr;          // [T][3][3]
    // outputs; a NULL pointer skips that record
    SpherePair* spheres = nullptr;
    LeafRecord* leaves = nullptr;
    LeafF* leaves_f = nullptr;
    PseudoNormals* normals = nullptr;
    float4* nodes_f = nullptr;
    int nodef_stride = 5;               // float4s per fp32 node record, 5..K8_MAX_NODEF_STRIDE
    WindLeaf* wind_leaves = nullptr;
    WindClusterPair* wind_clusters = nullptr;
};

// Queues every pass on `stream`.  k1 = false: only the K5 records (wind_*), for their first use after a refit.  The centre, half extent and
// finite flag land in r.bounds; the caller reads them back.
cudaError_t k8_launch_refit(const RefitDev& r, const std::vector<uint32_t>& level_begin, bool k1, cudaStream_t stream);

// the library's acos of the pseudonormal angles: k5_atan2(sqrt((1 - x) * (1 + x)), x)
double k8_acos_host(double x);

}  // namespace dgb
