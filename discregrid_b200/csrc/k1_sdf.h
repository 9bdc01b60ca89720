// Launch interface of the K1 kernels (k1_sdf.cu).  Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>
#include "bvh_build.h"
#include "dg_device.cuh"

namespace dgb {

#ifndef K1_THREADS_PER_BLOCK
#define K1_THREADS_PER_BLOCK 64
#endif
constexpr int K1_THREADS = K1_THREADS_PER_BLOCK;
// phase choice of the warp-synchronous traversal: the phase with the largest weight * #lanes runs
#ifndef K1_NODE_WEIGHT
#define K1_NODE_WEIGHT 2
#endif
#ifndef K1_LEAF_WEIGHT
#define K1_LEAF_WEIGHT 3
#endif
#ifndef K1_POP_WEIGHT
#define K1_POP_WEIGHT 4
#endif
#ifndef K1_POP_TRIES
#define K1_POP_TRIES 4          // deferred siblings re-tested per POP phase and lane
#endif
#ifndef K1_NODEF_STRIDE
#define K1_NODEF_STRIDE 5         // float4s per fp32 node record: 5 = packed 80 B, 6 = padded to 96 B
#endif
#ifndef K1_MIN_BLOCKS
#define K1_MIN_BLOCKS (1024 / K1_THREADS_PER_BLOCK)   // blocks per SM the register allocation must allow (32 warps)
#endif

// K1_PACKET 1 (default): the 32 queries of a brick walk the tree TOGETHER (one shared order, certified fp32
// pruning) and the reference's order-dependent accept rule is replayed afterwards on the few near-minimum triangles; lanes whose checks fail
// are walked again per lane (k1_sdf.cu, nearest_triangle_packet).  0: one query per lane in the reference's own order for the whole walk
// (the round-1 kernel; still what mesh_distance_kernel -- arbitrary points, no bricks -- and the fallback run).
//   K1_PKT_K          near-minimum candidates kept per query (8: with K = 6 bunny.obj's valence-7/8 vertices fall back to the per-lane walk)
//   K1_PKT_MIN_BLOCKS blocks per SM the register allocation of the node-loop kernel must allow (H100 80GB HBM3 at its 700 W limit,
//                     bunny.obj / torus 128^3: 14 -> 72 registers 40.2 / 28.6 ms; 12 -> 80 registers 42.2 / 30.2 ms; 10 or 8 -> 45.4 / 32.6 ms)
#ifndef K1_PACKET
#define K1_PACKET 1
#endif
#ifndef K1_PKT_MIN_BLOCKS
#define K1_PKT_MIN_BLOCKS 14
#endif

// One of the four row-major 3-D node arrays of the grid (vertex nodes, x-/y-/z-edge nodes), restricted to the
// slow-planes [s0, s1) that a node range touches.  l = l_base + (s*Dm + m)*Df + f.
// The warp's brick is chosen per node array at launch time: the power-of-two shape (f x m x s, 32 nodes) whose PHYSICAL diagonal is
// shortest.  On cubic cells that is 4 x 4 x 2 (x-edge arrays: their node spacing along f is half a cell); on strongly anisotropic cells
// (a flat bounding box sampled with a cubic resolution) a flatter brick keeps the 32 queries closer together than a fixed 4 x 4 x 2
// (CPU schedule model: -6 % issued instructions on the bench torus).
struct K1Segment {
    unsigned l_base, Ds, Dm, Df, s0, s1, tiles_f, tiles_m, tiles_s, block_begin;
    unsigned lf, lm;               // log2 of the brick's extents along f and m (s extent = 32 >> (lf + lm))
    unsigned pl_stride;            // plane groups between consecutive brick layers (1 = contiguous slab, n_parts = interleaved deal)
    unsigned out_base;             // interleaved mode: element offset of this array inside the part's exchange slot
    int kind;                      // 0 vertex (s,m,f)=(k,j,i); 1 x-edge (k,j,2i+b); 2 y-edge (i,k,2j+b); 3 z-edge (j,i,2k+b)
};
struct K1Work {
    K1Segment seg[4];
    int nseg;
    unsigned l_begin, l_end;
    int compact;                   // 0: out[l - l_begin]; 1: interleaved exchange slot (see k1_launch_sample_interleaved)
};

struct DeviceBvh {                 // device mirrors of HostBvh, uploaded once by dg_mesh_create
    const SpherePair* spheres = nullptr;
    const LeafRecord* leaves = nullptr;
    const PseudoNormals* normals = nullptr;
    const LeafF* leaves_f = nullptr;            // fp32 triangle shadows (the packet walk's leaf bound)
    const float4* nodes_f = nullptr;          // fp32 record per internal node, K1_NODEF_STRIDE float4s: SpherePairF (2) + BoxPairF (3) [+ pad]
    double ctr[3] = {0, 0, 0};
    float half_extent = 0.f;
    int n_tri = 0;
    int stack_depth = 1;           // deferred-sibling slots per lane (= tree levels - 1, at least 1)
};

cudaError_t k1_configure(int stack_depth);
cudaError_t k1_launch_sample_nodes(const DeviceBvh& m, const GridDev& g, double sign, uint64_t l_begin, uint64_t count,
                                   double* d_out, cudaStream_t stream);
// narrow-band form of k1_launch_sample_nodes (addFunction with pred(x) = |distance| <= band): the node-range [l_begin, l_begin + count) is
// written exactly as by k1_launch_sample_nodes where |distance| <= band and DBL_MAX elsewhere; nodes outside the range are never written.
// A classifier drops the blocks that provably hold no node within the band before the node loop runs (k1_sdf.cu, NARROW-BAND CLASSIFIER).
// d_scratch: k1_band_scratch_bytes(g, l_begin, count) bytes of device memory, used in stream order (one buffer per concurrent stream).
size_t k1_band_scratch_bytes(const GridDev& g, uint64_t l_begin, uint64_t count);
cudaError_t k1_launch_sample_nodes_band(const DeviceBvh& m, const GridDev& g, double sign, double band, uint64_t l_begin, uint64_t count,
                                        double* d_out, void* d_scratch, cudaStream_t stream);
// slab form: planes [plane_begin[a], plane_end[a]) of node array a (a = 0..3), written at d_full[l]
cudaError_t k1_launch_sample_slab(const DeviceBvh& m, const GridDev& g, double sign, const unsigned plane_begin[4], const unsigned plane_end[4],
                                  double* d_full, cudaStream_t stream);
// interleaved deal of plane pairs (SURVEY H7 / 8e P1): part `part` owns pairs part, part + n_parts, ... of every node array and writes
// them compactly into its exchange slot; k1_launch_unpack_interleaved scatters the gathered slots into node order.
struct InterleavedLayout {
    unsigned n_parts = 1;
    unsigned rot[4];               // plane group p of array a belongs to part (p + rot[a]) % n_parts: the deal is rotated per array so that the
                                   // parts that get one plane group more differ from array to array (129 planes = 65 pairs over 8 parts: 9:8 in
                                   // every array without the rotation, 33:32 over the four arrays with it)
    unsigned off[4][16];           // off[a][part]: element offset of array a in part's slot
    unsigned pairs[4];             // plane pairs of array a
    unsigned plane[4];             // elements per plane of array a
    uint64_t slot_elems = 0;       // elements per slot (max over parts)
    unsigned lf[4], lm[4];         // brick shape of array a (its plane groups are 32 >> (lf + lm) planes thick)
};
bool k1_interleaved_layout(const GridDev& g, unsigned n_parts, InterleavedLayout& L);
cudaError_t k1_launch_sample_interleaved(const DeviceBvh& m, const GridDev& g, double sign, const InterleavedLayout& L, unsigned part,
                                         double* d_slot, cudaStream_t stream);
void k1_interleaved_node_slots(const GridDev& g, const InterleavedLayout& L, uint64_t l_begin, uint64_t count, uint32_t* part_out, uint64_t* pos_out);
struct K1Run { uint64_t slot_pos, node_begin, count; };      // slot[slot_pos .. +count) == nodes[node_begin .. +count)
void k1_interleaved_runs(const GridDev& g, const InterleavedLayout& L, unsigned part, std::vector<K1Run>& runs);
cudaError_t k1_launch_unpack_interleaved(const GridDev& g, const InterleavedLayout& L, const double* d_slots, double* d_nodes, cudaStream_t stream);
cudaError_t k1_launch_distance(const DeviceBvh& m, const double* d_pts, uint64_t count, int is_signed, double* d_dist,
                               double* d_near, int* d_ent, int* d_tri, cudaStream_t stream);
// the same query that also writes the weights d_bary[count][3] of the nearest point (K10's forward; mesh_distance_bary_kernel)
cudaError_t k1_launch_distance_bary(const DeviceBvh& m, const double* d_pts, uint64_t count, int is_signed, double* d_dist,
                                    double* d_near, int* d_ent, int* d_tri, double* d_bary, cudaStream_t stream);
cudaError_t k1_launch_node_positions(const GridDev& g, uint64_t l_begin, uint64_t count, double* d_x, cudaStream_t stream);
cudaError_t k1_launch_build_cells(const GridDev& g, uint64_t c_begin, uint64_t count, unsigned* d_cells, cudaStream_t stream);
cudaError_t k1_launch_fp64_rate_probe(int blocks, int iters, double* d_out, cudaStream_t stream);
cudaError_t k1_launch_fma_probe(double a, double b, double c, double* d_out, cudaStream_t stream);

}  // namespace dgb
