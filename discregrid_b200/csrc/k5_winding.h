// Launch interface of K5 (k5_winding.cu): generalized winding numbers over the mesh's sphere tree.  Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "bvh_build.h"
#include "dg_device.cuh"

namespace dgb {

constexpr int K5_THREADS = 128;
constexpr int K5_MAX_STACK = 32;   // deferred right children per lane; a tree of < 2^25 triangles has at most 26 levels

struct WindLeaf { double v[9]; };                        // v0, v1, v2 of the triangle at this leaf position: V[F[t]] as uploaded
static_assert(sizeof(WindLeaf) == 72, "WindLeaf must be 72 bytes");
struct WindCluster { double p[3], n[3], M[9], r; };      // p~, n~, M (row-major, M[j][k] = sum (c - p~)_j (a n)_k), r_c
static_assert(sizeof(WindCluster) == 128, "WindCluster must be 128 bytes");
struct alignas(64) WindClusterPair { WindCluster l, r; }; // children of the internal node whose split position is the index; root: [0].l
static_assert(sizeof(WindClusterPair) == 256, "WindClusterPair must be 256 bytes");

struct WindDev {                   // device records of the winding mode, built and uploaded at first use
    const WindLeaf* leaves = nullptr;
    const WindClusterPair* clusters = nullptr;
    int n_tri = 0;
    int stack_depth = 1;           // as DeviceBvh::stack_depth (= tree levels - 1, at least 1)
};

// The leaf and cluster records of `h` (which must still hold V, F and order, as dg_mesh keeps them): leaves[T], clusters[T].
void build_winding_records(const HostBvh& h, RawVec<WindLeaf>& leaves, RawVec<WindClusterPair>& clusters);

// IEEE + - * / sqrt only (k5_winding.cu): the same bits on the device, in the CPU emulation and in a numpy restatement
double k5_atan2_host(double y, double x);

// w[i] = winding number of d_pts[i] (n x 3); beta >= 1 or +inf (checked by the caller)
cudaError_t k5_launch_winding(const WindDev& m, const double* d_pts, uint64_t n, double beta, double* d_w, cudaStream_t stream);
// node pass over [l_begin, l_begin + count): d_vals holds what K1 wrote with sign = +1 (dense: band = +inf; band form: its band); every
// value becomes the winding-signed one, sign * (w > 0.5 ? -d_u : d_u), and the sentinels become what K1 writes with `sign`
cudaError_t k5_launch_sign_nodes(const WindDev& m, const GridDev& g, double sign, double band, double beta, uint64_t l_begin, uint64_t count,
                                 double* d_vals, cudaStream_t stream);
// point pass: d_dist holds unsigned distances of d_pts (mesh_distance_kernel, is_signed = 0); each becomes w > 0.5 ? -d : d (DBL_MAX stays)
cudaError_t k5_launch_sign_points(const WindDev& m, const double* d_pts, uint64_t n, double beta, double* d_dist, cudaStream_t stream);

}  // namespace dgb
