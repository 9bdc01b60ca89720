// Launch interface of K6 (k6_isosurface.cu): level sets of a field by marching tetrahedra.  Host-callable, no kernel code here.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "dg_device.cuh"

namespace dgb {

constexpr unsigned K6_MAX_SUBDIVISIONS = 16;
constexpr unsigned long long K6_CHUNK = 1ull << 24;      // lattice points per values pass: 384 MiB of positions

struct K6Lattice {               // the lattice of a grid subdivided s times (contract in k6_isosurface.cu)
    double mn[3], mx[3], cell[3];
    unsigned s;
    unsigned np[3];              // lattice points per axis: s * n + 1
};

// the corner mask (bit 0 = +x, bit 1 = +y, bit 2 = +z) of edge direction d = 0..6: (1,0,0), (0,1,0), (0,0,1), (1,1,0), (1,0,1), (0,1,1), (1,1,1)
DG_HD unsigned mask_of_dir(unsigned d) { return ((1u | (2u << 3) | (4u << 6) | (3u << 9) | (5u << 12) | (6u << 15) | (7u << 18)) >> (3 * d)) & 7u; }
// coordinate a of lattice index i: mn + cell * (i / s), clamped to mx (the bits of the lattice positions, shared with K13)
DG_HD double lat_coord(const K6Lattice& L, int a, unsigned i)
{
    const double x = L.mn[a] + L.cell[a] * ((double)i / (double)L.s);
    return x > L.mx[a] ? L.mx[a] : x;
}
// lin offset of the cell corner with mask m
DG_HD unsigned corner_offset(const K6Lattice& L, unsigned m)
{
    return (m & 1u) + L.np[0] * (((m >> 1) & 1u) + L.np[1] * (m >> 2));
}

// the lattice of `g` at subdivision s, and its number of points (64-bit: the caller refuses 2^31 or more before anything else)
K6Lattice k6_lattice(const GridDev& g, unsigned s, uint64_t& n_points);
unsigned k6_tile();                                      // entries per tile of the count scan and of the emit passes
// d_x[3 * i + a] = position of lattice point begin + i, i < n
cudaError_t k6_launch_positions(const K6Lattice& L, uint64_t begin, uint64_t n, double* d_x, cudaStream_t stream);
// per lattice cell: d_count[c] = triangles of its emitting tetrahedra (0..12); d_flags[7 * lin(p) + d] = 1 for their crossing edges.
// d_flags must be zero on entry (7 bytes per lattice point)
cudaError_t k6_launch_classify(const K6Lattice& L, const double* d_values, double iso, unsigned char* d_count, unsigned char* d_flags,
                               cudaStream_t stream);
// d_tile (ceil(n / k6_tile()) entries) <- exclusive scan of the counts per tile; total = sum of all counts (64-bit).  Synchronises `stream`.
// The tile offsets are 32-bit: they are only meaningful when total < 2^32, which the caller checks.
cudaError_t k6_scan_counts(const unsigned char* d_count, uint64_t n, unsigned* d_tile, uint64_t& total, cudaStream_t stream);
// vertex of every flagged edge, and its edge id 7 * lin(p) + d, at its rank (d_edge_tile: k4_scan_flags of d_flags); d_chunk[e / 32] = rank
// of the first flag of e's 32-edge chunk, for the triangle pass.  n_edges = 7 * lattice points
cudaError_t k6_launch_vertices(const K6Lattice& L, const double* d_values, double iso, const unsigned char* d_flags, uint64_t n_edges,
                               const unsigned* d_edge_tile, unsigned* d_chunk, double* d_vertices, uint64_t* d_edge_ids, cudaStream_t stream);
// triangles of every cell at the scanned slots (d_tri_tile: k6_scan_counts of d_count), vertex ids from d_flags + d_chunk
cudaError_t k6_launch_triangles(const K6Lattice& L, const double* d_values, double iso, const unsigned char* d_count, const unsigned* d_tri_tile,
                                const unsigned char* d_flags, const unsigned* d_chunk, unsigned* d_triangles, cudaStream_t stream);

}  // namespace dgb
