// K6: the level set {phi = iso} of a field as a triangle mesh, by marching tetrahedra on a lattice that subdivides every grid cell s times.
//
// The reference has no such function, so this contract is the library's own.  It fixes what is emitted, in which order and with which bits;
// tests/isosurface_ref.py restates it in numpy and the tests compare bit for bit.
//
// Lattice.  The grid has n = (nx, ny, nz) cells, the subdivision is s (1 <= s <= 16).  Lattice points P = (I, J, K), 0 <= I <= s*nx (J, K
//   alike), numbered lin(P) = I + (s*nx + 1) * (J + (s*ny + 1) * K).  Position per axis a: x_a = mn[a] + cell[a] * ((double)I_a / (double)s),
//   replaced by mx[a] when it exceeds mx[a].  For s = 1 these are the bits of the vertex nodes of node_position (dg_device.cuh) wherever that
//   position lies inside the domain.  A lattice of 2^31 points or more is refused before anything is allocated.
// Values.  f_P has the bits of the value-only dg_interpolate_batch of the field at x_P (K2 evaluates the lattice, unchanged).  P is valid iff
//   f_P is finite and != DBL_MAX; P is negative iff f_P < iso (strict: -0.0 and values equal to iso are non-negative).  On a reduced field a
//   point whose lookup cell was removed gets DBL_MAX and is invalid -- including a point on a face that the lookup rule (K2: floor of
//   (x - mn) * inv, clamped to the last cell) assigns to the removed neighbour of a kept cell.
// Tetrahedra.  Lattice cell c = (I, J, K) (each index below s*n) is split into the 6 Kuhn tetrahedra: for t = 0..5, the permutations pi of
//   (0, 1, 2) in lexicographic order, v0 = c, v1 = v0 + e_pi0, v2 = v1 + e_pi1, v3 = c + (1, 1, 1).  The split is the same in every cell, so
//   shared faces match.  A tetrahedron emits only if its four vertices are valid.
// Edges and vertices.  Every tetrahedron edge is (p, p + delta) with delta one of 7 directions, d = 0..6 <-> (1,0,0), (0,1,0), (0,0,1),
//   (1,1,0), (1,0,1), (0,1,1), (1,1,1); edge id 7 * lin(p) + d.  An edge crosses iff exactly one endpoint is negative.  A vertex is emitted
//   for a crossing edge iff an emitting tetrahedron contains the edge (no vertex is unreferenced); vertices are ordered by edge id, and the
//   edge id of every vertex is written beside it (ascending; K13 differentiates the vertex through it, k13_isosurface_grad.cu).  With p
//   the lower endpoint and q = p + delta: t = (iso - f_p) / (f_q - f_p), then x_a = x_p,a + t * (x_q,a - x_p,a), in that order, no FMA.
//   Monotone rounding keeps t in [0, 1] while both differences are finite; near +-DBL_MAX they can overflow and t can become 0 or NaN -- the
//   contract keeps whatever that arithmetic gives.
// Triangles.  The case of a tetrahedron is its 4-bit negative mask (bit i = v_i negative).  One negative vertex (or one non-negative vertex)
//   gives one triangle on the three edges at that vertex.  Two negative vertices {a, b}, non-negative {c, d} (a < b, c < d) give the quad
//   ac, ad, bd, bc, split along ac-bd.  The normal (p1 - p0) x (p2 - p0) points from the negative to the non-negative side (outward for an
//   SDF).  Orientation comes from this table and the parity of pi only, never from a floating-point cross product.  The table below is
//   oriented for the even permutations (positively oriented tetrahedra, t = 0, 3, 4); for the odd ones (t = 1, 2, 5) the 2nd and 3rd vertex
//   of every triangle are swapped.  Edges as vertex pairs of the tetrahedron:
//      case  triangles                                  case  triangles
//       0    -                                            8    (03 23 13)
//       1    (01 02 03)                                   9    (01 02 23) (01 23 13)
//       2    (01 13 12)                                  10    (01 23 12) (01 03 23)
//       3    (02 03 13) (02 13 12)                       11    (02 23 12)
//       4    (02 12 23)                                  12    (02 12 13) (02 13 03)
//       5    (01 23 03) (01 12 23)                       13    (01 12 13)
//       6    (01 13 23) (01 23 02)                       14    (01 03 02)
//       7    (03 13 23)                                  15    -
//   Triangle order: by lattice cell c (numbered I + s*nx * (J + s*ny * K)), then t, then position in the table entry.  Indices are 0-based
//   uint32 into the vertex array (the layout dg_mesh_create takes).
// Not done, on purpose: coincident points are not welded (when f_q == iso several edges give vertices at x_q, and zero-area triangles are
//   kept, so the mesh stays closed when counted by vertex ids); no normals (interpolate with gradient=True at the vertices gives them); no
//   simplification.
// Closedness.  Every triangle edge lies in a tetrahedron face; a face with a sign change contributes one segment, shared by the two tetrahedra
//   on that face.  So when the negative region touches neither the lattice boundary nor an invalid tetrahedron, every undirected mesh edge is
//   used by exactly two triangles, in opposite directions.
//
// Passes (the host side is dg_isosurface_create in dg_api.cu): lattice positions per chunk of K6_CHUNK points, evaluated by K2's value-only
// kernel; classify (one thread per lattice cell: triangle count byte, idempotent byte flags of the crossing edges); scans (K4's flag scan over
// the 7 * Np edge flags, a warp-synchronous scan of the counts over the four bit planes of 0..12); emit (one warp per tile of edges writes the
// vertices and their edge ids at their ranks and the rank of every 32-edge chunk; one warp per tile of cells writes the triangles).  Integer work apart from the
// positions and the vertex arithmetic above; nothing depends on block or chunk size.  Warp-synchronous (ballot / popc only), so tests/emu
// runs it unchanged.
#include "k6_isosurface.h"
#include "dg_launch.h"

#include <cfloat>
#include <cmath>
#include <vector>

namespace dgb {
namespace {

constexpr unsigned TILE = 1024;                       // entries per warp in the count scan and the emit passes

// the case table of the header: bits 0-1 = triangles, then 3 bits per edge (pair code: 01 02 03 12 13 23 = 0..5), triangle k at bit 2 + 9k
#define K6_TRI(a, b, c) ((a) | (b) << 3 | (c) << 6)
DG_HD unsigned k6_case(unsigned m)
{
    switch (m) {
    case 1: return 1u | K6_TRI(0u, 1u, 2u) << 2;
    case 2: return 1u | K6_TRI(0u, 4u, 3u) << 2;
    case 3: return 2u | K6_TRI(1u, 2u, 4u) << 2 | K6_TRI(1u, 4u, 3u) << 11;
    case 4: return 1u | K6_TRI(1u, 3u, 5u) << 2;
    case 5: return 2u | K6_TRI(0u, 5u, 2u) << 2 | K6_TRI(0u, 3u, 5u) << 11;
    case 6: return 2u | K6_TRI(0u, 4u, 5u) << 2 | K6_TRI(0u, 5u, 1u) << 11;
    case 7: return 1u | K6_TRI(2u, 4u, 5u) << 2;
    case 8: return 1u | K6_TRI(2u, 5u, 4u) << 2;
    case 9: return 2u | K6_TRI(0u, 1u, 5u) << 2 | K6_TRI(0u, 5u, 4u) << 11;
    case 10: return 2u | K6_TRI(0u, 5u, 3u) << 2 | K6_TRI(0u, 2u, 5u) << 11;
    case 11: return 1u | K6_TRI(1u, 5u, 3u) << 2;
    case 12: return 2u | K6_TRI(1u, 3u, 4u) << 2 | K6_TRI(1u, 4u, 2u) << 11;
    case 13: return 1u | K6_TRI(0u, 3u, 4u) << 2;
    case 14: return 1u | K6_TRI(0u, 2u, 1u) << 2;
    default: return 0u;
    }
}
#undef K6_TRI

// pair code -> its lower / upper vertex of the tetrahedron (01 02 03 12 13 23)
DG_HD unsigned pair_lo(unsigned p) { return (0x940u >> (2 * p)) & 3u; }
DG_HD unsigned pair_hi(unsigned p) { return (0xFB9u >> (2 * p)) & 3u; }
// corners of a lattice cell as 3-bit masks (bit 0 = +x, bit 1 = +y, bit 2 = +z); tetrahedron t: v0 = 0, v1 = e_pi0, v2 = v1 + e_pi1, v3 = 7
DG_HD unsigned tet_corner(unsigned t, unsigned i)
{
    const unsigned pi0 = (0xA50u >> (2 * t)) & 3u;     // pi0 = 0 0 1 1 2 2
    const unsigned pi1 = (0x489u >> (2 * t)) & 3u;     // pi1 = 1 2 0 2 0 1
    return i == 0 ? 0u : i == 1 ? (1u << pi0) : i == 2 ? ((1u << pi0) | (1u << pi1)) : 7u;
}
DG_HD bool tet_odd(unsigned t) { return (0x26u >> t) & 1u; }               // t = 1, 2, 5
// direction d of an edge whose endpoints differ by the corner mask m (1..7); mask_of_dir (k6_isosurface.h) is its inverse
DG_HD unsigned dir_of_mask(unsigned m) { return (((0u << 3) | (1u << 6) | (3u << 9) | (2u << 12) | (4u << 15) | (5u << 18) | (6u << 21)) >> (3 * m)) & 7u; }

// finite and not the sentinel
DG_HD bool value_valid(double v) { return fabs(v) <= DBL_MAX && v != DBL_MAX; }

// valid / negative bits of the 8 corners of lattice cell c, and the lin of its corner 0
DG_HD void cell_corners(const K6Lattice& L, const double* __restrict__ values, double iso, unsigned c, unsigned& l0, unsigned& valid, unsigned& neg)
{
    const unsigned m0 = L.np[0] - 1, m1 = L.np[1] - 1;
    const unsigned I = c % m0, r = c / m0, J = r % m1, K = r / m1;
    l0 = I + L.np[0] * (J + L.np[1] * K);
    valid = 0; neg = 0;
    for (unsigned k = 0; k < 8; k++) {
        const double v = values[l0 + corner_offset(L, k)];
        valid |= (value_valid(v) ? 1u : 0u) << k;
        neg |= (v < iso ? 1u : 0u) << k;
    }
}

// the case of tetrahedron t of a cell, or 0 when one of its vertices is invalid
DG_HD unsigned tet_mask(unsigned t, unsigned valid, unsigned neg, bool& emits)
{
    unsigned ok = 1u, m = 0u;
    for (unsigned i = 0; i < 4; i++) {
        const unsigned cv = tet_corner(t, i);
        ok &= (valid >> cv) & 1u;
        m |= ((neg >> cv) & 1u) << i;
    }
    emits = ok != 0u;
    return m;
}

DG_HD unsigned long long edge_id(const K6Lattice& L, unsigned l0, unsigned t, unsigned p)
{
    const unsigned a = tet_corner(t, pair_lo(p)), b = tet_corner(t, pair_hi(p));
    return 7ull * (unsigned long long)(l0 + corner_offset(L, a)) + dir_of_mask(a ^ b);
}

__global__ void positions_kernel(K6Lattice L, unsigned long long begin, unsigned long long n, double* __restrict__ x)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned l = (unsigned)(begin + i);
    const unsigned I = l % L.np[0], r = l / L.np[0], J = r % L.np[1], K = r / L.np[1];
    x[3 * i] = lat_coord(L, 0, I);
    x[3 * i + 1] = lat_coord(L, 1, J);
    x[3 * i + 2] = lat_coord(L, 2, K);
}

__global__ void classify_kernel(K6Lattice L, const double* __restrict__ values, double iso, unsigned n_cells, unsigned char* __restrict__ count,
                                unsigned char* __restrict__ flags)
{
    const unsigned long long c = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_cells) return;
    unsigned l0, valid, neg;
    cell_corners(L, values, iso, (unsigned)c, l0, valid, neg);
    unsigned cnt = 0;
    if (valid != 0u && neg != 0u && neg != 0xffu) {
        for (unsigned t = 0; t < 6; t++) {
            bool emits;
            const unsigned m = tet_mask(t, valid, neg, emits);
            const unsigned nt = k6_case(m) & 3u;
            if (!emits || nt == 0u) continue;
            cnt += nt;
            for (unsigned p = 0; p < 6; p++)
                if (((m >> pair_lo(p)) ^ (m >> pair_hi(p))) & 1u) flags[edge_id(L, l0, t, p)] = 1;
        }
    }
    count[c] = (unsigned char)cnt;
}

// sum of the counts per tile of TILE cells (one warp per tile): four ballots over the bit planes of 0..12
__global__ void count_tiles_kernel(const unsigned char* __restrict__ count, unsigned long long n, unsigned* __restrict__ tile_sum)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long base = tile * TILE;
    if (base >= n) return;                            // whole warps
    unsigned sum = 0;
    for (unsigned k = 0; k < TILE; k += 32) {
        const unsigned long long i = base + k + lane;
        const unsigned v = i < n ? count[i] : 0u;
        for (unsigned b = 0; b < 4; b++) sum += (unsigned)__popc(__ballot_sync(0xffffffffu, (v >> b) & 1u)) << b;
    }
    if (lane == 0) tile_sum[tile] = sum;
}

// flags set in [e & ~31, e): the chunk's bytes are 0 / 1, read as four 8-byte words
DG_HD unsigned flags_before(const unsigned char* __restrict__ flags, unsigned long long e)
{
    const unsigned long long* w = reinterpret_cast<const unsigned long long*>(flags + (e & ~31ull));
    const unsigned r = (unsigned)(e & 31ull);
    unsigned n = 0;
    for (unsigned q = 0; q < 4 && 8 * q < r; q++) {
        unsigned long long x = w[q];
        const unsigned keep = r - 8 * q;
        if (keep < 8) x &= (1ull << (8 * keep)) - 1ull;
        n += (unsigned)((x * 0x0101010101010101ull) >> 56);     // byte sum
    }
    return n;
}

__global__ void vertices_kernel(K6Lattice L, const double* __restrict__ values, double iso, const unsigned char* __restrict__ flags,
                                unsigned long long n_edges, const unsigned* __restrict__ edge_tile, unsigned* __restrict__ chunk,
                                double* __restrict__ vout, unsigned long long* __restrict__ eout)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long base = tile * TILE;
    if (base >= n_edges) return;                      // whole warps
    unsigned run = edge_tile[tile];
    const unsigned lt = (1u << lane) - 1u;
    for (unsigned k = 0; k < TILE; k += 32) {
        const unsigned long long e = base + k + lane;
        const bool set = e < n_edges && flags[e] != 0;
        const unsigned m = __ballot_sync(0xffffffffu, set);
        if (lane == 0 && base + k < n_edges) chunk[(base + k) >> 5] = run;
        if (set) {
            const unsigned lp = (unsigned)(e / 7ull), dm = mask_of_dir((unsigned)(e % 7ull));
            const unsigned lq = lp + corner_offset(L, dm);
            const unsigned I = lp % L.np[0], r = lp / L.np[0], J = r % L.np[1], K = r / L.np[1];
            const unsigned ip[3] = {I, J, K};
            const double fp = values[lp], fq = values[lq];
            const double t = (iso - fp) / (fq - fp);
            const unsigned rank = run + (unsigned)__popc(m & lt);
            double* v = vout + 3ull * rank;
            eout[rank] = e;
            for (int a = 0; a < 3; a++) {
                const double xp = lat_coord(L, a, ip[a]), xq = lat_coord(L, a, ip[a] + ((dm >> a) & 1u));
                v[a] = xp + t * (xq - xp);
            }
        }
        run += (unsigned)__popc(m);
    }
}

__global__ void triangles_kernel(K6Lattice L, const double* __restrict__ values, double iso, const unsigned char* __restrict__ count,
                                 unsigned n_cells, const unsigned* __restrict__ tri_tile, const unsigned char* __restrict__ flags,
                                 const unsigned* __restrict__ chunk, unsigned* __restrict__ tout)
{
    const unsigned long long tile = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned long long base = tile * TILE;
    if (base >= n_cells) return;                      // whole warps
    unsigned run = tri_tile[tile];
    const unsigned lt = (1u << lane) - 1u;
    for (unsigned k = 0; k < TILE; k += 32) {
        const unsigned long long c = base + k + lane;
        const unsigned cnt = c < n_cells ? count[c] : 0u;
        unsigned before = 0, total = 0;
        for (unsigned b = 0; b < 4; b++) {
            const unsigned m = __ballot_sync(0xffffffffu, (cnt >> b) & 1u);
            before += (unsigned)__popc(m & lt) << b;
            total += (unsigned)__popc(m) << b;
        }
        if (cnt) {
            unsigned l0, valid, neg;
            cell_corners(L, values, iso, (unsigned)c, l0, valid, neg);
            unsigned* out = tout + 3ull * (run + before);
            for (unsigned t = 0; t < 6; t++) {
                bool emits;
                const unsigned m = tet_mask(t, valid, neg, emits);
                const unsigned cs = k6_case(m);
                if (!emits) continue;
                for (unsigned j = 0; j < (cs & 3u); j++) {
                    unsigned id[3];
                    for (unsigned q = 0; q < 3; q++) {
                        const unsigned long long e = edge_id(L, l0, t, (cs >> (2 + 9 * j + 3 * q)) & 7u);
                        id[q] = chunk[e >> 5] + flags_before(flags, e);
                    }
                    const bool odd = tet_odd(t);
                    out[0] = id[0]; out[1] = odd ? id[2] : id[1]; out[2] = odd ? id[1] : id[2];
                    out += 3;
                }
            }
        }
        run += total;
    }
}

inline unsigned blocks_for(unsigned long long threads, unsigned block) { return (unsigned)((threads + block - 1) / block); }

}  // namespace

K6Lattice k6_lattice(const GridDev& g, unsigned s, uint64_t& n_points)
{
    K6Lattice L;
    for (int a = 0; a < 3; a++) {
        L.mn[a] = g.mn[a]; L.mx[a] = g.mx[a]; L.cell[a] = g.cell[a];
        L.np[a] = s * g.n[a] + 1;                     // g.n < 2^16 (dg_grid_num_nodes), s <= 16: no overflow
    }
    L.s = s;
    n_points = (uint64_t)L.np[0] * L.np[1] * L.np[2];
    return L;
}

unsigned k6_tile() { return TILE; }

cudaError_t k6_launch_positions(const K6Lattice& L, uint64_t begin, uint64_t n, double* d_x, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(positions_kernel, blocks_for(n, 256), 256, 0, stream, L, (unsigned long long)begin, (unsigned long long)n, d_x);
    return DG_AFTER_LAUNCH();
}

cudaError_t k6_launch_classify(const K6Lattice& L, const double* d_values, double iso, unsigned char* d_count, unsigned char* d_flags,
                               cudaStream_t stream)
{
    const unsigned long long n_cells = (unsigned long long)(L.np[0] - 1) * (L.np[1] - 1) * (L.np[2] - 1);
    if (n_cells == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(classify_kernel, blocks_for(n_cells, 256), 256, 0, stream, L, d_values, iso, (unsigned)n_cells, d_count, d_flags);
    return DG_AFTER_LAUNCH();
}

cudaError_t k6_scan_counts(const unsigned char* d_count, uint64_t n, unsigned* d_tile, uint64_t& total, cudaStream_t stream)
{
    total = 0;
    if (n == 0) return cudaSuccess;
    const uint64_t tiles = (n + TILE - 1) / TILE;
    DG_KERNEL_LAUNCH(count_tiles_kernel, blocks_for(tiles * 32ull, 128), 128, 0, stream, d_count, (unsigned long long)n, d_tile);
    cudaError_t e = DG_AFTER_LAUNCH();
    if (e != cudaSuccess) return e;
    std::vector<unsigned> cnt(tiles);
    e = cudaMemcpyAsync(cnt.data(), d_tile, tiles * sizeof(unsigned), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return e;
    for (uint64_t t = 0; t < tiles; t++) { const unsigned c = cnt[t]; cnt[t] = (unsigned)total; total += c; }
    e = cudaMemcpyAsync(d_tile, cnt.data(), tiles * sizeof(unsigned), cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);          // cnt goes out of scope
    return e;
}

cudaError_t k6_launch_vertices(const K6Lattice& L, const double* d_values, double iso, const unsigned char* d_flags, uint64_t n_edges,
                               const unsigned* d_edge_tile, unsigned* d_chunk, double* d_vertices, uint64_t* d_edge_ids, cudaStream_t stream)
{
    if (n_edges == 0) return cudaSuccess;
    const uint64_t tiles = (n_edges + TILE - 1) / TILE;
    DG_KERNEL_LAUNCH(vertices_kernel, blocks_for(tiles * 32ull, 128), 128, 0, stream, L, d_values, iso, d_flags, (unsigned long long)n_edges,
                     d_edge_tile, d_chunk, d_vertices, reinterpret_cast<unsigned long long*>(d_edge_ids));
    return DG_AFTER_LAUNCH();
}

cudaError_t k6_launch_triangles(const K6Lattice& L, const double* d_values, double iso, const unsigned char* d_count, const unsigned* d_tri_tile,
                                const unsigned char* d_flags, const unsigned* d_chunk, unsigned* d_triangles, cudaStream_t stream)
{
    const unsigned long long n_cells = (unsigned long long)(L.np[0] - 1) * (L.np[1] - 1) * (L.np[2] - 1);
    if (n_cells == 0) return cudaSuccess;
    const uint64_t tiles = (n_cells + TILE - 1) / TILE;
    DG_KERNEL_LAUNCH(triangles_kernel, blocks_for(tiles * 32ull, 128), 128, 0, stream, L, d_values, iso, d_count, (unsigned)n_cells, d_tri_tile,
                     d_flags, d_chunk, d_triangles);
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
