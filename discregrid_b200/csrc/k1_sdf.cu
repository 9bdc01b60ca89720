// K1: nearest-triangle query + pseudonormal sign on the reference's own tree, bit-identical to the reference.
//
// Replaces TriangleMeshDistance::signed_distance / unsigned_distance / _query / point_triangle_sq_unsigned
// (TriangleMeshDistance.h:269-328, 514-562, 564-820) and, fused in front of it, indexToNodePosition
// (cubic_lagrange_discrete_grid.cpp:604-665) for the addFunction node loop (:806-817).
//
// What makes this more than a nearest-neighbour search: _query keeps the FIRST strictly smaller triangle in nearer-child-first
// order, compares d2 against fl(sqrt(best))^2 (:528) and prunes with the running best (:542-560), so the winner among triangles
// whose d2 differ by a few ulps (hence the nearest point, the entity, the sign and occasionally the last bit of the distance)
// depends on each query's own visit order.  Two walks live here:
//   * nearest_triangle        -- one query per lane, every lane in the reference's own order with its own stack; the warp shares the
//                                code path (one loop, phases chosen by vote) and the caches.  Round 1's node loop; now the kernel for
//                                arbitrary points, the fallback of the packet walk and the -DK1_PACKET=0 build.
//   * nearest_triangle_packet -- the 32 queries of a brick walk the tree together (certified fp32 pruning only), keep the few
//                                near-minimum triangles, and the reference's choice among them is replayed exactly afterwards; a lane
//                                whose checks fail is handed to nearest_triangle.  The node loop since round 2.
//
// Data (see bvh_build.h): implicit tree over leaf ranges [b,e); per internal node one 80-byte fp32 record (child spheres +
// child boxes, relative to the mesh centre) that DECIDES, the 64-byte fp64 sphere pair at spheres[(b+e)>>1] for the rare
// undecided case, one 128-byte fp64 record per triangle for the leaf test, one 7x3 pseudonormal block per triangle.  The
// per-lane stack of deferred siblings (packed range + fp32 sphere distance, 8 bytes) lives in shared memory, laid out
// [depth][lane] so it is bank-conflict-free whatever depth each lane is at.
//
// Structure of this file: tri_dist2 (leaf test) -> finish_query (nearest point + sign) -> leaf_lower_bound (certified fp32
// triangle bound) -> nearest_triangle (the warp-synchronous per-lane traversal: NODE / LEAF / POP phases, fp32 interval
// filter, exact-preserving shortcuts) -> nearest_triangle_packet -> the two kernels (grid nodes in bricks of 32; arbitrary points) -> launchers.
// The tuning constants are listed in k1_sdf.h.
#include "dg_device.cuh"
#include "bvh_build.h"
#include "k1_sdf.h"

#include <cfloat>
#include <mutex>
#include <vector>
#include <algorithm>

#include "dg_launch.h"       // DG_KERNEL_LAUNCH: <<<>>> on the device, fibers under tests/emu (DG_EMU)
#define SEG_BF(S) (1u << (S).lf)
#define SEG_BM(S) (1u << (S).lm)
#define SEG_BS(S) (32u >> ((S).lf + (S).lm))
#define LAY_BS(L, a) (32u >> ((L).lf[a] + (L).lm[a]))
#ifdef DG_EMU
#define DG_EMU_COUNT(i) (dg_emu::g_counters[(i)]++)        // event counters of the emulation (tests/emu, tools): nothing on the device
#define DG_EMU_ADD(i, v) (dg_emu::g_counters[(i)] += (unsigned long long)(v))
#define DG_EMU_TRACE_BLOCK(b) do { if (threadIdx.x == 0) dg_emu::g_block_trace.push_back(b); } while (0)
#else
#define DG_EMU_COUNT(i)
#define DG_EMU_ADD(i, v)
#define DG_EMU_TRACE_BLOCK(b)
#endif

namespace dgb {

namespace {

struct QueryResult {
    double dist;        // unsigned distance (sqrt of best d2)
    double s, t;        // barycentric parameters of the nearest point on the winning triangle
    int pos;            // leaf position of the winning triangle (-1 if none)
    int entity;         // dg_nearest_entity
};

__device__ __forceinline__ double2 ldg2(const double* p) { return __ldg(reinterpret_cast<const double2*>(p)); }

// point_triangle_sq_unsigned (TriangleMeshDistance.h:564-820) on a precomputed record.  Returns d2 and the
// (s, t, entity) the reference would use for nearest_point (:818); the point itself is only needed for the
// final winner, so it is reconstructed after the traversal.
//
// The reference is a 7-region decision tree whose leaves are only SEVEN distinct outcomes -- V0, V1, V2, E01, E02,
// E12, F -- each of them several times.  Run as written, 32 lanes scatter over ~20 short branches and the warp pays
// for all of them.  Here the decision tree is evaluated as pure predicate logic (same comparisons, same order, so
// NaNs fall the same way) producing the outcome code, and the arithmetic is done ONCE for the whole warp: one
// division (E01: -b0/a00, E02: -b1/a11, E12: numer/denom), one quadratic form (E12 and F), selected per lane.
// Every value a lane finally uses is produced by exactly the reference's operations in the reference's order.
__device__ __forceinline__ double tri_dist2(const LeafRecord* __restrict__ rec,
                                            double px, double py, double pz, double& s_out, double& t_out, int& ent_out)
{
    const double* r = reinterpret_cast<const double*>(rec);
    const double2 q0 = ldg2(r + 0), q1 = ldg2(r + 2), q2 = ldg2(r + 4), q3 = ldg2(r + 6);
    const double2 q4 = ldg2(r + 8), q5 = ldg2(r + 10), q6 = ldg2(r + 12), q7 = ldg2(r + 14);
    const double v0x = q0.x, v0y = q0.y, v0z = q1.x;
    const double e0x = q1.y, e0y = q2.x, e0z = q2.y;
    const double e1x = q3.x, e1y = q3.y, e1z = q4.x;
    const double a00 = q4.y, a01 = q5.x, a11 = q5.y;
    const double det = q6.x, inv_det = q6.y, denom = q7.x;

    const double dx = v0x - px, dy = v0y - py, dz = v0z - pz;          // diff = v0 - point  (:566)
    const double b0 = dx * e0x + dy * e0y + dz * e0z;                  // :572
    const double b1 = dx * e1x + dy * e1y + dz * e1z;                  // :573
    const double c = dx * dx + dy * dy + dz * dz;                      // :574
    const double s0 = a01 * b1 - a11 * b0;                             // :576
    const double t0 = a01 * b0 - a00 * b1;                             // :577

    // ---- outcome code (0..6 = V0 V1 V2 E01 E12 E02 F), predicate logic only
    const bool lower = (s0 + t0 <= det);                               // :581
    const bool sneg = (s0 < 0), tneg = (t0 < 0);
    const double tmp1_2 = a11 + b1, tmp0_2 = a01 + b0;                 // region 2 (:688-689)
    const double tmp1_6 = a00 + b0, tmp0_6 = a01 + b1;                 // region 6 (:735-736)
    const double numer_2 = tmp1_2 - tmp0_2, numer_6 = tmp1_6 - tmp0_6; // :692, :739
    const double numer_1 = tmp1_2 - a01 - b0;                          // region 1: a11 + b1 - a01 - b0 (:782)
    const int chain_b1 = (b1 >= 0) ? 0 : ((-b1 >= a11) ? 2 : 5);      // V0 / V2 / E02 (:606-623, :629-646)
    const int chain_b0 = (b0 >= 0) ? 0 : ((-b0 >= a00) ? 1 : 3);      // V0 / V1 / E01 (:652-669)
    const int ent_r4 = (b0 < 0) ? ((-b0 >= a00) ? 1 : 3) : chain_b1;   // :587-624
    const int ent_r2 = (tmp1_2 > tmp0_2) ? ((numer_2 >= denom) ? 1 : 4) : ((tmp1_2 <= 0) ? 2 : ((b1 >= 0) ? 0 : 5));   // :690-731
    const int ent_r6 = (tmp1_6 > tmp0_6) ? ((numer_6 >= denom) ? 2 : 4) : ((tmp1_6 <= 0) ? 1 : ((b0 >= 0) ? 0 : 3));   // :737-778
    const int ent_r1 = (numer_1 <= 0) ? 2 : ((numer_1 >= denom) ? 1 : 4);                                               // :783-808
    // The compiler places the branches of what follows.  Forcing it straight-line (every lane pays the division and the quadratic form),
    // or into one guarded block for the division and one for the quadratic form, was measured slower.
    int ent = lower ? (sneg ? (tneg ? ent_r4 : chain_b1) : (tneg ? chain_b0 : 6))
                    : (sneg ? ent_r2 : (tneg ? ent_r6 : ent_r1));
    const bool region6 = !lower && !sneg && tneg;
    const double numer = sneg ? numer_2 : (tneg ? numer_6 : numer_1);  // only read when ent == 4 (upper regions)

    // ---- one division for the three edge outcomes
    double num = (ent == 3) ? -b0 : ((ent == 5) ? -b1 : ((ent == 4) ? numer : 0.0));
    double den = (ent == 3) ? a00 : ((ent == 5) ? a11 : ((ent == 4) ? denom : 1.0));
    double q = num / den;
    // ---- (s, t) of the nearest point
    const double sF = s0 * inv_det, tF = t0 * inv_det;                 // :675-677 (read when ent == 6)
    const double omq = 1 - q;                                          // :705, :752, :804 (read when ent == 4)
    double s = (ent == 6) ? sF : ((ent == 4) ? (region6 ? omq : q) : ((ent == 1) ? 1.0 : ((ent == 3) ? q : 0.0)));
    double t = (ent == 6) ? tF : ((ent == 4) ? (region6 ? q : omq) : ((ent == 2) ? 1.0 : ((ent == 5) ? q : 0.0)));
    // ---- d2
    double quad = s * (a00 * s + a01 * t + 2 * b0) + t * (a01 * s + a11 * t + 2 * b1) + c;   // :678, :706, :753, :805
    double dv1 = a00 + 2 * b0 + c, dv2 = a11 + 2 * b1 + c;            // :594, :616
    double de1 = b0 * q + c, de2 = b1 * q + c;                         // :600, :622
    double d2 = (ent == 6 || ent == 4) ? quad : ((ent == 0) ? c : ((ent == 1) ? dv1 : ((ent == 2) ? dv2 : ((ent == 3) ? de1 : de2))));
    if (d2 < 0) d2 = 0;                                                // :812-816
    s_out = s; t_out = t; ent_out = ent;
    return d2;
}

// nearest_point (TriangleMeshDistance.h:818) and the pseudonormal sign (:274-305)
__device__ __forceinline__ void finish_query(const LeafRecord* __restrict__ leaves, const PseudoNormals* __restrict__ normals,
                                             const QueryResult& r, double px, double py, double pz, bool is_signed,
                                             double& dist, double& qx, double& qy, double& qz, int& tri_id)
{
    if (r.pos < 0) {            // nothing accepted (NaN input); the reference would index triangles[-1]
        dist = r.dist; qx = qy = qz = 0.0; tri_id = -1;
        return;
    }
    const double* rec = reinterpret_cast<const double*>(leaves + r.pos);
    const double v0x = __ldg(rec + 0), v0y = __ldg(rec + 1), v0z = __ldg(rec + 2);
    const double e0x = __ldg(rec + 3), e0y = __ldg(rec + 4), e0z = __ldg(rec + 5);
    const double e1x = __ldg(rec + 6), e1y = __ldg(rec + 7), e1z = __ldg(rec + 8);
    tri_id = __ldg(&leaves[r.pos].tri_id);
    qx = v0x + r.s * e0x + r.t * e1x;                  // v0 + s*edge0 + t*edge1
    qy = v0y + r.s * e0y + r.t * e1y;
    qz = v0z + r.s * e0z + r.t * e1z;
    dist = r.dist;
    if (is_signed) {
        const double* n = normals[r.pos].n[r.entity];
        const double nx = __ldg(n), ny = __ldg(n + 1), nz = __ldg(n + 2);
        const double ux = px - qx, uy = py - qy, uz = pz - qz;
        const double d = ux * nx + uy * ny + uz * nz;
        dist = dist * ((d >= 0.0) ? 1.0 : -1.0);       // :305
    }
}

// Stack entry = 8 bytes: the sibling's sphere distance rounded to fp32 + its leaf range packed in 32 bits.  A node at depth k
// covers either floor(T/2^k) or that + 1 leaves (halving splits), so (begin, depth, +1 flag) identifies the range; bit 31
// says whether the entry is its parent's LEFT child (needed to find its fp64 sphere again when the fp32 value cannot decide).
__device__ __forceinline__ unsigned pack_range(int b, int e, int depth, int n_tri, bool is_left)
{
    return (unsigned)b | ((unsigned)depth << 25) | ((unsigned)((e - b) - (n_tri >> depth)) << 30) | ((unsigned)is_left << 31);
}

// fp64 sphere distance exactly as the reference computes it (TriangleMeshDistance.h:539-540)
__device__ __forceinline__ double sphere_dist(double px, double py, double pz, double cx, double cy, double cz, double r)
{
    const double x = px - cx, y = py - cy, z = pz - cz;
    return sqrt(x * x + y * y + z * z) - r;
}

// ---------------------------------------------------------------------------------------------------------------
// FP32 INTERVAL FILTER.  The traversal only needs the sphere distances for three yes/no questions:
// which child is nearer (:542), is a child nearer than the best so far (:545-557).  Both are decided from an fp32 shadow
// of the spheres whenever the fp32 interval [d_f - E, d_f + E] -- which provably contains the reference's fp64 value -- lies
// entirely on one side; otherwise (ties, near-ties: a few per thousand) the lane recomputes that node in fp64 exactly as the
// reference does.  The decision taken is therefore ALWAYS the reference's decision, and every number that reaches the
// output (best, d2, s, t) is still computed in fp64 in the leaf test: results stay bit-identical.
//   Error bound.  Coordinates are taken relative to the mesh centre and rounded to fp32: |err| <= 2^-24 Mq per coordinate,
//   Mq = max(mesh half extent, |p - ctr|_inf).  With D = |p - c| <= 2 sqrt(3) Mq and r <= 2 sqrt(3) Mq the fp32 value of
//   sqrt(dx^2+dy^2+dz^2) - r differs from the real one by < 2^-24 (sqrt(3) 2 Mq + 8 D + r) < 35 * 2^-24 Mq (sqrt.approx: 2 ulp);
//   the reference's own fp64 rounding adds < 1e-15 Mq.  E = 64 * 2^-24 * Mq.
//   Range.  The relative bound above assumes normal fp32 numbers.  Below them the errors are absolute: a square under 2^-126 is subnormal
//   (off by up to 2^-149, its root by up to 2^-74.5), and sqrt.approx.ftz reads it as 0, so a distance below 2^-63 comes out as 0.
//   The spare (64 - 35) 2^-24 Mq of E covers both once Mq >= 2^-40 (a factor 14 over 2^-63).  Above, squares of lengths 1e18+ overflow.
//   So the budget holds for 2^-40 <= Mq < 1e18; outside that range E = +inf (filter_slack): every fp32 test is undecided and every
//   decision is made in fp64, exactly as the reference makes it (the packet walk hands such a lane to the per-lane walk).
// The fp64 chains (two IEEE square roots per node, ~10 cycles per dependent instruction) were the critical path of the kernel.
// ---------------------------------------------------------------------------------------------------------------
// E for a query with Mq = max(half extent, |q - ctr|_inf) in fp32: 64 * 2^-24 * Mq rounded up where the budget holds, else +inf.  (A NaN
// query does not reach Mq -- fmaxf drops NaN -- and is caught by the callers.)
__device__ __forceinline__ float filter_slack(float Mq)
{
    return (Mq >= 9.094947017729282379e-13f /* 2^-40 */ && Mq < 1.0e18f) ? __fmul_ru(Mq, 3.814697265625e-06f) : __int_as_float(0x7f800000);
}

struct MeshDev {
    const SpherePair* spheres;
    const float4* nodes_f;                 // [T][K1_NODEF_STRIDE]: sphere pair (2 float4) + box pair (3 float4)
    const LeafF* leaves_f;                 // [T] fp32 triangle shadows
    const LeafRecord* leaves;
    double cx, cy, cz;
    float half_extent;
    int n_tri;
};

__device__ __forceinline__ float sqrt_approx(float x)
{
#ifdef DG_EMU
    return dg_emu_ftz(std::sqrt(dg_emu_ftz(x)));     // the flush of .ftz (the 2-ulp error of .approx is not modelled: the budget covers it)
#else
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#endif
}


// LEAF BOUND of the packet walk: certified fp32 LOWER bound of the distance from the query to a triangle.
//   * distance to each of the three closed edges (clamped parameter => an actual point of the edge, so each value is an upper
//     bound of that edge's true distance up to rounding; their minimum is the true distance whenever the closest point is on the
//     boundary, i.e. whenever the projection of the query falls outside the triangle);
//   * distance to the supporting plane (<= the true distance always);
//   * the projection is declared "outside" only if one edge function is negative beyond a tolerance that covers the fp32 rounding
//     of the products and the 2^-24-relative perturbation of every coordinate (so: classified outside => truly outside).
//   bound = outside ? min(edge distances) : min(plane distance, edge distances), minus 4E for the fp32 evaluation itself.
// Range: the bound is valid wherever E is finite (2^-40 <= Mq < 1e18, filter_slack).  The shadow's normal is a unit vector, so (w.n)^2 is a
// squared distance (< 1e38), never inf or NaN: with plane2 = inf, min(inf, mseg) = mseg would NOT be a lower bound when the projection falls
// inside.  |e|^2 < 1.2e37 stays below the 2^126 where __fdividef returns 0.  Products of the outside test that overflow make tol = inf (never
// "outside"); products that go subnormal lose their relative error bound, and the 2^-146 floor of tol covers them (meshes of size ~1e-11
// need it).  A zero normal (zero area) gives plane2 = 0: no plane bound.
// The caller rejects the leaf only if bound > best_hi + 2E (same slack accounting as the box skip).  On bunny/dragon this rejects
// 83-90 % of the leaf tests; the rest (accepted ones, ties, near misses) take the exact fp64 test.  Prototype with 0 invalid
// rejections in 3 M leaf tests: see DESIGN.md.  The per-lane walk does not use it: there, as a phase of its own, it cost more
// iterations than the fp64 tests it saved.
__device__ __forceinline__ float dot3f(float ax, float ay, float az, float bx, float by, float bz) { return fmaf(az, bz, fmaf(ay, by, ax * bx)); }

__device__ __forceinline__ float leaf_lower_bound(const LeafF* __restrict__ rec, float qx, float qy, float qz, float E)
{
    const float4* r4 = reinterpret_cast<const float4*>(rec);
    const float4 a = __ldg(r4), b = __ldg(r4 + 1), c = __ldg(r4 + 2), d = __ldg(r4 + 3);
    // a = v0.xyz e0.x | b = e0.yz e1.xy | c = e1.z d00 d01 d11 | d = d22 n.xyz
    const float e0x = a.w, e0y = b.x, e0z = b.y, e1x = b.z, e1y = b.w, e1z = c.x;
    const float d00 = c.y, d01 = c.z, d11 = c.w, d22 = d.x;
    const float wx = qx - a.x, wy = qy - a.y, wz = qz - a.z;                       // w = q - v0
    const float w0 = dot3f(wx, wy, wz, e0x, e0y, e0z), w1 = dot3f(wx, wy, wz, e1x, e1y, e1z);
    // edge 01: v0 + t e0
    float t = (d00 > 0.f) ? __fdividef(w0, d00) : 0.f; t = fminf(fmaxf(t, 0.f), 1.f);
    float rx = wx - t * e0x, ry = wy - t * e0y, rz = wz - t * e0z;
    float mseg = dot3f(rx, ry, rz, rx, ry, rz);
    // edge 02: v0 + t e1
    t = (d11 > 0.f) ? __fdividef(w1, d11) : 0.f; t = fminf(fmaxf(t, 0.f), 1.f);
    rx = wx - t * e1x; ry = wy - t * e1y; rz = wz - t * e1z;
    mseg = fminf(mseg, dot3f(rx, ry, rz, rx, ry, rz));
    // edge 12: v1 + t (e1 - e0), w' = w - e0
    const float e2x = e1x - e0x, e2y = e1y - e0y, e2z = e1z - e0z;
    const float ux = wx - e0x, uy = wy - e0y, uz = wz - e0z;
    const float u2 = dot3f(ux, uy, uz, e2x, e2y, e2z);
    t = (d22 > 0.f) ? __fdividef(u2, d22) : 0.f; t = fminf(fmaxf(t, 0.f), 1.f);
    rx = ux - t * e2x; ry = uy - t * e2y; rz = uz - t * e2z;
    mseg = fminf(mseg, dot3f(rx, ry, rz, rx, ry, rz));
    // plane (n is a unit normal, or 0: no plane bound)
    const float nn = dot3f(d.y, d.z, d.w, d.y, d.z, d.w), wn = dot3f(wx, wy, wz, d.y, d.z, d.w);
    const float plane2 = (nn > 0.f) ? __fdividef(wn * wn, nn) : 0.f;
    // is the projection certainly outside the triangle?
    const float p1 = d11 * w0, p2 = d01 * w1, p3 = d00 * w1, p4 = d01 * w0, p5 = d00 * d11, p6 = d01 * d01;
    const float numv = p1 - p2, numu = p3 - p4, den = p5 - p6;
    const float S = d00 + d11, W = sqrt_approx(dot3f(wx, wy, wz, wx, wy, wz));
    const float tol = 32.f * (1.2e-7f * (fabsf(p1) + fabsf(p2) + fabsf(p3) + fabsf(p4) + p5 + p6) + 0.25f * E * S * (W + sqrt_approx(S)))
                    + 1.1210387714598537e-44f;                                   // 2^-146: 16 half-ulps of the subnormal products
    const bool outside = (numv < -tol) || (numu < -tol) || (den - numu - numv < -tol);
    const float lb2 = outside ? mseg : fminf(plane2, mseg);
    return sqrt_approx(fmaxf(lb2, 0.f)) - 4.f * E;      // NaN (degenerate input) compares false in the caller: no rejection
}

// _query (TriangleMeshDistance.h:514-562), iterative and WARP-SYNCHRONOUS.
//
// All 32 lanes of a warp call this together, each with its own query (`alive`).  Every lane walks the tree in the
// reference's own order with its own stack of deferred siblings, but the warp executes ONE PHASE per iteration, chosen
// by ballot so that each straight-line block runs converged:
//   NODE : lanes at an internal node: two sphere tests, then descend + defer the sibling, or prune
//   LEAF : lanes at a leaf: point-triangle test, accept if strictly closer
//   POP  : lanes that pruned / finished a leaf: re-test deferred siblings (`d < result.distance`, :549/:557)
// The phase holding the largest cost-weighted share of lanes runs; the other lanes idle for that iteration.  All lanes
// start at the root together and -- being 32 adjacent grid nodes -- take mostly the same decisions, so the phases stay
// largely aligned.  (Letting a finished lane start its next query immediately was tried and is ~1.6x SLOWER: lanes
// then sit at unrelated depths of the tree and both phase alignment and cache sharing are lost.)
// Stack layout [depth][lane] in shared memory: conflict-free whatever depth each lane is at.
__device__ __forceinline__ QueryResult nearest_triangle(const MeshDev& M, bool alive, double px, double py, double pz,
                                                        unsigned* stack_rng, float* stack_d, int stride)
{
    enum { NODE = 0, LEAF = 1, POP = 2, DONE = 3 };
    const int n_tri = M.n_tri;
    QueryResult res;
    res.dist = DBL_MAX; res.s = 0; res.t = 0; res.pos = -1; res.entity = 0;
    double best = DBL_MAX;             // result.distance
    double best_sq = best * best;      // result.distance * result.distance (= +inf initially), :528
    float best_lo = __double2float_rd(best), best_hi = __double2float_ru(best);   // fp32 bracket of best
    // query point relative to the mesh centre, in fp32, and the interval half-width for this query
    const float qx = (float)(px - M.cx), qy = (float)(py - M.cy), qz = (float)(pz - M.cz);
    const float Mq = fmaxf(fmaxf(M.half_extent, fabsf(qx)), fmaxf(fabsf(qy), fabsf(qz)));
    // outside the budget's range (below 2^-40 or beyond ~1e18) the filter is off for this query: E = inf leaves every test undecided
    const float E = filter_slack(Mq);
    const float E2 = E + E;
    // BOX SKIP.  A subtree may be skipped when visiting it provably changes nothing: no triangle in it can be
    // accepted, i.e. every d2 the reference would compute there is >= best_sq.  With L = (fp32 distance to the subtree's
    // outward-rounded box) - E <= true distance to every triangle, the reference's d2 >= L^2 - 240 eps64 R^2 (fp64 rounding of
    // its formula, R <= 7 Mq) and best_sq <= best^2 (1 + 2^-53): both slacks are below E * best once best >= 1e-6 Mq, so
    // "box distance > best_hi + 2E" suffices; for queries practically on the surface (best < 1e-6 Mq) nothing is skipped.
    // The running best only shrinks, so a subtree found hopeless stays hopeless and its deferred re-test can be dropped too.
    const float tiny_best = 1.0e-6f * Mq;
    float skip_sq = __int_as_float(0x7f800000);              // (best_hi + 2E)^2 rounded up; +inf = never skip
    int b = 0, e = n_tri, depth = 0, sp = 0;
    int state = alive ? ((n_tri == 1) ? LEAF : NODE) : DONE;
    for (;;) {
        // one warp-wide integer sum carries the three lane counts (8 bits each: NODE | LEAF << 8 | POP << 16; DONE adds nothing), which
        // costs less than ballots and popcounts: the loop head is ~19 % of the issued instructions
        const unsigned tally = __reduce_add_sync(0xffffffffu, (state < DONE) ? (1u << (8 * state)) : 0u);
        if (tally == 0u) break;                                                // every lane DONE
        const int w_node = K1_NODE_WEIGHT * (int)(tally & 0xffu), w_pop = K1_POP_WEIGHT * (int)(tally >> 16);
        const int w_leaf = K1_LEAF_WEIGHT * (int)((tally >> 8) & 0xffu);
        // (max with 0 changes no value, but without it the loop head compiles to other instructions than the timed ones)
        const int w_max = max(max(w_node, w_pop), max(0, w_leaf));
        DG_EMU_COUNT(0);
        if (w_pop == w_max) {
            if (state == POP) {
                // deferred siblings: the reference's second `if (d < result.distance)` (:549, :557) with the updated best
#pragma unroll 1
                for (int attempt = 0; attempt < K1_POP_TRIES; attempt++) {
                    if (sp == 0) { state = DONE; break; }
                    sp--;
                    DG_EMU_COUNT(5);
                    const float df = stack_d[sp * stride];
                    bool visit = (df + E < best_lo);                           // certainly d < best
                    const bool skip = (df - E >= best_hi);                     // certainly d >= best
                    if (!(visit || skip)) {                                    // undecided in fp32: the reference's fp64 value
                        DG_EMU_COUNT(6);
                        const unsigned r = stack_rng[sp * stride];
                        const int rb = (int)(r & 0x01ffffffu), rd = (int)((r >> 25) & 31u);
                        const int re = rb + (n_tri >> rd) + (int)((r >> 30) & 1u);
                        const bool is_left = (r >> 31) != 0u;
                        const double* s8 = reinterpret_cast<const double*>(M.spheres + (is_left ? re : rb)) + (is_left ? 0 : 4);
                        const double2 c0 = ldg2(s8), c1 = ldg2(s8 + 2);
                        visit = sphere_dist(px, py, pz, c0.x, c0.y, c1.x, c1.y) < best;
                    }
                    if (visit) {
                        const unsigned r = stack_rng[sp * stride];
                        const int rb = (int)(r & 0x01ffffffu), rd = (int)((r >> 25) & 31u);
                        const int re = rb + (n_tri >> rd) + (int)((r >> 30) & 1u);
                        {   // the best has usually shrunk since this sibling was deferred: box test against the current best
                            // the child's box sits in two of the record's three box quads (l_lo.xyz l_hi.x | l_hi.yz r_lo.xy | r_lo.z r_hi.xyz): two
                            // 16-byte loads instead of six scalar ones (fewer L1 tag requests)
                            const bool is_left = (r >> 31) != 0u;
                            const float4* bq = M.nodes_f + (size_t)(is_left ? re : rb) * K1_NODEF_STRIDE + (is_left ? 2 : 3);
                            const float4 u = __ldg(bq), v = __ldg(bq + 1);
                            const float lox = is_left ? u.x : u.z, loy = is_left ? u.y : u.w, loz = is_left ? u.z : v.x;
                            const float hix = is_left ? u.w : v.y, hiy = is_left ? v.x : v.z, hiz = is_left ? v.y : v.w;
                            const float gx = fmaxf(fmaxf(lox - qx, qx - hix), 0.f), gy = fmaxf(fmaxf(loy - qy, qy - hiy), 0.f), gz = fmaxf(fmaxf(loz - qz, qz - hiz), 0.f);
                            if (__fmaf_rd(gz, gz, __fmaf_rd(gy, gy, __fmul_rd(gx, gx))) > skip_sq) { DG_EMU_COUNT(7); continue; }   // visiting it could not change anything
                        }
                        b = rb; depth = rd; e = re;
                        state = (e - b == 1) ? LEAF : NODE;
                        break;
                    }
                }
            }
        } else if (w_node == w_max) {
            if (state == NODE) {                                                // internal (:537-561)
                DG_EMU_COUNT(1);
                const int m = (b + e) >> 1;
                bool left_first, go_first, go_second = false, defer = true;
                float d_second_f;
                bool decided = false;
                {
                    const float4* f4 = M.nodes_f + (size_t)m * K1_NODEF_STRIDE;
                    const float4 l4 = __ldg(f4), r4 = __ldg(f4 + 1);
                    // the box loads go out with the sphere loads (latency), not after the sphere decision that may need them
                    const float4 b0 = __ldg(f4 + 2), b1 = __ldg(f4 + 3), b2 = __ldg(f4 + 4);   // l_lo.xyz l_hi.x | l_hi.yz r_lo.xy | r_lo.z r_hi.xyz
                    const float lx = qx - l4.x, ly = qy - l4.y, lz = qz - l4.z;
                    const float rx = qx - r4.x, ry = qy - r4.y, rz = qz - r4.z;
                    const float dl = sqrt_approx(fmaf(lz, lz, fmaf(ly, ly, lx * lx))) - l4.w;
                    const float dr = sqrt_approx(fmaf(rz, rz, fmaf(ry, ry, rx * rx))) - r4.w;
                    left_first = dl < dr;
                    const float d_first_f = left_first ? dl : dr;
                    d_second_f = left_first ? dr : dl;
                    const bool order_sure = (d_first_f + E2 < d_second_f);      // |dl - dr| > 2E
                    go_first = (d_first_f + E < best_lo);                       // certainly d_first < best
                    const bool skip_first = (d_first_f - E >= best_hi);         // certainly d_first >= best (then d_second >= best too)
                    decided = order_sure && (go_first || skip_first);
                    // a sibling that is already certainly not nearer than the best can never pass its re-test (best only
                    // shrinks): the reference would pop it and skip it (:549/:557), so it is not stacked at all
                    defer = !(d_second_f - E >= best_hi);
                    if (decided && go_first) {
                        const float lgx = fmaxf(fmaxf(b0.x - qx, qx - b0.w), 0.f), lgy = fmaxf(fmaxf(b0.y - qy, qy - b1.x), 0.f),
                                    lgz = fmaxf(fmaxf(b0.z - qz, qz - b1.y), 0.f);
                        const float rgx = fmaxf(fmaxf(b1.z - qx, qx - b2.y), 0.f), rgy = fmaxf(fmaxf(b1.w - qy, qy - b2.z), 0.f),
                                    rgz = fmaxf(fmaxf(b2.x - qz, qz - b2.w), 0.f);
                        // squared box distances rounded DOWN (a smaller value only skips less)
                        const float l2 = __fmaf_rd(lgz, lgz, __fmaf_rd(lgy, lgy, __fmul_rd(lgx, lgx)));
                        const float r2 = __fmaf_rd(rgz, rgz, __fmaf_rd(rgy, rgy, __fmul_rd(rgx, rgx)));
                        const bool hopeless_first = (left_first ? l2 : r2) > skip_sq;
                        const bool hopeless_second = (left_first ? r2 : l2) > skip_sq;
                        if (hopeless_second) defer = false;
                        if (hopeless_first) {
                            // the first child would be visited without effect; what the reference does next is the re-test of the second
                            const bool second_yes = (d_second_f + E < best_lo), second_no = (d_second_f - E >= best_hi);
                            if (second_yes || second_no) {
                                go_first = false;
                                go_second = second_yes && !hopeless_second;
                            }                                   // undecided re-test: simply do not use the shortcut
                        }
                    }
                }
                if (!decided) {                                                 // fp64, exactly the reference
                    DG_EMU_COUNT(2);
                    const double* sp8 = reinterpret_cast<const double*>(M.spheres + m);
                    const double2 a0 = ldg2(sp8), a1 = ldg2(sp8 + 2), a2 = ldg2(sp8 + 4), a3 = ldg2(sp8 + 6);
                    const double d_left = sphere_dist(px, py, pz, a0.x, a0.y, a1.x, a1.y);      // :539
                    const double d_right = sphere_dist(px, py, pz, a2.x, a2.y, a3.x, a3.y);     // :540
                    left_first = d_left < d_right;                                            // :542
                    const double d_first = left_first ? d_left : d_right;
                    const double d_second = left_first ? d_right : d_left;
                    go_first = d_first < best;                                                // :545 / :554
                    go_second = !go_first && (d_second < best);     // only reachable through NaNs; kept for fidelity (:549 / :557)
                    d_second_f = (float)d_second;                   // |rounding| <= 2^-24 |d| << E: the stored value stays a valid filter input
                    defer = (d_second < best);
                }
                depth++;
                if (go_first) {                        // visit first now; second is re-tested when popped (:545-551)
                    if (defer) {
                        DG_EMU_COUNT(9);
                        stack_rng[sp * stride] = left_first ? pack_range(m, e, depth, n_tri, false) : pack_range(b, m, depth, n_tri, true);
                        stack_d[sp * stride] = d_second_f;
                        sp++;
                    }
                    if (left_first) e = m; else b = m;
                    state = (e - b == 1) ? LEAF : NODE;
                } else if (go_second) {
                    if (left_first) b = m; else e = m;
                    state = (e - b == 1) ? LEAF : NODE;
                } else {
                    state = POP;
                }
            }
        } else {
            if (state == LEAF) {                                                // leaf (:517-534)
                double s, t; int ent;
                DG_EMU_COUNT(3);
                const double d2 = tri_dist2(M.leaves + b, px, py, pz, s, t, ent);
                if (d2 < best_sq) {
                    DG_EMU_COUNT(4);
                    best = sqrt(d2);
                    best_sq = best * best;
                    best_lo = __double2float_rd(best); best_hi = __double2float_ru(best);
                    { const float th = __fadd_ru(best_hi, E2); skip_sq = (best_lo >= tiny_best) ? __fmul_ru(th, th) : __int_as_float(0x7f800000); }
                    res.s = s; res.t = t; res.pos = b; res.entity = ent;
                }
                state = POP;
            }
        }
    }
    res.dist = best;
    return res;
}

#if K1_PACKET
// =====================================================================================================================================
// PACKET TRAVERSAL (K1_PACKET): the 32 queries of a brick walk the tree TOGETHER -- one node per step for all lanes, one shared order
// (majority of the lanes that still want the node), one stack -- and the reference's ORDER-DEPENDENT result is reconstructed afterwards.
//
// Why this is admissible although _query's result depends on each query's own visit order (file header): the order only matters among the
// handful of triangles whose d2 lies within a few ulps of the minimum.  Write v_T for the d2 the reference computes for triangle T (a pure
// function of T and the query: tri_dist2), D(v) = fl(sqrt(v)), g(v) = fl(D(v) * D(v)).  The reference accepts T in state v' iff v_T < g(v')
// (:528) and g(v') lies in [v'(1 - 3 eps), v'(1 + 3 eps)].  Let m be the smallest v_T over ALL triangles and C the closure of {m} under
// "x <= c (1 + 2^-49) for some c in C" (a chain of values a few ulps apart).  If every other triangle has v > cmax (1 + 2^-49), then
//   (i)  a state outside C accepts every member of C (g(v') > cmax), a state inside C never accepts anything outside C, so the reference's
//        final state is the fold of C's members alone, in the reference's order, the first of them accepted unconditionally;
//   (ii) the reference does visit every member T of C provided none of T's ancestors n fails `d_n < result.distance` (:545-557) for the
//        smallest state that can ever occur, D(m): certified here by  max over ancestors (fp32 sphere distance + E)  <  best_lo;
//   (iii) the reference's order of two visited leaves is decided at their lowest common ancestor by `d_left < d_right` (:542), evaluated
//        here in fp64 exactly as the reference does (ref_visits_first).
// So the packet walk only has to (a) evaluate, with the reference's own fp64 leaf test, every triangle whose v could be <= m (1 + 1e-6)
// -- subtrees and leaves are dropped only by the CERTIFIED fp32 bounds of the box skip (true distance > best_hi + 2E  =>  v > m (1 + 2e-6),
// error budget at BOX SKIP above) -- (b) keep the K1_PKT_K smallest values near the minimum with their leaf position, the largest ancestor
// certificate of any of them, and the smallest value it did not keep, (c) form C, check (i) and (ii), order C by (iii) and replay the reference's
// accept rule.  A lane for which any check fails (on-surface queries below tiny_best, more than K1_PKT_K near-ties, a sphere that is tight
// to within E, non-finite input) is walked again by nearest_triangle() -- the per-lane reference-order traversal above -- so the result is
// the reference's in every case; the checks decide only how fast it is obtained.
// =====================================================================================================================================
#ifndef K1_PKT_K
#define K1_PKT_K 8
#endif
#ifdef DG_EMU
#define DG_NOINLINE
#else
#define DG_NOINLINE __noinline__
#endif

// does the reference reach leaf position pa before leaf position pb (pa != pb, both visited)?
__device__ DG_NOINLINE bool ref_visits_first(const SpherePair* __restrict__ spheres, int n_tri, int pa, int pb, double px, double py, double pz)
{
    int b = 0, e = n_tri;
    for (;;) {
        const int m = (b + e) >> 1;
        const bool al = pa < m, bl = pb < m;
        if (al != bl) {
            const double* sp8 = reinterpret_cast<const double*>(spheres + m);
            const double2 a0 = ldg2(sp8), a1 = ldg2(sp8 + 2), a2 = ldg2(sp8 + 4), a3 = ldg2(sp8 + 6);
            const double d_left = sphere_dist(px, py, pz, a0.x, a0.y, a1.x, a1.y);      // :539
            const double d_right = sphere_dist(px, py, pz, a2.x, a2.y, a3.x, a3.y);     // :540
            return al == (d_left < d_right);                                            // :542
        }
        if (al) e = m; else b = m;
    }
}

__device__ __forceinline__ QueryResult nearest_triangle_packet(const MeshDev& M, bool alive, double px, double py, double pz,
                                                               unsigned* wstack, unsigned* stack_rng, float* stack_pm, float* stack_key, double* cv, int* cpos, int stride)
{
    const unsigned FULL = 0xffffffffu;
    const int n_tri = M.n_tri;
    const float INF = __int_as_float(0x7f800000);
    const double DINF = (double)INF;
    QueryResult res;
    res.dist = DBL_MAX; res.s = 0; res.t = 0; res.pos = -1; res.entity = 0;
    const float qx = (float)(px - M.cx), qy = (float)(py - M.cy), qz = (float)(pz - M.cz);
    const float Mq = fmaxf(fmaxf(M.half_extent, fabsf(qx)), fmaxf(fabsf(qy), fabsf(qz)));
    const float E = filter_slack(Mq), E2 = E + E;      // as in nearest_triangle
    const float tiny_best = 1.0e-6f * Mq;
    bool need_fb = false;
    bool act = alive;                                   // lane still takes part in the shared walk
    // no certified pruning outside the budget's range (E = inf) or for NaN input: the per-lane walk decides everything in fp64
    if (alive && (!(E < INF) || !(qx == qx) || !(qy == qy) || !(qz == qz) || n_tri < 2)) { need_fb = true; act = false; }
    float skip_lin = INF, skip_sq = INF, best_lo = INF;
    double dropped = DINF;                              // smallest evaluated value that is NOT in the list
    int cnt = 0;                                        // list: cv[0] <= cv[1] <= ... (stride apart), all within 1e-6 of the minimum when inserted
    float pm_list = -INF;                               // max of the ancestor certificates (pm) of the entries inserted since the list last restarted
    float pm = -INF;                                    // max over the ancestors on the current path of (fp32 sphere distance + E)
    int b = 0, e = n_tri, depth = 0, sp = 0;            // warp-uniform
    bool have = true;
    for (;;) {
        if (!have) {
            if (sp == 0) break;
            sp--;
            DG_EMU_COUNT(16);
            // the deferred child's certified lower bound was stored per lane when it was pushed; only the running best has moved since
            const bool want = act && !(stack_key[sp * stride] > skip_lin);
            if (!__any_sync(FULL, want)) continue;
            DG_EMU_COUNT(17);
            const unsigned r = wstack[sp];                   // one copy per warp: every lane stored the same word
            const int rb = (int)(r & 0x01ffffffu), rd = (int)((r >> 25) & 31u);
            b = rb; e = rb + (n_tri >> rd) + (int)((r >> 30) & 1u); depth = rd; pm = stack_pm[sp * stride];
            have = true;
        }
        if (e - b == 1) {
            // ---- leaf: certified fp32 lower bound for all lanes, the reference's fp64 test for the lanes it cannot rule out
            DG_EMU_COUNT(18);
            const float lb = leaf_lower_bound(M.leaves_f + b, qx, qy, qz, E);
            const bool pass = act && !(lb > skip_lin);
            if (__any_sync(FULL, pass)) {
                DG_EMU_COUNT(19);
                if (pass) {
                    DG_EMU_COUNT(20);
                    double s, t; int ent;
                    const double x = tri_dist2(M.leaves + b, px, py, pz, s, t, ent);
                    const double v0 = cnt ? cv[0] : DINF;
                    bool insert = false;
                    if (x < v0) {
                        if (!(v0 <= x + x * 1e-6)) {                    // clear improvement (or empty list): the list restarts
                            dropped = fmin(dropped, v0);
                            cnt = 1; cv[0] = x; cpos[0] = b; pm_list = pm;
                        } else insert = true;
                        const double best = sqrt(x);
                        best_lo = __double2float_rd(best);
                        const float th = __fadd_ru(__double2float_ru(best), E2);
                        if (best_lo >= tiny_best) { skip_lin = th; skip_sq = __fmul_ru(th, th); }
                        else { need_fb = true; act = false; DG_EMU_COUNT(15); }           // practically on the surface: no certified pruning possible
                    } else if (x <= v0 + v0 * 1e-6) insert = true;
                    else dropped = fmin(dropped, x);                    // NaN falls through: never accepted by the reference either
                    if (insert) {
                        int i = cnt;
                        bool room = true;
                        if (cnt == K1_PKT_K) {
                            const double last = cv[(K1_PKT_K - 1) * stride];
                            if (x < last) { dropped = fmin(dropped, last); i = K1_PKT_K - 1; }
                            else { dropped = fmin(dropped, x); room = false; }
                        } else cnt++;
                        if (room) {
                            while (i > 0 && x < cv[(i - 1) * stride]) {
                                cv[i * stride] = cv[(i - 1) * stride]; cpos[i * stride] = cpos[(i - 1) * stride];
                                i--;
                            }
                            cv[i * stride] = x; cpos[i * stride] = b; pm_list = fmaxf(pm_list, pm);
                        }
                    }
                }
            }
            have = false;
            continue;
        }
        // ---- internal node: both children's certified bounds for all lanes
        DG_EMU_COUNT(21);
        const int m = (b + e) >> 1;
        const float4* f4 = M.nodes_f + (size_t)m * K1_NODEF_STRIDE;
        const float4 l4 = __ldg(f4), r4 = __ldg(f4 + 1);
        const float4 b0 = __ldg(f4 + 2), b1 = __ldg(f4 + 3), b2 = __ldg(f4 + 4);   // l_lo.xyz l_hi.x | l_hi.yz r_lo.xy | r_lo.z r_hi.xyz
        const float lx = qx - l4.x, ly = qy - l4.y, lz = qz - l4.z;
        const float rx = qx - r4.x, ry = qy - r4.y, rz = qz - r4.z;
        const float dl = sqrt_approx(fmaf(lz, lz, fmaf(ly, ly, lx * lx))) - l4.w;
        const float dr = sqrt_approx(fmaf(rz, rz, fmaf(ry, ry, rx * rx))) - r4.w;
        const float lgx = fmaxf(fmaxf(b0.x - qx, qx - b0.w), 0.f), lgy = fmaxf(fmaxf(b0.y - qy, qy - b1.x), 0.f), lgz = fmaxf(fmaxf(b0.z - qz, qz - b1.y), 0.f);
        const float rgx = fmaxf(fmaxf(b1.z - qx, qx - b2.y), 0.f), rgy = fmaxf(fmaxf(b1.w - qy, qy - b2.z), 0.f), rgz = fmaxf(fmaxf(b2.x - qz, qz - b2.w), 0.f);
        const float l2 = __fmaf_rd(lgz, lgz, __fmaf_rd(lgy, lgy, __fmul_rd(lgx, lgx)));
        const float r2 = __fmaf_rd(rgz, rgz, __fmaf_rd(rgy, rgy, __fmul_rd(rgx, rgx)));
        const bool wl = act && !(dl - E > skip_lin) && !(l2 > skip_sq);
        const bool wr = act && !(dr - E > skip_lin) && !(r2 > skip_sq);
        const unsigned ml = __ballot_sync(FULL, wl), mr = __ballot_sync(FULL, wr);
        if ((ml | mr) == 0u) { have = false; continue; }
        const unsigned pl = __ballot_sync(FULL, (wl || wr) && (dl < dr));
        const bool left_first = 2 * __popc(pl) >= __popc(ml | mr);
        depth++;
        const unsigned m1 = left_first ? ml : mr, m2 = left_first ? mr : ml;
        const float d1u = __fadd_ru(left_first ? dl : dr, E), d2u = __fadd_ru(left_first ? dr : dl, E);
        if (m1) {
            if (m2) {
                wstack[sp] = left_first ? pack_range(m, e, depth, n_tri, false) : pack_range(b, m, depth, n_tri, true);
                stack_pm[sp * stride] = fmaxf(pm, d2u);
                // lower bound of the true distance to anything in the deferred child: sphere (fp32 value - E) or box (sqrt.approx is within
                // 2 ulp: scaled down by 1 - 2^-21 it is a lower bound of the root of the squared box distance, itself rounded down)
                stack_key[sp * stride] = fmaxf((left_first ? dr : dl) - E, __fmul_rd(sqrt_approx(left_first ? r2 : l2), 0.99999952f));
                sp++;
            }
            pm = fmaxf(pm, d1u);
            if (left_first) e = m; else b = m;
        } else {
            pm = fmaxf(pm, d2u);
            if (left_first) b = m; else e = m;
        }
    }
    // ---- the closure C of the minimum, the checks (i) (ii), the reference's order (iii) and its accept rule
    bool ok = alive && !need_fb;
    if (ok && cnt == 0) { need_fb = true; ok = false; }
    int win = -1; double D = DBL_MAX;
    int ncmp = 0; (void)ncmp;
    if (ok) {
        const double EPSC = 1.7763568394002505e-15;     // 2^-49
        const double v0 = cv[0];
        double cmax = v0; int nC = 1;
        while (nC < cnt) { const double nx = cv[nC * stride]; if (nx <= cmax + cmax * EPSC) { cmax = nx; nC++; } else break; }
        bool good = (dropped > cmax + cmax * EPSC) && (cmax <= v0 + v0 * 1e-7);
        if (!(dropped > cmax + cmax * EPSC)) DG_EMU_COUNT(29);
        if (!(cmax <= v0 + v0 * 1e-7)) DG_EMU_COUNT(30);
        if (!(pm_list < best_lo)) DG_EMU_COUNT(31);
        good = good && (pm_list < best_lo);             // (ii) for every entry of the list, hence for every member of C
        if (!good) { need_fb = true; ok = false; }
        else if (nC == 1) { win = cpos[0]; D = sqrt(v0); }
        else {
            // order-free shortcut: with g monotone, "v1 >= g(v0)" means no member can displace the minimum once it is the state, and
            // "v0 < g(v1)" means the minimum is accepted from every other member's state: the fold ends at cv[0] whatever the order
            const double D0 = sqrt(v0), v1 = cv[stride], D1 = sqrt(v1);
            if (v1 >= D0 * D0 && v0 < D1 * D1) { win = cpos[0]; D = D0; }
            else {
            // tie shortcut: the k members equal to the minimum, every other member neither able to displace that state (v >= g(v0)) nor
            // to refuse it (v0 < g(v), monotone: checked on the smallest of them).  The state enters the tie group at its first member in
            // the reference's order and then moves on at every further member iff v0 < g(v0): winner = first or last of the group.
            int k = 1;
            while (k < nC && cv[k * stride] == v0) k++;
            bool tie_case = true;
            if (k < nC) { const double vk = cv[k * stride], Dk = sqrt(vk); tie_case = (vk >= D0 * D0) && (v0 < Dk * Dk); }
            if (tie_case) {
                DG_EMU_COUNT(26); DG_EMU_ADD(27, k - 1);
                const bool want_last = v0 < D0 * D0;
                int w = cpos[0];
                for (int i = 1; i < k; i++) {
                    const int p = cpos[i * stride];
                    ncmp++;
                    if (ref_visits_first(M.spheres, n_tri, p, w, px, py, pz) != want_last) w = p;
                }
                win = w; D = D0;
            } else {
            DG_EMU_COUNT(22);
            for (int i = 1; i < nC; i++) {              // insertion sort of C by the reference's visit order
                const double x = cv[i * stride]; const int p = cpos[i * stride];
                int j = i;
                while (j > 0 && (ncmp++, ref_visits_first(M.spheres, n_tri, p, cpos[(j - 1) * stride], px, py, pz))) {
                    DG_EMU_COUNT(23);
                    cv[j * stride] = cv[(j - 1) * stride]; cpos[j * stride] = cpos[(j - 1) * stride];
                    j--;
                }
                cv[j * stride] = x; cpos[j * stride] = p;
            }
            double thr = DINF;                          // result.distance = max(): max() * max() = +inf (:528)
            for (int i = 0; i < nC; i++) {
                const double x = cv[i * stride];
                if (x < thr) { win = cpos[i * stride]; D = sqrt(x); thr = D * D; }
            }
            }
            }
        }
    }
#ifdef DG_EMU
    {   // emulation only: the warp pays for its slowest lane -- max over lanes of the comparator calls
        int mx = 0;
        for (int bit = 5; bit >= 0; bit--) { const unsigned msk = __ballot_sync(FULL, ncmp >= (mx | (1 << bit))); if (msk) mx |= 1 << bit; }
        if ((threadIdx.x & 31u) == 0u) DG_EMU_ADD(28, mx);
    }
#endif
    if (__any_sync(FULL, ok)) {
        if (ok) {                                       // (s, t, entity) of the winner: the same function of (T, query) the reference stored at :529-530
            double s, t; int ent;
            (void)tri_dist2(M.leaves + win, px, py, pz, s, t, ent);
            res.dist = D; res.s = s; res.t = t; res.pos = win; res.entity = ent;
        }
    }
    if (__any_sync(FULL, need_fb)) {                    // the lanes the checks could not clear: the per-lane reference-order walk
        DG_EMU_COUNT(24);
        DG_EMU_ADD(25, need_fb ? 1 : 0);
        const QueryResult r2 = nearest_triangle(M, need_fb, px, py, pz, stack_rng, stack_pm, stride);
        if (need_fb) res = r2;
    }
    return res;
}
#endif  // K1_PACKET

#ifdef DG_EMU
extern unsigned char k1_smem[];                    // defined by the emulation TU (one block runs at a time)
#else
extern __shared__ __align__(16) unsigned char k1_smem[];
#endif

// addFunction node loop: out[l - l_begin] = sign * signed_distance(indexToNodePosition(l)).distance.
// Thread mapping: the node array is four row-major 3-D arrays (vertices, x-, y-, z-edge nodes; K1Segment).  A warp
// owns a brick of 32 nodes (fast x mid x slow, shaped per array: k1_sdf.h) of one of them and a block K1_THREADS / 32 bricks
// side by side along the fast axis, so the 32 queries of a warp are spatial neighbours: they visit nearly the same tree nodes (L1 hits) and
// take similar numbers of steps.  Whole slow-planes are covered; nodes outside [l_begin, l_end) are masked.
// BAND = true is the narrow-band form (sdf_sample_nodes_band_kernel): same walk, same replay, same fallback; only the block id comes from the
// classifier's list and the epilogue keeps the value where |distance| <= band and writes DBL_MAX elsewhere.
template <bool BAND>
__device__ __forceinline__ void sample_nodes_body(MeshDev mesh, const PseudoNormals* __restrict__ normals, int stack_depth, GridDev g,
                                                  K1Work w, double sign, double* __restrict__ out, unsigned this_block, double band)
{
    DG_EMU_TRACE_BLOCK(this_block);
    float* stack_d = reinterpret_cast<float*>(k1_smem);
    unsigned* stack_rng = reinterpret_cast<unsigned*>(k1_smem + (size_t)stack_depth * K1_THREADS * sizeof(float));
    // which segment does this block belong to (<= 4, uniform per block)
    int sg = 0;
#pragma unroll
    for (int k = 1; k < 4; k++) if (k < w.nseg && this_block >= w.seg[k].block_begin) sg = k;
    const K1Segment& S = w.seg[sg];
    unsigned t = this_block - S.block_begin;
    const unsigned tf = t % S.tiles_f; t /= S.tiles_f;
    const unsigned tm = t % S.tiles_m; const unsigned ts = t / S.tiles_m;
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const unsigned f = tf * (SEG_BF(S) * (unsigned)(K1_THREADS / 32)) + warp * SEG_BF(S) + (lane & (SEG_BF(S) - 1u));
    const unsigned m = tm * SEG_BM(S) + ((lane >> S.lf) & (SEG_BM(S) - 1u));
    const unsigned lane_s = lane >> (S.lf + S.lm);
    const unsigned sl = S.s0 + ts * S.pl_stride * SEG_BS(S) + lane_s;
    const unsigned l = S.l_base + (sl * S.Dm + m) * S.Df + f;
    const bool alive = (f < S.Df) && (m < S.Dm) && (sl < S.s1) && (l >= w.l_begin) && (l < w.l_end);

    // indexToNodePosition (cubic_lagrange_discrete_grid.cpp:604-665) from the array coordinates
    unsigned i, j, k;
    const unsigned par = f & 1u, fh = f >> 1;
    if (S.kind == 0) { i = f; j = m; k = sl; }
    else if (S.kind == 1) { i = fh; j = m; k = sl; }
    else if (S.kind == 2) { i = sl; k = m; j = fh; }
    else { j = sl; i = m; k = fh; }
    double px = g.mn[0] + g.cell[0] * (double)i;
    double py = g.mn[1] + g.cell[1] * (double)j;
    double pz = g.mn[2] + g.cell[2] * (double)k;
    const double fr = (1.0 + (double)par) / 3.0;
    if (S.kind == 1) px = px + fr * g.cell[0];
    else if (S.kind == 2) py = py + fr * g.cell[1];
    else if (S.kind == 3) pz = pz + fr * g.cell[2];

#if K1_PACKET
    double* cand_v = reinterpret_cast<double*>(k1_smem + (size_t)stack_depth * K1_THREADS * (sizeof(float) + sizeof(unsigned)));
    int* cand_pos = reinterpret_cast<int*>(cand_v + (size_t)K1_PKT_K * K1_THREADS);
    // shared memory: [stack_d | stack_rng] as the per-lane walk (the fallback) needs them; the packet walk keeps its per-lane certificate in the
    // first and the deferred children's lower bounds in the second, its own (warp-uniform) range stack once per warp behind the candidates
    unsigned* wstack = reinterpret_cast<unsigned*>(cand_pos + (size_t)K1_PKT_K * K1_THREADS) + (size_t)(threadIdx.x >> 5) * stack_depth;
    const QueryResult r = nearest_triangle_packet(mesh, alive, px, py, pz, wstack, stack_rng + threadIdx.x, stack_d + threadIdx.x,
                                                  reinterpret_cast<float*>(stack_rng) + threadIdx.x,
                                                  cand_v + threadIdx.x, cand_pos + threadIdx.x, K1_THREADS);
#else
    const QueryResult r = nearest_triangle(mesh, alive, px, py, pz, stack_rng + threadIdx.x, stack_d + threadIdx.x, K1_THREADS);
#endif
    if (!alive) return;
    double dist, qx, qy, qz; int tri;
    finish_query(mesh.leaves, normals, r, px, py, pz, true, dist, qx, qy, qz, tri);
    const unsigned out_idx = w.compact ? S.out_base + ((ts * SEG_BS(S) + lane_s) * S.Dm + m) * S.Df + f : l - w.l_begin;
    if (BAND)   // addFunction's predicate (cubic_lagrange_discrete_grid.cpp:811-817): |md.signed_distance(x).distance| <= band, else DBL_MAX
        out[out_idx] = (fabs(dist) <= band) ? ((sign == 1.0) ? dist : sign * dist) : DBL_MAX;
    else
        out[out_idx] = (sign == 1.0) ? dist : sign * dist;       // cmd/generate_sdf/main.cpp:97 (-1.0 * d) / :101
}

__global__ void __launch_bounds__(K1_THREADS, K1_PACKET ? K1_PKT_MIN_BLOCKS : K1_MIN_BLOCKS)
sdf_sample_nodes_kernel(MeshDev mesh, const PseudoNormals* __restrict__ normals, int stack_depth, GridDev g, K1Work w, double sign,
                        double* __restrict__ out)
{
    // blocks run in launch order: neighbouring bricks running at the same time share tree nodes in L1, which orders that end a launch with
    // short walks (plane groups from the outside in, heaviest distance class first) give up.
    sample_nodes_body<false>(mesh, normals, stack_depth, g, w, sign, out, blockIdx.x, 0.0);
}

// narrow band: block i of the launch is block list[i] of the node-loop geometry (the classifier's order-preserving list of the blocks that
// may hold a node within the band); the launch is sized for every block and the blocks past *n_list return at once
__global__ void __launch_bounds__(K1_THREADS, K1_PACKET ? K1_PKT_MIN_BLOCKS : K1_MIN_BLOCKS)
sdf_sample_nodes_band_kernel(MeshDev mesh, const PseudoNormals* __restrict__ normals, int stack_depth, GridDev g, K1Work w, double sign,
                             double band, const unsigned* __restrict__ list, const unsigned* __restrict__ n_list, double* __restrict__ out)
{
    if (blockIdx.x >= *n_list) return;
    sample_nodes_body<true>(mesh, normals, stack_depth, g, w, sign, out, list[blockIdx.x], band);
}

// grid node of lane `ln` of brick unit `unit` (= K1_THREADS / 32 * block + warp of the node-loop kernel's launch geometry): position,
// output index.  Used by the narrow-band classifier.
__device__ __forceinline__ bool brick_node(const GridDev& g, const K1Work& w, unsigned unit, unsigned ln, double& px, double& py, double& pz, unsigned& out_idx)
{
    const unsigned this_block = unit / (unsigned)(K1_THREADS / 32), warp = unit % (unsigned)(K1_THREADS / 32);
    int sg = 0;
#pragma unroll
    for (int k = 1; k < 4; k++) if (k < w.nseg && this_block >= w.seg[k].block_begin) sg = k;
    const K1Segment& S = w.seg[sg];
    unsigned t = this_block - S.block_begin;
    const unsigned tf = t % S.tiles_f; t /= S.tiles_f;
    const unsigned tm = t % S.tiles_m; const unsigned ts = t / S.tiles_m;
    const unsigned f = tf * (SEG_BF(S) * (unsigned)(K1_THREADS / 32)) + warp * SEG_BF(S) + (ln & (SEG_BF(S) - 1u));
    const unsigned m = tm * SEG_BM(S) + ((ln >> S.lf) & (SEG_BM(S) - 1u));
    const unsigned lane_s = ln >> (S.lf + S.lm);
    const unsigned sl = S.s0 + ts * S.pl_stride * SEG_BS(S) + lane_s;
    const unsigned l = S.l_base + (sl * S.Dm + m) * S.Df + f;
    const bool alive = (f < S.Df) && (m < S.Dm) && (sl < S.s1) && (l >= w.l_begin) && (l < w.l_end);
    unsigned i, j, k;
    const unsigned par = f & 1u, fh = f >> 1;
    if (S.kind == 0) { i = f; j = m; k = sl; }
    else if (S.kind == 1) { i = fh; j = m; k = sl; }
    else if (S.kind == 2) { i = sl; k = m; j = fh; }
    else { j = sl; i = m; k = fh; }
    px = g.mn[0] + g.cell[0] * (double)i;                 // indexToNodePosition (cubic_lagrange_discrete_grid.cpp:604-665)
    py = g.mn[1] + g.cell[1] * (double)j;
    pz = g.mn[2] + g.cell[2] * (double)k;
    const double fr = (1.0 + (double)par) / 3.0;
    if (S.kind == 1) px = px + fr * g.cell[0];
    else if (S.kind == 2) py = py + fr * g.cell[1];
    else if (S.kind == 3) pz = pz + fr * g.cell[2];
    out_idx = w.compact ? S.out_base + ((ts * SEG_BS(S) + lane_s) * S.Dm + m) * S.Df + f : l - w.l_begin;
    return alive;
}

// =====================================================================================================================================
// NARROW-BAND CLASSIFIER.  addFunction(func, pred) with pred(x) = |md.signed_distance(x).distance| <= band (cubic_lagrange_discrete_grid.cpp:
// 806-817) stores DBL_MAX wherever pred is false.  Before the node loop runs, every block of its launch geometry (K1_THREADS / 32 bricks of
// 32 nodes) is classified: a block may be DROPPED only when every one of its nodes has a reference distance > band; its nodes then get
// DBL_MAX here and it is never sampled.  The kept blocks form an order-preserving list (launch order matters, see the node-loop kernel) that
// sdf_sample_nodes_band_kernel walks.  Dropping is certified; keeping is free to be conservative (it costs time, never bits).
//   Bound.  Per brick: the fp64 box of its in-range node positions, taken relative to the mesh centre and rounded OUTWARD to fp32.  The tree's
//   fp32 child boxes are rounded outward too (bvh_build.h), so the box-to-box gap, evaluated with round-down operations, is a lower bound L of
//   the true distance from every node of the brick to every triangle of the subtree (up to the fp64 rounding of p - centre, < 2^-52 Mq).  A
//   subtree is pruned when L > thr = band + 2E (E = filter_slack(Mq), Mq = max(half extent, |box|_inf)); the brick is kept as soon as a leaf
//   survives.  If no leaf survives, every triangle T has true distance d_T > band + 2E to every node.  The reference's d2 for T is >= d_T^2 -
//   240 eps64 R^2 with R <= 7 Mq (the box-skip budget above), i.e. its distance is >= d_T - 1.3e-12 Mq^2 / d_T > d_T - 1.4e-6 Mq since
//   d_T > 2E >= 7.6e-6 Mq: so every distance the reference can compute, hence the one it returns, is > band and pred(x) is false.
//   Range: E must be finite (2^-40 <= Mq < 1e18, filter_slack); otherwise the brick is kept.  A mesh with non-finite vertices has half
//   extent +inf (bvh_build.cpp): every brick is kept.  NaN positions or band = +inf keep the brick too (no comparison can prune).
// Passes (all warp-synchronous -- ballot / popc / redux -- so tests/emu runs them): classify (one thread per brick) -> count per chunk of
// K1_BAND_CHUNK blocks -> compact (one warp per chunk; its offset = sum of the earlier chunks' counts) -> the band form of the node loop.
// =====================================================================================================================================
constexpr unsigned K1_BRICKS = K1_THREADS / 32;                  // bricks per block of the node-loop kernel
static_assert(K1_BRICKS >= 1 && K1_BRICKS <= 32 && (K1_BRICKS & (K1_BRICKS - 1)) == 0, "a block's bricks must share a warp of the classifier");
constexpr unsigned K1_BAND_CHUNK = 1024;                         // blocks per warp in the count / compaction passes
constexpr unsigned K1_BAND_THREADS = 128;

// squared gap between two fp32 boxes, rounded down
__device__ __forceinline__ float box_gap2_rd(float alx, float aly, float alz, float ahx, float ahy, float ahz, const float* lo, const float* hi)
{
    const float gx = fmaxf(fmaxf(__fmaf_rd(alx, 1.f, -hi[0]), __fmaf_rd(lo[0], 1.f, -ahx)), 0.f);
    const float gy = fmaxf(fmaxf(__fmaf_rd(aly, 1.f, -hi[1]), __fmaf_rd(lo[1], 1.f, -ahy)), 0.f);
    const float gz = fmaxf(fmaxf(__fmaf_rd(alz, 1.f, -hi[2]), __fmaf_rd(lo[2], 1.f, -ahz)), 0.f);
    return __fmaf_rd(gz, gz, __fmaf_rd(gy, gy, __fmul_rd(gx, gx)));
}

// may some triangle lie within sqrt(thr2) of the box [lo, hi] (fp32, relative to the mesh centre)?  Depth-first over the implicit tree; true
// at the first leaf whose box is not certainly farther.  NaN gaps compare false: not pruned.
__device__ bool band_box_near_mesh(const MeshDev M, const float* lo, const float* hi, float thr2)
{
    if (M.n_tri < 2) return true;
    int stk_b[32], stk_e[32];                                    // one deferred sibling per level; node ids hold 25 bits (pack_range)
    int b = 0, e = M.n_tri, sp = 0;
    for (;;) {
        const int m = (b + e) >> 1;
        const float4* f4 = M.nodes_f + (size_t)m * K1_NODEF_STRIDE;
        const float4 b0 = __ldg(f4 + 2), b1 = __ldg(f4 + 3), b2 = __ldg(f4 + 4);   // l_lo.xyz l_hi.x | l_hi.yz r_lo.xy | r_lo.z r_hi.xyz
        const bool wl = !(box_gap2_rd(b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, lo, hi) > thr2);
        const bool wr = !(box_gap2_rd(b1.z, b1.w, b2.x, b2.y, b2.z, b2.w, lo, hi) > thr2);
        if ((wl && m - b == 1) || (wr && e - m == 1)) return true;
        if (wl && wr) { stk_b[sp] = m; stk_e[sp] = e; sp++; e = m; }
        else if (wl) e = m;
        else if (wr) b = m;
        else {
            if (sp == 0) return false;
            sp--; b = stk_b[sp]; e = stk_e[sp];
        }
    }
}

// one thread per brick (unit = K1_BRICKS * block + warp, as brick_node numbers them); keep[block] = any of its bricks may be in the band;
// the in-range nodes of a dropped block get DBL_MAX
__global__ void __launch_bounds__(K1_BAND_THREADS)
band_classify_kernel(MeshDev M, GridDev g, K1Work w, unsigned n_blocks, double band, double* __restrict__ out, unsigned char* __restrict__ keep)
{
    const unsigned FULL = 0xffffffffu;
    const float INF = __int_as_float(0x7f800000);
    const unsigned unit = blockIdx.x * K1_BAND_THREADS + threadIdx.x, lane = threadIdx.x & 31u;
    const bool live = unit < n_blocks * K1_BRICKS;
    double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
    bool any = false, finite = true;
    if (live) {
        for (unsigned ln = 0; ln < 32u; ln++) {
            double p[3]; unsigned oi;
            if (!brick_node(g, w, unit, ln, p[0], p[1], p[2], oi)) continue;
            any = true;
            for (int k = 0; k < 3; k++) {
                if (!(fabs(p[k]) <= DBL_MAX)) finite = false;
                lo[k] = fmin(lo[k], p[k]); hi[k] = fmax(hi[k], p[k]);
            }
        }
    }
    bool near = false;
    if (any) {
        if (!finite) near = true;
        else {
            const double ctr[3] = {M.cx, M.cy, M.cz};
            float flo[3], fhi[3];
            float Mq = M.half_extent;
            for (int k = 0; k < 3; k++) {
                flo[k] = __double2float_rd(lo[k] - ctr[k]); fhi[k] = __double2float_ru(hi[k] - ctr[k]);
                Mq = fmaxf(Mq, fmaxf(fabsf(flo[k]), fabsf(fhi[k])));
            }
            const float E = filter_slack(Mq);                       // +inf outside the budget's range (and for a non-finite mesh)
            const float thr = __fadd_ru(__double2float_ru(band), __fadd_ru(E, E));
            const float thr2 = __fmul_ru(thr, thr);
            near = !(thr2 < INF) || band_box_near_mesh(M, flo, fhi, thr2);
        }
    }
    // the K1_BRICKS bricks of a block are adjacent lanes of one warp
    const unsigned votes = __ballot_sync(FULL, near);
    const unsigned group = (K1_BRICKS == 32u ? FULL : ((1u << K1_BRICKS) - 1u)) << (lane & ~(K1_BRICKS - 1u));
    const bool block_kept = (votes & group) != 0u;
    if (live && (lane & (K1_BRICKS - 1u)) == 0u) keep[unit / K1_BRICKS] = block_kept ? 1 : 0;
    if (any && !block_kept) {
        for (unsigned ln = 0; ln < 32u; ln++) {
            double px, py, pz; unsigned oi;
            if (brick_node(g, w, unit, ln, px, py, pz, oi)) out[oi] = DBL_MAX;
        }
    }
}

// kept blocks per chunk of K1_BAND_CHUNK blocks (one warp per chunk)
__global__ void __launch_bounds__(K1_BAND_THREADS) band_count_kernel(const unsigned char* __restrict__ keep, unsigned n_blocks, unsigned* __restrict__ chunk_count)
{
    const unsigned chunk = (blockIdx.x * K1_BAND_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    const unsigned long long base = (unsigned long long)chunk * K1_BAND_CHUNK;
    if (base >= n_blocks) return;                                // whole warps
    unsigned cnt = 0;
    for (unsigned k = 0; k < K1_BAND_CHUNK; k += 32) {
        const unsigned long long i = base + k + lane;
        cnt += (unsigned)__popc(__ballot_sync(0xffffffffu, i < n_blocks && keep[i] != 0));
    }
    if (lane == 0) chunk_count[chunk] = cnt;
}

// list of the kept blocks in launch order (one warp per chunk); the warp of the last chunk writes the list length
__global__ void __launch_bounds__(K1_BAND_THREADS) band_compact_kernel(const unsigned char* __restrict__ keep, unsigned n_blocks,
                                                                       const unsigned* __restrict__ chunk_count, unsigned* __restrict__ list,
                                                                       unsigned* __restrict__ n_list)
{
    const unsigned chunk = (blockIdx.x * K1_BAND_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    const unsigned long long base = (unsigned long long)chunk * K1_BAND_CHUNK;
    if (base >= n_blocks) return;
    unsigned run = 0;
    for (unsigned c = 0; c < chunk; c += 32) run += __reduce_add_sync(0xffffffffu, (c + lane < chunk) ? chunk_count[c + lane] : 0u);
    const unsigned lt = (1u << lane) - 1u;
    for (unsigned k = 0; k < K1_BAND_CHUNK; k += 32) {
        const unsigned long long i = base + k + lane;
        const bool kept = i < n_blocks && keep[i] != 0;
        const unsigned msk = __ballot_sync(0xffffffffu, kept);
        if (kept) list[run + (unsigned)__popc(msk & lt)] = (unsigned)i;
        run += (unsigned)__popc(msk);
    }
    if (lane == 0 && base + K1_BAND_CHUNK >= n_blocks) *n_list = run;
}

// batched TriangleMeshDistance::{signed,unsigned}_distance on arbitrary points (a warp = 32 consecutive points)
__global__ void __launch_bounds__(K1_THREADS, K1_MIN_BLOCKS)
mesh_distance_kernel(MeshDev mesh, const PseudoNormals* __restrict__ normals, int stack_depth,
                     const double* __restrict__ pts, unsigned long long count, int is_signed,
                     double* __restrict__ dist_out, double* __restrict__ near_out, int* __restrict__ ent_out,
                     int* __restrict__ tri_out)
{
    float* stack_d = reinterpret_cast<float*>(k1_smem);
    unsigned* stack_rng = reinterpret_cast<unsigned*>(k1_smem + (size_t)stack_depth * K1_THREADS * sizeof(float));
    const unsigned long long idx = (unsigned long long)blockIdx.x * K1_THREADS + threadIdx.x;
    const bool alive = idx < count;
    const unsigned long long ix = alive ? idx : 0ull;
    const double px = pts[3 * ix], py = pts[3 * ix + 1], pz = pts[3 * ix + 2];
    const QueryResult r = nearest_triangle(mesh, alive, px, py, pz, stack_rng + threadIdx.x, stack_d + threadIdx.x, K1_THREADS);
    if (!alive) return;
    double dist, qx, qy, qz; int tri;
    finish_query(mesh.leaves, normals, r, px, py, pz, is_signed != 0, dist, qx, qy, qz, tri);
    if (dist_out) dist_out[idx] = dist;
    if (near_out) { near_out[3 * idx] = qx; near_out[3 * idx + 1] = qy; near_out[3 * idx + 2] = qz; }
    if (ent_out) ent_out[idx] = r.entity;
    if (tri_out) tri_out[idx] = tri;
}

// mesh_distance_kernel that also writes the barycentric weights (fl(fl(1 - s) - t), s, t) of the nearest point (dg_mesh_distance_bary, K10's
// forward; NaN when nothing was accepted).  A separate kernel rather than a flag, so that mesh_distance_kernel's code stays as it is; the
// walk and finish_query are the same inlined functions, hence the same distance, nearest point, entity and triangle id.
__global__ void __launch_bounds__(K1_THREADS, K1_MIN_BLOCKS)
mesh_distance_bary_kernel(MeshDev mesh, const PseudoNormals* __restrict__ normals, int stack_depth,
                          const double* __restrict__ pts, unsigned long long count, int is_signed,
                          double* __restrict__ dist_out, double* __restrict__ near_out, int* __restrict__ ent_out,
                          int* __restrict__ tri_out, double* __restrict__ bary_out)
{
    float* stack_d = reinterpret_cast<float*>(k1_smem);
    unsigned* stack_rng = reinterpret_cast<unsigned*>(k1_smem + (size_t)stack_depth * K1_THREADS * sizeof(float));
    const unsigned long long idx = (unsigned long long)blockIdx.x * K1_THREADS + threadIdx.x;
    const bool alive = idx < count;
    const unsigned long long ix = alive ? idx : 0ull;
    const double px = pts[3 * ix], py = pts[3 * ix + 1], pz = pts[3 * ix + 2];
    const QueryResult r = nearest_triangle(mesh, alive, px, py, pz, stack_rng + threadIdx.x, stack_d + threadIdx.x, K1_THREADS);
    if (!alive) return;
    double dist, qx, qy, qz; int tri;
    finish_query(mesh.leaves, normals, r, px, py, pz, is_signed != 0, dist, qx, qy, qz, tri);
    if (dist_out) dist_out[idx] = dist;
    if (near_out) { near_out[3 * idx] = qx; near_out[3 * idx + 1] = qy; near_out[3 * idx + 2] = qz; }
    if (ent_out) ent_out[idx] = r.entity;
    if (tri_out) tri_out[idx] = tri;
    if (bary_out) {
        const double nan = __longlong_as_double(0x7ff8000000000000ll);
        bary_out[3 * idx] = r.pos < 0 ? nan : (1.0 - r.s) - r.t;
        bary_out[3 * idx + 1] = r.pos < 0 ? nan : r.s;
        bary_out[3 * idx + 2] = r.pos < 0 ? nan : r.t;
    }
}


__global__ void node_positions_kernel(GridDev g, unsigned l_begin, unsigned long long count, double* __restrict__ x)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    double px, py, pz;
    node_position(g, l_begin + (unsigned)idx, px, py, pz);
    x[3 * idx] = px; x[3 * idx + 1] = py; x[3 * idx + 2] = pz;
}

// closed-form cell table (cubic_lagrange_discrete_grid.cpp:833-886): one thread per (cell, local node)
__global__ void build_cells_kernel(GridDev g, unsigned c_begin, unsigned long long count32, unsigned* __restrict__ cells)
{
    const unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count32) return;
    const unsigned c = c_begin + (unsigned)(idx >> 5), jn = (unsigned)(idx & 31u);
    const unsigned nxy = g.n[0] * g.n[1];
    const unsigned k = c / nxy, t = c - k * nxy, j = t / g.n[0], i = t - j * g.n[0];
    cells[idx] = cell_node_id(g, i, j, k, jn);
}

// FMA-contraction probe: a*b+c with operands for which the fused and unfused roundings differ.
__global__ void fma_probe_kernel(double a, double b, double c, double* out) { out[0] = a * b + c; }

// fp64 issue-rate probe: 8 independent chains of x = x * a + b per thread, compiled (like the whole library) WITHOUT contraction,
// i.e. one DMUL + one DADD per step -- the instruction mix the bit-exact kernels are restricted to.  Used by bench.py as the measured
// denominator of K1's / K3's fp64 roofline (there is no fp64 figure in MEASURED_PEAKS.json).
__global__ void __launch_bounds__(256) fp64_rate_probe_kernel(double a, double b, int iters, double* out)
{
    double x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
#pragma unroll 4
    for (int i = 0; i < iters; i++) {
        x0 = x0 * a + b; x1 = x1 * a + b; x2 = x2 * a + b; x3 = x3 * a + b;
        x4 = x4 * a + b; x5 = x5 * a + b; x6 = x6 * a + b; x7 = x7 * a + b;
    }
    const double s = ((x0 + x1) + (x2 + x3)) + ((x4 + x5) + (x6 + x7));
    if (s == 123.456) out[0] = s;                      // never true: keeps the chains alive
}

}  // namespace

static inline size_t k1_smem_bytes(int stack_depth)
{
    size_t n = (size_t)stack_depth * K1_THREADS * (sizeof(float) + sizeof(unsigned));
#if K1_PACKET
    n += (size_t)K1_PKT_K * K1_THREADS * (sizeof(double) + sizeof(int));                        // candidate lists of the packet walk
    n += (size_t)(K1_THREADS / 32) * stack_depth * sizeof(unsigned);                            // the warp-uniform range stack
#endif
    return n;
}
static inline MeshDev mesh_dev(const DeviceBvh& m)
{
    return MeshDev{m.spheres, m.nodes_f, m.leaves_f, m.leaves, m.ctr[0], m.ctr[1], m.ctr[2], m.half_extent, m.n_tri};
}

// The opt-in limit for dynamic shared memory is a per-function attribute: keep it at the maximum any live mesh has needed
// (per device; meshes with different tree depths can coexist).
cudaError_t k1_configure(int stack_depth)
{
#ifdef DG_EMU
    (void)stack_depth; return cudaSuccess;
#else
    static std::mutex mu;
    static int configured[64] = {0};              // per device: stack depth the attribute currently allows
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    if (dev >= 0 && dev < 64 && configured[dev] >= stack_depth) return cudaSuccess;
    const size_t bytes = k1_smem_bytes(stack_depth);
    e = cudaFuncSetAttribute(sdf_sample_nodes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(sdf_sample_nodes_band_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(mesh_distance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(mesh_distance_bary_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess && dev >= 0 && dev < 64) configured[dev] = stack_depth;
    return e;
#endif
}

// brick shape of node array `kind`: (lf, lm, ls) with lf + lm + ls = 5 and lf >= 1 minimising the physical diagonal of the 32 nodes.
// Node spacing along (f, m, s): vertices (cx, cy, cz); x-edge nodes (cx/2, cy, cz); y-edge (cy/2, cz, cx); z-edge (cz/2, cx, cy).
static void choose_brick(const GridDev& g, int kind, unsigned& lf, unsigned& lm)
{
    const double c[3] = {g.cell[0], g.cell[1], g.cell[2]};
    const double h[4][3] = {{c[0], c[1], c[2]}, {0.5 * c[0], c[1], c[2]}, {0.5 * c[1], c[2], c[0]}, {0.5 * c[2], c[0], c[1]}};
    lf = 2; lm = 2;                                               // 4 x 4 x 2: kept on ties
    auto diag2 = [&](unsigned a, unsigned b) { const double x = (double)(1u << a) * h[kind][0], y = (double)(1u << b) * h[kind][1],
                                                              z = (double)(32u >> (a + b)) * h[kind][2]; return x * x + y * y + z * z; };
    double best = diag2(lf, lm);
    for (unsigned a = 1; a <= 4; a++)
        for (unsigned b = 0; a + b <= 5; b++) {
            const double d = diag2(a, b);
            if (d < best * (1.0 - 1e-9)) { best = d; lf = a; lm = b; }
        }
}

// Splits [l_begin, l_begin+count) into the (at most four) node arrays it touches and tiles whole slow-planes of each.
static unsigned node_range_work(const GridDev& g, uint64_t l_begin, uint64_t count, K1Work& w)
{
    const uint64_t l_end = l_begin + count;
    const unsigned nx = g.n[0], ny = g.n[1], nz = g.n[2];
    // {base, Ds, Dm, Df} of the four row-major node arrays (cubic_lagrange_discrete_grid.cpp:618-662)
    const uint64_t base[5] = {0, g.nv, (uint64_t)g.nv + 2ull * g.ne_x, (uint64_t)g.nv + 2ull * (g.ne_x + (uint64_t)g.ne_y),
                              (uint64_t)g.nv + 2ull * ((uint64_t)g.ne_x + g.ne_y + g.ne_z)};
    const unsigned dims[4][3] = {{nz + 1, ny + 1, nx + 1}, {nz + 1, ny + 1, 2 * nx}, {nx + 1, nz + 1, 2 * ny}, {ny + 1, nx + 1, 2 * nz}};
    w.nseg = 0; w.l_begin = (unsigned)l_begin; w.l_end = (unsigned)l_end; w.compact = 0;
    unsigned blocks = 0;
    for (int k = 0; k < 4; k++) {
        const uint64_t a = l_begin > base[k] ? l_begin : base[k];
        const uint64_t b = l_end < base[k + 1] ? l_end : base[k + 1];
        if (a >= b) continue;
        K1Segment& S = w.seg[w.nseg++];
        S.kind = k; S.l_base = (unsigned)base[k];
        S.Ds = dims[k][0]; S.Dm = dims[k][1]; S.Df = dims[k][2];
        const uint64_t plane = (uint64_t)S.Dm * S.Df;
        S.pl_stride = 1u; S.out_base = 0u;
        S.s0 = (unsigned)((a - base[k]) / plane);
        S.s1 = (unsigned)((b - 1 - base[k]) / plane) + 1;
        choose_brick(g, S.kind, S.lf, S.lm);
        const unsigned bf = SEG_BF(S) * (K1_THREADS / 32);
        S.tiles_f = (S.Df + bf - 1) / bf; S.tiles_m = (S.Dm + SEG_BM(S) - 1) / SEG_BM(S);
        const unsigned tiles_s = (S.s1 - S.s0 + SEG_BS(S) - 1) / SEG_BS(S);
        S.block_begin = blocks; S.tiles_s = tiles_s;
        blocks += S.tiles_f * S.tiles_m * tiles_s;
    }
    for (int k = w.nseg; k < 4; k++) { w.seg[k] = w.seg[0]; w.seg[k].block_begin = 0xffffffffu; }
    return blocks;
}

cudaError_t k1_launch_sample_nodes(const DeviceBvh& m, const GridDev& g, double sign, uint64_t l_begin, uint64_t count,
                                   double* d_out, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    K1Work w;
    const unsigned blocks = node_range_work(g, l_begin, count, w);
    DG_KERNEL_LAUNCH(sdf_sample_nodes_kernel, blocks, K1_THREADS, k1_smem_bytes(m.stack_depth), stream, mesh_dev(m), m.normals, m.stack_depth, g, w, sign, d_out);
    return DG_AFTER_LAUNCH();
}

// scratch of the band form: keep flag per block (bytes), count per chunk, the list, its length
static void band_scratch_layout(unsigned blocks, size_t off[4], size_t& total)
{
    const unsigned chunks = (blocks + K1_BAND_CHUNK - 1) / K1_BAND_CHUNK;
    off[0] = 0;
    off[1] = ((size_t)blocks + 255) / 256 * 256;
    off[2] = off[1] + ((size_t)chunks * sizeof(unsigned) + 255) / 256 * 256;
    off[3] = off[2] + ((size_t)blocks * sizeof(unsigned) + 255) / 256 * 256;
    total = off[3] + 256;
}

size_t k1_band_scratch_bytes(const GridDev& g, uint64_t l_begin, uint64_t count)
{
    if (count == 0) return 0;
    K1Work w;
    size_t off[4], total;
    band_scratch_layout(node_range_work(g, l_begin, count, w), off, total);
    return total;
}

cudaError_t k1_launch_sample_nodes_band(const DeviceBvh& m, const GridDev& g, double sign, double band, uint64_t l_begin, uint64_t count,
                                        double* d_out, void* d_scratch, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    K1Work w;
    const unsigned blocks = node_range_work(g, l_begin, count, w);
    size_t off[4], total;
    band_scratch_layout(blocks, off, total);
    unsigned char* keep = static_cast<unsigned char*>(d_scratch) + off[0];
    unsigned* chunk_count = reinterpret_cast<unsigned*>(static_cast<unsigned char*>(d_scratch) + off[1]);
    unsigned* list = reinterpret_cast<unsigned*>(static_cast<unsigned char*>(d_scratch) + off[2]);
    unsigned* n_list = reinterpret_cast<unsigned*>(static_cast<unsigned char*>(d_scratch) + off[3]);
    const unsigned long long units = (unsigned long long)blocks * K1_BRICKS, chunks = (blocks + K1_BAND_CHUNK - 1) / K1_BAND_CHUNK;
    DG_KERNEL_LAUNCH(band_classify_kernel, (unsigned)((units + K1_BAND_THREADS - 1) / K1_BAND_THREADS), K1_BAND_THREADS, 0, stream,
                     mesh_dev(m), g, w, blocks, band, d_out, keep);
    const unsigned warps_blocks = (unsigned)((chunks * 32ull + K1_BAND_THREADS - 1) / K1_BAND_THREADS);
    DG_KERNEL_LAUNCH(band_count_kernel, warps_blocks, K1_BAND_THREADS, 0, stream, keep, blocks, chunk_count);
    DG_KERNEL_LAUNCH(band_compact_kernel, warps_blocks, K1_BAND_THREADS, 0, stream, keep, blocks, chunk_count, list, n_list);
    DG_KERNEL_LAUNCH(sdf_sample_nodes_band_kernel, blocks, K1_THREADS, k1_smem_bytes(m.stack_depth), stream, mesh_dev(m), m.normals, m.stack_depth,
                     g, w, sign, band, list, n_list, d_out);
    return DG_AFTER_LAUNCH();
}

cudaError_t k1_launch_sample_slab(const DeviceBvh& m, const GridDev& g, double sign, const unsigned plane_begin[4], const unsigned plane_end[4],
                                  double* d_full, cudaStream_t stream)
{
    const unsigned nx = g.n[0], ny = g.n[1], nz = g.n[2];
    const uint64_t base[4] = {0, g.nv, (uint64_t)g.nv + 2ull * g.ne_x, (uint64_t)g.nv + 2ull * (g.ne_x + (uint64_t)g.ne_y)};
    const unsigned dims[4][3] = {{nz + 1, ny + 1, nx + 1}, {nz + 1, ny + 1, 2 * nx}, {nx + 1, nz + 1, 2 * ny}, {ny + 1, nx + 1, 2 * nz}};
    K1Work w;
    w.nseg = 0; w.l_begin = 0u; w.l_end = 0xffffffffu; w.compact = 0;   // whole planes: nothing to mask, out[l] is the final position
    unsigned blocks = 0;
    for (int k = 0; k < 4; k++) {
        if (plane_begin[k] >= plane_end[k]) continue;
        K1Segment& S = w.seg[w.nseg++];
        S.kind = k; S.l_base = (unsigned)base[k];
        S.Ds = dims[k][0]; S.Dm = dims[k][1]; S.Df = dims[k][2];
        S.s0 = plane_begin[k]; S.s1 = plane_end[k]; S.pl_stride = 1u; S.out_base = 0u;
        choose_brick(g, S.kind, S.lf, S.lm);
        const unsigned bf = SEG_BF(S) * (K1_THREADS / 32);
        S.tiles_f = (S.Df + bf - 1) / bf; S.tiles_m = (S.Dm + SEG_BM(S) - 1) / SEG_BM(S);
        const unsigned tiles_s = (S.s1 - S.s0 + SEG_BS(S) - 1) / SEG_BS(S);
        S.block_begin = blocks; S.tiles_s = tiles_s;
        blocks += S.tiles_f * S.tiles_m * tiles_s;
    }
    if (w.nseg == 0) return cudaSuccess;
    for (int k = w.nseg; k < 4; k++) { w.seg[k] = w.seg[0]; w.seg[k].block_begin = 0xffffffffu; }
    DG_KERNEL_LAUNCH(sdf_sample_nodes_kernel, blocks, K1_THREADS, k1_smem_bytes(m.stack_depth), stream, mesh_dev(m), m.normals, m.stack_depth, g, w, sign, d_full);
    return DG_AFTER_LAUNCH();
}

static void node_arrays(const GridDev& g, uint64_t base[4], unsigned dims[4][3])
{
    const unsigned nx = g.n[0], ny = g.n[1], nz = g.n[2];
    base[0] = 0; base[1] = g.nv; base[2] = (uint64_t)g.nv + 2ull * g.ne_x; base[3] = (uint64_t)g.nv + 2ull * (g.ne_x + (uint64_t)g.ne_y);
    const unsigned d[4][3] = {{nz + 1, ny + 1, nx + 1}, {nz + 1, ny + 1, 2 * nx}, {nx + 1, nz + 1, 2 * ny}, {ny + 1, nx + 1, 2 * nz}};
    for (int a = 0; a < 4; a++) for (int k = 0; k < 3; k++) dims[a][k] = d[a][k];
}

bool k1_interleaved_layout(const GridDev& g, unsigned n_parts, InterleavedLayout& L)
{
    if (n_parts == 0 || n_parts > 16) return false;
    uint64_t base[4]; unsigned dims[4][3];
    node_arrays(g, base, dims);
    L.n_parts = n_parts; L.slot_elems = 0;
    for (int a = 0; a < 4; a++) choose_brick(g, a, L.lf[a], L.lm[a]);
    for (int a = 0; a < 4; a++) { L.pairs[a] = (dims[a][0] + LAY_BS(L, a) - 1) / LAY_BS(L, a); L.plane[a] = dims[a][1] * dims[a][2]; L.rot[a] = ((unsigned)a * (n_parts >= 4 ? n_parts / 4 : 1u)) % n_parts; }
    for (unsigned part = 0; part < n_parts; part++) {
        uint64_t off = 0;
        for (int a = 0; a < 4; a++) {
            L.off[a][part] = (unsigned)off;
            const unsigned r = (part + n_parts - L.rot[a]) % n_parts;                                    // first plane group of this part in array a
            const uint64_t mine = (L.pairs[a] > r) ? (L.pairs[a] - r + n_parts - 1) / n_parts : 0;      // groups r, r + n_parts, ...
            off += mine * LAY_BS(L, a) * (uint64_t)L.plane[a];
        }
        if (off > 0xffffffffull) return false;
        if (off > L.slot_elems) L.slot_elems = off;
    }
    for (unsigned part = n_parts; part < 16; part++) for (int a = 0; a < 4; a++) L.off[a][part] = 0;
    return true;
}

cudaError_t k1_launch_sample_interleaved(const DeviceBvh& m, const GridDev& g, double sign, const InterleavedLayout& L, unsigned part,
                                         double* d_slot, cudaStream_t stream)
{
    uint64_t base[4]; unsigned dims[4][3];
    node_arrays(g, base, dims);
    K1Work w;
    w.nseg = 0; w.l_begin = 0u; w.l_end = 0xffffffffu; w.compact = 1;
    unsigned blocks = 0;
    for (int k = 0; k < 4; k++) {
        const unsigned first = (part + L.n_parts - L.rot[k]) % L.n_parts;                               // this part's first plane group of array k
        const unsigned mine = (L.pairs[k] > first) ? (L.pairs[k] - first + L.n_parts - 1) / L.n_parts : 0;
        if (mine == 0) continue;
        K1Segment& S = w.seg[w.nseg++];
        S.kind = k; S.l_base = (unsigned)base[k];
        S.Ds = dims[k][0]; S.Dm = dims[k][1]; S.Df = dims[k][2];
        S.lf = L.lf[k]; S.lm = L.lm[k];
        S.s0 = first * SEG_BS(S); S.s1 = S.Ds; S.pl_stride = L.n_parts; S.out_base = L.off[k][part];
        const unsigned bf = SEG_BF(S) * (K1_THREADS / 32);
        S.tiles_f = (S.Df + bf - 1) / bf; S.tiles_m = (S.Dm + SEG_BM(S) - 1) / SEG_BM(S);
        S.block_begin = blocks; S.tiles_s = mine;
        blocks += S.tiles_f * S.tiles_m * mine;
    }
    if (w.nseg == 0) return cudaSuccess;
    for (int k = w.nseg; k < 4; k++) { w.seg[k] = w.seg[0]; w.seg[k].block_begin = 0xffffffffu; }
    DG_KERNEL_LAUNCH(sdf_sample_nodes_kernel, blocks, K1_THREADS, k1_smem_bytes(m.stack_depth), stream, mesh_dev(m), m.normals, m.stack_depth, g, w, sign, d_slot);
    return DG_AFTER_LAUNCH();
}

// node id -> (part, position inside that part's slot): the one statement of the exchange layout, shared by the unpack kernel and the host
__host__ __device__ inline unsigned long long interleaved_slot_of(const GridDev& g, const InterleavedLayout& L, unsigned long long l, unsigned& part)
{
    const unsigned long long b1 = g.nv, b2 = b1 + 2ull * g.ne_x, b3 = b2 + 2ull * g.ne_y;
    const int a = (l < b1) ? 0 : ((l < b2) ? 1 : ((l < b3) ? 2 : 3));
    const unsigned long long rel = l - ((a == 0) ? 0ull : ((a == 1) ? b1 : ((a == 2) ? b2 : b3)));
    const unsigned plane = L.plane[a];
    const unsigned s = (unsigned)(rel / plane), inplane = (unsigned)(rel - (unsigned long long)s * plane);
    const unsigned bs = LAY_BS(L, a);
    const unsigned pair = s / bs, j = pair / L.n_parts;
    part = (pair + L.rot[a]) % L.n_parts;
    return (unsigned long long)L.off[a][part] + (unsigned long long)(j * bs + (s % bs)) * plane + inplane;
}

namespace {
// gathered slots [n_parts][slot_elems] -> coefficient array in the reference's node order
__global__ void unpack_interleaved_kernel(GridDev g, InterleavedLayout L, unsigned long long n_nodes, const double* __restrict__ slots,
                                          double* __restrict__ nodes)
{
    const unsigned long long l = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n_nodes) return;
    unsigned r;
    const unsigned long long pos = interleaved_slot_of(g, L, l, r);
    nodes[l] = slots[(size_t)r * L.slot_elems + pos];
}
}  // namespace

void k1_interleaved_node_slots(const GridDev& g, const InterleavedLayout& L, uint64_t l_begin, uint64_t count, uint32_t* part_out, uint64_t* pos_out)
{
    for (uint64_t i = 0; i < count; i++) {
        unsigned r;
        const unsigned long long pos = interleaved_slot_of(g, L, l_begin + i, r);
        if (part_out) part_out[i] = r;
        if (pos_out) pos_out[i] = pos;
    }
}

// The contiguous runs of part `part`: every plane group it owns is one run, contiguous both in the slot and in the node array.
void k1_interleaved_runs(const GridDev& g, const InterleavedLayout& L, unsigned part, std::vector<K1Run>& runs)
{
    uint64_t base[4]; unsigned dims[4][3];
    node_arrays(g, base, dims);
    runs.clear();
    for (int a = 0; a < 4; a++) {
        const unsigned bs = LAY_BS(L, a);
        for (unsigned pair = (part + L.n_parts - L.rot[a]) % L.n_parts; pair < L.pairs[a]; pair += L.n_parts) {
            const unsigned s0 = pair * bs, s1 = std::min(dims[a][0], s0 + bs);
            K1Run r;
            r.node_begin = base[a] + (uint64_t)s0 * L.plane[a];
            r.count = (uint64_t)(s1 - s0) * L.plane[a];
            unsigned owner;
            r.slot_pos = interleaved_slot_of(g, L, r.node_begin, owner);
            runs.push_back(r);
        }
    }
}

cudaError_t k1_launch_unpack_interleaved(const GridDev& g, const InterleavedLayout& L, const double* d_slots, double* d_nodes, cudaStream_t stream)
{
    const unsigned long long n = (unsigned long long)g.nv + 2ull * ((unsigned long long)g.ne_x + g.ne_y + g.ne_z);
    DG_KERNEL_LAUNCH(unpack_interleaved_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, g, L, n, d_slots, d_nodes);
    return DG_AFTER_LAUNCH();
}

cudaError_t k1_launch_distance(const DeviceBvh& m, const double* d_pts, uint64_t count, int is_signed, double* d_dist,
                               double* d_near, int* d_ent, int* d_tri, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((count + K1_THREADS - 1) / K1_THREADS);
    DG_KERNEL_LAUNCH(mesh_distance_kernel, blocks, K1_THREADS, k1_smem_bytes(m.stack_depth), stream, mesh_dev(m), m.normals, m.stack_depth, d_pts, (unsigned long long)count, is_signed, d_dist, d_near, d_ent, d_tri);
    return DG_AFTER_LAUNCH();
}

cudaError_t k1_launch_distance_bary(const DeviceBvh& m, const double* d_pts, uint64_t count, int is_signed, double* d_dist,
                                    double* d_near, int* d_ent, int* d_tri, double* d_bary, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((count + K1_THREADS - 1) / K1_THREADS);
    DG_KERNEL_LAUNCH(mesh_distance_bary_kernel, blocks, K1_THREADS, k1_smem_bytes(m.stack_depth), stream, mesh_dev(m), m.normals, m.stack_depth,
                     d_pts, (unsigned long long)count, is_signed, d_dist, d_near, d_ent, d_tri, d_bary);
    return DG_AFTER_LAUNCH();
}

cudaError_t k1_launch_node_positions(const GridDev& g, uint64_t l_begin, uint64_t count, double* d_x, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    DG_KERNEL_LAUNCH(node_positions_kernel, (unsigned)((count + 255) / 256), 256, 0, stream, g, (unsigned)l_begin, (unsigned long long)count, d_x);
    return DG_AFTER_LAUNCH();
}

cudaError_t k1_launch_build_cells(const GridDev& g, uint64_t c_begin, uint64_t count, unsigned* d_cells, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    const unsigned long long n32 = (unsigned long long)count * 32ull;
    DG_KERNEL_LAUNCH(build_cells_kernel, (unsigned)((n32 + 255) / 256), 256, 0, stream, g, (unsigned)c_begin, n32, d_cells);
    return DG_AFTER_LAUNCH();
}

cudaError_t k1_launch_fp64_rate_probe(int blocks, int iters, double* d_out, cudaStream_t stream)
{
    DG_KERNEL_LAUNCH(fp64_rate_probe_kernel, blocks, 256, 0, stream, 0.999999, 1.0e-6, iters, d_out);
    return DG_AFTER_LAUNCH();
}

cudaError_t k1_launch_fma_probe(double a, double b, double c, double* d_out, cudaStream_t stream)
{
    DG_KERNEL_LAUNCH(fma_probe_kernel, 1, 1, 0, stream, a, b, c, d_out);
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
