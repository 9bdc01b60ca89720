// K7: the first crossing of a level set {phi = iso} along each of n rays (or segments), isolated cell by cell.  One thread per ray.
//
// The reference has no such function, so this contract is the library's own.  tests/raycast_ref.py restates it in numpy and the tests compare
// t_lo, t_hi and status bit for bit.
//
// Why it works.  Inside one grid cell the interpolant restricted to a line is a polynomial of degree <= 5 in t (corner functions: a quadratic
// times a trilinear term; edge functions: a cubic times a bilinear term).  Six samples of a piece of line inside one cell therefore determine
// the restriction, and its Bernstein coefficients bound it (the polynomial is a convex combination of them).  A piece whose samples and
// coefficients all lie on one side of iso cannot cross it, whatever the field is (SDF, density map, user function): no Lipschitz bound and no
// step size are involved.
//
// Inputs.  A field; rays i = 0..n-1 with origin o[3] and direction d[3]; iso finite; t_min <= t_max, neither NaN, either may be infinite.  A
//   segment x0 -> x1 is the ray (x0, x1 - x0) with t in [0, 1].
// Samples.  x_a(t) = o_a + t * d_a (no FMA), clamped to [mn_a, mx_a] (the clamp keeps the rounding at the domain entry from making boundary
//   samples invalid).  f(t) has the bits of the value-only dg_interpolate_batch at x(t).  A value is valid iff it is finite and != DBL_MAX; it
//   is negative iff f < iso (strict), as in K6.
// Clip.  The ray misses if o or d is not finite, or d = 0.  For each axis with d_a != 0: u = (mn_a - o_a) / d_a, v = (mx_a - o_a) / d_a,
//   lo_a = u < v ? u : v, hi_a = u < v ? v : u; an axis with d_a == 0 misses unless mn_a <= o_a <= mx_a.  t_enter = t_min, then for a = 0, 1,
//   2: t_enter = t_enter < lo_a ? lo_a : t_enter; t_exit = t_max, then t_exit = hi_a < t_exit ? hi_a : t_exit.  The ray misses unless both
//   are finite and t_enter < t_exit.
// Segments.  Breakpoints: t_enter, t_exit, and every t_{a,m} = (p_{a,m} - o_a) / d_a with t_enter < t_{a,m} < t_exit, where
//   p_{a,m} = mn_a + (double)m * cell_a, m = 1..n_a - 1 (the `lo` values of K2's axis table).  Sorted, duplicates merged; segments are
//   consecutive pairs, visited in increasing t (at most nx + ny + nz per ray).
// Nodes.  A node [a, b] has six samples s_0 = a, s_5 = b, s_k = a + (b - a) * w_k with w_k = (double)k / 5.0 (k = 1..4), values F_k = f(s_k),
//   and Bernstein coefficients beta = M F, M the inverse of the 6 x 6 Bernstein collocation matrix at k/5 (entries: the doubles nearest the
//   exact rationals, row sums of |M| <= 33.54); row j is the left fold beta_j = M_j0 * F_0, then beta_j = beta_j + M_jk * F_k for k = 1..5.
//   Rows 0 and 5 are F_0 and F_5 themselves.
// Pruning.  A node is pruned iff one of its samples is invalid, or all F_k and all beta_j lie on one side (all >= iso, or all < iso).  A NaN
//   beta lies on neither side.  Since the samples are part of the test, a side change the samples show is never pruned.
// Descent.  Depth 0 is a segment.  A node that is not pruned, has depth < D (K7_DEPTH = 5) and whose midpoint m = a + (b - a) * 0.5 satisfies
//   a < m < b has the children [a, m] and [m, b], the left one first.  Otherwise (not pruned) it is a leaf: the first k with F_k and F_{k+1}
//   on different sides is bisected on [s_k, s_{k+1}] and reported; with no such k (a tangency, or two crossings closer than the leaf's
//   sample spacing, 1/(5 * 2^D) of the segment) nothing is reported and the walk continues.
// Bisection.  Repeat: m = a + (b - a) * 0.5; stop unless a < m < b; stop if f(m) is invalid; replace a (if f(m) is on a's side) or else b by m.
// Outputs.  t_lo, t_hi: the final bracket.  status = DG_RAY_ENTER (1) when f(t_lo) is non-negative and f(t_hi) negative, DG_RAY_LEAVE (2) for
//   the reverse; a ray with no crossing reported gives DG_RAY_MISS (0) and t_lo = t_hi = +inf.  A ray that starts inside reports its first
//   LEAVE.
//
// Implementation (the choices below change no result).  Each lane stages the 32 coefficients of the cell of its last evaluation in its own
// 272-byte shared-memory slot (256 bytes + 16 of bank padding, as K2) and refetches only when an evaluation lands in another cell, so a face
// sample whose lookup K2 assigns to the neighbour gets the neighbour's block.  The value arithmetic is K2's value-only expression sequence,
// copied (k2_interp.cu is left unchanged; the tests pin the copy to K2 bit for bit).  A segment's first sample is its predecessor's last one;
// a node's first sample is its parent's first (left child) or the previous node's last (right child), so a node costs five evaluations.
// The axis breakpoints are produced in increasing t by one cursor per axis, started from an estimate of the entry cell and corrected on the
// exact t values (t_{a,m} is monotone in m), and merged.  The right siblings of the descent sit on a stack of at most D doubles.
#include "k7_raycast.h"
#include "dg_launch.h"

#include <cfloat>
#include <climits>
#include <cmath>

namespace dgb {
namespace {

constexpr int K7_SLOT = 17;                           // double2 per lane: 256-byte block + 16 bytes of padding (bank spreading)
constexpr int K7_MISS = 0, K7_ENTER = 1, K7_LEAVE = 2;        // DG_RAY_MISS, DG_RAY_ENTER, DG_RAY_LEAVE of the C-ABI

// finite and not the sentinel
__device__ __forceinline__ bool k7_valid(double v) { return fabs(v) <= DBL_MAX && v != DBL_MAX; }

struct Ray {
    double o[3], d[3];
};

// the field and the lane's staged block
struct Eval {
    const FieldDev* f;
    double2* slot;
    unsigned cached;                                  // cell whose block is in the slot (UINT_MAX: none)
};

// f(t): K2's value-only interpolate (k2_interp.cu, interpolate_kernel<false, false>) at the clamped x(t)
__device__ __forceinline__ double k7_value(Eval& e, const Ray& r, double t)
{
    const GridDev& g = e.f->g;
    double p[3];
    for (int a = 0; a < 3; a++) {
        const double x = r.o[a] + t * r.d[a];
        p[a] = x < g.mn[a] ? g.mn[a] : (x > g.mx[a] ? g.mx[a] : x);
    }
    const double x = p[0], y = p[1], z = p[2];
    if (!((g.mn[0] <= x) && (x <= g.mx[0]) && (g.mn[1] <= y) && (y <= g.mx[1]) && (g.mn[2] <= z) && (z <= g.mx[2]))) return DBL_MAX;
    unsigned mi0 = (unsigned)((x - g.mn[0]) * g.inv[0]);
    unsigned mi1 = (unsigned)((y - g.mn[1]) * g.inv[1]);
    unsigned mi2 = (unsigned)((z - g.mn[2]) * g.inv[2]);
    if (mi0 >= g.n[0]) mi0 = g.n[0] - 1;
    if (mi1 >= g.n[1]) mi1 = g.n[1] - 1;
    if (mi2 >= g.n[2]) mi2 = g.n[2] - 1;
    const unsigned i = g.n[1] * g.n[0] * mi2 + g.n[0] * mi1 + mi0;
    const unsigned cell = e.f->cell_map ? __ldg(e.f->cell_map + i) : i;
    if (cell == UINT_MAX) return DBL_MAX;                                  // removed by reduceField
    if (cell != e.cached) {
        const double2* src = reinterpret_cast<const double2*>(e.f->packed + (size_t)cell * 32);
#pragma unroll
        for (int k = 0; k < 16; k++) e.slot[k] = __ldg(src + k);
        e.cached = cell;
    }
    const double2 tx = __ldg(e.f->tab + mi0), ty = __ldg(e.f->tab + g.n[0] + mi1), tz = __ldg(e.f->tab + g.n[0] + g.n[1] + mi2);
    const double X = tx.x * x - tx.y, Y = ty.x * y - ty.y, Z = tz.x * z - tz.y;
    const double x2 = X * X, y2 = Y * Y, z2 = Z * Z;
    const double _1mx = 1.0 - X, _1my = 1.0 - Y, _1mz = 1.0 - Z;
    const double _1px = 1.0 + X, _1py = 1.0 + Y, _1pz = 1.0 + Z;
    const double _1m3x = 1.0 - 3.0 * X, _1m3y = 1.0 - 3.0 * Y, _1m3z = 1.0 - 3.0 * Z;
    const double _1p3x = 1.0 + 3.0 * X, _1p3y = 1.0 + 3.0 * Y, _1p3z = 1.0 + 3.0 * Z;
    const double mxmy = _1mx * _1my, mxpy = _1mx * _1py, pxmy = _1px * _1my, pxpy = _1px * _1py;
    const double mxmz = _1mx * _1mz, mxpz = _1mx * _1pz, pxmz = _1px * _1mz, pxpz = _1px * _1pz;
    const double mymz = _1my * _1mz, mypz = _1my * _1pz, pymz = _1py * _1mz, pypz = _1py * _1pz;
    const double _1mx2 = 1.0 - x2, _1my2 = 1.0 - y2, _1mz2 = 1.0 - z2;
    const double facc = 1.0 / 64.0 * (9.0 * (x2 + y2 + z2) - 19.0);
    const double fx = 9.0 / 64.0 * _1mx2, fy = 9.0 / 64.0 * _1my2, fz = 9.0 / 64.0 * _1mz2;
    const double fxm = fx * _1m3x, fxp = fx * _1p3x, fym = fy * _1m3y, fyp = fy * _1p3y, fzm = fz * _1m3z, fzp = fz * _1p3z;
    const double2* cb = e.slot;
    double phi = 0.0;
    bool missing = false;
#define K7_TERM(cj, n)                   \
    {                                    \
        const double c_ = (cj);          \
        missing |= (c_ == DBL_MAX);      \
        phi = phi + c_ * (n);            \
    }
    double2 c;
    c = cb[0];  K7_TERM(c.x, facc * mxmy * _1mz) K7_TERM(c.y, facc * pxmy * _1mz)
    c = cb[1];  K7_TERM(c.x, facc * mxpy * _1mz) K7_TERM(c.y, facc * pxpy * _1mz)
    c = cb[2];  K7_TERM(c.x, facc * mxmy * _1pz) K7_TERM(c.y, facc * pxmy * _1pz)
    c = cb[3];  K7_TERM(c.x, facc * mxpy * _1pz) K7_TERM(c.y, facc * pxpy * _1pz)
    c = cb[4];  K7_TERM(c.x, fxm * mymz) K7_TERM(c.y, fxp * mymz)
    c = cb[5];  K7_TERM(c.x, fxm * mypz) K7_TERM(c.y, fxp * mypz)
    c = cb[6];  K7_TERM(c.x, fxm * pymz) K7_TERM(c.y, fxp * pymz)
    c = cb[7];  K7_TERM(c.x, fxm * pypz) K7_TERM(c.y, fxp * pypz)
    c = cb[8];  K7_TERM(c.x, fym * mxmz) K7_TERM(c.y, fyp * mxmz)
    c = cb[9];  K7_TERM(c.x, fym * pxmz) K7_TERM(c.y, fyp * pxmz)
    c = cb[10]; K7_TERM(c.x, fym * mxpz) K7_TERM(c.y, fyp * mxpz)
    c = cb[11]; K7_TERM(c.x, fym * pxpz) K7_TERM(c.y, fyp * pxpz)
    c = cb[12]; K7_TERM(c.x, fzm * mxmy) K7_TERM(c.y, fzp * mxmy)
    c = cb[13]; K7_TERM(c.x, fzm * mxpy) K7_TERM(c.y, fzp * mxpy)
    c = cb[14]; K7_TERM(c.x, fzm * pxmy) K7_TERM(c.y, fzp * pxmy)
    c = cb[15]; K7_TERM(c.x, fzm * pxpy) K7_TERM(c.y, fzp * pxpy)
#undef K7_TERM
    return missing ? DBL_MAX : phi;
}

// the breakpoints of one axis in increasing t: t_{a,m} for m = first, first + step, ... while t < t_exit
struct Cursor {
    int m, step, last;
    double p0, cell, o, d;
    double t;                                         // current breakpoint, +inf when exhausted
};

__device__ __forceinline__ double cursor_t(const Cursor& c, int m) { return ((c.p0 + (double)m * c.cell) - c.o) / c.d; }

__device__ __forceinline__ void cursor_settle(Cursor& c, double t_exit)
{
    const bool in = c.m >= 1 && c.m <= c.last;
    const double t = in ? cursor_t(c, c.m) : INFINITY;
    c.t = t < t_exit ? t : INFINITY;
}

// first m (in increasing t) with t_{a,m} > t_enter: an estimate from the entry position, corrected on the exact values
__device__ __forceinline__ void cursor_init(Cursor& c, const GridDev& g, int a, const Ray& r, double t_enter, double t_exit)
{
    c.last = (int)g.n[a] - 1;
    c.p0 = g.mn[a]; c.cell = g.cell[a]; c.o = r.o[a]; c.d = r.d[a];
    c.step = r.d[a] > 0.0 ? 1 : -1;
    if (r.d[a] == 0.0 || c.last < 1) { c.m = 0; c.t = INFINITY; return; }
    const double e = ((r.o[a] + t_enter * r.d[a]) - g.mn[a]) * g.inv[a];
    int m = !(e >= 1.0) ? 1 : (e >= (double)c.last ? c.last : (int)e);
    if (c.step > 0) {
        while (m > 1 && cursor_t(c, m - 1) > t_enter) m--;
        while (m <= c.last && !(cursor_t(c, m) > t_enter)) m++;
    } else {
        while (m < c.last && cursor_t(c, m + 1) > t_enter) m++;
        while (m >= 1 && !(cursor_t(c, m) > t_enter)) m--;
    }
    c.m = m;
    cursor_settle(c, t_exit);
}

// advances past every breakpoint equal to b (duplicates are merged)
__device__ __forceinline__ void cursor_pass(Cursor& c, double b, double t_exit)
{
    while (c.t == b) { c.m += c.step; cursor_settle(c, t_exit); }
}

__device__ __forceinline__ bool k7_neg(double v, double iso) { return v < iso; }

// bisection on [lo, hi], whose ends lie on different sides (neg_lo: the side of lo)
__device__ __forceinline__ void k7_bisect(Eval& e, const Ray& r, double iso, double& lo, double& hi, bool neg_lo)
{
    for (;;) {
        const double m = lo + (hi - lo) * 0.5;
        if (!(lo < m && m < hi)) return;
        const double v = k7_value(e, r, m);
        if (!k7_valid(v)) return;
        if (k7_neg(v, iso) == neg_lo) lo = m; else hi = m;
    }
}

// Bernstein coefficient j (1..4) of the six samples: row j of M as a left fold
__device__ __forceinline__ double k7_beta(int j, const double F[6])
{
    // M = inverse of the Bernstein collocation matrix at k/5, rows 1..4 (rows 0 and 5 are the unit rows)
    const double M[4][6] = {
        {-1.2833333333333334, 5.0, -5.0, 3.3333333333333335, -1.25, 0.2},
        {1.1208333333333333, -6.041666666666667, 12.291666666666666, -9.583333333333334, 3.8541666666666665, -0.6416666666666667},
        {-0.6416666666666667, 3.8541666666666665, -9.583333333333334, 12.291666666666666, -6.041666666666667, 1.1208333333333333},
        {0.2, -1.25, 3.3333333333333335, -5.0, 5.0, -1.2833333333333334},
    };
    double b = M[j - 1][0] * F[0];
#pragma unroll
    for (int k = 1; k < 6; k++) b = b + M[j - 1][k] * F[k];
    return b;
}

// walks segment [a, b] whose f(a) = fa; returns true with the bracket and status when it reports a crossing, else leaves f(b) in fa
__device__ __forceinline__ bool k7_segment(Eval& e, const Ray& r, double iso, double a, double b, double& fa, double& lo, double& hi, int& status)
{
    double stk[K7_DEPTH];                                                   // ends of the pending right siblings
    unsigned dstk = 0;                                                      // and their depths, 3 bits each
    int sp = 0, dep = 0;
    for (;;) {
        double F[6];
        F[0] = fa;
        const double w = b - a;
#pragma unroll
        for (int k = 1; k < 5; k++) F[k] = k7_value(e, r, a + w * ((double)k / 5.0));
        F[5] = k7_value(e, r, b);
        bool pruned = false;
#pragma unroll
        for (int k = 0; k < 6; k++) pruned |= !k7_valid(F[k]);
        if (!pruned) {
            bool ge = true, lt = true;
#pragma unroll
            for (int k = 0; k < 6; k++) { ge &= F[k] >= iso; lt &= F[k] < iso; }
#pragma unroll
            for (int j = 1; j < 5; j++) { const double bj = k7_beta(j, F); ge &= bj >= iso; lt &= bj < iso; }
            pruned = ge || lt;
        }
        if (!pruned) {
            const double m = a + (b - a) * 0.5;
            if (dep < K7_DEPTH && a < m && m < b) {
                stk[sp++] = b;
                dstk = (dstk << 3) | (unsigned)++dep;
                b = m;
                continue;
            }
            for (int k = 0; k < 5; k++) {                                   // leaf: the first side change of the samples
                if (k7_neg(F[k], iso) != k7_neg(F[k + 1], iso)) {
                    lo = k == 0 ? a : a + w * ((double)k / 5.0);
                    hi = k == 4 ? b : a + w * ((double)(k + 1) / 5.0);
                    const bool neg_lo = k7_neg(F[k], iso);
                    k7_bisect(e, r, iso, lo, hi, neg_lo);
                    status = neg_lo ? K7_LEAVE : K7_ENTER;
                    return true;
                }
            }
        }
        fa = F[5];                                                          // next node: the right sibling of the nearest ancestor
        if (sp == 0) return false;
        a = b;
        b = stk[--sp];
        dep = (int)(dstk & 7u);
        dstk >>= 3;
    }
}

__global__ void __launch_bounds__(K7_THREADS)
raycast_kernel(FieldDev f, const double* __restrict__ o_in, const double* __restrict__ d_in, unsigned long long n, double iso, double t_min,
               double t_max, double* __restrict__ t_lo_out, double* __restrict__ t_hi_out, int* __restrict__ status_out)
{
    __shared__ __align__(16) double2 stage[K7_THREADS * K7_SLOT];
    const unsigned long long q = (unsigned long long)blockIdx.x * K7_THREADS + threadIdx.x;
    if (q >= n) return;
    const GridDev& g = f.g;
    Ray r;
    // ---- clip
    bool finite = true, nonzero = false;
    for (int a = 0; a < 3; a++) {
        r.o[a] = o_in[3 * q + a]; r.d[a] = d_in[3 * q + a];
        finite &= fabs(r.o[a]) <= DBL_MAX && fabs(r.d[a]) <= DBL_MAX;
        nonzero |= r.d[a] != 0.0;
    }
    double t_enter = t_min, t_exit = t_max;
    bool ok = finite && nonzero;
    for (int a = 0; a < 3 && ok; a++) {
        if (r.d[a] != 0.0) {
            const double u = (g.mn[a] - r.o[a]) / r.d[a], v = (g.mx[a] - r.o[a]) / r.d[a];
            const double lo = u < v ? u : v, hi = u < v ? v : u;
            t_enter = t_enter < lo ? lo : t_enter;
            t_exit = hi < t_exit ? hi : t_exit;
        } else if (!(g.mn[a] <= r.o[a] && r.o[a] <= g.mx[a])) {
            ok = false;
        }
    }
    ok = ok && fabs(t_enter) <= DBL_MAX && fabs(t_exit) <= DBL_MAX && t_enter < t_exit;
    double lo = INFINITY, hi = INFINITY;
    int status = K7_MISS;
    if (ok) {
        Eval e{&f, stage + threadIdx.x * K7_SLOT, UINT_MAX};
        Cursor c[3];
        for (int a = 0; a < 3; a++) cursor_init(c[a], g, a, r, t_enter, t_exit);
        double a0 = t_enter, fa = k7_value(e, r, t_enter);
        for (;;) {
            double b = c[0].t < c[1].t ? c[0].t : c[1].t;
            b = c[2].t < b ? c[2].t : b;
            b = b < t_exit ? b : t_exit;
            for (int a = 0; a < 3; a++) cursor_pass(c[a], b, t_exit);
            if (k7_segment(e, r, iso, a0, b, fa, lo, hi, status)) break;
            if (b == t_exit) break;
            a0 = b;
        }
        if (status == K7_MISS) { lo = INFINITY; hi = INFINITY; }
    }
    t_lo_out[q] = lo;
    t_hi_out[q] = hi;
    status_out[q] = status;
}

}  // namespace

cudaError_t k7_launch_raycast(const FieldDev& f, const double* d_o, const double* d_d, uint64_t n, double iso, double t_min, double t_max,
                              double* d_t_lo, double* d_t_hi, int32_t* d_status, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((n + K7_THREADS - 1) / K7_THREADS);
    DG_KERNEL_LAUNCH(raycast_kernel, blocks, K7_THREADS, 0, stream, f, d_o, d_d, (unsigned long long)n, iso, t_min, t_max, d_t_lo, d_t_hi,
                     (int*)d_status);
    return DG_AFTER_LAUNCH();
}

}  // namespace dgb
