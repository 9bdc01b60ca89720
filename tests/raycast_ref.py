"""Numpy restatement of K7's contract (discregrid_b200/csrc/k7_raycast.cu): the first crossing of {phi = iso} along rays -- clip, segments,
samples, the Bernstein matrix M, pruning, descent and bisection -- in IEEE fp64 Python floats (one rounding per operation, no FMA).

The field enters only through an evaluator x[n, 3] -> f[n] (the tests pass the library's host interpolate, which is pinned to the reference
class elsewhere, or the device route of the same).  Every ray is a generator that asks for the values at a few points at a time; all rays
advance in lockstep, so one evaluator call serves every ray's request of a round.  The same walk counts segments, nodes and evaluations per
ray (for the benchmark's cost figures)."""
from fractions import Fraction
from math import comb

import numpy as np

DBL_MAX = float(np.finfo(np.float64).max)
INF = float("inf")
DEPTH = 5
MISS, ENTER, LEAVE = 0, 1, 2


def _bernstein_inverse():
    A = [[Fraction(comb(5, j)) * Fraction(k, 5) ** j * (1 - Fraction(k, 5)) ** (5 - j) for j in range(6)] for k in range(6)]
    M = [row[:] + [Fraction(int(i == j)) for j in range(6)] for i, row in enumerate(A)]
    for c in range(6):
        p = next(r for r in range(c, 6) if M[r][c] != 0)
        M[c], M[p] = M[p], M[c]
        M[c] = [x / M[c][c] for x in M[c]]
        for r in range(6):
            if r != c and M[r][c] != 0:
                f = M[r][c]
                M[r] = [a - f * b for a, b in zip(M[r], M[c])]
    return [row[6:] for row in M]


M_EXACT = _bernstein_inverse()
M = [[float(x) for x in row] for row in M_EXACT]          # the doubles nearest the exact rationals
W = [k / 5.0 for k in range(6)]                            # w_k = (double)k / 5.0


def valid(v):
    return abs(v) <= DBL_MAX and v != DBL_MAX              # finite and not the sentinel (NaN fails the first test)


class Grid:
    """the domain and cells of a grid: mn, mx, cell (3 floats each), n (3 ints)"""

    def __init__(self, mn, mx, cell, n):
        self.mn = [float(v) for v in mn]
        self.mx = [float(v) for v in mx]
        self.cell = [float(v) for v in cell]
        self.n = [int(v) for v in n]

    @classmethod
    def of_desc(cls, d):
        return cls(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.resolution[:])

    @classmethod
    def of_grid(cls, g):
        return cls.of_desc(g._desc)


def clip(g, o, d, t_min, t_max):
    """(t_enter, t_exit), or None for a miss"""
    if not all(abs(v) <= DBL_MAX for v in list(o) + list(d)) or all(v == 0.0 for v in d):
        return None
    te, tx = t_min, t_max
    for a in range(3):
        if d[a] != 0.0:
            u = (g.mn[a] - o[a]) / d[a]
            v = (g.mx[a] - o[a]) / d[a]
            lo, hi = (u, v) if u < v else (v, u)
            te = lo if te < lo else te
            tx = hi if hi < tx else tx
        elif not (g.mn[a] <= o[a] and o[a] <= g.mx[a]):
            return None
    if not (abs(te) <= DBL_MAX and abs(tx) <= DBL_MAX and te < tx):
        return None
    return te, tx


def breakpoints(g, o, d, te, tx):
    """the segment ends after t_enter, in increasing t, duplicates merged, ending with t_exit"""
    heads = []
    for a in range(3):
        if d[a] == 0.0:
            continue
        ts = [((g.mn[a] + float(m) * g.cell[a]) - o[a]) / d[a] for m in range(1, g.n[a])]
        ts = [t for t in (ts if d[a] > 0.0 else ts[::-1]) if te < t < tx]
        heads.append(ts)
    out = []
    while True:
        cand = [h[0] for h in heads if h]
        b = INF
        for t in cand:                                     # the first of equal heads in axis order wins, as the kernel's ternaries
            b = t if t < b else b
        b = b if b < tx else tx
        for h in heads:
            while h and h[0] == b:
                h.pop(0)
        out.append(b)
        if b == tx:
            return out


def position(g, o, d, t):
    p = []
    for a in range(3):
        x = o[a] + t * d[a]
        p.append(g.mn[a] if x < g.mn[a] else (g.mx[a] if x > g.mx[a] else x))
    return p


def _beta(j, F):
    b = M[j][0] * F[0]
    for k in range(1, 6):
        b = b + M[j][k] * F[k]
    return b


def _ray(g, o, d, iso, t_min, t_max, stats, bernstein=True):
    """generator: yields lists of positions, receives their values; returns (t_lo, t_hi, status)"""
    c = clip(g, o, d, t_min, t_max)
    if c is None:
        return INF, INF, MISS
    te, tx = c

    def f(ts):
        stats["evaluations"] += len(ts)
        return (yield [position(g, o, d, t) for t in ts])

    neg = lambda v: v < iso
    a = te
    fa = (yield from f([te]))[0]
    for b_seg in breakpoints(g, o, d, te, tx):
        stats["segments"] += 1
        b, depth, stack = b_seg, 0, []
        while True:
            stats["nodes"] += 1
            w = b - a
            s = [a] + [a + w * W[k] for k in range(1, 5)] + [b]
            F = [fa] + (yield from f(s[1:]))
            pruned = not all(valid(v) for v in F)
            if not pruned:
                vals = F + ([_beta(j, F) for j in range(1, 5)] if bernstein else [])
                pruned = all(v >= iso for v in vals) or all(v < iso for v in vals)
            if not pruned:
                m = a + (b - a) * 0.5
                if depth < DEPTH and a < m < b:
                    depth += 1
                    stack.append((b, depth))
                    b = m
                    continue
                for k in range(5):
                    if neg(F[k]) != neg(F[k + 1]):
                        lo, hi, neg_lo = s[k], s[k + 1], neg(F[k])
                        while True:
                            m = lo + (hi - lo) * 0.5
                            if not (lo < m < hi):
                                break
                            v = (yield from f([m]))[0]
                            if not valid(v):
                                break
                            if neg(v) == neg_lo:
                                lo = m
                            else:
                                hi = m
                        return lo, hi, (LEAVE if neg_lo else ENTER)
            fa = F[5]
            if not stack:
                break
            a, (b, depth) = b, stack.pop()
        a = b_seg
    return INF, INF, MISS


def raycast(g, evaluate, origins, directions, iso=0.0, t_min=0.0, t_max=INF, bernstein=True, with_stats=False):
    """(t_lo, t_hi, status) of every ray as the contract defines them; evaluate(x[n, 3]) -> f[n].  with_stats adds a dict of arrays
    segments, nodes, evaluations per ray.  bernstein=False prunes on the six samples alone (a plain sampled marcher, for comparison)."""
    O = np.ascontiguousarray(origins, np.float64).reshape(-1, 3)
    Dr = np.ascontiguousarray(directions, np.float64).reshape(-1, 3)
    n = len(O)
    t_lo, t_hi, status = np.full(n, INF), np.full(n, INF), np.zeros(n, np.int32)
    stats = [{"segments": 0, "nodes": 0, "evaluations": 0} for _ in range(n)]
    gens, want = {}, {}
    for i in range(n):
        gen = _ray(g, [float(v) for v in O[i]], [float(v) for v in Dr[i]], float(iso), float(t_min), float(t_max), stats[i], bernstein)
        try:
            want[i] = next(gen)
            gens[i] = gen
        except StopIteration as e:
            t_lo[i], t_hi[i], status[i] = e.value
    while gens:
        ids = list(gens)
        X = np.array([p for i in ids for p in want[i]], np.float64).reshape(-1, 3)
        vals = np.asarray(evaluate(X), np.float64)
        at = 0
        for i in ids:
            k = len(want[i])
            got = [float(v) for v in vals[at:at + k]]
            at += k
            try:
                want[i] = gens[i].send(got)
            except StopIteration as e:
                t_lo[i], t_hi[i], status[i] = e.value
                del gens[i], want[i]
    if with_stats:
        return t_lo, t_hi, status, {k: np.array([s[k] for s in stats]) for k in ("segments", "nodes", "evaluations")}
    return t_lo, t_hi, status
