"""numpy restatement of the level-set contract of K6 (discregrid_b200/csrc/k6_isosurface.cu, DESIGN §3): lattice positions, validity,
the Kuhn split, edges, the case table with its orientation, the order of vertices and triangles and the vertex arithmetic (IEEE fp64, one
rounding per operation, no FMA).  Its input is the lattice values; get them from the library's host interpolate at Lattice.points() (lattice_values)."""
import numpy as np

DBL_MAX = np.finfo(np.float64).max

# pair codes of a tetrahedron's edges: 01 02 03 12 13 23
PAIRS = np.array([(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)], np.int64)
# the case table of the kernel's header, oriented for the even permutations: case -> triangles as pair codes
CASES = {
    1: [(0, 1, 2)], 2: [(0, 4, 3)], 3: [(1, 2, 4), (1, 4, 3)], 4: [(1, 3, 5)], 5: [(0, 5, 2), (0, 3, 5)], 6: [(0, 4, 5), (0, 5, 1)],
    7: [(2, 4, 5)], 8: [(2, 5, 4)], 9: [(0, 1, 5), (0, 5, 4)], 10: [(0, 5, 3), (0, 2, 5)], 11: [(1, 5, 3)], 12: [(1, 3, 4), (1, 4, 2)],
    13: [(0, 3, 4)], 14: [(0, 2, 1)],
}
NTRI = np.array([len(CASES.get(m, [])) for m in range(16)], np.int64)
TABLE = np.zeros((16, 2, 3), np.int64)
for _m, _tris in CASES.items():
    for _k, _t in enumerate(_tris):
        TABLE[_m, _k] = _t
# permutations of (0, 1, 2) in lexicographic order; odd ones swap the 2nd and 3rd vertex of every triangle
PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]
ODD = np.array([False, True, True, False, False, True])
# tetrahedron t's corners as cell-corner masks (bit 0 = +x, bit 1 = +y, bit 2 = +z)
TET = np.array([[0, 1 << p[0], (1 << p[0]) | (1 << p[1]), 7] for p in PERMS], np.int64)
# direction d of an edge from the corner mask of its offset, and back
DIR_OF_MASK = np.array([-1, 0, 1, 3, 2, 4, 5, 6], np.int64)
MASK_OF_DIR = np.array([1, 2, 4, 3, 5, 6, 7], np.int64)


class Lattice:
    def __init__(self, mn, mx, cell, res, s):
        self.mn, self.mx, self.cell = (np.asarray(a, np.float64) for a in (mn, mx, cell))
        self.s = int(s)
        self.np = np.array([self.s * int(r) + 1 for r in res], np.int64)
        self.n_points = int(np.prod(self.np))
        self.n_cells = int(np.prod(self.np - 1))

    @classmethod
    def of_grid(cls, grid, s):
        d = grid._desc
        return cls(d.domain_min[:], d.domain_max[:], d.cell_size[:], d.resolution[:], s)

    def coord(self, a, i):
        """x_a = mn + cell * (I / s), clamped to mx"""
        i = np.asarray(i, np.int64)
        x = self.mn[a] + self.cell[a] * (i.astype(np.float64) / float(self.s))
        return np.where(x > self.mx[a], self.mx[a], x)

    def lin(self, I, J, K):
        return I + self.np[0] * (J + self.np[1] * K)

    def unlin(self, l):
        l = np.asarray(l, np.int64)
        return l % self.np[0], (l // self.np[0]) % self.np[1], l // (self.np[0] * self.np[1])

    def points(self, begin=0, end=None):
        end = self.n_points if end is None else end
        I, J, K = self.unlin(np.arange(begin, end, dtype=np.int64))
        return np.stack([self.coord(0, I), self.coord(1, J), self.coord(2, K)], axis=1)

    def corner_offset(self, m):
        m = np.asarray(m, np.int64)
        return (m & 1) + self.np[0] * (((m >> 1) & 1) + self.np[1] * (m >> 2))


def lattice_values(grid, field_id, L, chunk=1 << 22):
    """f_P: the host interpolate of the field at the lattice points"""
    out = np.empty(L.n_points)
    for b in range(0, L.n_points, chunk):
        e = min(L.n_points, b + chunk)
        out[b:e] = grid.interpolate(field_id, L.points(b, e))
    return out


def _cell_edges(L, valid, neg, c0, c1):
    """edge ids of the triangles of lattice cells [c0, c1), (m, 3), in (cell, t, table position) order, and the cell of each triangle"""
    m0, m1 = L.np[0] - 1, L.np[1] - 1
    c = np.arange(c0, c1, dtype=np.int64)
    l0 = L.lin(c % m0, (c // m0) % m1, c // (m0 * m1))
    off = L.corner_offset(np.arange(8))
    corner_valid = valid[l0[:, None] + off[None, :]]                       # (cells, 8)
    corner_neg = neg[l0[:, None] + off[None, :]].astype(np.uint8)
    emits = corner_valid[:, TET].all(axis=2)                               # (cells, 6)
    tn = corner_neg[:, TET]                                                # (cells, 6, 4)
    case = tn[..., 0] | (tn[..., 1] << 1) | (tn[..., 2] << 2) | (tn[..., 3] << 3)
    ntri = np.where(emits, NTRI[case], 0)
    cc, tt = np.nonzero(ntri)                                              # C order: by cell, then t
    case = case[cc, tt]
    nt = ntri[cc, tt]
    tris = TABLE[case]                                                     # (k, 2, 3) pair codes
    keep = np.arange(2)[None, :] < nt[:, None]                             # (k, 2)
    rows = np.arange(len(tt))[:, None, None]
    lo = TET[tt][rows, PAIRS[tris][..., 0]]                                # corner masks of each edge's lower / upper vertex
    hi = TET[tt][rows, PAIRS[tris][..., 1]]
    eid = 7 * (l0[cc][:, None, None] + L.corner_offset(lo)) + DIR_OF_MASK[lo ^ hi]
    odd = ODD[tt]
    eid[odd] = eid[odd][:, :, [0, 2, 1]]
    return eid[keep], np.broadcast_to(c[cc][:, None], keep.shape)[keep]


def _classify(f, iso):
    f = np.asarray(f, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return (np.abs(f) <= DBL_MAX) & (f != DBL_MAX), f < float(iso)


def _vertices(L, uniq, fp, fq, iso):
    """vertex arithmetic on the edges uniq: t = (iso - f_p) / (f_q - f_p), x = x_p + t * (x_q - x_p)"""
    lp = uniq // 7
    dm = MASK_OF_DIR[uniq % 7]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        t = (float(iso) - fp) / (fq - fp)
        ip = L.unlin(lp)
        V = np.empty((len(uniq), 3))
        for a in range(3):
            xp = L.coord(a, ip[a])
            xq = L.coord(a, ip[a] + ((dm >> a) & 1))
            V[:, a] = xp + t * (xq - xp)
    return V


def extract(L, f, iso, chunk=1 << 21):
    """(vertices (n, 3) float64, triangles (m, 3) uint32) of the contract, from the lattice values f[Np]"""
    f = np.asarray(f, np.float64)
    valid, neg = _classify(f, iso)
    eid = np.concatenate([_cell_edges(L, valid, neg, b, min(L.n_cells, b + chunk))[0] for b in range(0, L.n_cells, chunk)] or
                         [np.zeros((0, 3), np.int64)])
    uniq, inv = np.unique(eid.reshape(-1), return_inverse=True)           # vertices by increasing edge id
    T = inv.reshape(-1, 3).astype(np.uint32)
    lp = uniq // 7
    lq = lp + L.corner_offset(MASK_OF_DIR[uniq % 7])
    return _vertices(L, uniq, f[lp], f[lq], iso), T


def extract_windows(L, windows, iso):
    """extract() restricted to the lattice cells inside index boxes: windows = [(lo, hi, f_box)], lo and hi the first and last lattice
    point of the box per axis, f_box the values of the box's points (I fastest).  Lattice points, edge ids, cells and coordinates stay
    those of L, so when no tetrahedron outside the boxes changes sign or is invalid next to a crossing (and the boxes share no lattice
    cell), the result equals extract(L, f, iso) of the whole lattice, without its values.  -> (V, T, the edge id of every vertex)"""
    eids, cells, lins, vals = [], [], [], []
    for lo, hi, fb in windows:
        lo, hi = np.asarray(lo, np.int64), np.asarray(hi, np.int64)
        W = Lattice(np.zeros(3), np.zeros(3), np.zeros(3), hi - lo, 1)       # the box's own numbering
        valid, neg = _classify(fb, iso)
        e, c = _cell_edges(W, valid, neg, 0, W.n_cells)
        I, J, K = W.unlin(e // 7)
        eids.append(7 * L.lin(I + lo[0], J + lo[1], K + lo[2]) + e % 7)
        m0, m1 = W.np[0] - 1, W.np[1] - 1
        g0, g1 = L.np[0] - 1, L.np[1] - 1
        cells.append(c % m0 + lo[0] + g0 * ((c // m0) % m1 + lo[1] + g1 * (c // (m0 * m1) + lo[2])))
        I, J, K = W.unlin(np.arange(W.n_points))
        lins.append(L.lin(I + lo[0], J + lo[1], K + lo[2]))
        vals.append(np.asarray(fb, np.float64))
    eid = np.concatenate(eids or [np.zeros((0, 3), np.int64)])
    eid = eid[np.argsort(np.concatenate(cells or [np.zeros(0, np.int64)]), kind="stable")]   # triangles by cell, then t and table position
    uniq, inv = np.unique(eid.reshape(-1), return_inverse=True)
    lin, val = np.concatenate(lins or [np.zeros(0, np.int64)]), np.concatenate(vals or [np.zeros(0)])
    order = np.argsort(lin)
    lin, val = lin[order], val[order]
    lp = uniq // 7
    lq = lp + L.corner_offset(MASK_OF_DIR[uniq % 7])
    fp, fq = val[np.searchsorted(lin, lp)], val[np.searchsorted(lin, lq)]
    return _vertices(L, uniq, fp, fq, iso), inv.reshape(-1, 3).astype(np.uint32), uniq


def case_counts(L, f, iso, chunk=1 << 21):
    """how often each case (the 4-bit negative mask) occurs among the tetrahedra whose four vertices are valid: (16, 2) counts, column 0
    the even permutations (t = 0, 3, 4), column 1 the odd ones"""
    valid, neg = _classify(f, iso)
    out = np.zeros((16, 2), np.int64)
    m0, m1 = L.np[0] - 1, L.np[1] - 1
    off = L.corner_offset(np.arange(8))
    for b in range(0, L.n_cells, chunk):
        c = np.arange(b, min(L.n_cells, b + chunk), dtype=np.int64)
        l0 = L.lin(c % m0, (c // m0) % m1, c // (m0 * m1))
        cv = valid[l0[:, None] + off[None, :]][:, TET].all(axis=2)
        tn = neg[l0[:, None] + off[None, :]].astype(np.int64)[:, TET]
        case = tn[..., 0] | (tn[..., 1] << 1) | (tn[..., 2] << 2) | (tn[..., 3] << 3)
        for odd in (0, 1):
            sel = cv & (ODD[None, :] == bool(odd))
            out[:, odd] += np.bincount(case[sel], minlength=16)
    return out


# ---- mesh checks -------------------------------------------------------------------------------------------------------------------
def directed_edges(T):
    T = np.asarray(T, np.int64)
    return np.concatenate([T[:, [0, 1]], T[:, [1, 2]], T[:, [2, 0]]])


def edge_use(T):
    """(every undirected edge used by exactly two triangles, every directed edge used once): closed and consistently oriented"""
    d = directed_edges(T)
    und = np.sort(d, axis=1)
    _, cu = np.unique(und, axis=0, return_counts=True)
    _, cd = np.unique(d, axis=0, return_counts=True)
    return bool(len(cu) and (cu == 2).all()), bool(len(cd) and (cd == 1).all())


def edge_use_counts(T):
    und = np.sort(directed_edges(T), axis=1)
    _, cu = np.unique(und, axis=0, return_counts=True)
    return np.bincount(cu)


def euler_characteristic(V, T):
    und = np.unique(np.sort(directed_edges(T), axis=1), axis=0)
    used = np.unique(np.asarray(T, np.int64))
    return len(used) - len(und) + len(T)


def signed_volume(V, T):
    T = np.asarray(T, np.int64)
    p0, p1, p2 = V[T[:, 0]], V[T[:, 1]], V[T[:, 2]]
    return float(np.einsum("ij,ij->i", p0, np.cross(p1, p2)).sum() / 6.0)


def normals(V, T):
    T = np.asarray(T, np.int64)
    p0, p1, p2 = V[T[:, 0]], V[T[:, 1]], V[T[:, 2]]
    return np.cross(p1 - p0, p2 - p0)
