"""Symmetric quasidefinite matrices whose assembly tree contains chosen fronts: the shapes at which the multifrontal
LDL^T's kernels switch code paths (pivot counts around the 4x4 register blocks, row counts around the 64-row tiles,
the 128-row R tasks, the 96-row big-front threshold and the 256-row solve slab; every kind of child record).

A matrix is built from dense blocks of vertices ("groups") coupled to each other; the elimination order is the order
in which the groups are listed.  Building blocks (the symbolic analysis with its default options, max_panel 64):
- a dense group of ns <= 64 vertices with no children becomes one front (a relaxed subtree);
- its rows into the parent are the separator vertices it is coupled to: a contiguous range of them lands
  contiguously in the parent front, a strided subset lands scattered;
- `lift` puts a dense 64-vertex group in front of a group, coupled to all of its columns: the group's subtree then
  exceeds relax_subtree (64), so it is no longer a relaxed subtree, and the relaxed merge of the two declines (the
  merge would add too many explicit zeros), so the group becomes a front above level 0;
- a lifted 64-vertex "blocker" coupled only to the separator's first vertex, placed right before the separator,
  stops the relaxed amalgamation along the separator's last-child chain (without it the separator absorbs the group
  before it);
- the separator is one dense group, split by the analysis into balanced panels of at most 64 columns: a chain.
The fronts that come out are read back from the symbolic analysis; nothing here assumes the tree.

Values: off-diagonals uniform in [-1, 1]; vertex v has a sign s_v and the diagonal s_v (1.1 rowsum_v + 1), rowsum_v
the sum of the magnitudes of row v's off-diagonals.  The matrix is strictly diagonally dominant, so elimination in
any order keeps every pivot's sign: nothing is regularised, the positive inertia is the number of + signs and the
condition number stays modest.  `flip` gives chosen vertices the opposite diagonal sign while their expected sign
stays: those pivots are regularised."""
import numpy as np


class Shape:
    """upper-triangular CSC (N, cp, rv, nz) with expected pivot signs ds and an elimination order perm (perm[k] =
    vertex eliminated k-th), plus the vertex sets of the named groups (labels as stored)"""

    def __init__(self, name, N, cp, rv, nz, ds, perm, groups):
        self.name, self.N, self.cp, self.rv, self.nz, self.ds, self.perm, self.groups = name, N, cp, rv, nz, ds, perm, groups

    def dense(self, dtype=np.float64):
        K = np.zeros((self.N, self.N), dtype)
        cols = np.repeat(np.arange(self.N), np.diff(self.cp))
        K[self.rv, cols] = self.nz
        K[cols, self.rv] = self.nz
        return K


class Builder:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.sizes, self.names, self.edges = [], [], []

    def group(self, ns, name=None):
        g = len(self.sizes)
        self.sizes.append(ns)
        self.names.append(name)
        self.edges.append((g, None, None, None))   # dense inside
        return g

    def couple(self, a, b, ia=None, ib=None):
        """couple vertices ia of group a (all when None) with vertices ib of group b"""
        self.edges.append((a, b, ia, ib))

    def lift(self, g):
        """a dense 64-vertex group coupled to all columns of g: g becomes a front above level 0"""
        h = self.group(64)
        self.couple(h, g)
        return h

    def build(self, name, order, minus=0.5, flip=()):
        """order: the groups in elimination order; minus: share of - signs; flip: (group, local index) pairs whose
        diagonal gets the sign opposite to its expected one (and whose couplings are scaled by 1e-4, so that the
        regularised pivot's tiny value does not blow up the pivots after it)"""
        assert sorted(order) == list(range(len(self.sizes)))
        start = np.zeros(len(self.sizes), np.int64)
        pos = 0
        for g in order:
            start[g] = pos
            pos += self.sizes[g]
        N = pos
        ids = lambda g, i: start[g] + (np.arange(self.sizes[g]) if i is None else np.asarray(i, np.int64))
        r, c = [], []
        for a, b, ia, ib in self.edges:
            if b is None:
                v = ids(a, None)
                I, J = np.meshgrid(v, v, indexing="ij")
                keep = I < J
                r.append(I[keep]); c.append(J[keep])
            else:
                I, J = np.meshgrid(ids(a, ia), ids(b, ib), indexing="ij")
                r.append(I.ravel()); c.append(J.ravel())
        r, c = np.concatenate(r), np.concatenate(c)
        lo, hi = np.minimum(r, c), np.maximum(r, c)
        key = np.unique(lo * N + hi)
        lo, hi = key // N, key % N
        val = self.rng.uniform(-1.0, 1.0, size=len(key))
        fl = np.array([start[g] + i for g, i in flip], np.int64)
        val[np.isin(lo, fl) | np.isin(hi, fl)] *= 1e-4
        rowsum = np.zeros(N)
        np.add.at(rowsum, lo, np.abs(val))
        np.add.at(rowsum, hi, np.abs(val))
        sign = np.where(self.rng.random(N) < minus, -1, 1).astype(np.int8)
        diag = sign * (1.1 * rowsum + 1.0)
        diag[fl] = -diag[fl]
        # random labels: the vertex eliminated k-th is stored as label[k]
        label = self.rng.permutation(N)
        R = np.concatenate([label[lo], label])
        C = np.concatenate([label[hi], label])
        V = np.concatenate([val, diag])
        R, C = np.minimum(R, C), np.maximum(R, C)
        o = np.lexsort((R, C))
        R, C, V = R[o], C[o], V[o]
        cp = np.zeros(N + 1, np.int64)
        np.add.at(cp, C + 1, 1)
        cp = np.cumsum(cp)
        ds = np.empty(N, np.int8)
        ds[label] = sign
        groups = {nm: label[ids(g, None)] for g, nm in enumerate(self.names) if nm}
        groups.update({"flip%d" % k: label[[v]] for k, v in enumerate(fl)})
        return Shape(name, N, cp, R.astype(np.int64), V, ds, label.astype(np.int64), groups)


SEP = 300   # the separator: five panels of 60, a chain of wide fronts; nr up to 257 fits, and the blocker still blocks


def _spread(lo, hi, k):
    """k separator indices spread over [lo, hi), first and last included"""
    return np.unique(np.round(np.linspace(lo, hi - 1, k)).astype(np.int64))


def _blocked(b, sep, order):
    """the blocker and the separator after the groups in order.  The blocker is coupled to the separator's first
    vertex only and lifted: the postorder puts the children of a vertex in ascending subtree size, so the blocker's
    subtree (128 vertices, at least as large as any other child of the separator's first vertex, and later in the
    order) comes right before the separator, where it is the child the relaxed amalgamation looks at and declines"""
    blk = b.group(64)
    b.couple(blk, sep, None, [0])
    return order + [b.lift(blk), blk, sep]


def big_fronts(seed=1):
    """groups under one separator, at the (ns, nr) pairs where the factor and solve kernels switch paths"""
    b = Builder(seed)
    sep = b.group(SEP, "sep")
    order = []

    def block(ns, rows, lift, name):
        g = b.group(ns, name)
        b.couple(g, sep, None, rows)
        if lift:
            order.append(b.lift(g))
        order.append(g)
        return g

    # level 0: leaf1 / leafn / leafw leaves, the three k_factor_level classes, big fronts factored by D/R/T tasks
    block(1, np.arange(40, 135), False, "l0_1_95")        # k_factor_leaf1, nr 95
    block(1, np.arange(10, 106), False, "l0_1_96")        # big at level 0
    block(3, _spread(0, 200, 63), False, "l0_3_63")       # leafn, k_factor_level class 1
    block(5, np.arange(3, 8), False, "l0_5_5")            # k_factor_level class 0 (64-thread CTA)
    block(64, np.arange(0, 95), False, "l0_64_95")        # leafw, k_factor_level class 2
    block(9, np.arange(100, 197), False, "l0_9_97")       # big at level 0, leafw
    # above level 0: F tasks (nr < 96) and big fronts at every pivot count 1..9, 63, 64 and every row count boundary
    block(9, np.arange(150, 245), True, "f_9_95")
    block(2, _spread(0, 280, 40), True, "f_2_40")
    block(1, np.arange(0, 96), True, "d_1_96")
    block(2, np.arange(20, 117), True, "d_2_97")
    block(3, _spread(0, 300, 127), True, "d_3_127")
    block(4, np.arange(50, 178), True, "d_4_128")
    block(5, _spread(0, 299, 257), True, "d_5_257")       # narrow front, nr > 256
    block(6, np.arange(0, 129), True, "d_6_129")
    block(7, _spread(1, 300, 255), True, "d_7_255")
    block(8, np.arange(44, 300), True, "d_8_256")
    block(9, _spread(0, 300, 257), True, "d_9_257")       # wide, nr > 256 rows: a row task beyond the slab cap
    block(63, np.arange(10, 106), True, "d_63_96")
    block(64, np.arange(100, 229), True, "d_64_129")      # wide: partial slab and row tasks
    block(64, np.arange(30, 286), True, "d_64_256")
    block(33, _spread(0, 300, 127), True, "d_33_127")
    return b.build("big_fronts", _blocked(b, sep, order))


def child_records(seed=2):
    """one big front (16 pivots, 200 rows) under every kind of child: child records with contig 0..3, dense children
    alone in a tile and beside scattered ones, sorted small-child lists longer than 512 entries (panel and tile); and
    a second big front with 34 children in its pivot block (more than 32 child records in one task)"""
    b = Builder(seed)
    sep = b.group(SEP, "sep")
    order = []
    P = b.group(16, "P")
    b.couple(P, sep, None, np.arange(0, 200))
    R = np.arange(0, 200)     # P's rows, as separator indices

    def kid(ns, pcols, rows, name=None):
        k = b.group(ns, name)
        b.couple(k, P, None, pcols)
        b.couple(k, sep, None, rows)
        order.append(k)
        return k

    kid(3, np.arange(0, 8), np.r_[R[0:20], R[150:170]], "k_dense")        # contiguous: contig 3, dense in its tiles
    kid(2, np.arange(0, 16, 2), R[0:120:3], "k_scatter")                  # contig 0
    kid(2, np.arange(8, 16), R[1:110:4], "k_rows_strided")                # R tasks: columns contiguous, rows not
    kid(2, np.arange(1, 16, 3), R[70:100], "k_cols_strided")              # R tasks: rows contiguous, columns not
    for i in range(4):
        kid(1, np.arange(16), [], None)                                      # small, 16 rows in the pivot block
    for i in range(5):
        kid(1, [i], R[100:115], None)                                      # small, 15 rows in tile row 1
    order.append(b.lift(P))
    order.append(P)

    Q = b.group(40, "Q")
    b.couple(Q, sep, None, np.arange(100, 196))
    for i in range(34):
        k = b.group(1)
        b.couple(k, Q, None, (np.arange(17) * 2 + i) % 40)
        order.append(k)
    order.append(b.lift(Q))
    order.append(Q)
    return b.build("child_records", _blocked(b, sep, order))


def all_shapes():
    return [big_fronts(), child_records()]


# where a regularised pivot lands: (group, pivot index inside the group)
REG_SITES = [("leaf1", 0), ("level", 3), ("F", 4), ("D", 0), ("D", 1), ("D", 2), ("D", 3), ("D", 8)]


def regularised(group, j, seed=3):
    """a small matrix (N 317) with one wrong-signed diagonal: pivot j of group `group`, which becomes a front
    factored by k_factor_leaf1 ("leaf1", 1 x 5), k_factor_level ("level", 6 x 10), an F task ("F", 9 x 25 above level
    0) or D/R/T tasks ("D", 9 x 96 at level 0)"""
    b = Builder(seed)
    sep = b.group(100, "sep")
    order = []
    g = {}
    for name, ns, rows, lift in [("leaf1", 1, np.arange(1, 6), False), ("level", 6, np.arange(2, 12), False),
                                 ("F", 9, np.arange(5, 30), True), ("D", 9, np.arange(1, 97), False)]:
        g[name] = b.group(ns, name)
        b.couple(g[name], sep, None, rows)
        if lift:
            order.append(b.lift(g[name]))
        order.append(g[name])
    return b.build("reg_%s_%d" % (group, j), _blocked(b, sep, order), flip=[(g[group], j)])
