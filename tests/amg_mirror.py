"""Host mirror (numpy / scipy) of the smoothed-aggregation multigrid preconditioner of ipc_b200/csrc/amg.cu, the preconditioner of
ipcgpu_solve_pcg_amg.  Test infrastructure: it decides on the CPU whether the hierarchy saves iterations, and it is what the kernels'
aggregates, level matrices, spectral radii and application are compared with on the GPU.

Every level is a block CSR matrix of 3 x 3 vertex blocks (ia, ja ascending within a row, blocks).  The set-up, step by step:
  1. level 0 keeps the blocks of the full symmetric matrix with a nonzero among their 9 entries;
  2. rows i != j are connected when block (i, j) is kept; a row without a connection is in no aggregate (its row of P is zero);
  3. aggregates from a distance-2 maximal independent set: priority (splitmix64(row), row); each round an undecided row whose key
     (state, priority) is the largest in its distance-2 neighbourhood becomes a root, an undecided row whose largest key there is a root is
     taken out; a root and its neighbours form an aggregate, every other connected row joins the aggregate of its assigned (distance-1)
     neighbour of largest priority; aggregates are numbered by ascending root;
  4. P = (I - omega D^-1 A) P_tent, P_tent the 3 x 3 identity at (i, agg(i)), omega = (4/3) / rho_G, rho_G the largest absolute row sum of
     D^-1 A; a row of P lists its neighbours' aggregates in storage order, equal columns summed in that order, stored by ascending column;
  5. A_{l+1} = P^T (A_l P), both products by one block SpGEMM (every output block the sum, in enumeration order, of the products of the
     left row's blocks in storage order with the right rows' blocks in storage order), P^T by a stable counting sort;
  6. D^-1 by a 3 x 3 Cholesky factorization of every diagonal block;
  7. rho_l of D^-1 A by 100 power steps from b_0[i] = splitmix64(i) mapped to [-1, 1); Chebyshev interval [2 rho_l / 120, 2 rho_l];
  8. at most 6 levels; the first level with at most 1000 block rows is the last, and so is a level whose coarsening would keep more than
     4/5 of its rows or make no aggregate.
The preconditioner is one W-cycle (two visits of every coarse level, the last level two smoothing applications alone) with a degree-16
D^-1-scaled Chebyshev smoother before and after the coarse correction, every level starting from x = 0."""
import numpy as np
import scipy.sparse as sp

MAX_LEVELS = 6
COARSE_ENOUGH = 1000  # block rows
DEGREE = 16
POWER_STEPS = 100
NCYCLE = 2


def splitmix64(i):
    z = np.asarray(i, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def power_start(n):
    """b_0 of the power iteration: splitmix64(i) >> 11 as a 53-bit fraction, mapped to [-1, 1)"""
    return (splitmix64(np.arange(n)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -52 - 1.0


class BlockCSR:
    def __init__(self, ia, ja, blk, ncols):
        self.ia, self.ja, self.blk = np.asarray(ia, dtype=np.int64), np.asarray(ja, dtype=np.int64), np.asarray(blk, dtype=np.float64)
        self.n, self.ncols = self.ia.size - 1, ncols
        self.rows = np.repeat(np.arange(self.n), np.diff(self.ia))

    def scipy(self):
        return sp.bsr_matrix((self.blk, self.ja, self.ia), shape=(3 * self.n, 3 * self.ncols)).tocsr()

    def transpose(self):
        """stable counting sort by column: every row of the transpose lists its blocks by ascending row of the original"""
        order = np.argsort(self.ja, kind="stable")
        ia = np.zeros(self.ncols + 1, dtype=np.int64)
        np.add.at(ia, self.ja + 1, 1)
        return BlockCSR(np.cumsum(ia), self.rows[order], self.blk[order].transpose(0, 2, 1), self.n)


def from_entries(n, ncols, row, col, val):
    """block CSR of the (row, col, 3 x 3) list, entries of one (row, col) summed in list order (a stable sort by (row, col))"""
    order = np.lexsort((col, row))
    row, col, val = row[order], col[order], val[order]
    if row.size == 0:
        return BlockCSR(np.zeros(n + 1, dtype=np.int64), row, val, ncols)
    head = np.flatnonzero(np.r_[True, (row[1:] != row[:-1]) | (col[1:] != col[:-1])])
    out = np.zeros((head.size, 3, 3))
    bounds = np.r_[head, row.size]
    # summed one term after another in order (the device's loop), not pairwise
    cur = val[head].copy()
    length = np.diff(bounds)
    for t in range(1, length.max()):
        more = length > t
        cur[more] += val[head[more] + t]
    out[:] = cur
    ia = np.zeros(n + 1, dtype=np.int64)
    np.add.at(ia, row[head] + 1, 1)
    return BlockCSR(np.cumsum(ia), col[head], out, ncols)


def spgemm(L, R):
    """the block SpGEMM of step 5"""
    cnt = np.diff(R.ia)[L.ja]
    e = np.repeat(np.arange(L.ja.size), cnt)
    start = np.repeat(np.cumsum(cnt) - cnt, cnt)
    r = R.ia[L.ja[e]] + np.arange(e.size) - start
    return from_entries(L.n, R.ncols, L.rows[e], R.ja[r], np.einsum("eij,ejk->eik", L.blk[e], R.blk[r]))


def level0(H):
    """step 1: the kept 3 x 3 blocks of the full symmetric matrix H (scipy, vertex-interleaved)"""
    C = sp.coo_matrix(H)
    nb = H.shape[0] // 3
    nz = C.data != 0.0
    keep = np.unique((C.row[nz] // 3) * nb + C.col[nz] // 3)
    key = (C.row // 3) * nb + C.col // 3
    pos = np.searchsorted(keep, key)
    inside = (pos < keep.size) & (keep[np.minimum(pos, keep.size - 1)] == key)
    blk = np.zeros((keep.size, 3, 3))
    np.add.at(blk, (pos[inside], C.row[inside] % 3, C.col[inside] % 3), C.data[inside])
    ia = np.zeros(nb + 1, dtype=np.int64)
    np.add.at(ia, keep // nb + 1, 1)
    return BlockCSR(np.cumsum(ia), keep % nb, blk, nb)


def aggregate(A):
    """steps 2-3: (agg, roots, rounds); agg = -1 for a row without a connection"""
    n = A.n
    off = A.ja != A.rows
    connected = np.bincount(A.rows[off], minlength=n) > 0
    # closed neighbourhoods: the row itself, then its connections
    rows_c = np.r_[np.arange(n), A.rows[off]]
    cols_c = np.r_[np.arange(n), A.ja[off]]
    order = np.argsort(rows_c, kind="stable")
    rows_c, cols_c = rows_c[order], cols_c[order]
    start = np.searchsorted(rows_c, np.arange(n))
    prio = np.empty(n, dtype=np.int64)  # priority rank: splitmix64 is a bijection, so the row index never breaks a tie
    prio[np.argsort(splitmix64(np.arange(n)), kind="stable")] = np.arange(n)
    state = np.where(connected, 1, 0)  # 0 out (or unconnected), 1 undecided, 2 root
    rounds = 0
    while (state == 1).any():
        key = state * n + prio
        k1 = np.maximum.reduceat(key[cols_c], start)
        k2 = np.maximum.reduceat(k1[cols_c], start)
        und = state == 1
        new = state.copy()
        new[und & (k2 == key)] = 2
        new[und & (k2 >= 2 * n)] = 0
        state = new
        rounds += 1
    roots = state == 2
    ids = np.cumsum(roots) - 1
    agg = np.full(n, -1, dtype=np.int64)
    agg[roots] = ids[roots]
    i, j = A.rows[off], A.ja[off]
    near = roots[j]
    agg[i[near]] = ids[j[near]]  # unique: roots are at least 3 apart
    agg1 = agg.copy()
    far = connected[i] & (agg1[i] < 0) & (agg1[j] >= 0)
    i2, j2 = i[far], j[far]
    best = np.lexsort((prio[j2], i2))  # per row, the assigned neighbour of largest priority last
    last = np.r_[i2[best][1:] != i2[best][:-1], True] if i2.size else np.zeros(0, dtype=bool)
    agg[i2[best][last]] = agg1[j2[best][last]]
    assert (agg[connected] >= 0).all() and (agg[~connected] < 0).all()
    return agg, np.flatnonzero(roots), rounds


def cholesky_inverse(D):
    """step 6: inverses of the (n, 3, 3) SPD blocks; (Dinv, every pivot > 0)"""
    ok = True
    try:
        L = np.linalg.cholesky(D)
    except np.linalg.LinAlgError:
        return None, False
    Linv = np.linalg.inv(L)
    return np.einsum("nki,nkj->nij", Linv, Linv), ok


class Level:
    def __init__(self, A):
        self.A = A
        self.n = A.n
        diag = A.ja == A.rows
        assert np.array_equal(A.rows[diag], np.arange(A.n)), "every row holds its diagonal block"
        self.Dinv, ok = cholesky_inverse(A.blk[diag])
        if not ok:
            raise np.linalg.LinAlgError("a 3 x 3 diagonal block is not positive definite")
        self.S = A.scipy()
        self.DinvA = np.einsum("eij,ejk->eik", self.Dinv[A.rows], A.blk)  # D^-1 A, block by block
        b = power_start(3 * A.n)
        for _ in range(POWER_STEPS):
            y = self.dinv(self.S @ b)
            ny = np.linalg.norm(y)
            self.rho = ny / np.linalg.norm(b)
            b = y / ny
        self.hi = 2.0 * self.rho
        self.lo = self.hi / 120.0
        self.agg = self.P = self.R = None

    def dinv(self, v):
        return np.einsum("nij,nj->ni", self.Dinv, v.reshape(-1, 3)).ravel()

    def coarsen(self):
        """steps 2-5 from this level: the next level's matrix, or None when this level is the last"""
        A = self.A
        self.agg, self.roots, self.rounds = aggregate(A)
        nagg = self.roots.size
        if nagg == 0 or 5 * nagg > 4 * self.n:
            self.agg = None
            return None
        absrow = np.zeros((A.n, 3))
        np.add.at(absrow, A.rows, np.abs(self.DinvA).sum(axis=2))
        self.rho_g = absrow.max()
        self.omega = (4.0 / 3.0) / self.rho_g
        has = self.agg[A.ja] >= 0
        val = -self.omega * self.DinvA[has]
        eye = (A.ja == A.rows)[has]
        val[eye] += np.eye(3)
        self.P = from_entries(A.n, nagg, A.rows[has], self.agg[A.ja[has]], val)
        self.R = self.P.transpose()
        self.Ps, self.Rs = self.P.scipy(), self.R.scipy()
        return spgemm(self.R, spgemm(A, self.P))

    def chebyshev(self, f, x=None):
        theta, delta = 0.5 * (self.hi + self.lo), 0.5 * (self.hi - self.lo)
        sigma = theta / delta
        rho_prev = 1.0 / sigma
        r = self.dinv(f if x is None else f - self.S @ x)
        d = r / theta
        x = np.zeros_like(f) if x is None else x.copy()
        for k in range(1, DEGREE + 1):
            x += d
            if k < DEGREE:
                r -= self.dinv(self.S @ d)
                rho_k = 1.0 / (2.0 * sigma - rho_prev)
                d = rho_k * rho_prev * d + (2.0 * rho_k / delta) * r
                rho_prev = rho_k
        return x


class AMG:
    """the hierarchy of the symmetric matrix H (scipy sparse, 3 nV rows, vertex-interleaved)"""

    def __init__(self, H):
        self.n = H.shape[0]
        self.lv = [Level(level0(H))]
        while len(self.lv) < MAX_LEVELS and self.lv[-1].n > COARSE_ENOUGH:
            A = self.lv[-1].coarsen()
            if A is None:
                break
            self.lv.append(Level(A))
        self.levels = len(self.lv)

    def cycle(self, l, f, x=None):
        lv = self.lv[l]
        if l == self.levels - 1:
            return lv.chebyshev(f, lv.chebyshev(f, x))
        x = lv.chebyshev(f, x)
        fc = lv.Rs @ (f - lv.S @ x)
        xc = None
        for _ in range(NCYCLE):
            xc = self.cycle(l + 1, fc, xc)
        return lv.chebyshev(f, x + lv.Ps @ xc)

    def apply(self, r):
        return self.cycle(0, r)
