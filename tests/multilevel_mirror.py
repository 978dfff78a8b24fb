"""Host mirror (numpy / scipy) of the multilevel additive Schwarz preconditioner of ipc_b200/csrc/multilevel.cu, and of the PCG
recurrences it is used in.  Test infrastructure: it decides on the CPU how many iterations the hierarchy saves against block-Jacobi, and it
is what the kernels' level matrices, stored inverses, application and iteration counts are compared with on the GPU.

The hierarchy: vertices sorted by a 30-bit Morton code of their current position (ties keep ascending ids); at level l the aggregates are
the runs of 32^l consecutive ranks and the domains the runs of 32 consecutive aggregates; A_l[D] is the 96 x 96 Galerkin matrix of domain D
for piecewise-constant translations of its aggregates; z = sum_l P_l^T A_l^-1 P_l r.  Vertices without degrees of freedom (Dirichlet, obstacle
tail) are in their level-0 domain only and in no aggregate of the levels >= 1; an aggregate without a free vertex is identity rows."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

DOMAIN = 32  # aggregates per domain, children per aggregate


def morton_codes(V):
    """30-bit codes of the (nV, 3) positions: 10 bits per axis of the cube over the largest extent of their bounding box (one cell size on
    every axis), x in the lowest bit of every triple"""
    V = np.asarray(V, dtype=np.float64)
    lo, hi = V.min(axis=0), V.max(axis=0)
    ext = (hi - lo).max()
    scale = 1024.0 / ext if ext > 0.0 else 0.0
    q = np.minimum(1023, ((V - lo) * scale).astype(np.int64))
    code = np.zeros(V.shape[0], dtype=np.int64)
    for b in range(10):
        for c in range(3):
            code |= ((q[:, c] >> b) & 1) << (3 * b + c)
    return code


def morton_order(V):
    """(order, rank): order[k] = vertex at place k, rank[v] = place of vertex v"""
    order = np.argsort(morton_codes(V), kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    return order, rank


def level_sizes(nV):
    """domains per level, up to the first level with one domain"""
    out, span = [], DOMAIN
    while True:
        out.append(-(-nV // span))
        if out[-1] == 1:
            return out
        span *= DOMAIN


class Multilevel:
    """the hierarchy of the symmetric matrix H (scipy sparse, 3 nV rows, vertex-interleaved) at the (nV, 3) positions V; fixed: mask of the
    vertices without degrees of freedom"""

    def __init__(self, H, V, fixed=None):
        H = sp.csr_matrix(H)
        self.n = H.shape[0]
        self.nV = self.n // 3
        self.order, self.rank = morton_order(V)
        self.domains = level_sizes(self.nV)
        self.levels = len(self.domains)
        comp = np.tile(np.arange(3), self.nV)
        free = np.ones(self.nV) if fixed is None else 1.0 - np.asarray(fixed, dtype=np.float64)
        self.P, self.A, self.Ainv = [], [], []
        for l, nD in enumerate(self.domains):
            agg = np.repeat(self.rank >> (5 * l), 3) * 3 + comp  # coarse row of every fine row
            P = sp.csr_matrix((np.repeat(free, 3) if l else np.ones(self.n), (agg, np.arange(self.n))), shape=(96 * nD, self.n))
            P.eliminate_zeros()
            G = sp.coo_matrix(P @ H @ P.T)
            A = np.zeros((nD, 96, 96))
            same = (G.row // 96) == (G.col // 96)
            np.add.at(A, (G.row[same] // 96, G.row[same] % 96, G.col[same] % 96), G.data[same])
            if l == 0:
                pad = np.arange(3 * self.nV, 96 * nD)  # past the last vertex: identity rows
                A[pad // 96, pad % 96, pad % 96] = 1.0
            else:  # an aggregate without a free vertex (a zero diagonal): identity rows
                d, i = np.nonzero(np.einsum("dii->di", A) == 0.0)
                A[d, i, i] = 1.0
            self.P.append(P)
            self.A.append(A)
            self.Ainv.append(np.linalg.inv(A))

    def apply(self, r):
        z = np.zeros(self.n)
        for P, Ainv in zip(self.P, self.Ainv):
            rl = (P @ r).reshape(-1, 96)
            z += P.T @ np.einsum("dij,dj->di", Ainv, rl).ravel()
        return z

    def operator(self):
        return spla.LinearOperator((self.n, self.n), matvec=self.apply, dtype=np.float64)

    def stored_bytes(self):
        return 8 * 96 * 96 * sum(self.domains)


def block_jacobi(H):
    """the preconditioner of ipcgpu_solve_pcg: inverse of every vertex's 3 x 3 diagonal block"""
    H = sp.csr_matrix(H)
    nV = H.shape[0] // 3
    i = np.arange(nV)
    D = np.zeros((nV, 3, 3))
    for a in range(3):
        for b in range(3):
            D[:, a, b] = np.asarray(H[3 * i + a, 3 * i + b]).ravel()
    Dinv = np.linalg.inv(D)
    return lambda r: np.einsum("vij,vj->vi", Dinv, r.reshape(-1, 3)).ravel()


def pcg(H, b, precond, rel_tol, max_iter, check_every=25):
    """the recurrences of the device loop, with its convergence test every `check_every` iterations: (x, iterations, |r| / |b|)"""
    x = np.zeros_like(b)
    r = b.copy()
    z = precond(r)
    p = z.copy()
    rz, bb = r @ z, b @ b
    rr, it = bb, 0
    if bb > 0.0:
        while it < max_iter:
            for _ in range(min(check_every, max_iter - it)):
                q = H @ p
                pq = p @ q
                alpha = rz / pq if pq != 0.0 else 0.0
                x += alpha * p
                r -= alpha * q
                z = precond(r)
                rz_new, rr = r @ z, r @ r
                beta = rz_new / rz if rz != 0.0 else 0.0
                p = z + beta * p
                rz = rz_new
                it += 1
            if not rr == rr or np.sqrt(rr) <= rel_tol * np.sqrt(bb):
                break
    return x, it, np.sqrt(rr / bb) if bb > 0.0 else 0.0


def newton_system(m, dHat, kappa, dt2, V=None):
    """the oracle's Newton system of mesh m (elasticity + mass + barrier, projected) at positions V: (ia, ja, a, g, H, sets), 1-based upper
    triangular CSR on the contact-augmented pattern, the gradient, the full symmetric matrix and the constraint sets (mm, pa, pe)"""
    import oracle as orc
    from stagecheck import contact_pattern_pairs
    s, o = (orc.Surf(m), orc.Elastic(m)) if V is None else (orc.Surf(m, V=V), orc.Elastic(m, V=V))
    mm, pa, pe, _ = s.constraint_set(dHat, nthreads=8)
    ia, ja = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe))
    g = s.barrier_gradient(mm, pa, pe, dHat, kappa, g=o.gradient(dt2, 1))
    a = o.hessian_csr(dt2, ia, ja, 1, 1, 1)
    a[np.asarray(ia[:-1], dtype=np.int64) - 1] += np.repeat(m.mass, 3)
    a = s.barrier_hessian_csr(mm, pa, pe, dHat, kappa, ia, ja, 1, 1, a=a)
    return ia, ja, a, g, full_matrix(ia, ja, a, 3 * m.nV), (mm, pa, pe)


def full_matrix(ia, ja, a, n, base=1):
    U = sp.csr_matrix((a, np.asarray(ja) - base, np.asarray(ia) - base), shape=(n, n))
    return (U + sp.triu(U, 1).T).tocsr()
