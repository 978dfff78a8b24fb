"""numpy restatements of the damping, Neumann and augmented-Lagrangian Dirichlet terms (TEST INFRASTRUCTURE ONLY).

- D (computeDampingMtr, Optimizer.cpp:3723-3734) is the CPU oracle's elastic CSR Hessian (projectSPD = projectDBC = 1) on the mesh-only pattern;
- LinSysSolver::multiply (LinSysSolver.hpp:238-253) over the upper-triangular CSR;
- the damping energy / gradient (Optimizer.cpp:3381-3400, :3519-3540), the Neumann forces (:3241-3250, :3452-3461) and
  AnimScripter's augmentMDBC* / updateLambda / computeCompletedStepSize (AnimScripter.cpp:2286-2344)."""
import numpy as np
import scipy.sparse as sp

import oracle as orc


def damping_matrix(m, V, coef):
    """(ia, ja, a) of D on the mesh-only pattern (1-based), at positions V (nV, 3)"""
    ia, ja = m.csr_pattern(1)
    return ia, ja, orc.Elastic(m, V=V).hessian_csr(coef, ia, ja, 1, 1, 1)


def multiply(ia, ja, a, x, base=1):
    """LinSysSolver::multiply: Ax over the stored upper triangle, every off-diagonal entry used twice"""
    n = ia.size - 1
    Ax = np.zeros(n)
    for r in range(n):
        for k in range(ia[r] - base, ia[r + 1] - base):
            c = ja[k] - base
            Ax[r] += a[k] * x[c]
            if r != c:
                Ax[c] += a[k] * x[r]
    return Ax


def multiply_fast(ia, ja, a, x, base=1):
    """the same product through scipy (the whole symmetric matrix), for the larger scenes"""
    return full_matrix(ia, ja, a, base) @ x


def full_matrix(ia, ja, a, base=1):
    n = ia.size - 1
    U = sp.csr_matrix((a, ja - base, ia - base), shape=(n, n))
    return U + sp.triu(U, 1).T


def _disp(V, Vprev, zero):
    d = (np.asarray(V) - np.asarray(Vprev)).copy()
    d[zero] = 0.0
    return d.ravel()


def projected(dbc, projectDBC):
    """Mesh::isProjectDBCVertex (Mesh.hpp:135-143)"""
    return (dbc == 1) | ((dbc == 2) & bool(projectDBC))


def damping_energy(D, V, Vprev, dbc):
    """1/2 d^T D d, every Dirichlet row of d zeroed"""
    d = _disp(V, Vprev, dbc != 0)
    return 0.5 * float(d @ multiply_fast(*D, d))


def damping_gradient(D, V, Vprev, dbc, projectDBC):
    """D d with the projected Dirichlet rows of d zeroed"""
    return multiply_fast(*D, _disp(V, Vprev, projected(dbc, projectDBC)))


def neumann_energy(V, f, mass, dbc, coef):
    f = np.asarray(f).reshape(-1, 3)
    free = dbc == 0
    dot = (V[:, 0] * f[:, 0] + V[:, 1] * f[:, 1]) + V[:, 2] * f[:, 2]
    return float(np.sum(-((coef * mass) * dot)[free]))


def neumann_gradient(f, mass, dbc, coef):
    f = np.asarray(f).reshape(-1, 3)
    g = -(coef * mass)[:, None] * f
    g[dbc != 0] = 0.0
    return g.ravel()


def mdbc_energy(V, vid, tgt, lam, mass, rho):
    if rho == 0.0:
        return 0.0
    dx = V[vid] - tgt
    m = mass[vid]
    return float(np.sum(rho / 2.0 * m * np.sum(dx * dx, axis=1) - np.sqrt(m) * np.sum(lam * dx, axis=1)))


def mdbc_gradient(V, vid, tgt, lam, mass, rho, nV):
    g = np.zeros((nV, 3))
    if rho != 0.0:
        m = mass[vid][:, None]
        g[vid] = -np.sqrt(m) * lam + rho * m * (V[vid] - tgt)
    return g.ravel()


def mdbc_hessian_diag(vid, mass, rho, nV):
    """augmentMDBCHessian: the 3nV diagonal increments"""
    h = np.zeros((nV, 3))
    if rho != 0.0:
        h[vid] = (rho * mass[vid])[:, None]
    return h.ravel()


def mdbc_update_lambda(V, vid, tgt, lam, mass, rho):
    return lam - (rho * np.sqrt(mass[vid]))[:, None] * (V[vid] - tgt)


def mdbc_completed_step(V, vid, tgt, dist2Tol):
    if dist2Tol == 0.0:
        return 1.0
    dx = V[vid] - tgt
    return 1.0 - np.sqrt(float(np.sum(np.sum(dx * dx, axis=1))) / (dist2Tol * 1.0e6))


def scatter(ia_from, ja_from, a_from, ia_to, ja_to, base=1):
    """the entries of an upper CSR moved into a pattern that contains it"""
    pos = {}
    n = ia_to.size - 1
    for r in range(n):
        for k in range(ia_to[r] - base, ia_to[r + 1] - base):
            pos[(r, ja_to[k] - base)] = k
    out = np.zeros(ja_to.size)
    for r in range(n):
        for k in range(ia_from[r] - base, ia_from[r + 1] - base):
            out[pos[(r, ja_from[k] - base)]] += a_from[k]
    return out
