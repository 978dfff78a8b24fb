"""CPU checks of the damping, Neumann and Dirichlet-penalty restatements (tests/oracle_damping.py) that the GPU tests compare against:
the restated LinSysSolver::multiply against scipy, finite differences of the three energies against the restated gradients, and the
identity that computeDampingMtr leaves on the diagonal of every Dirichlet vertex."""
import numpy as np

import oracle_damping as OD
from ipc_b200 import mesh as M


def small_mesh():
    V, T = M.grid_tets(2, 2, 2, h=0.5)
    m = M.Mesh(V, T, energy=1, density=1.0)
    M.deform(m, 4, twist=0.2, amp=0.02, noise=0.02)
    m.dbc[[0, 1]] = 1
    m.dbc[[2]] = 2
    return m


def test_multiply_equals_the_full_symmetric_product():
    m = small_mesh()
    D = OD.damping_matrix(m, m.V, 0.3)
    x = np.random.default_rng(0).standard_normal(3 * m.nV)
    full = OD.full_matrix(*D).toarray()
    assert np.allclose(full, full.T)
    np.testing.assert_allclose(OD.multiply(*D, x), full @ x, rtol=0, atol=1e-12 * np.abs(full).max() * np.abs(x).max() * 10)


def test_dirichlet_diagonal_is_the_identity():
    """addBlockToMatrix's setCoeff (IglUtils.hpp:45-52): D holds 1.0 on the diagonal of a Dirichlet vertex and nothing else in its rows;
    the system matrix therefore gets 2.0 there, and with projectDBC = 0, D d adds x_v - x_prev,v to the vertex's gradient rows"""
    m = small_mesh()
    ia, ja, a = OD.damping_matrix(m, m.V, 0.3)
    full = OD.full_matrix(ia, ja, a).toarray()
    for v in np.flatnonzero(m.dbc):
        rows = full[3 * v:3 * v + 3]
        assert np.array_equal(rows[:, 3 * v:3 * v + 3], np.eye(3))
        rest = rows.copy()
        rest[:, 3 * v:3 * v + 3] = 0.0
        assert not rest.any()
    # (identity + D: the elastic assembly sets 1.0, adding D makes 2.0)
    assert all(full[3 * v + r, 3 * v + r] + 1.0 == 2.0 for v in np.flatnonzero(m.dbc) for r in range(3))
    rng = np.random.default_rng(1)
    Vp = m.V - 0.01 * rng.standard_normal(m.V.shape)
    g = OD.damping_gradient((ia, ja, a), m.V, Vp, m.dbc, 0).reshape(-1, 3)
    for v in np.flatnonzero(m.dbc == 2):  # NONZERO Dirichlet vertex, not projected: its displacement comes through the identity
        assert np.allclose(g[v], m.V[v] - Vp[v], rtol=0, atol=1e-15)
    g1 = OD.damping_gradient((ia, ja, a), m.V, Vp, m.dbc, 1).reshape(-1, 3)
    assert not g1[m.dbc != 0].any()


def fd_check(energy, grad, V, rows, h=1e-6):
    """central differences of energy(V) against grad (interleaved) on the vertex rows `rows`"""
    for v in rows:
        for c in range(3):
            Vp, Vm = V.copy(), V.copy()
            Vp[v, c] += h
            Vm[v, c] -= h
            fd = (energy(Vp) - energy(Vm)) / (2 * h)
            assert abs(fd - grad[3 * v + c]) <= 1e-6 * max(1.0, abs(grad[3 * v + c])), (v, c, fd, grad[3 * v + c])


def test_damping_gradient_is_the_energy_derivative_on_free_rows():
    m = small_mesh()
    rng = np.random.default_rng(2)
    D = OD.damping_matrix(m, m.V, 0.3)
    Vp = m.V - 0.05 * rng.standard_normal(m.V.shape)
    V = m.V + 0.02 * rng.standard_normal(m.V.shape)
    g = OD.damping_gradient(D, V, Vp, m.dbc, 1)
    fd_check(lambda X: OD.damping_energy(D, X, Vp, m.dbc), g, V, np.flatnonzero(m.dbc == 0))


def test_neumann_gradient_is_the_energy_derivative():
    m = small_mesh()
    rng = np.random.default_rng(3)
    f = rng.standard_normal((m.nV, 3))
    g = OD.neumann_gradient(f, m.mass, m.dbc, 0.01)
    fd_check(lambda X: OD.neumann_energy(X, f, m.mass, m.dbc, 0.01), g, m.V, range(m.nV))
    assert not g.reshape(-1, 3)[m.dbc != 0].any()


def test_dirichlet_gradient_and_hessian_are_the_energy_derivatives():
    m = small_mesh()
    rng = np.random.default_rng(4)
    vid = np.array([0, 1, 2, 5])
    tgt = m.V[vid] + 0.03 * rng.standard_normal((4, 3))
    lam = rng.standard_normal((4, 3))
    rho = 50.0
    g = OD.mdbc_gradient(m.V, vid, tgt, lam, m.mass, rho, m.nV)
    fd_check(lambda X: OD.mdbc_energy(X, vid, tgt, lam, m.mass, rho), g, m.V, range(m.nV))
    h = OD.mdbc_hessian_diag(vid, m.mass, rho, m.nV)
    for v in vid:  # the energy is quadratic with the diagonal Hessian rho m
        for c in range(3):
            e = np.zeros_like(m.V)
            e[v, c] = 1e-3
            g1 = OD.mdbc_gradient(m.V + e, vid, tgt, lam, m.mass, rho, m.nV)
            assert abs((g1[3 * v + c] - g[3 * v + c]) / 1e-3 - h[3 * v + c]) <= 1e-6 * h[3 * v + c]
    assert OD.mdbc_energy(m.V, vid, tgt, lam, m.mass, 0.0) == 0.0 and not OD.mdbc_gradient(m.V, vid, tgt, lam, m.mass, 0.0, m.nV).any()
    # completed step: 1 at the targets, 0 at the distance sqrt(dist2Tol 1e6)
    assert OD.mdbc_completed_step(tgt, np.arange(4), tgt, 1e-8) == 1.0 and OD.mdbc_completed_step(m.V, vid, tgt, 0.0) == 1.0
    dx2 = float(np.sum((m.V[vid] - tgt) ** 2))
    assert abs(OD.mdbc_completed_step(m.V, vid, tgt, dx2 * 1e-6)) <= 1e-15
