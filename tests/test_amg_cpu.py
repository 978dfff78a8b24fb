"""The host mirror of the smoothed-aggregation multigrid preconditioner (tests/amg_mirror.py) on the oracle's matrices: its aggregates cover
every connected row once and are connected, its roots are pairwise at distance >= 3, P_tent reproduces translations, every level matrix is
SPD, the W-cycle is a symmetric positive definite operator, rows without degrees of freedom stay exactly 0, PCG with it reaches the direct
solve, and on ball_on_mat it needs no more iterations than the multilevel additive Schwarz mirror."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csg
import scipy.sparse.linalg as spla

import amg_mirror as am
import multilevel_mirror as mlm
from gpu_common import rel
from ipc_b200 import scenes
from test_multilevel_cpu import DT2, ball_on_mat_system


@pytest.fixture(scope="module")
def pile():
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    return (m,) + mlm.newton_system(m, info["dHat"], 1e6, DT2)


@pytest.fixture(scope="module")
def mat():
    return ball_on_mat_system()


def graph(A):
    off = A.ja != A.rows
    return sp.csr_matrix((np.ones(off.sum()), (A.rows[off], A.ja[off])), shape=(A.n, A.n))


def check_aggregates(A, agg, roots):
    G = graph(A)
    connected = np.diff(G.indptr) > 0
    assert np.array_equal(agg >= 0, connected)  # every connected row exactly once, unconnected rows nowhere
    assert np.array_equal(np.unique(agg[agg >= 0]), np.arange(roots.size))
    assert np.array_equal(agg[roots], np.arange(roots.size)) and (np.diff(roots) > 0).all()  # numbered by ascending root
    d = csg.shortest_path(G, unweighted=True, indices=roots)[:, roots]
    np.fill_diagonal(d, np.inf)
    assert d.min() >= 3
    for a in range(roots.size):  # every aggregate is connected
        rows = np.flatnonzero(agg == a)
        assert csg.connected_components(G[rows][:, rows], directed=False)[0] == 1


def test_level0_keeps_the_nonzero_blocks(pile):
    m, ia, ja, a, g, H, sets = pile
    A = am.level0(H)
    assert A.n == m.nV and np.allclose(A.scipy().toarray(), H.toarray(), rtol=0, atol=0)
    # explicit zeros of the pattern do not make blocks or connections
    C = sp.coo_matrix(H)
    Hz = sp.csr_matrix((np.r_[C.data, 0.0], (np.r_[C.row, 0], np.r_[C.col, 3 * (m.nV - 1)])), shape=H.shape)  # (an explicitly stored zero)
    assert (A.rows != A.ja).any() and not ((am.level0(Hz).rows == 0) & (am.level0(Hz).ja == m.nV - 1)).any()


@pytest.mark.parametrize("scene", ["pile", "mat"])
def test_aggregates_and_level_matrices(scene, request):
    sysm = request.getfixturevalue(scene)
    H = sysm[5] if scene == "pile" else sysm[1]
    M = am.AMG(H)
    assert M.levels >= 2 and M.lv[-1].n <= am.COARSE_ENOUGH or M.levels == am.MAX_LEVELS
    for l, lv in enumerate(M.lv):
        S = lv.S.toarray()
        assert np.abs(S - S.T).max() <= 1e-12 * np.abs(S).max()
        assert np.linalg.eigvalsh(0.5 * (S + S.T)).min() > 0.0
        assert 0.0 < lv.rho and np.isfinite(lv.rho)
        if l + 1 < M.levels:
            check_aggregates(lv.A, lv.agg, lv.roots)
            # P_tent reproduces translations: every connected row's translation is its aggregate's
            t = np.tile(np.eye(3), (lv.roots.size, 1))
            Pt = sp.csr_matrix((np.ones(3 * (lv.agg >= 0).sum()), (np.flatnonzero(np.repeat(lv.agg >= 0, 3)), (3 * np.repeat(lv.agg[lv.agg >= 0], 3) + np.tile(np.arange(3), (lv.agg >= 0).sum())))),
                               shape=(3 * lv.n, 3 * lv.roots.size))
            assert np.array_equal((Pt @ t).reshape(-1, 3, 3)[lv.agg >= 0], np.tile(np.eye(3), ((lv.agg >= 0).sum(), 1, 1)))
            # P = (I - omega D^-1 A) P_tent, the Galerkin product
            DinvA = sp.block_diag([sp.csr_matrix(D) for D in lv.Dinv]).tocsr() @ lv.S
            P = (sp.eye(3 * lv.n) - lv.omega * DinvA) @ Pt
            assert abs(np.abs(P - lv.Ps).max()) <= 1e-14 * np.abs(P).max()
            C = (lv.Ps.T @ lv.S @ lv.Ps).toarray()
            assert np.abs(C - M.lv[l + 1].S.toarray()).max() <= 1e-12 * np.abs(C).max()
            assert np.array_equal(lv.Rs.toarray(), lv.Ps.T.toarray())


def test_cycle_is_symmetric_positive_definite(pile):
    m, ia, ja, a, g, H, sets = pile
    M = am.AMG(H)
    rng = np.random.default_rng(0)
    for _ in range(5):
        u, v = rng.standard_normal(H.shape[0]), rng.standard_normal(H.shape[0])
        Mu, Mv = M.apply(u), M.apply(v)
        assert abs(u @ Mv - v @ Mu) <= 1e-10 * np.linalg.norm(u) * np.linalg.norm(Mv)
        assert u @ Mu > 0.0


def test_rows_without_degrees_of_freedom_stay_exactly_zero(pile):
    m, ia, ja, a, g, H, sets = pile
    fixed_v = np.zeros(m.nV, dtype=bool)
    fixed_v[::7] = True
    fixed_v[40:80] = True
    rows = np.flatnonzero(np.repeat(fixed_v, 3))
    Hf = H.tolil()
    Hf[rows, :] = 0.0
    Hf[:, rows] = 0.0
    Hf[rows, rows] = 1.0
    Hf = Hf.tocsr()
    M = am.AMG(Hf)
    assert (M.lv[0].agg[fixed_v] == -1).all()
    b = -g.copy()
    b[rows] = 0.0
    assert (M.apply(b)[rows] == 0.0).all()
    x, it, res = mlm.pcg(Hf, b, M.apply, 1e-6, 5000)
    assert res <= 1e-6 and (x[rows] == 0.0).all() and rel(x, spla.spsolve(Hf.tocsc(), b)) <= 1e-4


def test_mirror_pcg_equals_the_direct_solve(pile):
    m, ia, ja, a, g, H, sets = pile
    M = am.AMG(H)
    x, it, res = mlm.pcg(H, -g, M.apply, 1e-10, 5000)
    assert res <= 1e-10 and 0 < it < 5000
    assert rel(x, spla.spsolve(H.tocsc(), -g)) <= 1e-7


def test_not_positive_definite_is_detected():
    H = sp.csr_matrix(np.diag(np.r_[np.ones(3), -np.ones(3)]))
    with pytest.raises(np.linalg.LinAlgError):
        am.AMG(H)


def test_iterations_against_the_multilevel_mirror(pile, mat, record_property):
    """the gate of the configuration: on ball_on_mat at 1e-6 no more iterations than the multilevel additive Schwarz mirror (107)"""
    m, ia, ja, a, g, H, sets = pile
    counts = {}
    for name, (mesh, sysH, rhs) in {"ball_pile": (m, H, -g), "ball_on_mat": mat}.items():
        M, ML = am.AMG(sysH), mlm.Multilevel(sysH, mesh.V)
        for tol in (1e-6, 1e-10):
            counts[f"{name}@{tol:g}"] = (mlm.pcg(sysH, rhs, M.apply, tol, 5000, check_every=1)[1],
                                         mlm.pcg(sysH, rhs, ML.apply, tol, 5000, check_every=1)[1])
    record_property("amg_vs_multilevel_iterations", counts)
    print("iterations (AMG, multilevel):", counts)
    amg, mas = counts["ball_on_mat@1e-06"]
    assert mas == 107 and amg <= mas, counts
