"""The host mirror of the multilevel additive Schwarz preconditioner (tests/multilevel_mirror.py) on the oracle's matrices: its order is a
stable permutation, its operator symmetric positive definite, PCG with it reaches the direct solve, and it needs fewer iterations than
block-Jacobi -- at most half on ball_on_mat, the scene whose count the device test repeats."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

import multilevel_mirror as mlm
from gpu_common import rel
from ipc_b200 import scenes

DT2 = 0.025 ** 2


@pytest.fixture(scope="module")
def pile():
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    return (m,) + mlm.newton_system(m, info["dHat"], 1e6, DT2)


def test_morton_order_is_a_stable_permutation():
    rng = np.random.default_rng(0)
    V = rng.uniform(-1.0, 2.0, (500, 3))
    V[100:140] = V[7]  # ties: the same position, hence the same code
    V[300] = V[7]
    order, rank = mlm.morton_order(V)
    assert np.array_equal(np.sort(order), np.arange(500)) and np.array_equal(order[rank], np.arange(500))
    code = mlm.morton_codes(V)
    assert (np.diff(code[order]) >= 0).all() and code.max() < 1 << 30
    tied = np.flatnonzero(code == code[7])
    assert tied.size >= 42 and (np.diff(rank[tied]) > 0).all()  # ascending ids keep ascending places
    # a pure function of the positions; the cube's cell size is one on every axis: a thin sheet is not cut along its thin axis first
    assert np.array_equal(order, mlm.morton_order(V.copy())[0])
    flat = np.column_stack([rng.uniform(0, 1, 400), rng.uniform(0, 1, 400), rng.uniform(0, 1e-3, 400)])
    assert ((mlm.morton_codes(flat) >> 2) & 0x09249249).max() <= 1  # z takes one cell or two, not 1024
    assert mlm.level_sizes(257_000) == [8032, 251, 8, 1] and mlm.level_sizes(32) == [1] and mlm.level_sizes(33) == [2, 1]


def test_preconditioner_is_symmetric_positive_definite(pile):
    m, ia, ja, a, g, H, sets = pile
    ML = mlm.Multilevel(H, m.V)
    assert ML.domains == mlm.level_sizes(m.nV) and ML.stored_bytes() == 73728 * sum(ML.domains)
    M = np.column_stack([ML.apply(e) for e in np.eye(3 * m.nV)])
    assert np.abs(M - M.T).max() <= 1e-12 * np.abs(M).max()
    assert np.linalg.eigvalsh(0.5 * (M + M.T)).min() > 0.0
    for A in ML.A:  # every level matrix is SPD, padding included
        assert np.linalg.eigvalsh(A).min() > 0.0


def test_vertices_without_degrees_of_freedom_stay_exactly_zero(pile):
    m, ia, ja, a, g, H, sets = pile
    fixed_v = np.zeros(m.nV, dtype=bool)
    fixed_v[::7] = True
    fixed_v[40:80] = True  # (whole level-0 domains among them)
    rows = np.flatnonzero(np.repeat(fixed_v, 3))
    Hf = H.tolil()
    Hf[rows, :] = 0.0
    Hf[:, rows] = 0.0
    Hf[rows, rows] = 1.0
    Hf = Hf.tocsr()
    ML = mlm.Multilevel(Hf, m.V, fixed=fixed_v)
    for A in ML.A:
        assert np.linalg.eigvalsh(A).min() > 0.0
    b = -g.copy()
    b[rows] = 0.0
    assert (ML.apply(b)[rows] == 0.0).all()
    x, it, res = mlm.pcg(Hf, b, ML.apply, 1e-6, 5000)
    assert res <= 1e-6 and (x[rows] == 0.0).all() and rel(x, spla.spsolve(Hf.tocsc(), b)) <= 1e-4
    # without the mask the coarse corrections reach into the identity rows
    assert np.abs(mlm.pcg(Hf, b, mlm.Multilevel(Hf, m.V).apply, 1e-6, 5000)[0][rows]).max() > 0.0


def test_mirror_pcg_equals_the_direct_solve(pile):
    m, ia, ja, a, g, H, sets = pile
    ML = mlm.Multilevel(H, m.V)
    x, it, res = mlm.pcg(H, -g, ML.apply, 1e-10, 5000)
    assert res <= 1e-10 and 0 < it < 5000
    assert rel(x, spla.spsolve(H.tocsc(), -g)) <= 1e-7
    # the operator form gives scipy's CG the same preconditioner
    xs, info = spla.cg(H, -g, M=ML.operator(), rtol=1e-10, maxiter=5000)
    assert info == 0 and rel(xs, x) <= 1e-7


def test_iteration_counts_against_block_jacobi(pile, record_property):
    m, ia, ja, a, g, H, sets = pile
    counts = {}
    for name, (mesh, sysH, rhs) in {"ball_pile": (m, H, -g), "ball_on_mat": ball_on_mat_system()}.items():
        ML = mlm.Multilevel(sysH, mesh.V)
        for tol in (1e-6, 1e-10):
            mas = mlm.pcg(sysH, rhs, ML.apply, tol, 20000, check_every=1)[1]
            bj = mlm.pcg(sysH, rhs, mlm.block_jacobi(sysH), tol, 20000, check_every=1)[1]
            counts[f"{name}@{tol:g}"] = (mas, bj)
            assert mas < bj
    record_property("multilevel_vs_block_jacobi_iterations", counts)
    print("iterations (multilevel, block-Jacobi):", counts)
    for tol in ("1e-06", "1e-10"):
        mas, bj = counts[f"ball_on_mat@{tol}"]
        assert 2 * mas <= bj, counts


def ball_on_mat_system():
    m, info = scenes.ball_on_mat()
    ia, ja, a, g, H, sets = mlm.newton_system(m, info["dHat"], 1e8, DT2)
    return m, H, -g
