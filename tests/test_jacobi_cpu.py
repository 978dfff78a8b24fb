"""The diagonally preconditioned gradient (LinSysSolver::precondition_diag) and initX's option-5 Jacobi predictor, restated in
tests/oracle_jacobi.py, on small systems in the LinSysSolver layout: index base 0 and 1, projected and penalty-mode Dirichlet rows and an
obstacle tail.  The restatement is checked against a dense reading of the same CSR (Mesh.csr_pattern); its warm-start driver, which starts from a given
predictor, is checked to reproduce the time-integration driver's option predictors.  No GPU."""
import os
import re

import numpy as np
import pytest
import scipy.sparse as sp

import oracle as orc
import oracle_jacobi as OJ
import oracle_timestep as OT
from gpu_common import same_bits
from ipc_b200 import lib as L
from ipc_b200 import mesh as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COEF = 0.01 ** 2
N_TAIL = 5


def system(base, projectDBC):
    """a deformed grid with Dirichlet vertices and an obstacle tail (no tets, Dirichlet flag): g and the CSR values of the elastic term plus
    the mass diagonal, as the assembly leaves them (the tail's rows are identity rows when projected)"""
    V, T = M.grid_tets(3, 3, 2, h=0.25)
    rng = np.random.default_rng(7)
    tail = rng.standard_normal((N_TAIL, 3)) + [0.0, 0.0, 2.0]
    m = M.Mesh(np.vstack([V, tail]), T, energy=1, density=1.0)
    M.deform(m, 3)
    m.V[-N_TAIL:] = tail
    m.dbc[:4] = 1
    m.dbc[-N_TAIL:] = 1
    ia, ja = m.csr_pattern(base)
    o = orc.Elastic(m)
    g = o.gradient(COEF, projectDBC)
    a = o.hessian_csr(COEF, ia, ja, base, 1, projectDBC)
    rows = np.arange(3 * m.nV)
    fixed = np.repeat(m.dbc != 0, 3)
    diag = ia[:-1] - base
    a[diag[~fixed]] += np.repeat(m.mass, 3)[~fixed]
    if projectDBC:  # the Dirichlet identity rows of the assembly's diagonal pass
        a[diag[fixed]] = 1.0
    else:  # the tail has no term of its own: give its rows a diagonal, as a binding's penalty rows carry one
        a[diag[rows >= 3 * (m.nV - N_TAIL)]] += 1.0
    g = g + rng.standard_normal(g.size) * np.abs(g).max() * (~fixed if projectDBC else 1.0)
    return m, ia, ja, a, g


def dense_diagonal(ia, ja, a, base):
    n = len(ia) - 1
    U = sp.csr_matrix((a, ja - base, ia - base), shape=(n, n))
    return U.diagonal()


@pytest.mark.parametrize("base", [0, 1])
def test_every_row_starts_at_its_diagonal(base):
    m, ia, ja, _, _ = system(base, 1)
    assert np.array_equal(ja[ia[:-1] - base] - base, np.arange(3 * m.nV))


@pytest.mark.parametrize("projectDBC", [1, 0])
@pytest.mark.parametrize("base", [0, 1])
def test_precondition_diag_matches_a_dense_reading(base, projectDBC):
    m, ia, ja, a, g = system(base, projectDBC)
    d = dense_diagonal(ia, ja, a, base)
    assert (d != 0).all()
    fixed = np.repeat(m.dbc != 0, 3)
    for sign in (-1, 1):
        out = OJ.precondition_diag(g, ia, a, base, sign)
        assert same_bits(out, (sign * g) / d)
        assert np.isfinite(out).all()
        if projectDBC:  # identity rows with a zero gradient: 0 without a special case
            assert not out[fixed].any() and (d[fixed] == 1.0).all()
        else:  # penalty mode: those rows are divided like any other
            assert out[fixed].all()
    assert same_bits(OJ.precondition_diag(g, ia, a, base, -1), -OJ.precondition_diag(g, ia, a, base, 1))


def test_zero_and_negative_diagonals_are_divided():
    m, ia, ja, a, g = system(1, 1)
    r0, r1 = 3 * 5, 3 * 6 + 1
    a[ia[r0] - 1], a[ia[r1] - 1] = 0.0, -2.0
    out = OJ.precondition_diag(g, ia, a, 1, -1)
    assert np.isinf(out[r0]) and out[r1] == g[r1] / 2.0
    assert np.isfinite(np.delete(out, r0)).all()


@pytest.mark.parametrize("projectDBC", [1, 0])
@pytest.mark.parametrize("base", [0, 1])
def test_jacobi_predictor(base, projectDBC):
    m, ia, ja, a, g = system(base, projectDBC)
    p = OJ.jacobi_predictor(g, ia, a, base, m.dbc).reshape(-1, 3)
    q = OJ.precondition_diag(g, ia, a, base, -1).reshape(-1, 3)
    fixed = m.dbc != 0
    assert same_bits(p[~fixed], q[~fixed])
    assert (p[fixed].view(np.uint64) == 0).all()  # +0.0, whatever the row held (penalty mode: nonzero)
    assert fixed[-N_TAIL:].all()


def test_warm_start_driver_takes_a_predictor():
    """the driver from a given predictor gives what oracle_timestep's driver gives from an option's own predictor"""
    V1, T1 = M.grid_tets(2, 2, 2, h=0.5)
    V2, T2 = M.grid_tets(2, 2, 2, h=0.5, origin=(0.1, 0.05, 1.05))
    m = M.merge_meshes([(V1, T1), (V2, T2)], energy=1, density=1.0)
    P = OT.Params(OT.BE, 0.01)
    vel = np.zeros((m.nV, 3))
    vel[:len(V1), 2], vel[len(V1):, 2] = 4.0, -4.0
    dxe = np.random.default_rng(2).standard_normal((m.nV, 3)) * 1e-4
    evf, eee = np.full(3, 1e-9), np.full(3, 1e-9)
    ref = OT.warm_start(m, P, 2, vel, dxe, m.avgEdgeLen / 3.0, 1e-6, evf, eee)
    got = OJ.warm_start(m, OT.predictor(P, 2, vel, dxe, m.dbc).ravel(), m.avgEdgeLen / 3.0, 1e-6, evf, eee)
    assert ref["alpha"] < 1.0  # the bodies close: the bound binds
    for k in ("p", "V"):
        assert same_bits(got[k], ref[k]), k
    for k in ("alpha", "alpha_inversion", "alpha_swept_grid", "alpha_full_ccd", "counts", "status"):
        assert got[k] == ref[k], k


def test_signature_matches_the_header():
    import ctypes as C
    src = open(os.path.join(ROOT, "include", "ipcgpu.h")).read()
    mt = re.search(r"\bint\s+ipcgpu_precondition_diag\s*\(([^)]*)\)\s*;", src)
    assert mt, "ipcgpu_precondition_diag is not declared"
    args = [x.strip() for x in mt.group(1).split(",")]
    res, argtypes = L.SIGNATURES["ipcgpu_precondition_diag"]
    assert res is C.c_int and len(argtypes) == len(args) == 4
    assert argtypes[0] is C.c_void_p and argtypes[1] is C.c_int and argtypes[2] is C.POINTER(C.c_double) and argtypes[3] is C.c_int
    assert args[1].startswith("int") and args[2].startswith("double*") and args[3].startswith("int")
