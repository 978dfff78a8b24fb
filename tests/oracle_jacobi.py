"""Float64 restatement of the diagonally preconditioned gradient (the oracle of ipcgpu_precondition_diag and ipcgpu_warm_start option 5).
TEST INFRASTRUCTURE ONLY.

  - LinSysSolver::precondition_diag (LinSysSolver.hpp:411-420) over a gradient and a CSR value array in the LinSysSolver layout;
  - initX's option 5, Jacobi (Optimizer.cpp:1082-1110), and its step bound and backtracking loops (:1120-1215) from that predictor, through
    the driver of tests/oracle_timestep.py.
numpy rounds each elementwise operation once, so the device results must match bit for bit.
"""
import numpy as np

import oracle_timestep as OT


def precondition_diag(g, ia, a, base, sign=-1):
    """(sign g_i) / a(i,i), the diagonal being the first stored entry of row i in the LinSysSolver layout (upper-triangular CSR, every row
    starts at its diagonal).  One division per row, nothing skipped or clamped"""
    g = np.asarray(g, dtype=np.float64)
    d = np.asarray(a, dtype=np.float64)[np.asarray(ia, dtype=np.int64)[:-1] - base]
    with np.errstate(divide="ignore", invalid="ignore"):
        return (-g if sign < 0 else g) / d


def jacobi_predictor(g, ia, a, base, dbc=None):
    """initX option 5's searchDir, interleaved 3 nV: -g_i / H_ii, +0 on Dirichlet vertices (isDBCVertex; the obstacle tail carries the flag)"""
    p = precondition_diag(g, ia, a, base, -1).reshape(-1, 3)
    p[OT.fixed(dbc, len(p))] = 0.0
    return p.ravel()


def warm_start(m, p, voxel, tol, evf, eee, planes=None, alpha_inversion=None):
    """initX's bound and backtracking loops from the predictor p (interleaved 3 nV, 0 on Dirichlet vertices): oracle_timestep.warm_start with
    option 1 at dt = 1, whose predictor dt * velocity is the velocity itself, bit for bit, and 0 on the same vertices"""
    p3 = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    return OT.warm_start(m, OT.Params(OT.BE, 1.0), 1, p3, np.zeros_like(p3), voxel, tol, evf, eee, planes, alpha_inversion)
