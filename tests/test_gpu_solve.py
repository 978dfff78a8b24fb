"""Device-resident linear-solve hand-off (SURVEY 8(f) rank 1): the Hessian assembled on the device is solved there (block-Jacobi PCG) and
the solution matches a host direct solve of the oracle's matrix; the solution can be adopted as the search direction without a transfer."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import oracle as orc
from gpu_common import load_scene, rel, shared_ctx
from ipc_b200 import scenes
from stagecheck import contact_pattern_pairs

pytestmark = pytest.mark.gpu


def full_matrix(ia, ja, a, n):
    U = sp.csr_matrix((a, np.asarray(ja) - 1, np.asarray(ia) - 1), shape=(n, n))
    return (U + sp.triu(U, 1).T).tocsc()


def test_pcg_on_the_device_resident_hessian(shared_ctx):
    ctx = shared_ctx
    m, info = scenes.ball_pile(4, res=6, seed=5, height=4)
    dHat, p, kappa, dt2 = info["dHat"], info["p"], 1e6, 0.025 ** 2
    load_scene(ctx, m)
    mm, pa, pe, cand = ctx.constraint_set(dHat, 1)
    ia, ja = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe))
    ctx.set_csr(ia, ja, 1)
    # assemble g and H on the device (elastic + mass + barrier), nothing downloaded
    ctx.elastic_grad_hess(dt2, 1, 1, 1, None, None)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    x, iters, res = ctx.solve_pcg(None, rel_tol=1e-10, max_iter=5000)
    assert res <= 1e-10 and 0 < iters < 5000
    # host reference: oracle matrix and gradient, direct solve
    s, o = orc.Surf(m), orc.Elastic(m)
    g_ref = s.barrier_gradient(mm, pa, pe, dHat, kappa, g=o.gradient(dt2, 1))
    a_ref = o.hessian_csr(dt2, ia, ja, 1, 1, 1)
    a_ref[np.asarray(ia[:-1], dtype=np.int64) - 1] += np.repeat(m.mass, 3)
    a_ref = s.barrier_hessian_csr(mm, pa, pe, dHat, kappa, ia, ja, 1, 1, a=a_ref)
    x_ref = spla.spsolve(full_matrix(ia, ja, a_ref, 3 * m.nV), -g_ref)
    assert rel(x, x_ref) <= 1e-7
    # a host right-hand side, and adoption as the search direction: the step-bound stages then run on it without any upload
    b = np.linspace(-1.0, 1.0, 3 * m.nV)
    xb, _, resb = ctx.solve_pcg(b, rel_tol=1e-10, max_iter=5000)
    assert resb <= 1e-10 and rel(xb, spla.spsolve(full_matrix(ia, ja, a_ref, 3 * m.nV), b)) <= 1e-7
    _, _, _ = ctx.solve_pcg(None, rel_tol=1e-10, max_iter=5000, want_x=False, adopt=True)
    al = ctx.inversion_step(None, 0.2, 1.0)
    al_ref, _ = o.inversion_step(x, 0.2, 1.0)
    assert abs(al - al_ref) <= 1e-9 * al_ref
