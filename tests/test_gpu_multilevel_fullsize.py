"""The multilevel additive Schwarz PCG at BASELINE.json's full size: C5, the 1M-tet pile bench.py times, at the state and right-hand side
of profiles/step_control_timing.py (one implicit-Euler step under gravity, device-built pattern).  Both built-in solvers reach 1e-6 on the
same system; the hierarchy has the expected shape, two solves give identical bits, and the multilevel solve needs at most half of
block-Jacobi's iterations."""
import os
import sys

import numpy as np
import pytest

from gpu_common import load_scene, shared_ctx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
DT2 = 0.025 ** 2


class _Args:
    tets, res, scene = 1_000_000, 10, "c5"


def test_c5_newton_direction_in_half_the_iterations(shared_ctx):
    import bench
    ctx = shared_ctx
    m, info = bench.build_scene(_Args())
    dHat, kappa = info["dHat"], bench.KAPPA
    load_scene(ctx, m)
    ctx.set_canonical_order(0)
    ctx.enable_device_pattern(1)
    xt = m.V.copy()
    xt[:, 2] -= 9.81 * DT2
    ctx.set_xtilde(np.ascontiguousarray(xt.T).ravel())
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    ctx.inertia_gradient(1, None)
    x_ml, it_ml, res_ml = ctx.solve_pcg_multilevel(None, 1e-6, 10000)
    domains, nbytes = ctx.multilevel_info()
    assert domains == [8030, 251, 8, 1] and nbytes == 73728 * 8290
    x_2, it_2, res_2 = ctx.solve_pcg_multilevel(None, 1e-6, 10000)
    assert it_2 == it_ml and np.array_equal(x_ml.view(np.uint64), x_2.view(np.uint64))
    x_bj, it_bj, res_bj = ctx.solve_pcg(None, 1e-6, 10000)
    assert res_ml <= 1e-6 and res_bj <= 1e-6
    assert np.linalg.norm(x_ml - x_bj) <= 1e-2 * np.linalg.norm(x_bj)  # (both at a residual of 1e-6 of an ill-conditioned system)
    print(f"C5 iterations to 1e-6: multilevel {it_ml}, block-Jacobi {it_bj}")
    assert 2 * it_ml <= it_bj, (it_ml, it_bj)
