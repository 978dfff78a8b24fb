"""The smoothed-aggregation multigrid PCG at BASELINE.json's full size: C5, the 1M-tet pile bench.py times, at the state and right-hand side
of tests/test_gpu_multilevel_fullsize.py (one implicit-Euler step under gravity, device-built pattern).  The solve reaches 1e-6, the
hierarchy has at least 3 levels with a coarsest of at most 1000 block rows, two solves give identical bits, the solution is block-Jacobi's
to 1e-2, and it needs fewer iterations than the multilevel additive Schwarz solve."""
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


def test_c5_amg_direction(shared_ctx):
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
    x_amg, it_amg, res_amg = ctx.solve_pcg_amg(None, 1e-6, 10000)
    h = ctx.amg_info()
    assert res_amg <= 1e-6 and len(h["rows"]) >= 3 and h["rows"][-1] <= 1000, h
    x_2, it_2, res_2 = ctx.solve_pcg_amg(None, 1e-6, 10000)
    assert it_2 == it_amg and np.array_equal(x_amg.view(np.uint64), x_2.view(np.uint64))
    x_bj, it_bj, res_bj = ctx.solve_pcg(None, 1e-6, 10000)
    x_ml, it_ml, res_ml = ctx.solve_pcg_multilevel(None, 1e-6, 10000)
    assert res_bj <= 1e-6 and res_ml <= 1e-6
    assert np.linalg.norm(x_amg - x_bj) <= 1e-2 * np.linalg.norm(x_bj)  # (both at a residual of 1e-6 of an ill-conditioned system)
    print(f"C5 iterations to 1e-6: AMG {it_amg}, multilevel {it_ml}, block-Jacobi {it_bj}; AMG levels {h['rows']}, blocks {h['blocks']}, "
          f"rho {h['rho']}, {h['bytes'] / 2**20:.0f} MiB")
    assert it_amg < it_ml, (it_amg, it_ml)
