"""The reproducible mode (ipcgpu_set_canonical_order(ctx, 2)) at BASELINE.json's full size: C5, the 1M-tet pile bench.py times (~8.8k
contact pairs).  Two fresh contexts assemble the system of one implicit-Euler step and solve it with the multilevel PCG: the gradient, the
CSR values, the direction and the iteration count are the same bits in both."""
import os
import sys

import numpy as np
import pytest

from gpu_common import load_scene, own_context
from ipc_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
DT2 = 0.025 ** 2


class _Args:
    tets, res, scene = 1_000_000, 10, "c5"


def test_c5_two_contexts_same_bits():
    import bench
    m, info = bench.build_scene(_Args())
    dHat, kappa, n = info["dHat"], bench.KAPPA, 3 * m.nV
    xt = m.V.copy()
    xt[:, 2] -= 9.81 * DT2
    out = []
    for _ in range(2):
        with own_context() as ctx:
            load_scene(ctx, m)
            ctx.set_canonical_order(2)
            ctx.enable_device_pattern(1)
            ctx.set_xtilde(np.ascontiguousarray(xt.T).ravel())
            nC, nP, _ = ctx.constraint_set(dHat, 1, fetch=False)
            ctx.update_pattern(want=False)
            ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
            ctx.inertia_gradient(1, None)
            ctx.barrier_gradient(dHat, kappa, None)
            ctx.barrier_hessian(dHat, kappa, 1, None)
            x, iters, res = ctx.solve_pcg_multilevel(None, 1e-6, 10000)
            _, ja = ctx.get_pattern()
            out.append(dict(nC=nC, nP=nP, g=ctx.download(L.BUF_GRADIENT, n), a=ctx.download(L.BUF_CSR_VALUES, len(ja)), x=x, iters=iters, res=res))
    a, b = out
    assert a["nC"] > 5000 and (a["nC"], a["nP"]) == (b["nC"], b["nP"])
    assert a["res"] <= 1e-6 and a["iters"] == b["iters"], (a["iters"], b["iters"])
    for key in ("g", "a", "x"):
        assert np.array_equal(a[key].view(np.uint64), b[key].view(np.uint64)), key
